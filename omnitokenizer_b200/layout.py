"""Host-side index maps and one-time weight packing for the omnitok_b200 kernels.

Everything here is tiny integer / table work done once per (shape, checkpoint) and uploaded;
the per-token arithmetic all happens in the CUDA kernels.
"""
from __future__ import annotations

import functools
import math
import random
from typing import List, NamedTuple, Tuple

import numpy as np
import torch


class U8Norm(NamedTuple):
    """A data pipeline's uint8 -> fp32 normalisation, (u / 255 - mean_c) / std_c per channel in fp32.
    max_test: VideoNorm's `if max(clip) > 1: div_(255)` (OmniTokenizer/video_utils.py:53-54) -- a clip whose largest
    byte is <= 1 is only shifted and scaled, (u - mean_c) / std_c."""
    name: str
    mean: Tuple[float, ...]
    std: Tuple[float, ...]
    max_test: bool = False


def u8_norm_table(norm: U8Norm, channels: int) -> torch.Tensor:
    """fp32 [n_tab, channels, 256]: the value every byte of every channel stands for, computed on the host CPU with the
    pipelines' own torch expression and op order (ToTensor / to_tensor / VideoNorm: / 255; Normalize / VideoNorm:
    .sub_(mean).div_(std) with fp32 mean / std tensors).  Table 0 is the normal mapping; with max_test, table 1 is
    the undivided one.  Kernels only look values up, so they reproduce the pipeline's bits (CUDA would divide by
    multiplying with the reciprocal, which differs in about half of the byte values)."""
    if len(norm.mean) != channels or len(norm.std) != channels:
        raise ValueError(f"normalisation {norm.name!r} has {len(norm.mean)} channels, the model takes {channels}")
    mean = torch.tensor(norm.mean, dtype=torch.float32).view(channels, 1)
    std = torch.tensor(norm.std, dtype=torch.float32).view(channels, 1)
    u = torch.arange(256, dtype=torch.uint8).float().expand(channels, 256).contiguous()
    tabs = [(u / 255.0).sub_(mean).div_(std)]
    if norm.max_test:
        tabs.append(u.clone().sub_(mean).div_(std))
    return torch.stack(tabs).contiguous()


def u8_normalize(frames: torch.Tensor, norm: U8Norm) -> torch.Tensor:
    """(B, T, H, W, C) uint8 -> the (B, C, T, H, W) fp32 video the pipeline hands the model, by table lookup (exact on
    any device).  With max_test the table is chosen per sample from its largest byte, as VideoNorm sees one clip."""
    B, C = frames.shape[0], frames.shape[-1]
    tab = u8_norm_table(norm, C).to(frames.device)
    sel = torch.zeros(B, dtype=torch.long, device=frames.device)
    if norm.max_test and frames.numel() > 0:
        sel = (frames.reshape(B, -1).amax(dim=1) <= 1).long()
    x = frames.permute(0, 4, 1, 2, 3).long()
    return tab[sel.view(B, 1, 1, 1, 1), torch.arange(C, device=frames.device).view(1, C, 1, 1, 1), x]


class U8Resize(NamedTuple):
    """An image loader's geometric transform before ToTensor: torchvision Resize(size, filter) on the PIL image (Pillow's
    8-bit resize), then optionally RandomCrop(crop) and RandomHorizontalFlip(0.5), in that order."""
    size: Tuple[int, int]          # (height, width) after the resize
    filter: str = "bicubic"        # Pillow filter: "bicubic", "bilinear", "box" or "antialias" (LANCZOS)
    crop: int = 0                  # side of the square random crop of the resized image; 0: none
    flip: bool = False

    @property
    def out_size(self) -> Tuple[int, int]:
        return (self.crop, self.crop) if self.crop else (int(self.size[0]), int(self.size[1]))


def image_resize(resolution: int) -> U8Resize:
    """ImageDataset without --resizecrop (OmniTokenizer/data.py:93-99): Resize((res, res), BICUBIC)."""
    return U8Resize((resolution, resolution), "bicubic")


def resizecrop_resize(resolution: int) -> U8Resize:
    """ImageDataset with --resizecrop (OmniTokenizer/data.py:84-90): Resize((1.5 res, 1.5 res), BICUBIC), RandomCrop(res)."""
    side = int(resolution * 1.5)
    return U8Resize((side, side), "bicubic", crop=resolution)


def dit_resize(image_size: int) -> U8Resize:
    """DiT with the OmniTokenizer VAE (Diffusion/DiT/train.py:192-198): Resize((s, s)) -- torchvision's default filter,
    BILINEAR -- then RandomHorizontalFlip."""
    return U8Resize((image_size, image_size), "bilinear", flip=True)


def check_infer_downsample(d, what: str = "infer_downsample") -> int:
    """vqgan_eval.py's --infer_downsample (type=int): an integer factor d >= 1.  Returns it as an int."""
    if isinstance(d, bool) or not isinstance(d, (int, np.integer)):
        raise TypeError(f"{what}: infer_downsample must be an integer factor, got {d!r}")
    if d < 1:
        raise ValueError(f"{what}: infer_downsample must be >= 1, got {d}")
    return int(d)


def eval_downsample_resize(resolution: int, d: int) -> U8Resize:
    """vqgan_eval.py's image branch with --infer_downsample d (:207-208, :218-219): img.resize((res // d, res // d),
    Image.ANTIALIAS), Pillow's LANCZOS, of the saved input and reconstruction."""
    d = check_infer_downsample(d)
    side = int(resolution) // d
    if side < 1:
        raise ValueError(f"infer_downsample {d} leaves {resolution} // {d} = {side} pixels")
    return U8Resize((side, side), "antialias")


def check_resize(resize: U8Resize):
    if not isinstance(resize, U8Resize):
        raise TypeError(f"expected a layout.U8Resize, got {type(resize).__name__}")
    if resize.filter not in _FILTERS:
        raise ValueError(f"unknown resize filter {resize.filter!r}; choose from {sorted(_FILTERS)}")
    h, w = resize.size
    if h < 1 or w < 1 or resize.crop < 0 or resize.crop > min(h, w):
        raise ValueError(f"resize to {h}x{w} with a crop of {resize.crop}: the crop must fit the resized image")


# Resample.c's filters (bicubic a = -0.5) and supports, in its float64 operation order
def _bicubic(x):
    x = np.abs(x)
    a = -0.5
    return np.where(x < 1.0, ((a + 2.0) * x - (a + 3.0)) * x * x + 1,
                    np.where(x < 2.0, (((x - 5) * x + 8) * x - 4) * a, 0.0))


def _bilinear(x):
    x = np.abs(x)
    return np.where(x < 1.0, 1.0 - x, 0.0)


def _box(x):
    return np.where((x > -0.5) & (x <= 0.5), 1.0, 0.0)


def _sinc(x):
    """Resample.c sinc_filter: sin(pi x) / (pi x), 1 at 0.  sin from the C library, as Pillow calls it (numpy's own
    vectorised sin may differ in the last bit)."""
    px = x * math.pi
    s = np.array([math.sin(v) for v in px.reshape(-1)], dtype=np.float64).reshape(px.shape)
    return np.where(x == 0.0, 1.0, s / np.where(x == 0.0, 1.0, px))


def _lanczos(x):
    """Resample.c lanczos_filter: the sinc truncated to [-3, 3), windowed by sinc(x / 3)."""
    x = np.asarray(x, dtype=np.float64)
    return np.where((x >= -3.0) & (x < 3.0), _sinc(x) * _sinc(x / 3), 0.0)


# "antialias": Pillow's LANCZOS under the name vqgan_eval.py resizes with (Image.ANTIALIAS, LANCZOS's old alias)
_FILTERS = {"bicubic": (_bicubic, 2.0), "bilinear": (_bilinear, 1.0), "box": (_box, 0.5), "antialias": (_lanczos, 3.0)}
RESAMPLE_BITS = 22       # Resample.c PRECISION_BITS for 8-bit images


@functools.lru_cache(maxsize=1024)
def resample_coeffs(in_size: int, out_size: int, filter: str) -> Tuple[np.ndarray, np.ndarray]:
    """Pillow's per-axis tables for resizing an axis of in_size to out_size: (bounds int32 [out, 2] = (xmin, n) per output
    index, coefficients int32 [out, ksize], zero past n).  libImaging/Resample.c precompute_coeffs + normalize_coeffs_8bpc
    in float64, operation for operation: the weights of an output are summed tap by tap in order (numpy's pairwise sum
    rounds differently), then rounded to 22-bit fixed point with +-0.5 and truncation.  Computed on the host: a device
    compiler would contract these multiply-adds into FMAs and change the float64 results."""
    fn, support = _FILTERS[filter]
    scale = filterscale = in_size / out_size
    if filterscale < 1.0:
        filterscale = 1.0
    support = support * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    center = 0.0 + (np.arange(out_size, dtype=np.float64) + 0.5) * scale
    ss = 1.0 / filterscale
    xmin = np.maximum(np.trunc(center - support + 0.5), 0).astype(np.int64)
    xmax = np.minimum(np.trunc(center + support + 0.5), in_size).astype(np.int64)
    n = xmax - xmin
    x = np.arange(ksize, dtype=np.int64)[None, :]
    live = x < n[:, None]
    w = np.where(live, fn(((x + xmin[:, None]).astype(np.float64) - center[:, None] + 0.5) * ss), 0.0)
    ww = np.zeros(out_size, dtype=np.float64)
    for j in range(ksize):
        ww = ww + w[:, j]
    k = np.where(ww[:, None] != 0.0, w / np.where(ww == 0.0, 1.0, ww)[:, None], w)
    fixed = np.where(k < 0, np.trunc(-0.5 + k * (1 << RESAMPLE_BITS)), np.trunc(0.5 + k * (1 << RESAMPLE_BITS)))
    coeffs = np.where(live, fixed, 0).astype(np.int32)
    bounds = np.stack([xmin, n], axis=1).astype(np.int32)
    bounds.flags.writeable = False
    coeffs.flags.writeable = False
    return bounds, coeffs


def resize_params(n: int, resize: U8Resize) -> List[Tuple[int, int, bool]]:
    """(top, left, flip) of n images, drawn from torch's default CPU generator exactly as the loader's transforms draw them
    image after image: RandomCrop.get_params (torch.randint for the top, then the left; nothing when the crop is the
    whole image), then RandomHorizontalFlip (torch.rand(1) < 0.5)."""
    h, w = resize.size
    out = []
    for _ in range(n):
        i = j = 0
        if resize.crop and not (h == resize.crop and w == resize.crop):
            i = torch.randint(0, h - resize.crop + 1, size=(1,)).item()
            j = torch.randint(0, w - resize.crop + 1, size=(1,)).item()
        flip = bool(torch.rand(1) < 0.5) if resize.flip else False
        out.append((int(i), int(j), flip))
    return out


def check_resize_params(params, n: int, resize: U8Resize):
    if len(params) != n:
        raise ValueError(f"{len(params)} resize parameters for {n} images")
    (h, w), (oh, ow) = resize.size, resize.out_size
    for b, (i, j, flip) in enumerate(params):
        if not (0 <= i <= h - oh and 0 <= j <= w - ow) or (flip and not resize.flip) or ((i or j) and not resize.crop):
            raise ValueError(f"resize parameters of image {b} ({i}, {j}, {flip}) are not a draw of {resize}")


def _resample_axis(x: torch.Tensor, dim: int, out_size: int, filter: str) -> torch.Tensor:
    """One Pillow pass over axis `dim` of int64 bytes, tap by tap: 2^21 + sum of byte * coefficient, then clip8."""
    in_size = x.shape[dim]
    bounds, coeffs = resample_coeffs(in_size, out_size, filter)
    xmin = torch.from_numpy(bounds[:, 0].astype(np.int64))
    k = torch.from_numpy(coeffs.astype(np.int64))
    shape = [1] * x.ndim
    shape[dim] = out_size
    out_shape = list(x.shape)
    out_shape[dim] = out_size
    acc = torch.full(out_shape, 1 << (RESAMPLE_BITS - 1), dtype=torch.int64)
    for t in range(k.shape[1]):            # past n the coefficient is 0 (the clamped index is never counted)
        acc += x.index_select(dim, (xmin + t).clamp(max=in_size - 1)) * k[:, t].view(shape)
    return (acc >> RESAMPLE_BITS).clamp(0, 255)


def vertical_first(H: int, W: int, h: int, w: int) -> bool:
    """Pillow's Image.resize runs the vertical pass first (as a resize of its own) for an image taller than 100 times its
    width that shrinks in height; the two passes round differently in that order."""
    return H > W * 100 and h < H and w != W


def resize_u8(image: torch.Tensor, resize: U8Resize, param: Tuple[int, int, bool] = (0, 0, False)) -> torch.Tensor:
    """Host twin of omt_resample_u8 for one (H, W, C) uint8 image: Pillow's horizontal pass (skipped when the width stays),
    then its vertical pass (skipped when the height stays) -- swapped for vertical_first images --, then the crop at
    (top, left) and the flip -> (oh, ow, C) uint8, byte for byte what the loader's transforms make of the PIL image."""
    h, w = resize.size
    x = image.long()
    v_first = vertical_first(x.shape[0], x.shape[1], h, w)
    if v_first:
        x = _resample_axis(x, 0, h, resize.filter)
    if x.shape[1] != w:
        x = _resample_axis(x, 1, w, resize.filter)
    if x.shape[0] != h:
        x = _resample_axis(x, 0, h, resize.filter)
    (oh, ow), (i, j, flip) = resize.out_size, param
    x = x[i:i + oh, j:j + ow]
    if flip:
        x = x.flip(1)
    return x.to(torch.uint8).contiguous()


class ClipResize(NamedTuple):
    """A Latte video loader's geometric transform of a ToTensorVideo'd clip (Diffusion/Latte/datasets/__init__.py,
    video_transforms.py), bilinear F.interpolate with align_corners=False on the fp32 clip:
    - "scale_crop": UCFCenterCropVideo(size): scale_factor size / min(H, W), then a centre size x size crop;
    - "crop_resize": CenterCropResizeVideo(size): centre crop of the short edge, then resize to size x size;
    - "none": the clip keeps its H x W.
    flip: RandomHorizontalFlipVideo before the resize (Python's random.random() < 0.5, once per clip).
    in_workers: the transform runs where torch.get_num_threads() == 1, as in the DataLoader worker processes of Latte's
    configs (num_workers > 0); torch's CPU bilinear kernel picks its arithmetic by that (clip_interp_form)."""
    mode: str
    size: int = 0
    flip: bool = False
    in_workers: bool = True


def ucf_clip_resize(size: int) -> ClipResize:
    """ucf101 and ffs: ToTensorVideo, RandomHorizontalFlipVideo, UCFCenterCropVideo(size), Normalize."""
    return ClipResize("scale_crop", size, True)


def sky_clip_resize(size: int) -> ClipResize:
    """sky: ToTensorVideo, CenterCropResizeVideo(size), Normalize (no flip)."""
    return ClipResize("crop_resize", size, False)


def taichi_clip_resize() -> ClipResize:
    """taichi: ToTensorVideo, RandomHorizontalFlipVideo, Normalize (no resize)."""
    return ClipResize("none", 0, True)


_CLIP_MODES = ("scale_crop", "crop_resize", "none")


def check_clip_resize(resize: ClipResize):
    if not isinstance(resize, ClipResize):
        raise TypeError(f"expected a layout.ClipResize, got {type(resize).__name__}")
    if resize.mode not in _CLIP_MODES:
        raise ValueError(f"unknown clip resize mode {resize.mode!r}; choose from {list(_CLIP_MODES)}")
    if (resize.mode == "none") != (resize.size == 0) or resize.size < 0:
        raise ValueError(f"clip resize {resize.mode!r} with size {resize.size}: 'none' takes size 0, the others a size >= 1")


class ClipGeometry(NamedTuple):
    """Where one clip's transform reads and writes: the window (y0, x0, wh, ww) of the (flipped) source frame the resize
    reads, the resized size (rh, rw), the crop origin (cy, cx) in it, and the fp32 coordinate scale of each axis."""
    y0: int
    x0: int
    wh: int
    ww: int
    rh: int
    rw: int
    cy: int
    cx: int
    scale_h: float
    scale_w: float


@functools.lru_cache(maxsize=4096)
def scaled_size(H: int, W: int, size: int) -> Tuple[int, int]:
    """Output size of UCFCenterCropVideo's F.interpolate(scale_factor=size / min(H, W)), from torch's own shape rule."""
    x = torch.empty(1, 1, H, W, device="meta")
    y = torch.nn.functional.interpolate(x, scale_factor=size / min(H, W), mode="bilinear", align_corners=False)
    return int(y.shape[-2]), int(y.shape[-1])


def clip_geometry(H: int, W: int, resize: ClipResize) -> ClipGeometry:
    """The transform's geometry for an H x W source frame.  Raises center_crop's ValueError (video_transforms.py:85-86)
    where the reference does: UCFCenterCropVideo's scaled short side can come out one pixel short of the size."""
    if resize.mode == "none":
        return ClipGeometry(0, 0, H, W, H, W, 0, 0, 1.0, 1.0)
    s = resize.size
    if resize.mode == "scale_crop":
        rh, rw = scaled_size(H, W, s)
        if rh < s or rw < s:
            raise ValueError("height and width must be no smaller than crop_size")
        inv = float(np.float32(1.0 / (s / min(H, W))))     # torch: static_cast<float>(1.0 / scale_factor)
        # center_crop's offsets are Python's round-half-to-even of (h - th) / 2
        return ClipGeometry(0, 0, H, W, rh, rw, int(round((rh - s) / 2.0)), int(round((rw - s) / 2.0)), inv, inv)
    if H < W:                                                # center_crop_using_short_edge
        y0, x0, n = 0, int(round((W - H) / 2.0)), H
    else:
        y0, x0, n = int(round((H - W) / 2.0)), 0, W
    sc = float(np.float32(n) / np.float32(s))                # torch: (float)input_size / output_size
    return ClipGeometry(y0, x0, n, n, s, s, 0, 0, sc, sc)


def clip_out_size(H: int, W: int, resize: ClipResize) -> Tuple[int, int]:
    return (H, W) if resize.mode == "none" else (resize.size, resize.size)


INTERP_SEPARABLE, INTERP_WEIGHTS = 0, 1


def clip_interp_form(g: ClipGeometry, in_workers: bool) -> int:
    """Which of torch's CPU bilinear kernels (x86-64 with FMA) runs for a 3-channel clip resized to g.rh x g.rw:
    - INTERP_WEIGHTS, the channels-last kernel, when the output is small (rh + rw <= 128) or torch runs on one thread:
      w_ab = lambda_h_a * lambda_w_b, out = fma(x11, w11, fma(x10, w10, fma(x00, w00, x01 * w01)));
    - INTERP_SEPARABLE, the generic kernel, otherwise: t_r = fma(x_r0, l0w, x_r1 * l1w), out = fma(t_0, l0h, t_1 * l1h)."""
    return INTERP_WEIGHTS if in_workers or g.rh + g.rw <= 128 else INTERP_SEPARABLE


@functools.lru_cache(maxsize=1024)
def clip_axis_table(n_in: int, n_out: int, scale: float) -> np.ndarray:
    """int32 [n_out, 4]: (i0, i1, lambda0 bits, lambda1 bits) of every output index of one axis of torch's bilinear
    interpolation (align_corners=False), in fp32 as torch's CPU kernel computes them: src = max(fma(scale, d + 0.5,
    -0.5), 0) (the compiler contracts it); i0 = min(floor(src), n_in - 1); i1 = i0 + (i0 < n_in - 1);
    lambda1 = clamp(src - i0, 0, 1); lambda0 = 1 - lambda1.  Built on the host: the device must see these exact bits."""
    f32 = np.float32
    d = np.arange(n_out).astype(f32)
    src = np.maximum(fma32(f32(scale), d + f32(0.5), f32(-0.5)), f32(0))
    i0 = np.minimum(np.floor(src).astype(np.int64), n_in - 1)
    i1 = i0 + (i0 < n_in - 1)
    l1 = np.minimum(np.maximum(src - i0.astype(f32), f32(0)), f32(1))
    l0 = f32(1) - l1
    t = np.stack([i0.astype(np.int32), i1.astype(np.int32), l0.view(np.int32), l1.view(np.int32)], axis=1)
    t.flags.writeable = False
    return t


def fma32(a, b, c) -> np.ndarray:
    """fp32 a * b + c rounded once, elementwise (the CPU kernel's vector FMA; Python 3.12 has no math.fma).  The product
    is exact in fp64 and TwoSum gives the sum's exact error, so the fp64 sum is rounded to fp32 correctly except when it
    lands exactly on a midpoint between two fp32 values: there the sign of the error picks the side."""
    a, b, c = (np.asarray(t, dtype=np.float32) for t in (a, b, c))
    p = a.astype(np.float64) * b.astype(np.float64)
    c = c.astype(np.float64)
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    r = s.astype(np.float32)
    r64 = r.astype(np.float64)
    other = np.nextafter(r, np.where(s > r64, np.float32(np.inf), np.float32(-np.inf))).astype(np.float32)
    tie = (s != r64) & ((r64 + other.astype(np.float64)) * 0.5 == s) & (err != 0)
    return np.where(tie, np.where(err > 0, np.maximum(r, other), np.minimum(r, other)), r)


def byte_table() -> torch.Tensor:
    """fp32 [256]: to_tensor's clip.float() / 255.0 of every byte (video_transforms.py:143), computed by torch."""
    return torch.arange(256, dtype=torch.uint8).float() / 255.0


def clip_norm_table(norm: U8Norm) -> torch.Tensor:
    """fp32 [262] for omt_resample_clips: the 256 byte values, then mean[3], then std[3] as fp32."""
    if norm.max_test:
        raise ValueError(f"normalisation {norm.name!r} tests each clip's largest byte; the video loaders' Normalize does not")
    if len(norm.mean) != 3 or len(norm.std) != 3:
        raise ValueError(f"normalisation {norm.name!r} has {len(norm.mean)} channels, clips have 3")
    return torch.cat([byte_table(), torch.tensor(norm.mean, dtype=torch.float32), torch.tensor(norm.std, dtype=torch.float32)])


def clip_params(n: int, resize: ClipResize) -> List[bool]:
    """The flips of n clips, drawn as RandomHorizontalFlipVideo draws them clip after clip: random.random() < 0.5 from
    Python's generator (torch's generator is not touched); nothing is drawn without a flip."""
    return [random.random() < 0.5 for _ in range(n)] if resize.flip else [False] * n


def check_clip_params(params, n: int, resize: ClipResize):
    if len(params) != n:
        raise ValueError(f"{len(params)} clip parameters for {n} clips")
    for b, flip in enumerate(params):
        if not isinstance(flip, (bool, np.bool_)) or (flip and not resize.flip):
            raise ValueError(f"clip parameter {b} ({flip!r}) is not a draw of {resize}")


def resize_clip(clip: torch.Tensor, resize: ClipResize, flip: bool = False, norm: U8Norm = None) -> torch.Tensor:
    """Host twin of omt_resample_clips for one (F, H, W, 3) uint8 clip -> (F, 3, oh, ow) fp32: to_tensor, the flip, the
    window, the bilinear interpolation through clip_axis_table in the arithmetic of clip_interp_form, the crop, and
    (value - mean) / std when norm is given."""
    F_, H, W = (int(v) for v in clip.shape[:3])
    g = clip_geometry(H, W, resize)
    oh, ow = clip_out_size(H, W, resize)
    v = byte_table().numpy()[clip.numpy()]                 # (F, H, W, 3)
    if flip:
        v = v[:, :, ::-1]
    v = v[:, g.y0:g.y0 + g.wh, g.x0:g.x0 + g.ww]
    th = clip_axis_table(g.wh, g.rh, g.scale_h)[g.cy:g.cy + oh]
    tw = clip_axis_table(g.ww, g.rw, g.scale_w)[g.cx:g.cx + ow]
    l0h, l1h = (th[:, k].view(np.float32)[None, :, None, None] for k in (2, 3))
    l0w, l1w = (tw[:, k].view(np.float32)[None, None, :, None] for k in (2, 3))

    r0, r1 = v[:, th[:, 0]], v[:, th[:, 1]]
    x00, x01, x10, x11 = r0[:, :, tw[:, 0]], r0[:, :, tw[:, 1]], r1[:, :, tw[:, 0]], r1[:, :, tw[:, 1]]
    if clip_interp_form(g, resize.in_workers) == INTERP_WEIGHTS:
        out = fma32(x11, l1h * l1w, fma32(x10, l1h * l0w, fma32(x00, l0h * l0w, x01 * (l0h * l1w))))
    else:
        out = fma32(fma32(x00, l0w, x01 * l1w), l0h, fma32(x10, l0w, x11 * l1w) * l1h)
    if norm is not None:
        out = (out - np.asarray(norm.mean, np.float32)) / np.asarray(norm.std, np.float32)
    return torch.from_numpy(np.ascontiguousarray(out.transpose(0, 3, 1, 2)))


@functools.lru_cache(maxsize=1024)
def downsample_geometry(H: int, W: int, d: int) -> ClipGeometry:
    """vqgan_eval.py's F.interpolate(scale_factor=1 / d, mode="bilinear", align_corners=False) of an H x W frame: the
    output size from torch's own shape rule (floor of n * (1 / d) in double, so 63 at d = 3 gives 20), and the coordinate
    scale torch's CPU kernel uses for a given scale_factor, static_cast<float>(1.0 / scale_factor)."""
    x = torch.empty(1, 1, H, W, device="meta")
    y = torch.nn.functional.interpolate(x, scale_factor=1 / d, mode="bilinear", align_corners=False)
    rh, rw = int(y.shape[-2]), int(y.shape[-1])
    inv = float(np.float32(1.0 / (1 / d)))
    return ClipGeometry(0, 0, H, W, rh, rw, 0, 0, inv, inv)


def downsample_clips(src: torch.Tensor, d: int, one_thread: bool, value_table: torch.Tensor = None,
                     sel=None) -> torch.Tensor:
    """Host twin of omt_eval_downsample: (B, T, oh, ow, 3) uint8 = shift_dim(F.interpolate(v, scale_factor=1 / d) * 255,
    1, -1).byte() in torch's CPU arithmetic (the kernel form clip_interp_form picks for one_thread), of
    - src fp32 (B, 3, T, H, W), the decoder's reconstruction: v = clamp(src + 0.5, 0, 1) (value_table None);
    - src uint8 (B, T, H, W, 3), the loader's bytes: v = value_table[sel[b]][byte] (value_table fp32 [n_tab, 256],
      sel per clip, all 0 when None)."""
    if value_table is None:
        v = torch.clamp(src.float() + 0.5, 0, 1).permute(0, 2, 3, 4, 1).numpy()
    else:
        B = src.shape[0]
        sel = np.zeros(B, dtype=np.int64) if sel is None else np.asarray(sel, dtype=np.int64)
        v = value_table.numpy()[sel.reshape(B, 1, 1, 1, 1), src.numpy()]
    B, T, H, W, _ = v.shape
    g = downsample_geometry(H, W, d)
    th = clip_axis_table(H, g.rh, g.scale_h)
    tw = clip_axis_table(W, g.rw, g.scale_w)
    l0h, l1h = (th[:, k].view(np.float32)[None, None, :, None, None] for k in (2, 3))
    l0w, l1w = (tw[:, k].view(np.float32)[None, None, None, :, None] for k in (2, 3))
    r0, r1 = v[:, :, th[:, 0]], v[:, :, th[:, 1]]
    x00, x01, x10, x11 = r0[:, :, :, tw[:, 0]], r0[:, :, :, tw[:, 1]], r1[:, :, :, tw[:, 0]], r1[:, :, :, tw[:, 1]]
    if clip_interp_form(g, one_thread) == INTERP_WEIGHTS:
        out = fma32(x11, l1h * l1w, fma32(x10, l1h * l0w, fma32(x00, l0h * l0w, x01 * (l0h * l1w))))
    else:
        out = fma32(fma32(x00, l0w, x01 * l1w), l0h, fma32(x10, l0w, x11 * l1w) * l1h)
    # .byte(): the product truncated to int32, its low byte kept (x86-64)
    return torch.from_numpy((out * np.float32(255)).astype(np.int32).astype(np.uint8))


def peg_neighbour_table(T: int, h: int, w: int, temporal: bool, causal: bool) -> torch.Tensor:
    """int32 [T*h*w, 27]: canonical neighbour row (inside one batch element) of every tap of the
    PEG depthwise 3x3x3 stencil, -1 where the reference zero-pads.

    Spatial transformers see the true (t,h,w) volume.  Temporal transformers hand PEG a
    '(b h w) t d' tensor that the reference reshapes LITERALLY to (b,t,h,w,d)
    (modules/attention.py:313-319), i.e. flat position f = n*T + tau is unravelled over (T,h,w):
    the stencil runs in that scrambled space and is mapped back to canonical rows tau*N + n.
    Padding: (1,1) on h and w, (2,0) on t when causal else (1,1) (attention.py:323-325).
    """
    N = h * w
    tau = torch.arange(T).view(T, 1).expand(T, N).reshape(-1)
    n = torch.arange(N).view(1, N).expand(T, N).reshape(-1)
    f = (n * T + tau) if temporal else (tau * N + n)
    t2 = f // N
    h2 = (f % N) // w
    w2 = f % w
    out = torch.empty(T * N, 27, dtype=torch.int64)
    k = 0
    for kt in range(3):
        tt = t2 + kt - (2 if causal else 1)
        for kh in range(3):
            hh = h2 + kh - 1
            for kw in range(3):
                ww = w2 + kw - 1
                ok = (tt >= 0) & (tt < T) & (hh >= 0) & (hh < h) & (ww >= 0) & (ww < w)
                f2 = (tt * h + hh) * w + ww
                r2 = (f2 % T) * N + (f2 // T) if temporal else f2
                out[:, k] = torch.where(ok, r2, torch.full_like(r2, -1))
                k += 1
    return out.to(torch.int32)


def rope_tables(N: int, dim_head: int, theta: float = 10000.0) -> Tuple[torch.Tensor, torch.Tensor]:
    """(cos, sin) [N, dim_head/2] of the 2-D axial rope (modules/attention.py:28-44), computed with
    the same torch fp32 ops as the reference so the table is bit-identical to its freqs_cis."""
    H = int(N ** 0.5)
    pos = torch.arange(N)
    x_pos, y_pos = pos % H, pos // H
    freqs = 1.0 / (theta ** (torch.arange(0, dim_head, 4)[: (dim_head // 4)].float() / dim_head))
    xf = torch.outer(x_pos, freqs).float()
    yf = torch.outer(y_pos, freqs).float()
    x_cis = torch.polar(torch.ones_like(xf), xf)
    y_cis = torch.polar(torch.ones_like(yf), yf)
    cis = torch.cat([x_cis.unsqueeze(-1), y_cis.unsqueeze(-1)], dim=-1).reshape(N, -1)
    return cis.real.contiguous().float(), cis.imag.contiguous().float()


def window_bias(table: torch.Tensor, index: torch.Tensor, ws: int) -> torch.Tensor:
    """[heads, ws*ws, ws*ws] gathered relative position bias (modules/attention.py:277-279)."""
    n = ws * ws
    b = table[index.reshape(-1).long()].reshape(n, n, -1)
    return b.permute(2, 0, 1).contiguous().float()


def tf32_round(w: torch.Tensor) -> torch.Tensor:
    """Round fp32 to tf32 (10-bit mantissa), nearest / ties away -- the `cvt.rna.tf32.f32` rule."""
    i = w.contiguous().view(torch.int32)
    return ((i + 0x1000) & -8192).view(torch.float32)


F16X3_LO_SCALE = 2048.0


def split_f16(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Operand planes of the f16x3 tensor-core path (csrc/omt_common.cuh): hi = fp16(w) (round to nearest, saturating)
    and lo = fp16((w - hi) * 2^11); w ~= hi + lo * 2^-11 to 2^-23 |w|.  Same rounding as the device-side split."""
    w = w.float()
    hi = w.clamp(-65504.0, 65504.0).to(torch.float16)
    lo = ((w - hi.float()) * F16X3_LO_SCALE).clamp(-65504.0, 65504.0).to(torch.float16)
    return hi.contiguous(), lo.contiguous()


def split_f16_rs(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, float]:
    """Row-scaled form for a WEIGHT matrix (one scale for the whole matrix): w' = w * 2^e with max |w'| in [2^14, 2^15),
    hi = fp16(w'), lo = fp16(w' - hi) unscaled.  Returns (hi, lo, 2^-e)."""
    w = w.float()
    mx = float(w.abs().max())
    e = 14 - math.floor(math.log2(mx)) if mx > 0 else 0
    e = max(-100, min(100, e))
    ws = w * (2.0 ** e)
    hi = ws.clamp(-65504.0, 65504.0).to(torch.float16)
    lo = (ws - hi.float()).to(torch.float16)
    return hi.contiguous(), lo.contiguous(), 2.0 ** -e


def pow2_scale(bound: float) -> float:
    """The power of two that maps values bounded by `bound` into [2^14, 2^15) (fp16 range with headroom); 1.0 for 0."""
    if not (bound > 0.0) or not math.isfinite(bound):
        return 1.0
    return 2.0 ** max(-100, min(100, 14 - math.floor(math.log2(bound))))


def split_rows_rs(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Row-scaled form of an activation matrix, the host twin of csrc/omt_common.cuh row_scale(): per row the power of two
    that puts the largest magnitude in [2^14, 2^15).  Returns (hi, lo, inverse row scales [rows])."""
    x = x.float()
    eb = ((x.abs().amax(dim=1).contiguous().view(torch.int32) >> 23) & 0xFF).clamp(15, 254)
    scale = ((268 - eb) << 23).view(torch.float32)
    inv = ((eb - 14) << 23).view(torch.float32)
    xs = x * scale[:, None]
    hi = xs.clamp(-65504.0, 65504.0).to(torch.float16)
    lo = (xs - hi.float()).to(torch.float16)
    return hi.contiguous(), lo.contiguous(), inv.contiguous()


def join_f16(hi: torch.Tensor, lo: torch.Tensor) -> torch.Tensor:
    """fp32 value a pair of operand planes stands for (int16 views are reinterpreted as fp16)."""
    return hi.view(torch.float16).float() + lo.view(torch.float16).float() / F16X3_LO_SCALE


def pad_rows(w: torch.Tensor, mult: int) -> torch.Tensor:
    n = w.shape[0]
    n_pad = (n + mult - 1) // mult * mult
    if n_pad == n:
        return w.contiguous()
    out = torch.zeros(n_pad, w.shape[1], dtype=w.dtype, device=w.device)
    out[:n] = w
    return out


def pad_cols(w: torch.Tensor, k_pad: int) -> torch.Tensor:
    if w.shape[1] == k_pad:
        return w.contiguous()
    out = torch.zeros(w.shape[0], k_pad, dtype=w.dtype, device=w.device)
    out[:, : w.shape[1]] = w
    return out


def pack_geglu(w1: torch.Tensor, inner: int, ku: int) -> torch.Tensor:
    """Interleave FeedForward's first Linear (modules/attention.py:164, rows [value | gate]) so that
    packed rows (2j, 2j+1) = (value_j, gate_j); zero rows pad j up to ku."""
    out = torch.zeros(2 * ku, w1.shape[1], dtype=w1.dtype, device=w1.device)
    out[0: 2 * inner: 2] = w1[:inner]
    out[1: 2 * inner: 2] = w1[inner: 2 * inner]
    return out


def round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def isqrt_exact(n: int) -> int:
    r = int(math.sqrt(n))
    return r
