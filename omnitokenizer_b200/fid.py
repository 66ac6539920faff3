"""The FID metric's feature network on the device: pytorch-fid's InceptionV3 (evaluation/pytorch-fid/src/pytorch_fid/
inception.py, with the FIDInceptionA / C / E_1 / E_2 patches) up to the 2048-wide pool3 features, from device uint8
images, on the sm_90a kernels of csrc/i3d.cu and csrc/resample.cu.

Drop-in names for fid_score.py: load_fid_model(device, path), activation_statistics(features) (mu, sigma as
calculate_activation_statistics computes them), calculate_frechet_distance(mu1, sigma1, mu2, sigma2, eps) and
fid_given_paths(paths, model, batch_size) for directories of images (the `python3 .../pytorch_fid/__main__.py in recon`
line of vqgan_eval.py).

Activations are channels-last fp32 [B][H][W][Cs], Cs the channel count rounded up to a multiple of 32 (4 for the
network input, fvd.cpad); the pad columns are zero.  Every BasicConv2d (conv without bias, BatchNorm2d(eps=0.001),
ReLU) is one omt_conv3d launch with a kernel depth of 1 (3xTF32, BatchNorm folded into the weights at pack time); each
branch writes its slice of the block's concat buffer in place, and the pools run on omt_pool2d.
"""
from __future__ import annotations

import os
import pathlib
from typing import Dict, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _cabi
from . import layout as L
from .engine import CLIP_DESC_WORDS, run_graphed
from .fvd import cpad, pack_weight, real_byte_table

TARGET_RESOLUTION = (299, 299)     # inception.py:148
BN_EPS = 1e-3                      # torchvision BasicConv2d's BatchNorm2d(eps=0.001)
DIMS = 2048                        # fid_score.py --dims default: the pool3 features; the only width built here
POOL_MAX, POOL_AVG = 0, 1          # omt_pool2d modes
IMAGE_EXTENSIONS = ("bmp", "jpg", "jpeg", "pgm", "png", "ppm", "tif", "tiff", "webp", "JPEG")   # fid_score.py:94


class Conv(NamedTuple):
    """One BasicConv2d: its key prefix, input ("x": the block input, "p": the pooled block input, or another conv of
    the block), widths, kernel, stride, symmetric padding, and its concat-buffer column (None: its own buffer)."""
    name: str
    src: str
    cin: int
    cout: int
    k: Tuple[int, int]
    s: int
    p: Tuple[int, int]
    col: Optional[int]


class Pool(NamedTuple):
    """A pool: mode, window, stride, padding, and its concat-buffer column (None: the "p" input of branch_pool)."""
    mode: int
    k: int
    s: int
    p: int
    col: Optional[int]


def _c(name, src, cin, cout, k, s=1, p=0, col=None) -> Conv:
    k = (k, k) if isinstance(k, int) else tuple(k)
    p = (p, p) if isinstance(p, int) else tuple(p)
    return Conv(name, src, cin, cout, k, s, p, col)


# torchvision inception.py's Inception3 stem as pytorch-fid's blocks 0 and 1 use it (inception.py:86-101)
STEM = [_c("Conv2d_1a_3x3", "x", 3, 32, 3, s=2), _c("Conv2d_2a_3x3", "x", 32, 32, 3),
        _c("Conv2d_2b_3x3", "x", 32, 64, 3, p=1), Pool(POOL_MAX, 3, 2, 0, None),
        _c("Conv2d_3b_1x1", "x", 64, 80, 1), _c("Conv2d_4a_3x3", "x", 80, 192, 3), Pool(POOL_MAX, 3, 2, 0, None)]


def _block_a(cin, pool_features):        # FIDInceptionA: the pool averages without the padding
    return ([_c("branch1x1", "x", cin, 64, 1, col=0),
             _c("branch5x5_1", "x", cin, 48, 1), _c("branch5x5_2", "branch5x5_1", 48, 64, 5, p=2, col=64),
             _c("branch3x3dbl_1", "x", cin, 64, 1), _c("branch3x3dbl_2", "branch3x3dbl_1", 64, 96, 3, p=1),
             _c("branch3x3dbl_3", "branch3x3dbl_2", 96, 96, 3, p=1, col=128),
             _c("branch_pool", "p", cin, pool_features, 1, col=224)], Pool(POOL_AVG, 3, 1, 1, None), 224 + pool_features)


def _block_b(cin):                       # InceptionB (Mixed_6a): the max pool fills the last cin columns
    return ([_c("branch3x3", "x", cin, 384, 3, s=2, col=0),
             _c("branch3x3dbl_1", "x", cin, 64, 1), _c("branch3x3dbl_2", "branch3x3dbl_1", 64, 96, 3, p=1),
             _c("branch3x3dbl_3", "branch3x3dbl_2", 96, 96, 3, s=2, col=384)], Pool(POOL_MAX, 3, 2, 0, 480), 480 + cin)


def _block_c(cin, c7):                   # FIDInceptionC
    return ([_c("branch1x1", "x", cin, 192, 1, col=0),
             _c("branch7x7_1", "x", cin, c7, 1), _c("branch7x7_2", "branch7x7_1", c7, c7, (1, 7), p=(0, 3)),
             _c("branch7x7_3", "branch7x7_2", c7, 192, (7, 1), p=(3, 0), col=192),
             _c("branch7x7dbl_1", "x", cin, c7, 1), _c("branch7x7dbl_2", "branch7x7dbl_1", c7, c7, (7, 1), p=(3, 0)),
             _c("branch7x7dbl_3", "branch7x7dbl_2", c7, c7, (1, 7), p=(0, 3)),
             _c("branch7x7dbl_4", "branch7x7dbl_3", c7, c7, (7, 1), p=(3, 0)),
             _c("branch7x7dbl_5", "branch7x7dbl_4", c7, 192, (1, 7), p=(0, 3), col=384),
             _c("branch_pool", "p", cin, 192, 1, col=576)], Pool(POOL_AVG, 3, 1, 1, None), 768)


def _block_d(cin):                       # InceptionD (Mixed_7a)
    return ([_c("branch3x3_1", "x", cin, 192, 1), _c("branch3x3_2", "branch3x3_1", 192, 320, 3, s=2, col=0),
             _c("branch7x7x3_1", "x", cin, 192, 1),
             _c("branch7x7x3_2", "branch7x7x3_1", 192, 192, (1, 7), p=(0, 3)),
             _c("branch7x7x3_3", "branch7x7x3_2", 192, 192, (7, 1), p=(3, 0)),
             _c("branch7x7x3_4", "branch7x7x3_3", 192, 192, 3, s=2, col=320)], Pool(POOL_MAX, 3, 2, 0, 512), 512 + cin)


def _block_e(cin, pool_mode):            # FIDInceptionE_1 (average pool without the padding) / _E_2 (max pool)
    return ([_c("branch1x1", "x", cin, 320, 1, col=0),
             _c("branch3x3_1", "x", cin, 384, 1),
             _c("branch3x3_2a", "branch3x3_1", 384, 384, (1, 3), p=(0, 1), col=320),
             _c("branch3x3_2b", "branch3x3_1", 384, 384, (3, 1), p=(1, 0), col=704),
             _c("branch3x3dbl_1", "x", cin, 448, 1), _c("branch3x3dbl_2", "branch3x3dbl_1", 448, 384, 3, p=1),
             _c("branch3x3dbl_3a", "branch3x3dbl_2", 384, 384, (1, 3), p=(0, 1), col=1088),
             _c("branch3x3dbl_3b", "branch3x3dbl_2", 384, 384, (3, 1), p=(1, 0), col=1472),
             _c("branch_pool", "p", cin, 192, 1, col=1856)], Pool(pool_mode, 3, 1, 1, None), 2048)


# pytorch-fid's blocks 2 and 3 (inception.py:104-125, fid_inception_v3 :204-213): (name, convs, pool, output width)
BLOCKS = [("Mixed_5b",) + _block_a(192, 32), ("Mixed_5c",) + _block_a(256, 64), ("Mixed_5d",) + _block_a(288, 64),
          ("Mixed_6a",) + _block_b(288),
          ("Mixed_6b",) + _block_c(768, 128), ("Mixed_6c",) + _block_c(768, 160), ("Mixed_6d",) + _block_c(768, 160),
          ("Mixed_6e",) + _block_c(768, 192),
          ("Mixed_7a",) + _block_d(768),
          ("Mixed_7b",) + _block_e(1280, POOL_AVG), ("Mixed_7c",) + _block_e(2048, POOL_MAX)]


def conv_list() -> List[Conv]:
    """Every BasicConv2d with its full key prefix, in the network's order (94 of them)."""
    out = [c for c in STEM if isinstance(c, Conv)]
    for name, convs, _, _ in BLOCKS:
        out += [c._replace(name=f"{name}.{c.name}") for c in convs]
    return out


def out_size(n: int, k: int, s: int, p: int) -> int:
    """Output length of a conv / pool axis of length n (symmetric padding p, floor mode)."""
    return (n + 2 * p - k) // s + 1


def expected_keys() -> Dict[str, tuple]:
    keys = {}
    for c in conv_list():
        keys[c.name + ".conv.weight"] = (c.cout, c.cin) + c.k
        for f in ("weight", "bias", "running_mean", "running_var"):
            keys[f"{c.name}.bn.{f}"] = (c.cout,)
    return keys


def fold_bn(w: torch.Tensor, gamma, beta, mean, var) -> Tuple[torch.Tensor, torch.Tensor]:
    """BatchNorm2d (running statistics, eps 1e-3) folded into a conv weight (cout, cin, kh, kw), in float64:
    (W s, beta - mean s) with s = gamma / sqrt(var + eps), rounded to fp32."""
    s = gamma.double() / torch.sqrt(var.double() + BN_EPS)
    return (w.double() * s.view(-1, 1, 1, 1)).float(), (beta.double() - mean.double() * s).float()


class _Unit:
    """One BasicConv2d packed for omt_conv3d: tf32 hi / lo planes of W, the folded bias, its geometry."""

    def __init__(self, conv: Conv, w, bias, device):
        packed, self.K = pack_weight(w.unsqueeze(2))        # (cout, cin, 1, kh, kw): K = (dh, dw, c)
        hi = L.tf32_round(packed)
        self.w_hi, self.w_lo = hi.to(device), (packed - hi).to(device)
        self.bias, self.conv = bias.to(device), conv


def byte_lut(real_norm: Optional[L.U8Norm] = None) -> torch.Tensor:
    """fp32 [n_tab, 256]: the value the network's input takes for each byte before the resize: ToTensor's byte / 255
    (fid_score.py:146), or, for the loader's bytes of a real image, / 255 of the byte vqgan_eval.py saves for it,
    ((v + 0.5) * 255).astype(uint8) of the normalised value v (:205; fvd.real_byte_table)."""
    b = torch.arange(256, dtype=torch.float32).view(1, 256) if real_norm is None else real_byte_table(real_norm).float()
    return b / 255


class _Workspace:
    """Buffers, launch list and CUDA graph state of one (B, H, W, real_norm)."""

    def __init__(self, net: "FIDInception", B: int, H: int, W: int, real_norm: Optional[L.U8Norm] = None):
        dev = net.device
        self.graphs = {}
        self.u8 = torch.empty(B, H, W, 3, dtype=torch.uint8, device=dev)
        self.lut = byte_lut(real_norm).to(dev)
        self.sel = torch.empty(B, dtype=torch.int32, device=dev) if real_norm is not None and real_norm.max_test else None
        self.out = torch.empty(B, DIMS, device=dev)
        # inception.py:148 F.interpolate to 299 x 299 from torch's multi-threaded CPU kernel: the separable form
        oh, ow = TARGET_RESOLUTION
        tv = L.clip_axis_table(H, oh, float(np.float32(H) / np.float32(oh))).reshape(-1)
        th = L.clip_axis_table(W, ow, float(np.float32(W) / np.float32(ow))).reshape(-1)
        self.tab_host = torch.from_numpy(np.concatenate([tv, th]).astype(np.int32))
        desc = torch.zeros(B, CLIP_DESC_WORDS, dtype=torch.int32)
        desc[:, :2] = (torch.arange(B, dtype=torch.int64) * (H * W * 3)).view(torch.int32).view(B, 2)
        desc[:, 2:] = torch.tensor([H, W, 0, 0, H, W, oh, ow, 0, 0, 0, 0, tv.size, L.INTERP_SEPARABLE], dtype=torch.int32)
        self.desc_host = desc
        self.desc, self.tab = desc.to(dev), self.tab_host.to(dev)
        self.ops = []
        self.B = B

        x = self._act(oh, ow, 3)
        if self.sel is not None:
            self.ops.append(lambda: _cabi.call("omt_u8_norm_select", self.u8, B, H * W * 3, self.sel))
        self.ops.append(lambda: _cabi.call(
            "omt_fid_preprocess", self.u8, self.u8.numel(), self.desc, self.desc_host, self.tab, self.tab_host,
            self.tab_host.numel(), self.lut, self.sel, B, oh, ow, x))
        cur, c_cur, hw = x, 3, (oh, ow)
        for layer in STEM:
            if isinstance(layer, Conv):
                cur, hw = self._conv(net.units[layer.name], cur, hw)
                c_cur = layer.cout
            else:
                cur, hw = self._pool(layer, cur, c_cur, hw)
        for name, convs, pool, cout in BLOCKS:
            o = hw
            if pool.col is not None:                   # strided blocks: the output size is the pool's
                o = tuple(out_size(n, pool.k, pool.s, pool.p) for n in hw)
            y = self._act(*o, cout)
            bufs = {"x": cur}
            if pool.col is None:
                bufs["p"], _ = self._pool(pool, cur, c_cur, hw)
            else:
                self._pool(pool, cur, c_cur, hw, out=(y, pool.col))
            for c in convs:
                u = net.units[f"{name}.{c.name}"]
                if c.col is None:
                    bufs[c.name], _ = self._conv(u, bufs[c.src], hw)
                else:
                    _, got = self._conv(u, bufs[c.src], hw, out=(y, c.col))
                    if got != o:
                        raise AssertionError(f"{name}.{c.name}: output {got}, the block's is {o}")
            cur, c_cur, hw = y, cout, o
        if hw != (8, 8) or c_cur != DIMS:
            raise ValueError(f"the pool3 features need an [8, 8, {DIMS}] map, got {hw + (c_cur,)}")
        # AdaptiveAvgPool2d(1) of the 8 x 8 map (inception.py:123): one 8 x 8 window straight into the (B, 2048) output
        self._pool(Pool(POOL_AVG, 8, 1, 0, 0), cur, c_cur, hw, out=(self.out.view(B, 1, 1, DIMS), 0))

    def _act(self, H_, W_, c):
        # pad columns stay zero: no kernel writes them
        return torch.zeros(self.B, H_, W_, cpad(c), device=self.u8.device, dtype=torch.float32)

    def _conv(self, u: _Unit, x, hw, out=None):
        c = u.conv
        o = tuple(out_size(n, k, c.s, p) for n, k, p in zip(hw, c.k, c.p))
        y, col = (self._act(*o, c.cout), 0) if out is None else out
        ypt = y.data_ptr() + 4 * col
        B = self.B
        self.ops.append(lambda: _cabi.call(
            "omt_conv3d", x, x.shape[-1], B, 1, hw[0], hw[1], u.w_hi, u.w_lo, u.K, u.bias, c.cout,
            1, c.k[0], c.k[1], 1, c.s, c.s, 0, c.p[0], c.p[1], 1, o[0], o[1], ypt, y.shape[-1], 1))
        return y, o

    def _pool(self, pool: Pool, x, c, hw, out=None):
        o = tuple(out_size(n, pool.k, pool.s, pool.p) for n in hw)
        y, col = (self._act(*o, c), 0) if out is None else out
        ypt = y.data_ptr() + 4 * col
        B = self.B
        self.ops.append(lambda: _cabi.call(
            "omt_pool2d", x, x.shape[-1], c, B, hw[0], hw[1], pool.k, pool.k, pool.s,
            pool.s, pool.p, pool.p, o[0], o[1], ypt, y.shape[-1], pool.mode))
        return y, o

    def run(self):
        for op in self.ops:
            op()


class FIDInception:
    """pytorch-fid's InceptionV3([3]) (inception.py:16-161, fid_inception_v3's patched blocks) in eval mode, from a
    state_dict in the layout of its weight file pt_inception-2015-12-05-6726825d.pth, torchvision Inception3 keys
    (`Conv2d_1a_3x3.conv.weight`, `Mixed_7c.branch_pool.bn.running_var`, ...); `fc.*`, `AuxLogits.*` and
    `num_batches_tracked` are ignored.  BatchNorm is folded and the weights packed once, on `device`; every
    (B, H, W, real_norm) gets its own buffers and CUDA graph (the last few are kept)."""

    MAX_WORKSPACES = 4

    def __init__(self, state_dict: Dict[str, torch.Tensor], device="cuda"):
        sd = {k: v for k, v in state_dict.items()
              if not (k.endswith(".num_batches_tracked") or k.startswith(("fc.", "AuxLogits.")))}
        want = expected_keys()
        missing, unexpected = sorted(set(want) - set(sd)), sorted(set(sd) - set(want))
        if missing or unexpected:
            raise KeyError(f"FID InceptionV3 state_dict: missing keys {missing}, unexpected keys {unexpected}")
        for k, shape in want.items():
            if tuple(sd[k].shape) != shape:
                raise ValueError(f"FID InceptionV3 state_dict: {k} has shape {tuple(sd[k].shape)}, expected {shape}")
        self.device = torch.device(device)
        if self.device.type == "cuda" and self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        sd = {k: v.detach().float().cpu() for k, v in sd.items()}
        self.units = {}
        for c in conv_list():
            w, b = fold_bn(sd[c.name + ".conv.weight"], *(sd[f"{c.name}.bn.{f}"]
                                                          for f in ("weight", "bias", "running_mean", "running_var")))
            self.units[c.name] = _Unit(c, w, b, self.device)
        self._ws = {}

    @staticmethod
    def check_images(images: torch.Tensor):
        if not isinstance(images, torch.Tensor) or images.dtype != torch.uint8:
            raise TypeError(f"FIDInception.features takes a uint8 tensor, got {getattr(images, 'dtype', type(images))}")
        if images.dim() != 4 or images.shape[-1] != 3:
            raise ValueError(f"FIDInception.features takes (B, H, W, 3) images, got {tuple(images.shape)}")
        if min(images.shape[:3]) < 1:
            raise ValueError(f"empty image batch {tuple(images.shape)}")

    def features(self, images_u8: torch.Tensor, real_norm: Optional[L.U8Norm] = None) -> torch.Tensor:
        """(B, H, W, 3) uint8 on this network's device -> the pool3 features (B, 2048) fp32: get_activations of
        fid_score.py on the PNGs of these bytes.  real_norm: the images are the loader's bytes, and the network sees
        the bytes vqgan_eval.py saves of the normalised input, ((v + 0.5) * 255).astype(uint8) (byte_lut).
        The returned tensor is the workspace's static output: clone it before the next call of the same shape."""
        self.check_images(images_u8)
        if images_u8.device != self.device:
            raise ValueError(f"FIDInception.features: images on {images_u8.device}, the network is on {self.device}")
        if real_norm is not None:
            real_byte_table(real_norm)                       # refuses a per-channel normalisation before any launch
        key = tuple(int(v) for v in images_u8.shape[:3]) + (real_norm,)
        ws = self._ws.get(key)
        if ws is None:
            while len(self._ws) >= self.MAX_WORKSPACES:
                self._ws.pop(next(iter(self._ws)))
            ws = self._ws[key] = _Workspace(self, *key)
        ws.u8.copy_(images_u8)
        run_graphed(ws.graphs, self.device, "fid", ws.run)
        return ws.out


def _check_dims(dims: int):
    if dims != DIMS:
        raise ValueError(f"only the {DIMS}-wide pool3 features are built (fid_score.py's default --dims), got {dims}")


def load_fid_model(device, path: str, dims: int = DIMS) -> FIDInception:
    """InceptionV3([BLOCK_INDEX_BY_DIM[2048]]) (fid_score.py:294-296) with the weight file given by path
    (pt_inception-2015-12-05-6726825d.pth; the weights are not shipped and nothing is downloaded)."""
    _check_dims(dims)
    return FIDInception(torch.load(path, map_location="cpu"), device)


def activation_statistics(features) -> Tuple[np.ndarray, np.ndarray]:
    """calculate_activation_statistics' (mu, sigma) (fid_score.py:259-262) of (N, 2048) features, torch or numpy:
    np.mean and np.cov(rowvar=False) of the float64 features."""
    if isinstance(features, torch.Tensor):
        features = features.detach().cpu().numpy()
    act = np.asarray(features, dtype=np.float64)
    return np.mean(act, axis=0), np.cov(act, rowvar=False)


def calculate_frechet_distance(mu1, sigma1, mu2, sigma2, eps: float = 1e-6) -> float:
    """The Frechet distance between N(mu1, sigma1) and N(mu2, sigma2), |mu1 - mu2|^2 + tr(sigma1 + sigma2 -
    2 sqrt(sigma1 sigma2)), as fid_score.py:179-236 computes it: scipy.linalg.sqrtm of the product; if that is not
    finite, eps is added to both diagonals and the root taken again; a complex root whose diagonal has an imaginary
    part beyond 1e-3 is an error, otherwise its real part is used.  Runs once per split on the host."""
    from scipy import linalg
    mu1, mu2 = np.atleast_1d(mu1), np.atleast_1d(mu2)
    sigma1, sigma2 = np.atleast_2d(sigma1), np.atleast_2d(sigma2)
    if mu1.shape != mu2.shape:
        raise ValueError(f"mean vectors of different lengths: {mu1.shape} and {mu2.shape}")
    if sigma1.shape != sigma2.shape:
        raise ValueError(f"covariances of different shapes: {sigma1.shape} and {sigma2.shape}")
    diff = mu1 - mu2
    root = linalg.sqrtm(sigma1.dot(sigma2))          # scipy >= 1.16 has no `disp`; the root is the same either way
    if not np.isfinite(root).all():
        print(f"fid calculation produces singular product; adding {eps} to diagonal of cov estimates")
        offset = np.eye(sigma1.shape[0]) * eps
        root = linalg.sqrtm((sigma1 + offset).dot(sigma2 + offset))
    if np.iscomplexobj(root):
        if not np.allclose(np.diagonal(root).imag, 0, atol=1e-3):
            raise ValueError(f"Imaginary component {np.max(np.abs(root.imag))}")
        root = root.real
    return diff.dot(diff) + np.trace(sigma1) + np.trace(sigma2) - 2 * np.trace(root)


def image_files(path) -> List[pathlib.Path]:
    """fid_score.py:270-277: the sorted */*.ext files of a directory, or, if there are none, its sorted *.ext files."""
    path = pathlib.Path(path)
    files = sorted(f for ext in IMAGE_EXTENSIONS for f in path.glob(f"*/*.{ext}"))
    if not files:
        files = sorted(f for ext in IMAGE_EXTENSIONS for f in path.glob(f"*.{ext}"))
    return files


def path_features(files: Sequence, model: FIDInception, batch_size: int = 50) -> torch.Tensor:
    """get_activations (fid_score.py:113-176) of image files: decoded on the host (PIL, .convert("RGB")) in batches of
    batch_size (the whole list when it is shorter), copied to the device as uint8, features on the device.  Images of
    one batch that differ in size run as consecutive sub-batches of equal size.  Returns (N, 2048) fp32 on the device."""
    from PIL import Image
    files = list(files)
    if not files:
        raise ValueError("no image files")
    batch_size = min(batch_size, len(files))
    out = []
    for i in range(0, len(files), batch_size):
        ims = [torch.from_numpy(np.asarray(Image.open(f).convert("RGB"))) for f in files[i:i + batch_size]]
        j = 0
        while j < len(ims):
            e = j + 1
            while e < len(ims) and ims[e].shape == ims[j].shape:
                e += 1
            batch = torch.stack(ims[j:e]).to(model.device)
            out.append(model.features(batch).clone())
            j = e
    return torch.cat(out)


def fid_given_paths(paths: Sequence[str], model: FIDInception, batch_size: int = 50, dims: int = DIMS) -> float:
    """calculate_fid_given_paths (fid_score.py:288-306) with the model given: the FID between two directories of
    images (or .npz files holding mu and sigma), each listed as compute_statistics_of_path lists it."""
    _check_dims(dims)
    stats = []
    for p in paths:
        p = str(p)
        if not os.path.exists(p):
            raise RuntimeError(f"Invalid path: {p}")
        if p.endswith(".npz"):
            with np.load(p) as f:
                stats.append((f["mu"][:], f["sigma"][:]))
            continue
        files = image_files(p)
        if not files:
            raise ValueError(f"no images with extensions {IMAGE_EXTENSIONS} in {p}")
        stats.append(activation_statistics(path_features(files, model, batch_size)))
    (m1, s1), (m2, s2) = stats
    return calculate_frechet_distance(m1, s1, m2, s2)
