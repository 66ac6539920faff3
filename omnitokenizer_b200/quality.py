"""Per-frame reconstruction metrics on the device: PSNR and SSIM of evaluation/common_metrics_on_video_quality
(calculate_psnr.py, calculate_ssim.py) and LPIPS with the tokenizer's own VGG16 network (OmniTokenizer/modules/lpips.py,
the `perceptual_model` every OmniTokenizer checkpoint carries), on the sm_90a kernels of csrc/quality.cu and the VGG16
trunk on csrc/i3d.cu's omt_conv3d (3x3, pad 1, ReLU, 3xTF32) and omt_pool2d (2 x 2 max pools).

- frame_metrics(real_u8, fake_u8, lpips=None, real_norm=None): per-frame psnr / ssim (fp64) and lpips (fp32) of device
  uint8 (B, T, H, W, 3) frames;
- drop-ins with the suite's signatures and result dicts: calculate_psnr, calculate_ssim (videos (B, T, C, H, W) in
  [0, 1]) and calculate_lpips_vgg (the VGG LPIPS);
- calculate_lpips(videos1, videos2, device, model): the suite's own calculate_lpips, the lpips package's AlexNet with
  spatial=True (AlexLPIPS, load_lpips_alex: torchvision's AlexNet file and the package's lin file, taken by path): the
  five convs on omt_conv3d, the 3 x 3 / 2 max pools on omt_pool2d, each tap's per-pixel map (omt_lpips_map) and the
  maps upsampled, summed and averaged per frame (omt_lpips_upsample_mean);
- calculate_fvd(videos1, videos2, device, method, i3d): the suite's FVD at every prefix length, styleganv or videogpt,
  on fvd.I3D.features (csrc/resample.cu's omt_fvd_suite_preprocess and the I3D kernels).

Activations are channels-last fp32 [2P][h][w][C] (the network input [2P][H][W][4]); pair p is images p (real) and
p + P (reconstruction).  Each VGG tap's LPIPS head runs right after the tap's conv, so only two ping-pong activation
buffers live; AlexNet writes each tap's map right after the tap's conv in the same way.  The frames run in chunks of at
most LPIPS_ROWS / (2 H W) pairs; every (chunk, H, W, real_norm) gets its own buffers and CUDA graph.
"""
from __future__ import annotations

import math
from typing import Dict, List, NamedTuple, Optional, Tuple

import numpy as np
import torch

from . import _cabi
from . import layout as L
from .engine import run_graphed
from .fvd import I3D, SuiteClips
from .fvd import frechet_distance as fvd_frechet_distance
from .metricnet import FORM_F32 as FORM_FVD_F32, FORM_F32_TRUNC as FORM_FVD_F32_TRUNC, FORM_U8 as FORM_FVD_U8
from .metricnet import (MAX_WORKSPACES, PackedConv, bounded, byte_lut, check_state_dict, real_byte_table,
                        resolve_device)

FORM_U8, FORM_F32 = 0, 1           # OMT_Q_U8 / OMT_Q_F32
POOL_MAX = 0                       # omt_pool2d mode
SSIM_TAPS, SSIM_SIGMA = 11, 1.5    # calculate_ssim.py:11 cv2.getGaussianKernel(11, 1.5)
MIN_SSIM = SSIM_TAPS               # the valid map of an 11-tap window needs H, W >= 11
MIN_LPIPS = 16                     # four 2 x 2 pools leave a 1 x 1 relu5_3 map
PSNR_MAX, PSNR_MSE_FLOOR = 100.0, 1e-10   # calculate_psnr.py:11-12
NORM_EPS = 1e-10                   # lpips.py normalize_tensor
CHNS = (64, 128, 256, 512, 512)    # lpips.py:57, the channels of the five taps
# ScalingLayer's constructor values (lpips.py:113-114): used only for state dicts without its buffers
SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)
# int32 output rows of omt_conv3d: one chunk's first layer has 2 P H W rows (1 GiB of 64-channel activations)
LPIPS_ROWS = 1 << 22
MAX_CONV_ROWS = 0x7FFFFFFF
PLAIN_CHUNK = 1024                 # pairs per launch without LPIPS


class Conv(NamedTuple):
    """One VGG16 conv: its index in torchvision's vgg16().features, the lpips.py slice that holds it, its widths."""
    idx: int
    slice: int
    cin: int
    cout: int


# torchvision vgg16 features as lpips.py's vgg16 slices them (slice1 = features[0:4], ... slice5 = [23:30]): every
# slice but the first starts with MaxPool2d(2, 2); each ends at its tap (relu1_2, relu2_2, relu3_3, relu4_3, relu5_3)
SLICES: List[List[Conv]] = [
    [Conv(0, 1, 3, 64), Conv(2, 1, 64, 64)],
    [Conv(5, 2, 64, 128), Conv(7, 2, 128, 128)],
    [Conv(10, 3, 128, 256), Conv(12, 3, 256, 256), Conv(14, 3, 256, 256)],
    [Conv(17, 4, 256, 512), Conv(19, 4, 512, 512), Conv(21, 4, 512, 512)],
    [Conv(24, 5, 512, 512), Conv(26, 5, 512, 512), Conv(28, 5, 512, 512)],
]


# cv2.getGaussianKernel(11, 1.5) (calculate_ssim.py:11), CV_64F: OpenCV computes it in its own soft-float arithmetic,
# whose exp rounds some taps one ulp away from the C library's, so the taps are kept as its exact output (half of the
# symmetric kernel, centre last); gaussian_taps_formula restates the formula itself
_CV2_TAPS_11_1_5 = ("0x1.0d956b52a1d6ep-10", "0x1.f1fe01ae5a5b5p-8", "0x1.26eb175d83f66p-5", "0x1.bff0fe8e98418p-4",
                    "0x1.b43c3f52b19f3p-3", "0x1.106560aa892bfp-2")


def gaussian_taps() -> torch.Tensor:
    """The SSIM window's 1-D taps, fp64 [11]: cv2.getGaussianKernel(11, 1.5) bit for bit."""
    half = [float.fromhex(h) for h in _CV2_TAPS_11_1_5]
    return torch.tensor(half + half[-2::-1], dtype=torch.float64)


def gaussian_taps_formula(n: int = SSIM_TAPS, sigma: float = SSIM_SIGMA) -> torch.Tensor:
    """getGaussianKernel's formula for sigma > 0 in double: t_i = exp(-(x_i)^2 / (2 sigma^2)), x_i = i - (n - 1) / 2,
    each times 1 / sum t.  Within an ulp of OpenCV's soft-float result."""
    t = [math.exp(-0.5 / (sigma * sigma) * (i - (n - 1) * 0.5) ** 2) for i in range(n)]
    s = 1.0 / sum(t)
    return torch.tensor([v * s for v in t], dtype=torch.float64)


def psnr_from_sse(sse: torch.Tensor, n: int) -> torch.Tensor:
    """img_psnr (calculate_psnr.py:6-14) from the fp64 sum of squared differences over n = C H W values:
    mse = sse / n; 100 if mse < 1e-10, else 20 log10(1 / sqrt(mse))."""
    mse = sse.double() / n
    return torch.where(mse < PSNR_MSE_FLOOR, torch.full_like(mse, PSNR_MAX), 20 * torch.log10(1 / torch.sqrt(mse)))


def expected_keys() -> Dict[str, tuple]:
    """The LPIPS state_dict keys lpips.py's module holds (NetLinLayer's Dropout has no parameters)."""
    keys = {}
    for convs in SLICES:
        for c in convs:
            keys[f"net.slice{c.slice}.{c.idx}.weight"] = (c.cout, c.cin, 3, 3)
            keys[f"net.slice{c.slice}.{c.idx}.bias"] = (c.cout,)
    for k, ch in enumerate(CHNS):
        keys[f"lin{k}.model.1.weight"] = (1, ch, 1, 1)
    keys["scaling_layer.shift"] = (1, 3, 1, 1)
    keys["scaling_layer.scale"] = (1, 3, 1, 1)
    return keys


def lpips_state_dict(state_dict: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """The LPIPS keys of any of: a tokenizer checkpoint's state_dict (the `perceptual_model.` entries, the rest
    ignored), a bare LPIPS state_dict, or torchvision vgg16's `features.N.*` plus the LPIPS lin file's
    `lin{k}.model.1.weight` (`classifier.*` ignored; without `scaling_layer.*`, ScalingLayer's constructor values)."""
    sd = dict(state_dict)
    pre = "perceptual_model."
    if any(k.startswith(pre) for k in sd):
        sd = {k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}
    if any(k.startswith("features.") for k in sd):
        where = {c.idx: c.slice for convs in SLICES for c in convs}
        out = {}
        for k, v in sd.items():
            if k.startswith("classifier."):
                continue
            if k.startswith("features."):
                idx, rest = k[len("features."):].split(".", 1)
                if not idx.isdigit() or int(idx) not in where:
                    raise KeyError(f"LPIPS state_dict: unexpected torchvision key {k}")
                k = f"net.slice{where[int(idx)]}.{idx}.{rest}"
            out[k] = v
        sd = out
        sd.setdefault("scaling_layer.shift", torch.tensor(SHIFT).view(1, 3, 1, 1))
        sd.setdefault("scaling_layer.scale", torch.tensor(SCALE).view(1, 3, 1, 1))
    return sd


def check_net(net: str = "vgg", spatial: bool = False):
    if net != "vgg":
        raise NotImplementedError(f"LPIPS net {net!r} is not built here: this class is the tokenizer's VGG16 LPIPS "
                                  f"(lpips.py); the lpips package's net='alex', spatial=True is quality.AlexLPIPS")
    if spatial:
        raise NotImplementedError("LPIPS spatial=True is not built for the VGG LPIPS, which returns the spatial "
                                  "average; the lpips package's AlexNet with spatial=True is quality.AlexLPIPS")


def input_table(shift: torch.Tensor, scale: torch.Tensor, real_norm: Optional[L.U8Norm] = None) -> torch.Tensor:
    """fp32 [n_tab, 3, 256]: the network input each byte of each channel becomes, in torch's fp32 with the reference's
    ops: v = byte / 255 (or / 255 of the byte real_byte_table(real_norm) sends it to), x = v * 2 - 1
    (calculate_lpips.trans), then (x - shift_c) / scale_c (ScalingLayer)."""
    v = byte_lut(real_norm)                                          # [n_tab, 256]
    x = (v * 2 - 1).unsqueeze(1)
    return ((x - shift.float().view(1, 3, 1)) / scale.float().view(1, 3, 1)).contiguous()


class LPIPS:
    """lpips.py's LPIPS (VGG16 trunk, five lin layers, ScalingLayer) in eval mode, from a state_dict (see
    lpips_state_dict for the accepted layouts).  A missing or mis-shaped key is named in the error.  The weights are
    packed once, on `device`.  net / spatial: the lpips package's options; anything but VGG without the spatial map
    raises NotImplementedError."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device="cuda", net: str = "vgg", spatial: bool = False):
        check_net(net, spatial)
        sd = lpips_state_dict(state_dict)
        check_state_dict(sd, expected_keys(), "LPIPS")
        self.device = resolve_device(device)
        sd = {k: v.detach().float().cpu() for k, v in sd.items()}
        self.units = [[PackedConv(sd[f"net.slice{c.slice}.{c.idx}.weight"], sd[f"net.slice{c.slice}.{c.idx}.bias"],
                                  self.device) for c in convs] for convs in SLICES]
        self.lin = [sd[f"lin{k}.model.1.weight"].reshape(-1).contiguous().to(self.device) for k in range(len(CHNS))]
        self.shift, self.scale = sd["scaling_layer.shift"].reshape(3), sd["scaling_layer.scale"].reshape(3)
        self.shift_scale = torch.cat([self.shift, self.scale]).to(self.device)
        self._ws = {}


class _Workspace:
    """Buffers, launch list and CUDA graph state of one (form, P, H, W, real_norm) with or without LPIPS."""

    def __init__(self, device, form: int, P: int, H: int, W: int, real_norm: Optional[L.U8Norm],
                 lpips: Optional[LPIPS]):
        self.graphs = {}
        dt = torch.uint8 if form == FORM_U8 else torch.float32
        self.a = torch.empty(P, H, W, 3, dtype=dt, device=device)
        self.b = torch.empty(P, H, W, 3, dtype=dt, device=device)
        self.sel = (torch.zeros(P, dtype=torch.int32, device=device)
                    if real_norm is not None and real_norm.max_test else None)
        self.sse = torch.empty(P, dtype=torch.float64, device=device)
        self.ssim = torch.empty(P, dtype=torch.float64, device=device)
        self.taps = gaussian_taps().to(device)
        self.ops = []
        lut_a = lut_b = None
        if form == FORM_U8:
            lut_a, lut_b = byte_lut(real_norm).to(device), byte_lut().to(device)
        self.ops.append(lambda: _cabi.call("omt_psnr_ssim", self.a, lut_a, self.sel, self.b, lut_b, None, form, P, H, W,
                                           self.taps, self.sse, self.ssim))
        self.lp = None
        if lpips is None:
            return
        f = dict(device=device, dtype=torch.float32)
        self.lp_taps = torch.zeros(len(CHNS), P, **f)
        self.lp = torch.zeros(P, **f)
        x = torch.zeros(2 * P, H, W, 4, **f)
        big = 2 * P * H * W * CHNS[0]                 # the largest activation: 64 channels at full size
        bufs = [torch.zeros(big, **f), torch.zeros(big, **f)]
        half = P * H * W * 4
        if form == FORM_U8:
            in_a = input_table(lpips.shift, lpips.scale, real_norm).to(device)
            in_b = input_table(lpips.shift, lpips.scale).to(device)
            self.ops.append(lambda: _cabi.call("omt_lpips_input", self.a, in_a, self.sel, None, form, P, H, W, x))
            self.ops.append(lambda: _cabi.call("omt_lpips_input", self.b, in_b, None, None, form, P, H, W,
                                               x.data_ptr() + 4 * half))
        else:
            ss = lpips.shift_scale
            self.ops.append(lambda: _cabi.call("omt_lpips_input", self.a, None, None, ss, form, P, H, W, x))
            self.ops.append(lambda: _cabi.call("omt_lpips_input", self.b, None, None, ss, form, P, H, W,
                                               x.data_ptr() + 4 * half))
        cur, c_cur, h, w, nxt = x, 4, H, W, 0
        for s, units in enumerate(lpips.units):
            if s > 0:                                 # MaxPool2d(kernel_size=2, stride=2), floor mode
                ho, wo = h // 2, w // 2
                y = bufs[nxt][:2 * P * ho * wo * c_cur].view(2 * P, ho, wo, c_cur)
                self.ops.append(lambda x_=cur, y_=y, c=c_cur, h_=h, w_=w, ho_=ho, wo_=wo: _cabi.call(
                    "omt_pool2d", x_, c, c, 2 * P, h_, w_, 2, 2, 2, 2, 0, 0, ho_, wo_, y_, c, POOL_MAX))
                cur, h, w, nxt = y, ho, wo, 1 - nxt
            for u in units:                           # 3 x 3, padding 1, ReLU
                y = bufs[nxt][:2 * P * h * w * u.cout].view(2 * P, h, w, u.cout)
                self.ops.append(u.launch(cur, 2 * P, (1, h, w), (0, 1, 1), (1, h, w), y))
                cur, c_cur, nxt = y, u.cout, 1 - nxt
            last = s == len(lpips.units) - 1
            self.ops.append(lambda x_=cur, c=c_cur, h_=h, w_=w, k=s, tot=(self.lp if last else None): _cabi.call(
                "omt_lpips_head", x_, c, c, P, h_, w_, lpips.lin[k], k, self.lp_taps, tot))

    def run(self):
        for op in self.ops:
            op()


_PLAIN_WS: Dict[tuple, _Workspace] = {}


def chunk_pairs(P: int, H: int, W: int, with_lpips: bool) -> int:
    """Frame pairs per launch sequence: with LPIPS, as many as keep the first layer's 2 P H W rows within LPIPS_ROWS."""
    if not with_lpips:
        return min(P, PLAIN_CHUNK)
    return max(1, min(P, LPIPS_ROWS // (2 * H * W)))


def check_pair(a: torch.Tensor, b: torch.Tensor, dtype, what: str):
    """The refusals of every metric entry point, before any launch."""
    for name, t in (("first", a), ("second", b)):
        if not isinstance(t, torch.Tensor) or t.dtype != dtype:
            raise TypeError(f"{what}: the {name} frames must be a {dtype} tensor, got {getattr(t, 'dtype', type(t))}")
    if a.dim() != 5 or b.dim() != 5:
        raise ValueError(f"{what}: frames must have rank 5, got {tuple(a.shape)} and {tuple(b.shape)}")
    if a.shape != b.shape:
        raise ValueError(f"{what}: the two sides differ in shape: {tuple(a.shape)} and {tuple(b.shape)}")
    if a.device != b.device:
        raise ValueError(f"{what}: the two sides are on {a.device} and {b.device}")
    if min(a.shape[:2]) < 1:
        raise ValueError(f"{what}: empty batch {tuple(a.shape)}")


def _check_sizes(H: int, W: int, C: int, what: str, with_lpips: bool):
    if C != 3:
        raise ValueError(f"{what}: frames need 3 channels, got {C} (grayscale is not supported)")
    if H < MIN_SSIM or W < MIN_SSIM:
        raise ValueError(f"{what}: SSIM's 11 x 11 window needs H, W >= {MIN_SSIM}, got {H} x {W}")
    if with_lpips and (H < MIN_LPIPS or W < MIN_LPIPS):
        raise ValueError(f"{what}: LPIPS's four 2 x 2 pools need H, W >= {MIN_LPIPS}, got {H} x {W}")
    if with_lpips and 2 * H * W > MAX_CONV_ROWS:
        raise ValueError(f"{what}: {H} x {W} frames exceed the conv kernel's {MAX_CONV_ROWS} rows for one pair")


def _run(a: torch.Tensor, b: torch.Tensor, form: int, lpips: Optional[LPIPS], real_norm: Optional[L.U8Norm],
         sel: Optional[torch.Tensor]):
    """a, b: (P, H, W, 3) on the device.  Returns sse (P,) fp64, ssim (P,) fp64, lpips (P,) fp32 or None."""
    P, H, W = (int(v) for v in a.shape[:3])
    dev = a.device
    sse = torch.empty(P, dtype=torch.float64, device=dev)
    ssim = torch.empty(P, dtype=torch.float64, device=dev)
    lp = torch.empty(P, dtype=torch.float32, device=dev) if lpips is not None else None
    chunk = chunk_pairs(P, H, W, lpips is not None)
    for p0 in range(0, P, chunk):
        n = min(chunk, P - p0)
        key = (dev, form, n, H, W, real_norm)
        if lpips is None:
            ws = bounded(_PLAIN_WS, 8, key, lambda: _Workspace(dev, form, n, H, W, real_norm, None))
        else:
            ws = bounded(lpips._ws, MAX_WORKSPACES, key, lambda: _Workspace(dev, form, n, H, W, real_norm, lpips))
        ws.a.copy_(a[p0:p0 + n])
        ws.b.copy_(b[p0:p0 + n])
        if ws.sel is not None:
            ws.sel.copy_(sel[p0:p0 + n])
        run_graphed(ws.graphs, dev, "quality", ws.run)
        sse[p0:p0 + n] = ws.sse
        ssim[p0:p0 + n] = ws.ssim
        if lp is not None:
            lp[p0:p0 + n] = ws.lp
    return sse, ssim, lp


@torch.no_grad()
def frame_metrics(real_u8: torch.Tensor, fake_u8: torch.Tensor, lpips: Optional[LPIPS] = None,
                  real_norm: Optional[L.U8Norm] = None):
    """Per-frame PSNR, SSIM and (with an LPIPS model) VGG LPIPS of device uint8 frames (B, T, H, W, 3) (images:
    T = 1), each byte standing for byte / 255.  real_norm: the real frames are the loader's bytes, and the metrics see
    the bytes vqgan_eval.py makes of the normalised clip, ((v + 0.5) * 255).byte() (metricnet.real_byte_table), with
    real_norm's branch picked per clip on the device.  Returns psnr (B, T) fp64, ssim (B, T) fp64 and lpips (B, T)
    fp32 or None, on the device."""
    what = "frame_metrics"
    check_pair(real_u8, fake_u8, torch.uint8, what)
    B, T, H, W, C = (int(v) for v in real_u8.shape)
    _check_sizes(H, W, C, what, lpips is not None)
    if real_norm is not None:
        real_byte_table(real_norm)                  # refuses a per-channel normalisation before any launch
    if real_u8.device.type != "cuda":
        raise ValueError(f"{what}: frames must be on a CUDA device, got {real_u8.device}")
    if lpips is not None and real_u8.device != lpips.device:
        raise ValueError(f"{what}: frames on {real_u8.device}, the LPIPS network is on {lpips.device}")
    real = real_u8.contiguous().view(B * T, H, W, 3)
    fake = fake_u8.contiguous().view(B * T, H, W, 3)
    sel = None
    if real_norm is not None and real_norm.max_test:
        sel_clip = torch.empty(B, dtype=torch.int32, device=real.device)
        _cabi.call("omt_u8_norm_select", real, B, T * H * W * 3, sel_clip)
        sel = sel_clip.repeat_interleave(T)
    sse, ssim, lp = _run(real, fake, FORM_U8, lpips, real_norm, sel)
    psnr = psnr_from_sse(sse, 3 * H * W)
    return psnr.view(B, T), ssim.view(B, T), (lp.view(B, T) if lp is not None else None)


# ------------------------------------------------------------------------------------------------ drop-ins
def _videos_f32(videos1, videos2, what: str, with_lpips: bool, device=None):
    """(B, T, C, H, W) floats on the host or the device -> (B T, H, W, 3) fp32 on the device, both sides."""
    v1, v2 = (torch.as_tensor(v) for v in (videos1, videos2))
    for name, t in (("first", v1), ("second", v2)):
        if not t.is_floating_point():
            raise TypeError(f"{what}: the {name} videos must be floating point in [0, 1], got {t.dtype}")
    if v1.dim() != 5 or v2.dim() != 5:
        raise ValueError(f"{what}: videos must be (B, T, C, H, W), got {tuple(v1.shape)} and {tuple(v2.shape)}")
    if v1.shape != v2.shape:
        raise ValueError(f"{what}: the two sides differ in shape: {tuple(v1.shape)} and {tuple(v2.shape)}")
    B, T, C, H, W = (int(v) for v in v1.shape)
    if min(B, T) < 1:
        raise ValueError(f"{what}: empty batch {tuple(v1.shape)}")
    _check_sizes(H, W, C, what, with_lpips)
    if device is None:
        device = resolve_device(v1.device if v1.device.type == "cuda" else "cuda")
    out = [t.to(device=device, dtype=torch.float32).permute(0, 1, 3, 4, 2).reshape(B * T, H, W, 3).contiguous()
           for t in (v1, v2)]
    return out[0], out[1], (B, T), v1[0].shape


def result_dict(per_frame, video_setting) -> dict:
    """The suite's result dict of per-frame values (B, T): np.mean / np.std over the videos at each timestep."""
    r = np.asarray(per_frame, dtype=np.float64)
    return {
        "value": {t: np.mean(r[:, t]) for t in range(r.shape[1])},
        "value_std": {t: np.std(r[:, t]) for t in range(r.shape[1])},
        "video_setting": video_setting,
        "video_setting_name": "time, channel, heigth, width",
    }


@torch.no_grad()
def _psnr_ssim_f32(videos1, videos2, what):
    a, b, (B, T), setting = _videos_f32(videos1, videos2, what, False)
    sse, ssim, _ = _run(a, b, FORM_F32, None, None, None)
    return psnr_from_sse(sse, 3 * a.shape[1] * a.shape[2]).view(B, T), ssim.view(B, T), setting


def calculate_psnr(videos1, videos2) -> dict:
    """calculate_psnr.py's calculate_psnr: videos (B, T, C, H, W) in [0, 1], torch on the host or the device (taken as
    fp32).  The squared differences are summed in fp64."""
    psnr, _, setting = _psnr_ssim_f32(videos1, videos2, "calculate_psnr")
    return result_dict(psnr.cpu().numpy(), setting)


def calculate_ssim(videos1, videos2) -> dict:
    """calculate_ssim.py's calculate_ssim: videos (B, T, 3, H, W) in [0, 1], torch on the host or the device (taken as
    fp32), H, W >= 11."""
    _, ssim, setting = _psnr_ssim_f32(videos1, videos2, "calculate_ssim")
    return result_dict(ssim.cpu().numpy(), setting)


@torch.no_grad()
def calculate_lpips_vgg(videos1, videos2, model: LPIPS) -> dict:
    """calculate_lpips.py's loop and result dict with the tokenizer's VGG LPIPS (lpips.py) as the model: videos
    (B, T, 3, H, W) in [0, 1] (taken as fp32), trans's x * 2 - 1 then the network, one value per frame.  Not named
    calculate_lpips: the suite's function of that name means the lpips package's AlexNet with spatial=True."""
    if not isinstance(model, LPIPS):
        raise TypeError(f"calculate_lpips_vgg takes a quality.LPIPS model, got {type(model)}")
    a, b, (B, T), setting = _videos_f32(videos1, videos2, "calculate_lpips_vgg", True, model.device)
    _, _, lp = _run(a, b, FORM_F32, model, None, None)
    return result_dict(lp.view(B, T).cpu().numpy(), setting)


# ------------------------------------------------------------------------------------------------ AlexNet LPIPS
class AlexConv(NamedTuple):
    """One conv of torchvision's alexnet().features as the lpips package slices it (slice k = the conv and its ReLU,
    tap k): index, slice, widths, square kernel, stride, padding, and whether MaxPool2d(3, 2) precedes it."""
    idx: int
    slice: int
    cin: int
    cout: int
    k: int
    stride: int
    pad: int
    pool: bool


# lpips/pretrained_networks.py alexnet: slice1 = features[0:2], slice2 = [2:5], slice3 = [5:8], slice4 = [8:10],
# slice5 = [10:12]; the taps are relu1 ... relu5
ALEX = [AlexConv(0, 1, 3, 64, 11, 4, 2, False), AlexConv(3, 2, 64, 192, 5, 1, 2, True),
        AlexConv(6, 3, 192, 384, 3, 1, 1, True), AlexConv(8, 4, 384, 256, 3, 1, 1, False),
        AlexConv(10, 5, 256, 256, 3, 1, 1, False)]
ALEX_CHNS = tuple(c.cout for c in ALEX)
ALEX_POOL = (3, 2)                 # MaxPool2d(kernel_size=3, stride=2), floor mode
MIN_ALEX = 31                      # at 30 the second pool gets a 2 x 2 map


def alex_tap_sizes(H: int, W: int) -> List[Tuple[int, int]]:
    """(h, w) of relu1 ... relu5 of an H x W frame: conv1 (H + 4 - 11) // 4 + 1, each pool (n - 3) // 2 + 1, the 3 x 3
    pad-1 convs keep their size.  Raises ValueError where a pool would get less than its window."""
    sizes, h, w = [], H, W
    for c in ALEX:
        if c.pool:
            if min(h, w) < ALEX_POOL[0]:
                raise ValueError(f"AlexNet LPIPS: a {H} x {W} frame leaves a {h} x {w} map for a 3 x 3 pool; H, W >= "
                                 f"{MIN_ALEX}")
            h, w = (h - ALEX_POOL[0]) // ALEX_POOL[1] + 1, (w - ALEX_POOL[0]) // ALEX_POOL[1] + 1
        h, w = (h + 2 * c.pad - c.k) // c.stride + 1, (w + 2 * c.pad - c.k) // c.stride + 1
        if min(h, w) < 1:
            raise ValueError(f"AlexNet LPIPS: a {H} x {W} frame is smaller than conv1's 11 x 11 window")
        sizes.append((h, w))
    return sizes


def alex_expected_keys() -> Dict[str, tuple]:
    """The keys of the lpips package's LPIPS(net='alex') state_dict."""
    keys = {}
    for c in ALEX:
        keys[f"net.slice{c.slice}.{c.idx}.weight"] = (c.cout, c.cin, c.k, c.k)
        keys[f"net.slice{c.slice}.{c.idx}.bias"] = (c.cout,)
    for k, ch in enumerate(ALEX_CHNS):
        keys[f"lin{k}.model.1.weight"] = (1, ch, 1, 1)
    keys["scaling_layer.shift"] = (1, 3, 1, 1)
    keys["scaling_layer.scale"] = (1, 3, 1, 1)
    return keys


def alex_state_dict(state_dict: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """The lpips AlexNet keys of either layout: the lpips module's own state_dict, or torchvision alexnet's
    `features.{0,3,6,8,10}.*` plus the lpips lin file's `lin{k}.model.1.weight` (`classifier.*` ignored).  Without
    `scaling_layer.*`, ScalingLayer's constructor values."""
    sd = {}
    where = {c.idx: c.slice for c in ALEX}
    for k, v in state_dict.items():
        if k.startswith("classifier."):
            continue
        if k.startswith("features."):
            idx, rest = k[len("features."):].split(".", 1)
            if not idx.isdigit() or int(idx) not in where:
                raise KeyError(f"AlexNet LPIPS state_dict: unexpected torchvision key {k}")
            k = f"net.slice{where[int(idx)]}.{idx}.{rest}"
        sd[k] = v
    sd.setdefault("scaling_layer.shift", torch.tensor(SHIFT).view(1, 3, 1, 1))
    sd.setdefault("scaling_layer.scale", torch.tensor(SCALE).view(1, 3, 1, 1))
    return sd


class AlexLPIPS:
    """The lpips package's LPIPS(net='alex', spatial=True) (v0.1: ScalingLayer, torchvision's AlexNet trunk, five lin
    layers, each tap's map upsampled to the frame and the maps summed) in eval mode, from a state_dict (see
    alex_state_dict for the accepted layouts).  A missing or mis-shaped key is named in the error.  The convs are packed
    once, on `device`.  Only the configuration calculate_lpips.py builds exists: any other net or spatial raises
    NotImplementedError."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device="cuda", net: str = "alex", spatial: bool = True):
        if net != "alex":
            raise NotImplementedError(f"AlexLPIPS: net {net!r} is not built; only net='alex' (the suite's "
                                      f"calculate_lpips) is, and quality.LPIPS is the tokenizer's VGG LPIPS")
        if spatial is not True:
            raise NotImplementedError(f"AlexLPIPS: spatial={spatial!r} is not built; only spatial=True (the suite's "
                                      f"calculate_lpips) is")
        sd = alex_state_dict(state_dict)
        check_state_dict(sd, alex_expected_keys(), "AlexNet LPIPS")
        self.device = resolve_device(device)
        sd = {k: v.detach().float().cpu() for k, v in sd.items()}
        self.convs = [PackedConv(sd[f"net.slice{c.slice}.{c.idx}.weight"], sd[f"net.slice{c.slice}.{c.idx}.bias"],
                                 self.device, c, (1, c.stride, c.stride)) for c in ALEX]
        self.lin = [sd[f"lin{k}.model.1.weight"].reshape(-1).contiguous().to(self.device) for k in range(len(ALEX))]
        self.shift, self.scale = sd["scaling_layer.shift"].reshape(3), sd["scaling_layer.scale"].reshape(3)
        self.shift_scale = torch.cat([self.shift, self.scale]).to(self.device)
        self._ws = {}


def load_lpips_alex(device, alexnet_path: str, lin_path: str) -> AlexLPIPS:
    """AlexLPIPS from the two files lpips.LPIPS(net='alex') reads: torchvision's alexnet-owt-7be5be79.pth and the lpips
    package's weights/v0.1/alex.pth.  Not shipped; nothing is downloaded."""
    sd = dict(torch.load(alexnet_path, map_location="cpu", weights_only=True))
    sd.update(torch.load(lin_path, map_location="cpu", weights_only=True))
    return AlexLPIPS(sd, device)


class _AlexWorkspace:
    """Buffers, launch list and CUDA graph state of one (form, P, H, W): the network input, the trunk on two ping-pong
    activation buffers with each tap's map written right after its conv, then the upsampled sum and its per-pair mean."""

    def __init__(self, device, form: int, P: int, H: int, W: int, model: AlexLPIPS):
        self.graphs = {}
        f = dict(device=device, dtype=torch.float32)
        dt = torch.uint8 if form == FORM_U8 else torch.float32
        self.a = torch.empty(P, H, W, 3, dtype=dt, device=device)
        self.b = torch.empty(P, H, W, 3, dtype=dt, device=device)
        self.mean = torch.zeros(P, **f)
        sizes = alex_tap_sizes(H, W)
        self.maps = [torch.zeros(P, h, w, **f) for h, w in sizes]
        x = torch.zeros(2 * P, H, W, 4, **f)
        big, prev = 0, (H, W)
        for c, (h, w) in zip(ALEX, sizes):
            big = max(big, h * w * c.cout, prev[0] * prev[1] * c.cin if c.pool else 0)
            prev = (h, w)
        bufs = [torch.zeros(2 * P * big, **f), torch.zeros(2 * P * big, **f)]
        half = P * H * W * 4
        self.ops = []
        if form == FORM_U8:
            tab = input_table(model.shift, model.scale).to(device)
            self.ops.append(lambda: _cabi.call("omt_lpips_input", self.a, tab, None, None, form, P, H, W, x))
            self.ops.append(lambda: _cabi.call("omt_lpips_input", self.b, tab, None, None, form, P, H, W,
                                               x.data_ptr() + 4 * half))
        else:
            ss = model.shift_scale
            self.ops.append(lambda: _cabi.call("omt_lpips_input", self.a, None, None, ss, form, P, H, W, x))
            self.ops.append(lambda: _cabi.call("omt_lpips_input", self.b, None, None, ss, form, P, H, W,
                                               x.data_ptr() + 4 * half))
        pk, ps = ALEX_POOL
        cur, c_cur, h, w, nxt = x, 4, H, W, 0
        for k, (u, (ho, wo)) in enumerate(zip(model.convs, sizes)):
            c = u.conv
            if c.pool:
                ph, pw = (h - pk) // ps + 1, (w - pk) // ps + 1
                y = bufs[nxt][:2 * P * ph * pw * c_cur].view(2 * P, ph, pw, c_cur)
                self.ops.append(lambda x_=cur, y_=y, cc=c_cur, h_=h, w_=w, ph_=ph, pw_=pw: _cabi.call(
                    "omt_pool2d", x_, cc, cc, 2 * P, h_, w_, pk, pk, ps, ps, 0, 0, ph_, pw_, y_, cc, POOL_MAX))
                cur, h, w, nxt = y, ph, pw, 1 - nxt
            y = bufs[nxt][:2 * P * ho * wo * c.cout].view(2 * P, ho, wo, c.cout)
            self.ops.append(u.launch(cur, 2 * P, (1, h, w), (0, c.pad, c.pad), (1, ho, wo), y))
            cur, c_cur, h, w, nxt = y, c.cout, ho, wo, 1 - nxt
            self.ops.append(lambda x_=cur, cc=c_cur, h_=h, w_=w, k_=k: _cabi.call(
                "omt_lpips_map", x_, cc, cc, P, h_, w_, model.lin[k_], self.maps[k_]))
        taps = _cabi.lpips_taps([(m, m.shape[1], m.shape[2]) for m in self.maps])
        self.ops.append(lambda: _cabi.call("omt_lpips_upsample_mean", taps, len(ALEX), P, H, W, None, self.mean))

    def run(self):
        for op in self.ops:
            op()


def _alex_side(v, name: str):
    """One side of calculate_lpips -> its form, with the dtype and rank refusals."""
    if not isinstance(v, torch.Tensor):
        raise TypeError(f"calculate_lpips: {name} must be a torch tensor, got {type(v)}")
    if v.dtype == torch.uint8:
        if v.dim() != 5 or v.shape[-1] != 3:
            raise ValueError(f"calculate_lpips: uint8 {name} must be (B, T, H, W, 3), got {tuple(v.shape)}")
        return FORM_U8
    if v.dtype == torch.float32:
        if v.dim() != 5 or v.shape[2] not in (1, 3):
            raise ValueError(f"calculate_lpips: fp32 {name} must be (B, T, C, H, W) with C 1 or 3, got "
                             f"{tuple(v.shape)}")
        return FORM_F32
    raise TypeError(f"calculate_lpips: {name} must be fp32 (B, T, C, H, W) in [0, 1] or uint8 (B, T, H, W, 3), got "
                    f"{v.dtype}")


@torch.no_grad()
def lpips_alex_frames(videos1, videos2, device, model: AlexLPIPS) -> torch.Tensor:
    """calculate_lpips's per-frame values, (B, T) fp32 on the device, with its refusals (see calculate_lpips)."""
    if not isinstance(model, AlexLPIPS):
        raise TypeError(f"calculate_lpips needs the AlexNet LPIPS as model= (quality.load_lpips_alex), got "
                        f"{type(model)}")
    forms = [_alex_side(v, n) for v, n in ((videos1, "videos1"), (videos2, "videos2"))]
    if forms[0] != forms[1]:
        raise TypeError(f"calculate_lpips: videos1 is {videos1.dtype}, videos2 {videos2.dtype}")
    if videos1.shape != videos2.shape:
        raise ValueError(f"calculate_lpips: the two sides differ in shape: {tuple(videos1.shape)} and "
                         f"{tuple(videos2.shape)}")
    form = forms[0]
    if form == FORM_U8:
        B, T, H, W, C = (int(v) for v in videos1.shape)
    else:
        B, T, C, H, W = (int(v) for v in videos1.shape)
    if min(B, T) < 1:
        raise ValueError(f"calculate_lpips: empty batch {tuple(videos1.shape)}")
    if H < MIN_ALEX or W < MIN_ALEX:
        raise ValueError(f"calculate_lpips: AlexNet's pools need H, W >= {MIN_ALEX}, got {H} x {W}")
    if 2 * H * W > MAX_CONV_ROWS:
        raise ValueError(f"calculate_lpips: {H} x {W} frames exceed the conv kernel's {MAX_CONV_ROWS} rows for one pair")
    if torch.device(device).type != "cuda":
        raise ValueError(f"calculate_lpips runs on a CUDA device, got {device}")
    dev = resolve_device(device)
    if dev != model.device:
        raise ValueError(f"calculate_lpips: device {dev}, the AlexNet LPIPS network is on {model.device}")
    P = B * T
    if form == FORM_U8:
        a, b = (v.to(dev).contiguous().view(P, H, W, 3) for v in (videos1, videos2))
    else:
        a, b = (v.to(dev).permute(0, 1, 3, 4, 2).reshape(P, H, W, C).expand(P, H, W, 3).contiguous()
                for v in (videos1, videos2))
    out = torch.empty(P, dtype=torch.float32, device=dev)
    chunk = chunk_pairs(P, H, W, True)
    for p0 in range(0, P, chunk):
        n = min(chunk, P - p0)
        ws = bounded(model._ws, MAX_WORKSPACES, (dev, form, n, H, W),
                     lambda: _AlexWorkspace(dev, form, n, H, W, model))
        ws.a.copy_(a[p0:p0 + n])
        ws.b.copy_(b[p0:p0 + n])
        run_graphed(ws.graphs, dev, "lpips_alex", ws.run)
        out[p0:p0 + n] = ws.mean
    return out.view(B, T)


def calculate_lpips(videos1, videos2, device="cuda", model: Optional[AlexLPIPS] = None) -> dict:
    """calculate_lpips.py's calculate_lpips: per frame, the mean of the lpips package's AlexNet LPIPS map
    (model = load_lpips_alex(...)), and the suite's result dict.  videos: fp32 (B, T, C, H, W) in [0, 1] (C 1 or 3; host
    or device) or uint8 (B, T, H, W, 3) standing for byte / 255 (frames on the device stay there); both sides of one
    shape and dtype, H, W >= 31.  uint8 frames and fp32 frames of byte / 255 give the same bits, as do grey frames and
    the same frames repeated to 3 channels.  The frames run in chunks; the values do not depend on the chunking."""
    per = lpips_alex_frames(videos1, videos2, device, model)
    H, W = (videos1.shape[2:4] if videos1.dtype == torch.uint8 else videos1.shape[3:5])
    return result_dict(per.cpu().numpy(), torch.Size([per.shape[1], 3, int(H), int(W)]))


# ------------------------------------------------------------------------------------------------ calculate_fvd
FVD_METHODS = ("styleganv", "videogpt")
FVD_MIN_FRAMES = 10                # calculate_fvd.py:43: the first prefix length


def sqrtm_disp(a: np.ndarray, disp: bool = False):
    """scipy.linalg.sqrtm(a, disp=False) -> (root, error estimate) on every scipy: from 1.16 sqrtm takes no disp and
    returns the root alone (the estimate is then None)."""
    from scipy.linalg import sqrtm
    try:
        return sqrtm(a, disp=False)
    except TypeError:
        return sqrtm(a), None


def frechet_distance_styleganv(feats_fake: np.ndarray, feats_real: np.ndarray) -> float:
    """fvd/styleganv/fvd.py:75-90: numpy means and np.cov, scipy.linalg.sqrtm of the product, the real part; the mean
    term alone for one clip per side."""
    mu_gen, sigma_gen = feats_fake.mean(axis=0), np.cov(feats_fake, rowvar=False)
    mu_real, sigma_real = feats_real.mean(axis=0), np.cov(feats_real, rowvar=False)
    m = np.square(mu_gen - mu_real).sum()
    if feats_fake.shape[0] > 1:
        s, _ = sqrtm_disp(np.dot(sigma_gen, sigma_real))
        return float(np.real(m + np.trace(sigma_gen + sigma_real - s * 2)))
    return float(np.real(m))


def frechet_distance_videogpt(x1: torch.Tensor, x2: torch.Tensor) -> float:
    """fvd/videogpt/fvd.py:113-125: OmniTokenizer/fvd's torch distance (fvd.frechet_distance), with the mean term
    alone for one clip per side."""
    if x1.shape[0] > 1:
        return float(fvd_frechet_distance(x1, x2))
    return float(torch.sum((x1.flatten(start_dim=1).mean(dim=0) - x2.flatten(start_dim=1).mean(dim=0)) ** 2))


def _fvd_side(v, name: str):
    """One side of calculate_fvd -> SuiteClips on the device (uploaded once), with the refusals."""
    if not isinstance(v, torch.Tensor):
        raise TypeError(f"calculate_fvd: {name} must be a torch tensor, got {type(v)}")
    if v.dtype == torch.uint8:
        if v.dim() != 5 or v.shape[-1] != 3:
            raise ValueError(f"calculate_fvd: uint8 {name} must be (B, T, H, W, 3), got {tuple(v.shape)}")
        form = FORM_FVD_U8
    elif v.dtype == torch.float32:
        if v.dim() != 5 or v.shape[2] not in (1, 3):
            raise ValueError(f"calculate_fvd: fp32 {name} must be (B, T, C, H, W) with C 1 or 3, got {tuple(v.shape)}")
        form = FORM_FVD_F32
    else:
        raise TypeError(f"calculate_fvd: {name} must be fp32 (B, T, C, H, W) in [0, 1] or uint8 (B, T, H, W, 3), "
                        f"got {v.dtype}")
    if min(v.shape) < 1:
        raise ValueError(f"calculate_fvd: empty {name} {tuple(v.shape)}")
    return v, form


def _video_setting(v: torch.Tensor, form: int) -> torch.Size:
    """calculate_fvd.trans's shape: (B, 3, T, H, W) (grey repeated to 3 channels)."""
    if form == FORM_FVD_U8:
        B, T, H, W, _ = v.shape
    else:
        B, T, _, H, W = v.shape
    return torch.Size([B, 3, T, H, W])


@torch.no_grad()
def calculate_fvd(videos1, videos2, device="cuda", method: str = "styleganv", i3d=None) -> dict:
    """calculate_fvd.py's calculate_fvd: the FVD between the first t frames of videos1 and of videos2 for every
    t = 10 ... T (T: videos1's length; T < 10 gives an empty value and runs no network), with the suite's result dict.
    videos: fp32 (B, T, C, H, W) in [0, 1] (C 1 or 3; host or device) or uint8 (B, T, H, W, 3) standing for byte / 255;
    the two sides may differ in B and in H x W, and videos2 needs at least T frames.  uint8 clips and fp32 clips of
    byte / 255 give the same features.
    method: "styleganv" with i3d = fvd.load_i3d_styleganv(...), or "videogpt" (fvd_external.py's) with
    i3d = fvd.load_fvd_model(device, "i3d_pretrained_400.pt").  videogpt rounds fp32 clips to bytes first, as its
    preprocess does.  The features come to the host as float64 and the distance is the method's own host code."""
    if method not in FVD_METHODS:
        raise ValueError(f"calculate_fvd: unknown method {method!r}; expected one of {FVD_METHODS}")
    if not isinstance(i3d, I3D):
        raise TypeError(f"calculate_fvd needs the method's network as i3d= (fvd.load_i3d_styleganv or "
                        f"fvd.load_fvd_model), got {type(i3d)}")
    if i3d.variant != method:
        raise ValueError(f"calculate_fvd: method {method!r} with the {i3d.variant} network")
    if torch.device(device).type != "cuda":
        raise ValueError(f"calculate_fvd runs on a CUDA device, got {device}")
    sides = [_fvd_side(v, n) for v, n in ((videos1, "videos1"), (videos2, "videos2"))]
    T1, T2 = int(sides[0][0].shape[1]), int(sides[1][0].shape[1])
    if T2 < T1:
        raise ValueError(f"calculate_fvd: videos2 has {T2} frames, fewer than videos1's {T1}")
    result = {"value": {}, "video_setting": _video_setting(*sides[0]),
              "video_setting_name": "batch_size, channel, time, heigth, width"}
    if T1 < FVD_MIN_FRAMES:
        return result
    clips = []
    for v, form in sides:
        if form == FORM_FVD_F32 and method == "videogpt":
            form = FORM_FVD_F32_TRUNC
        clips.append(SuiteClips(v.to(i3d.device).contiguous(), form))
    for t in range(FVD_MIN_FRAMES, T1 + 1):
        f1, f2 = (i3d.features(c, t).double().cpu() for c in clips)
        if method == "styleganv":
            result["value"][t] = frechet_distance_styleganv(f1.numpy(), f2.numpy())
        else:
            result["value"][t] = frechet_distance_videogpt(f1, f2)
    return result
