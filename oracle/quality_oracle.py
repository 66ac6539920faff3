"""CPU restatement of the per-frame reconstruction metrics, written from their spec.  TEST INFRASTRUCTURE ONLY: the
product never imports it.

- psnr: calculate_psnr.py img_psnr, mse in float64, 100 below 1e-10.
- ssim: calculate_ssim.py ssim / calculate_ssim_function for 3 channels, in numpy float64 with the separable filter
  (the 11 taps along w, then along h), the valid (H - 10) x (W - 10) crop, C1 = 0.01^2, C2 = 0.03^2.
- lpips: OmniTokenizer/modules/lpips.py's LPIPS (VGG16 features[0:30] in five slices, normalize_tensor, the squared
  difference, NetLinLayer's 1x1 conv without bias, spatial_average, the taps summed in order) in torch fp32, after
  calculate_lpips.py's x * 2 - 1 and ScalingLayer.

The keyword arguments break one wiring each; tests use them to show the fixture detects it.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

CHNS = (64, 128, 256, 512, 512)
# features index of every conv per slice (torchvision vgg16: conv, ReLU pairs; a MaxPool2d(2, 2) opens slices 2-5)
VGG_SLICES: List[List[Tuple[int, int, int]]] = [
    [(0, 3, 64), (2, 64, 64)],
    [(5, 64, 128), (7, 128, 128)],
    [(10, 128, 256), (12, 256, 256), (14, 256, 256)],
    [(17, 256, 512), (19, 512, 512), (21, 512, 512)],
    [(24, 512, 512), (26, 512, 512), (28, 512, 512)],
]
SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)


def gaussian(n: int = 11, sigma: float = 1.5) -> np.ndarray:
    t = np.array([math.exp(-0.5 / (sigma * sigma) * (i - (n - 1) * 0.5) ** 2) for i in range(n)])
    return t * (1.0 / t.sum())


def psnr(a: np.ndarray, b: np.ndarray) -> float:
    mse = float(np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2))
    return 100.0 if mse < 1e-10 else 20 * math.log10(1 / math.sqrt(mse))


def _filter(x: np.ndarray, k: np.ndarray) -> np.ndarray:
    """Valid separable correlation of a 2-D float64 map: along w, then along h, taps added in order."""
    n = len(k)
    Ho, Wo = x.shape[0] - n + 1, x.shape[1] - n + 1
    h = np.zeros((x.shape[0], Wo))
    for j in range(n):
        h = h + k[j] * x[:, j:j + Wo]
    v = np.zeros((Ho, Wo))
    for j in range(n):
        v = v + k[j] * h[j:j + Ho, :]
    return v


def ssim_channel(x: np.ndarray, y: np.ndarray, taps: np.ndarray, same: bool = False) -> float:
    """same=True: the full-size map of cv2.filter2D's default border (reflect 101) instead of the valid crop."""
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    x, y = x.astype(np.float64), y.astype(np.float64)
    if same:
        r = len(taps) // 2
        x, y = np.pad(x, r, mode="reflect"), np.pad(y, r, mode="reflect")
    mu1, mu2 = _filter(x, taps), _filter(y, taps)
    mu1_sq, mu2_sq, mu1_mu2 = mu1 ** 2, mu2 ** 2, mu1 * mu2
    s1 = _filter(x * x, taps) - mu1_sq
    s2 = _filter(y * y, taps) - mu2_sq
    s12 = _filter(x * y, taps) - mu1_mu2
    m = ((2 * mu1_mu2 + C1) * (2 * s12 + C2)) / ((mu1_sq + mu2_sq + C1) * (s1 + s2 + C2))
    return float(m.mean())


def ssim(a: np.ndarray, b: np.ndarray, taps: Optional[np.ndarray] = None, same: bool = False,
         sigma: float = 1.5) -> float:
    """a, b: (3, H, W) values in [0, 1]."""
    if taps is None:
        taps = gaussian(11, sigma)
    return float(np.array([ssim_channel(a[c], b[c], taps, same) for c in range(3)]).mean())


# ------------------------------------------------------------------------------------------------ LPIPS
def make_state_dict(seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded LPIPS weights in lpips.py's module layout: He-scaled uniform conv weights (bound sqrt(6 / fan_in), so
    the ReLU trunk keeps every tap O(1)), small biases, lin weights uniform in [0, 1), ScalingLayer's constants.
    torch.rand plus exact arithmetic."""
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    for s, convs in enumerate(VGG_SLICES, 1):
        for idx, cin, cout in convs:
            b = math.sqrt(6.0 / (cin * 9))
            sd[f"net.slice{s}.{idx}.weight"] = (torch.rand(cout, cin, 3, 3, generator=g) * 2 - 1) * b
            sd[f"net.slice{s}.{idx}.bias"] = (torch.rand(cout, generator=g) * 2 - 1) * 0.05
    for k, c in enumerate(CHNS):
        sd[f"lin{k}.model.1.weight"] = torch.rand(1, c, 1, 1, generator=g)
    sd["scaling_layer.shift"] = torch.tensor(SHIFT).view(1, 3, 1, 1)
    sd["scaling_layer.scale"] = torch.tensor(SCALE).view(1, 3, 1, 1)
    return sd


def fingerprint(sd) -> float:
    """Order-independent float64 checksum of the weights."""
    tot = 0.0
    for k in sorted(sd):
        v = sd[k].double().flatten()
        tot += float((v * torch.arange(1, v.numel() + 1, dtype=torch.float64) % 7.0).sum())
    return tot


def vgg_taps(sd, x: torch.Tensor, pre_relu: bool = False) -> List[torch.Tensor]:
    """relu1_2 ... relu5_3 of (N, 3, H, W); pre_relu=True: each tap taken before its ReLU."""
    taps = []
    h = x
    for s, convs in enumerate(VGG_SLICES, 1):
        if s > 1:
            h = F.max_pool2d(h, 2, 2)
        for i, (idx, _, _) in enumerate(convs):
            z = F.conv2d(h, sd[f"net.slice{s}.{idx}.weight"], sd[f"net.slice{s}.{idx}.bias"], padding=1)
            h = F.relu(z)
            if i == len(convs) - 1:
                taps.append(z if pre_relu else h)
    return taps


def lpips(sd, a01: torch.Tensor, b01: torch.Tensor, scale_01: bool = False, pre_relu: bool = False,
          eps: float = 1e-10, drop_tap: Optional[int] = None, per_tap: Optional[list] = None,
          features: Optional[list] = None) -> torch.Tensor:
    """LPIPS of (N, 3, H, W) pairs in [0, 1] -> (N,) fp32.  scale_01: ScalingLayer applied to [0, 1] instead of [-1, 1];
    drop_tap: leave one tap out of the sum; per_tap / features: filled with each tap's (N,) value / feature maps."""
    shift, scale = sd["scaling_layer.shift"], sd["scaling_layer.scale"]
    xa, xb = (t if scale_01 else t * 2 - 1 for t in (a01, b01))
    fa = vgg_taps(sd, (xa - shift) / scale, pre_relu)
    fb = vgg_taps(sd, (xb - shift) / scale, pre_relu)
    if features is not None:
        features.extend(zip(fa, fb))
    val = None
    for k in range(len(CHNS)):
        na = fa[k] / (torch.sqrt(torch.sum(fa[k] ** 2, dim=1, keepdim=True)) + eps)
        nb = fb[k] / (torch.sqrt(torch.sum(fb[k] ** 2, dim=1, keepdim=True)) + eps)
        r = F.conv2d((na - nb) ** 2, sd[f"lin{k}.model.1.weight"]).mean([2, 3], keepdim=True)
        if per_tap is not None:
            per_tap.append(r.flatten())
        if k == drop_tap:
            continue
        val = r if val is None else val + r
    return val.flatten()


def lpips_head64(fa: torch.Tensor, fb: torch.Tensor, w: torch.Tensor, eps: float = 1e-10) -> torch.Tensor:
    """One tap's head in float64: (N, C, h, w) features, lin weight (C,) -> (N,)."""
    fa, fb, w = fa.double(), fb.double(), w.double().view(1, -1, 1, 1)
    na = fa / (torch.sqrt((fa ** 2).sum(1, keepdim=True)) + eps)
    nb = fb / (torch.sqrt((fb ** 2).sum(1, keepdim=True)) + eps)
    return ((na - nb) ** 2 * w).sum(1).mean((1, 2))


# ------------------------------------------------------------------------------------------------ frames
def frame_pair(spec) -> Tuple[torch.Tensor, torch.Tensor]:
    """Seeded uint8 (H, W, 3) pair of a fixture case spec (H, W, kind, seed):
    noise: b = clamp(a + uniform noise in [-20, 20]); same: b = a; const: 200 vs 190; one / two: b = a with one / two
    bytes raised by 1."""
    H, W, kind, seed = spec
    g = torch.Generator().manual_seed(seed)
    if kind == "const":
        return (torch.full((H, W, 3), 200, dtype=torch.uint8), torch.full((H, W, 3), 190, dtype=torch.uint8))
    a = torch.randint(0, 250, (H, W, 3), generator=g, dtype=torch.uint8)
    if kind == "noise":
        n = torch.randint(-20, 21, (H, W, 3), generator=g, dtype=torch.int16)
        return a, (a.to(torch.int16) + n).clamp(0, 255).to(torch.uint8)
    b = a.clone()
    if kind == "one":
        b[H // 2, W // 3, 1] += 1
    elif kind == "two":
        b[H // 2, W // 3, 1] += 1
        b[H // 4, W // 2, 2] += 1
    return a, b


def to01(u8: torch.Tensor) -> torch.Tensor:
    """(..., H, W, 3) uint8 -> (..., 3, H, W) fp32 byte / 255."""
    return u8.float().div(255).movedim(-1, -3).contiguous()
