"""CPU restatement of the lpips package's LPIPS(net='alex', spatial=True), v0.1, written from its spec.  TEST
INFRASTRUCTURE ONLY: the product never imports it.

The package is not in the reference tree, so its forward is restated here as a small nn.Module; the trunk is the
installed torchvision's own alexnet().features, sliced as lpips/pretrained_networks.py's alexnet slices it
(slice1 = features[0:2], slice2 = [2:5], slice3 = [5:8], slice4 = [8:10], slice5 = [10:12]; taps relu1 ... relu5).
lpips/lpips.py's LPIPS.forward then takes, per tap k:
  ScalingLayer         (x - shift) / scale before the trunk;
  normalize_tensor     f / (sqrt(sum_c f^2) + eps), eps = 1e-10, both images;
  (n0 - n1) ** 2, then NetLinLayer lin_k (Dropout, a 1x1 conv without bias);
  upsample             nn.Upsample(size=in0.shape[2:], mode='bilinear', align_corners=False);
and sums val = 0; val += res[k] for k = 0 ... 4, giving an (N, 1, H, W) map.

The keyword arguments break one wiring each; tests use them to show the fixture detects it.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F
import torchvision

from oracle.quality_oracle import SCALE, SHIFT, fingerprint  # noqa: F401  (fingerprint: the same checksum)

# (features index, slice, cin, cout, kernel) of every conv; slice k ends with the conv's ReLU (tap k)
ALEX_CONVS: List[Tuple[int, int, int, int, int]] = [(0, 1, 3, 64, 11), (3, 2, 64, 192, 5), (6, 3, 192, 384, 3),
                                                    (8, 4, 384, 256, 3), (10, 5, 256, 256, 3)]
SLICE_BOUNDS = [(0, 2), (2, 5), (5, 8), (8, 10), (10, 12)]
CHNS = tuple(c[3] for c in ALEX_CONVS)


def make_state_dict(seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded weights in the lpips module's layout: He-scaled uniform conv weights (bound sqrt(6 / fan_in)), small
    biases, lin weights uniform in [0, 1), ScalingLayer's constants.  torch.rand plus exact arithmetic."""
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    for idx, s, cin, cout, k in ALEX_CONVS:
        b = math.sqrt(6.0 / (cin * k * k))
        sd[f"net.slice{s}.{idx}.weight"] = (torch.rand(cout, cin, k, k, generator=g) * 2 - 1) * b
        sd[f"net.slice{s}.{idx}.bias"] = (torch.rand(cout, generator=g) * 2 - 1) * 0.05
    for k, c in enumerate(CHNS):
        sd[f"lin{k}.model.1.weight"] = torch.rand(1, c, 1, 1, generator=g)
    sd["scaling_layer.shift"] = torch.tensor(SHIFT).view(1, 3, 1, 1)
    sd["scaling_layer.scale"] = torch.tensor(SCALE).view(1, 3, 1, 1)
    return sd


def torchvision_state_dict(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """The conv weights of sd under torchvision alexnet's `features.N.*` names."""
    return {f"features.{idx}.{f}": sd[f"net.slice{s}.{idx}.{f}"] for idx, s, _, _, _ in ALEX_CONVS
            for f in ("weight", "bias")}


class AlexLPIPSOracle(nn.Module):
    """LPIPS(net='alex', spatial=True) forward of (N, 3, H, W) images in [-1, 1] -> (N, 1, H, W).
    Wiring breaks: align_corners=True; spatial_average=True (each tap's mean instead of its upsampled map, lpips's
    spatial=False); scaling=False (ScalingLayer skipped); pre_relu=True (each tap taken before its ReLU);
    drop_tap=k (tap k left out of the sum); eps (normalize_tensor's).  record: every forward's .mean() is appended,
    as calculate_lpips.py takes it (set it to None to record nothing)."""

    def __init__(self, sd: Dict[str, torch.Tensor], align_corners: bool = False, spatial_average: bool = False,
                 scaling: bool = True, pre_relu: bool = False, drop_tap: Optional[int] = None, eps: float = 1e-10):
        super().__init__()
        self.features = torchvision.models.alexnet(weights=None).features.eval()
        self.features.load_state_dict({k[len("features."):]: v for k, v in torchvision_state_dict(sd).items()})
        self.register_buffer("shift", sd["scaling_layer.shift"].clone())
        self.register_buffer("scale", sd["scaling_layer.scale"].clone())
        for k in range(len(CHNS)):                  # buffers, so .to(device) moves them as it moves the lpips module
            self.register_buffer(f"lin{k}", sd[f"lin{k}.model.1.weight"].clone())
        self.align_corners, self.spatial_average, self.scaling = align_corners, spatial_average, scaling
        self.pre_relu, self.drop_tap, self.eps = pre_relu, drop_tap, eps
        self.record: Optional[List[float]] = []      # None: nothing recorded (no extra host sync per frame)
        self.maps: Optional[list] = None              # set to a list to collect (tap maps, spatial map) per forward

    def taps(self, x: torch.Tensor) -> List[torch.Tensor]:
        out, h = [], x
        for a, b in SLICE_BOUNDS:
            for i in range(a, b):
                if i == b - 1 and self.pre_relu:
                    out.append(h.clone())             # the conv's output; the ReLU below is in place
                h = self.features[i](h)
            if not self.pre_relu:
                out.append(h)
        return out

    def forward(self, in0: torch.Tensor, in1: torch.Tensor) -> torch.Tensor:
        if self.scaling:
            in0, in1 = (in0 - self.shift) / self.scale, (in1 - self.shift) / self.scale
        f0, f1 = self.taps(in0), self.taps(in1)
        ds, res = [], []
        for k in range(len(CHNS)):
            n0 = f0[k] / (torch.sqrt(torch.sum(f0[k] ** 2, dim=1, keepdim=True)) + self.eps)
            n1 = f1[k] / (torch.sqrt(torch.sum(f1[k] ** 2, dim=1, keepdim=True)) + self.eps)
            d = F.conv2d((n0 - n1) ** 2, getattr(self, f"lin{k}"))
            ds.append(d)
            if self.spatial_average:
                res.append(d.mean([2, 3], keepdim=True))
            else:
                res.append(F.interpolate(d, size=in0.shape[2:], mode="bilinear", align_corners=self.align_corners))
        val = 0
        for k in range(len(CHNS)):
            if k != self.drop_tap:
                val += res[k]
        if self.maps is not None:
            self.maps.append((ds, val))
        if self.record is not None:
            self.record.append(val.mean().detach().cpu().tolist())
        return val


def trans(x: torch.Tensor) -> torch.Tensor:
    """calculate_lpips.py's trans: grey repeated to 3 channels, then x * 2 - 1."""
    if x.shape[-3] == 1:
        x = x.repeat(1, 1, 3, 1, 1)
    return x * 2 - 1


def suite_loop(net: nn.Module, videos1: torch.Tensor, videos2: torch.Tensor, device) -> torch.Tensor:
    """calculate_lpips.py's per-frame loop restated: (B, T) float64 of forward(img1, img2).mean() per frame."""
    v1, v2 = trans(videos1), trans(videos2)
    out = [[net.forward(v1[b, t].unsqueeze(0).to(device), v2[b, t].unsqueeze(0).to(device)).mean().detach().cpu()
            .tolist() for t in range(v1.shape[1])] for b in range(v1.shape[0])]
    return torch.tensor(out, dtype=torch.float64)


# ------------------------------------------------------------------------------------------------ inputs
def videos(spec) -> Tuple[torch.Tensor, torch.Tensor]:
    """fp32 (B, T, C, H, W) in [0, 1] of a fixture case spec (B, T, C, H, W, kind, seed):
    zeros_ones: the demo's zeros vs ones; bytes: byte / 255 of a uint8 pair, the second the first plus uniform noise
    in [-20, 20], clamped; border: bytes as for `bytes`, with the noise only in an 8-pixel border (where the upsample
    weights a tap map's edge differently from its spatial average); float: uniform values and a clamped Gaussian
    perturbation (not bytes); same: an identical pair of byte frames."""
    B, T, C, H, W, kind, seed = spec
    shape = (B, T, C, H, W)
    if kind == "zeros_ones":
        return torch.zeros(shape), torch.ones(shape)
    g = torch.Generator().manual_seed(seed)
    if kind == "float":
        a = torch.rand(shape, generator=g)
        return a, (a + 0.1 * torch.randn(shape, generator=g)).clamp(0, 1)
    a = torch.randint(0, 256, shape, generator=g, dtype=torch.int16)
    if kind == "same":
        b = a
    else:
        assert kind in ("bytes", "border"), kind
        n = torch.randint(-20, 21, shape, generator=g, dtype=torch.int16)
        if kind == "border":
            n[..., 8:-8, 8:-8] = 0
        b = (a + n).clamp(0, 255)
    return a.to(torch.uint8).float() / 255, b.to(torch.uint8).float() / 255


def to_u8(v: torch.Tensor) -> torch.Tensor:
    """(B, T, 3, H, W) byte / 255 values -> the uint8 (B, T, H, W, 3) frames they stand for."""
    u = (v * 255).round()
    assert torch.equal(u / 255, v), "not byte / 255 values"
    return u.to(torch.uint8).movedim(2, -1).contiguous()
