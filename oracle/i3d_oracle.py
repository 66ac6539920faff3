"""CPU fp32 restatement of the FVD metric's feature network and distance (OmniTokenizer/fvd/pytorch_i3d.py,
OmniTokenizer/fvd/fvd.py), written from their spec.  TEST INFRASTRUCTURE ONLY: the product never imports it.

- preprocess: fvd.py:18-29 -- bytes -> fp32, bilinear F.interpolate to 224 x 224 (align_corners=False), 2 y / 255 - 1.
- Unit3D: pytorch_i3d.py:59-131 -- TF-style SAME padding (compute_pad, pad // 2 in front, the rest behind), conv3d
  without bias, BatchNorm3d (eps 1e-5, running statistics), ReLU.  The logits unit has a bias, no BN and no ReLU.
- MaxPool3dSamePadding: pytorch_i3d.py:24-56 -- the same padding with F.pad's zeros, then max_pool3d.
- InceptionModule: pytorch_i3d.py:135-160 -- branches b0 | b1a->b1b | b2a->b2b | b3a->b3b concatenated on channels.
- InceptionI3d.forward: pytorch_i3d.py:355-365 -- the endpoints in order, AvgPool3d([2, 7, 7], stride 1), the logits
  unit, squeeze, mean over time.
- frechet_distance: fvd.py:55-112 -- torch.svd square roots, unbiased covariances.

The keyword arguments of `forward` / `preprocess` break one wiring each; tests use them to show the fixture detects it.
"""
from __future__ import annotations

import math
from typing import Dict, List, Tuple

import numpy as np
import torch
import torch.nn.functional as F

# (name, kind, spec): "unit" (cin, cout, kernel, stride), "pool" (kernel, stride), "mixed" (cin, 6 widths)
ARCH: List[Tuple[str, str, tuple]] = [
    ("Conv3d_1a_7x7", "unit", (3, 64, (7, 7, 7), (2, 2, 2))),
    ("MaxPool3d_2a_3x3", "pool", ((1, 3, 3), (1, 2, 2))),
    ("Conv3d_2b_1x1", "unit", (64, 64, (1, 1, 1), (1, 1, 1))),
    ("Conv3d_2c_3x3", "unit", (64, 192, (3, 3, 3), (1, 1, 1))),
    ("MaxPool3d_3a_3x3", "pool", ((1, 3, 3), (1, 2, 2))),
    ("Mixed_3b", "mixed", (192, (64, 96, 128, 16, 32, 32))),
    ("Mixed_3c", "mixed", (256, (128, 128, 192, 32, 96, 64))),
    ("MaxPool3d_4a_3x3", "pool", ((3, 3, 3), (2, 2, 2))),
    ("Mixed_4b", "mixed", (480, (192, 96, 208, 16, 48, 64))),
    ("Mixed_4c", "mixed", (512, (160, 112, 224, 24, 64, 64))),
    ("Mixed_4d", "mixed", (512, (128, 128, 256, 24, 64, 64))),
    ("Mixed_4e", "mixed", (512, (112, 144, 288, 32, 64, 64))),
    ("Mixed_4f", "mixed", (528, (256, 160, 320, 32, 128, 128))),
    ("MaxPool3d_5a_2x2", "pool", ((2, 2, 2), (2, 2, 2))),
    ("Mixed_5b", "mixed", (832, (256, 160, 320, 32, 128, 128))),
    ("Mixed_5c", "mixed", (832, (384, 192, 384, 48, 128, 128))),
]
# Inception branch units: name, input ("x" or another unit), width index, kernel
BRANCHES = [("b0", 0, 1), ("b1a", 1, 1), ("b1b", 2, 3), ("b2a", 3, 1), ("b2b", 4, 3), ("b3b", 5, 1)]


def units() -> List[Tuple[str, int, int, tuple, tuple]]:
    """Every Unit3D with BatchNorm: (prefix, cin, cout, kernel, stride)."""
    out = []
    for name, kind, spec in ARCH:
        if kind == "unit":
            out.append((name, spec[0], spec[1], spec[2], spec[3]))
        elif kind == "mixed":
            cin, w = spec
            ins = {"b0": cin, "b1a": cin, "b1b": w[1], "b2a": cin, "b2b": w[3], "b3b": cin}
            for b, wi, k in BRANCHES:
                out.append((f"{name}.{b}", ins[b], w[wi], (k, k, k), (1, 1, 1)))
    return out


def compute_pad(k: int, s: int, n: int) -> int:
    """pytorch_i3d.py:26-30 / 93-97."""
    return max(k - s, 0) if n % s == 0 else max(k - n % s, 0)


def same_pad(kernel, stride, dims, symmetric=False) -> Tuple[int, ...]:
    """F.pad's (w_f, w_b, h_f, h_b, t_f, t_b); symmetric=True is the broken k // 2 wiring."""
    pads = []
    for k, s, n in zip(kernel[::-1], stride[::-1], dims[::-1]):
        if symmetric:
            pads += [k // 2, k // 2]
        else:
            p = compute_pad(k, s, n)
            pads += [p // 2, p - p // 2]
    return tuple(pads)


def preprocess(videos, size=(224, 224), norm_first=False) -> torch.Tensor:
    """fvd.py:18-29: (b, t, h, w, c) uint8 -> (b, c, t, 224, 224) fp32 in [-1, 1].  norm_first: the broken order."""
    v = torch.as_tensor(np.asarray(videos))
    b, t, h, w, c = v.shape
    x = v.float().flatten(end_dim=1).permute(0, 3, 1, 2).contiguous()
    if norm_first:
        x = 2. * x / 255. - 1
    x = F.interpolate(x, size=size, mode="bilinear", align_corners=False)
    x = x.view(b, t, c, *size).transpose(1, 2).contiguous()
    return x if norm_first else 2. * x / 255. - 1


def unit3d(x, sd, prefix, kernel, stride, bn=True, relu=True, eps=1e-5, symmetric=False):
    x = F.pad(x, same_pad(kernel, stride, x.shape[2:], symmetric))
    x = F.conv3d(x, sd[prefix + ".conv3d.weight"], sd.get(prefix + ".conv3d.bias"), stride=stride)
    if bn:
        x = F.batch_norm(x, sd[prefix + ".bn.running_mean"], sd[prefix + ".bn.running_var"], sd[prefix + ".bn.weight"],
                         sd[prefix + ".bn.bias"], False, 0.0, eps)
    return F.relu(x) if relu else x


def maxpool(x, kernel, stride, symmetric=False):
    return F.max_pool3d(F.pad(x, same_pad(kernel, stride, x.shape[2:], symmetric)), kernel, stride)


def forward(sd: Dict[str, torch.Tensor], x: torch.Tensor, endpoints: dict = None, eps=1e-5, symmetric=False,
            branch_order=(0, 1, 2, 3)) -> torch.Tensor:
    """InceptionI3d.forward on (b, 3, t, 224, 224) -> logits (b, num_classes).  endpoints: filled with each endpoint's
    output (b, c, t, h, w)."""
    kw = dict(eps=eps, symmetric=symmetric)
    for name, kind, spec in ARCH:
        if kind == "unit":
            x = unit3d(x, sd, name, spec[2], spec[3], **kw)
        elif kind == "pool":
            x = maxpool(x, spec[0], spec[1], symmetric)
        else:
            k1, k3 = (1, 1, 1), (3, 3, 3)
            one = (1, 1, 1)
            br = [unit3d(x, sd, name + ".b0", k1, one, **kw),
                  unit3d(unit3d(x, sd, name + ".b1a", k1, one, **kw), sd, name + ".b1b", k3, one, **kw),
                  unit3d(unit3d(x, sd, name + ".b2a", k1, one, **kw), sd, name + ".b2b", k3, one, **kw),
                  unit3d(maxpool(x, k3, one, symmetric), sd, name + ".b3b", k1, one, **kw)]
            x = torch.cat([br[i] for i in branch_order], dim=1)
        if endpoints is not None:
            endpoints[name] = x
    x = F.avg_pool3d(x, (2, 7, 7), stride=1)
    x = F.conv3d(x, sd["logits.conv3d.weight"], sd["logits.conv3d.bias"])
    return x.squeeze(3).squeeze(3).mean(dim=2)


def frechet_distance(x1: torch.Tensor, x2: torch.Tensor) -> torch.Tensor:
    """fvd.py:101-112 with its helpers (:56-98)."""
    def sqrtm(mat, eps=1e-10):
        u, s, v = torch.svd(mat)
        si = torch.where(s < eps, s, torch.sqrt(s))
        return u @ torch.diag(si) @ v.t()

    def cov(m):
        m = m.t()
        mc = m - m.mean(dim=1, keepdim=True)
        return (1.0 / (m.size(1) - 1)) * (mc @ mc.t()).squeeze()

    x1, x2 = x1.flatten(start_dim=1), x2.flatten(start_dim=1)
    s1, s2 = cov(x1), cov(x2)
    r = sqrtm(s1)
    return torch.trace(s1 + s2) - 2.0 * torch.trace(sqrtm(r @ (s2 @ r))) + torch.sum((x1.mean(0) - x2.mean(0)) ** 2)


def make_state_dict(seed: int = 0, num_classes: int = 400) -> Dict[str, torch.Tensor]:
    """Seeded weights in the reference's state_dict layout: torch.rand plus exact arithmetic (as oracle/weights.py).
    BatchNorm statistics are placeholders (mean 0, var 1); the fixture stores calibrated ones (calibrate_bn)."""
    g = torch.Generator().manual_seed(seed)

    def uni(shape, lo, hi):
        return torch.rand(shape, generator=g) * (hi - lo) + lo

    sd: Dict[str, torch.Tensor] = {}
    for prefix, cin, cout, k, _ in units():
        b = 1.0 / math.sqrt(cin * k[0] * k[1] * k[2])
        sd[prefix + ".conv3d.weight"] = uni((cout, cin) + tuple(k), -b, b)
        sd[prefix + ".bn.weight"] = uni((cout,), 0.5, 1.5)
        sd[prefix + ".bn.bias"] = uni((cout,), -0.1, 0.1)
        sd[prefix + ".bn.running_mean"] = torch.zeros(cout)
        sd[prefix + ".bn.running_var"] = torch.ones(cout)
        sd[prefix + ".bn.num_batches_tracked"] = torch.tensor(0, dtype=torch.int64)
    b = 1.0 / math.sqrt(1024)
    sd["logits.conv3d.weight"] = uni((num_classes, 1024, 1, 1, 1), -b, b)
    sd["logits.conv3d.bias"] = uni((num_classes,), -b, b)
    return sd


def calibrate_bn(sd: Dict[str, torch.Tensor], x: torch.Tensor) -> None:
    """Set every unit's running statistics to its conv output's per-channel mean and variance on x, layer by layer, so
    that every unit's output is O(1) (random weights with mean 0 / var 1 statistics shrink or grow layer after layer).
    Rounded to 2^-12 so the stored vectors are short exact values."""
    q = lambda t: torch.round(t * 4096) / 4096

    def unit_cal(x, prefix, kernel, stride):
        y = F.conv3d(F.pad(x, same_pad(kernel, stride, x.shape[2:])), sd[prefix + ".conv3d.weight"], stride=stride)
        sd[prefix + ".bn.running_mean"] = q(y.mean(dim=(0, 2, 3, 4)))
        sd[prefix + ".bn.running_var"] = torch.clamp(q(y.var(dim=(0, 2, 3, 4))), min=2.0 ** -12)
        return unit3d(x, sd, prefix, kernel, stride)

    with torch.no_grad():
        for name, kind, spec in ARCH:
            if kind == "unit":
                x = unit_cal(x, name, spec[2], spec[3])
            elif kind == "pool":
                x = maxpool(x, spec[0], spec[1])
            else:
                k1, k3, one = (1, 1, 1), (3, 3, 3), (1, 1, 1)
                b0 = unit_cal(x, name + ".b0", k1, one)
                b1 = unit_cal(unit_cal(x, name + ".b1a", k1, one), name + ".b1b", k3, one)
                b2 = unit_cal(unit_cal(x, name + ".b2a", k1, one), name + ".b2b", k3, one)
                b3 = unit_cal(maxpool(x, k3, one), name + ".b3b", k1, one)
                x = torch.cat([b0, b1, b2, b3], dim=1)


def bn_stats(sd) -> Dict[str, torch.Tensor]:
    return {k: v for k, v in sd.items() if k.endswith((".running_mean", ".running_var"))}


def conv_fingerprint(sd) -> float:
    """Order-independent float64 checksum of the weights make_state_dict draws."""
    tot = 0.0
    for k in sorted(sd):
        if k.endswith((".running_mean", ".running_var", ".num_batches_tracked")):
            continue
        v = sd[k].double().flatten()
        tot += float((v * torch.arange(1, v.numel() + 1, dtype=torch.float64) % 7.0).sum())
    return tot


def fold_bn(sd, prefix, eps=1e-5) -> Tuple[torch.Tensor, torch.Tensor]:
    """BatchNorm folded into the conv in float64: W' = W s, b' = beta - mean s with s = gamma / sqrt(var + eps)."""
    w = sd[prefix + ".conv3d.weight"].double()
    s = sd[prefix + ".bn.weight"].double() / torch.sqrt(sd[prefix + ".bn.running_var"].double() + eps)
    b = sd[prefix + ".bn.bias"].double() - sd[prefix + ".bn.running_mean"].double() * s
    return (w * s.view(-1, 1, 1, 1, 1)).float(), b.float()


def endpoint_summary(x: torch.Tensor, seed: int, n: int = 64) -> Dict[str, torch.Tensor]:
    """Channel means and a seeded sample of elements of an endpoint (b, c, t, h, w), for localising a fault."""
    flat = x.flatten()
    idx = torch.randint(0, flat.numel(), (n,), generator=torch.Generator().manual_seed(seed))
    return {"channel_mean": x.mean(dim=(0, 2, 3, 4)), "idx": idx, "val": flat[idx]}
