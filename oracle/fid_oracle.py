"""CPU fp32 restatement of the FID metric's feature network and statistics (evaluation/pytorch-fid/src/pytorch_fid/
inception.py with torchvision's Inception3 blocks, fid_score.py), written from their spec.  TEST INFRASTRUCTURE ONLY:
the product never imports it.

- preprocess: fid_score.py:146 ToTensor (byte / 255, channel-planar), inception.py:147-151 -- bilinear F.interpolate
  to 299 x 299 (align_corners=False), then 2 x - 1.
- BasicConv2d: conv2d without bias (symmetric padding), BatchNorm2d (eps 1e-3, running statistics), ReLU.
- Blocks: Conv2d_1a..4a with two MaxPool2d(3, 2) (blocks 0, 1); Mixed_5b..5d FIDInceptionA, Mixed_6a InceptionB,
  Mixed_6b..6e FIDInceptionC, Mixed_7a InceptionD, Mixed_7b FIDInceptionE_1, Mixed_7c FIDInceptionE_2 (blocks 2, 3);
  the FID patches: the A / C / E_1 pool branches average without the padding, E_2's pool branch is a max pool.
- AdaptiveAvgPool2d(1) -> the (B, 2048) pool3 features.

The keyword arguments of `forward` / `preprocess` break one wiring each; tests use them to show the fixture detects it.
"""
from __future__ import annotations

import math
from typing import Dict, List, Tuple

import torch
import torch.nn.functional as F

# (block, kind, in channels, kind argument): A pool_features, C channels_7x7
BLOCKS: List[Tuple[str, str, int, int]] = [
    ("Mixed_5b", "A", 192, 32), ("Mixed_5c", "A", 256, 64), ("Mixed_5d", "A", 288, 64), ("Mixed_6a", "B", 288, 0),
    ("Mixed_6b", "C", 768, 128), ("Mixed_6c", "C", 768, 160), ("Mixed_6d", "C", 768, 160), ("Mixed_6e", "C", 768, 192),
    ("Mixed_7a", "D", 768, 0), ("Mixed_7b", "E1", 1280, 0), ("Mixed_7c", "E2", 2048, 0)]


def convs() -> List[Tuple[str, int, int, Tuple[int, int], int, Tuple[int, int]]]:
    """Every BasicConv2d: (prefix, cin, cout, kernel, stride, padding), in torchvision's module order."""
    out = [("Conv2d_1a_3x3", 3, 32, (3, 3), 2, (0, 0)), ("Conv2d_2a_3x3", 32, 32, (3, 3), 1, (0, 0)),
           ("Conv2d_2b_3x3", 32, 64, (3, 3), 1, (1, 1)), ("Conv2d_3b_1x1", 64, 80, (1, 1), 1, (0, 0)),
           ("Conv2d_4a_3x3", 80, 192, (3, 3), 1, (0, 0))]
    one, k3, p1 = (1, 1), (3, 3), (1, 1)
    for name, kind, cin, a in BLOCKS:
        if kind == "A":
            u = [("branch1x1", cin, 64, one, 1, (0, 0)), ("branch5x5_1", cin, 48, one, 1, (0, 0)),
                 ("branch5x5_2", 48, 64, (5, 5), 1, (2, 2)), ("branch3x3dbl_1", cin, 64, one, 1, (0, 0)),
                 ("branch3x3dbl_2", 64, 96, k3, 1, p1), ("branch3x3dbl_3", 96, 96, k3, 1, p1),
                 ("branch_pool", cin, a, one, 1, (0, 0))]
        elif kind == "B":
            u = [("branch3x3", cin, 384, k3, 2, (0, 0)), ("branch3x3dbl_1", cin, 64, one, 1, (0, 0)),
                 ("branch3x3dbl_2", 64, 96, k3, 1, p1), ("branch3x3dbl_3", 96, 96, k3, 2, (0, 0))]
        elif kind == "C":
            r, c = ((1, 7), (0, 3)), ((7, 1), (3, 0))
            u = [("branch1x1", cin, 192, one, 1, (0, 0)), ("branch7x7_1", cin, a, one, 1, (0, 0)),
                 ("branch7x7_2", a, a, r[0], 1, r[1]), ("branch7x7_3", a, 192, c[0], 1, c[1]),
                 ("branch7x7dbl_1", cin, a, one, 1, (0, 0)), ("branch7x7dbl_2", a, a, c[0], 1, c[1]),
                 ("branch7x7dbl_3", a, a, r[0], 1, r[1]), ("branch7x7dbl_4", a, a, c[0], 1, c[1]),
                 ("branch7x7dbl_5", a, 192, r[0], 1, r[1]), ("branch_pool", cin, 192, one, 1, (0, 0))]
        elif kind == "D":
            u = [("branch3x3_1", cin, 192, one, 1, (0, 0)), ("branch3x3_2", 192, 320, k3, 2, (0, 0)),
                 ("branch7x7x3_1", cin, 192, one, 1, (0, 0)), ("branch7x7x3_2", 192, 192, (1, 7), 1, (0, 3)),
                 ("branch7x7x3_3", 192, 192, (7, 1), 1, (3, 0)), ("branch7x7x3_4", 192, 192, k3, 2, (0, 0))]
        else:
            u = [("branch1x1", cin, 320, one, 1, (0, 0)), ("branch3x3_1", cin, 384, one, 1, (0, 0)),
                 ("branch3x3_2a", 384, 384, (1, 3), 1, (0, 1)), ("branch3x3_2b", 384, 384, (3, 1), 1, (1, 0)),
                 ("branch3x3dbl_1", cin, 448, one, 1, (0, 0)), ("branch3x3dbl_2", 448, 384, k3, 1, p1),
                 ("branch3x3dbl_3a", 384, 384, (1, 3), 1, (0, 1)), ("branch3x3dbl_3b", 384, 384, (3, 1), 1, (1, 0)),
                 ("branch_pool", cin, 192, one, 1, (0, 0))]
        out += [(f"{name}.{n}",) + tuple(rest) for n, *rest in u]
    return out


_GEOM = {p: (k, s, pad) for p, _, _, k, s, pad in convs()}


def preprocess(images, align_corners=False, norm_first=False, lut=None) -> torch.Tensor:
    """(B, H, W, 3) uint8 -> (B, 3, 299, 299) fp32: ToTensor, F.interpolate, 2 x - 1.  lut: fp32 [256] replacing
    byte / 255 (the real side's composed byte map).  align_corners / norm_first: the broken wirings."""
    u8 = torch.as_tensor(images).permute(0, 3, 1, 2).contiguous()
    x = u8.float().div(255) if lut is None else lut[u8.long()]
    if norm_first:
        x = 2 * x - 1
    x = F.interpolate(x, size=(299, 299), mode="bilinear", align_corners=align_corners)
    return x if norm_first else 2 * x - 1


def basic_conv(x, sd, prefix, eps=1e-3):
    k, s, p = _GEOM[prefix]
    x = F.conv2d(x, sd[prefix + ".conv.weight"], None, stride=s, padding=p)
    x = F.batch_norm(x, sd[prefix + ".bn.running_mean"], sd[prefix + ".bn.running_var"], sd[prefix + ".bn.weight"],
                     sd[prefix + ".bn.bias"], False, 0.0, eps)
    return F.relu(x)


def _block(x, sd, name, kind, conv, count_include_pad=False, e2_avg=False):
    c = lambda n, t: conv(t, f"{name}.{n}")

    def avg(t):
        return F.avg_pool2d(t, 3, 1, 1, count_include_pad=count_include_pad)

    if kind == "A":
        out = [c("branch1x1", x), c("branch5x5_2", c("branch5x5_1", x)),
               c("branch3x3dbl_3", c("branch3x3dbl_2", c("branch3x3dbl_1", x))), c("branch_pool", avg(x))]
    elif kind == "B":
        out = [c("branch3x3", x), c("branch3x3dbl_3", c("branch3x3dbl_2", c("branch3x3dbl_1", x))),
               F.max_pool2d(x, 3, 2)]
    elif kind == "C":
        b7 = c("branch7x7_3", c("branch7x7_2", c("branch7x7_1", x)))
        d = x
        for i in range(1, 6):
            d = c(f"branch7x7dbl_{i}", d)
        out = [c("branch1x1", x), b7, d, c("branch_pool", avg(x))]
    elif kind == "D":
        d = x
        for i in range(1, 5):
            d = c(f"branch7x7x3_{i}", d)
        out = [c("branch3x3_2", c("branch3x3_1", x)), d, F.max_pool2d(x, 3, 2)]
    else:
        b3 = c("branch3x3_1", x)
        dbl = c("branch3x3dbl_2", c("branch3x3dbl_1", x))
        pooled = avg(x) if (kind == "E1" or e2_avg) else F.max_pool2d(x, 3, 1, 1)
        out = [c("branch1x1", x), c("branch3x3_2a", b3), c("branch3x3_2b", b3), c("branch3x3dbl_3a", dbl),
               c("branch3x3dbl_3b", dbl), c("branch_pool", pooled)]
    return torch.cat(out, 1)


def forward(sd: Dict[str, torch.Tensor], x: torch.Tensor, endpoints: dict = None, eps=1e-3, count_include_pad=False,
            e2_avg=False) -> torch.Tensor:
    """InceptionV3([3]).forward after the preprocess: (B, 3, 299, 299) -> pool3 features (B, 2048).  endpoints: filled
    with each block's output (B, C, H, W).  eps / count_include_pad / e2_avg: the broken wirings."""
    conv = lambda t, p: basic_conv(t, sd, p, eps)
    for p in ("Conv2d_1a_3x3", "Conv2d_2a_3x3", "Conv2d_2b_3x3"):
        x = conv(x, p)
    x = F.max_pool2d(x, 3, 2)
    x = F.max_pool2d(conv(conv(x, "Conv2d_3b_1x1"), "Conv2d_4a_3x3"), 3, 2)
    if endpoints is not None:
        endpoints["stem"] = x
    for name, kind, _, _ in BLOCKS:
        x = _block(x, sd, name, kind, conv, count_include_pad, e2_avg)
        if endpoints is not None:
            endpoints[name] = x
    return F.adaptive_avg_pool2d(x, (1, 1)).flatten(1)


def make_state_dict(seed: int = 0, num_classes: int = 1008) -> Dict[str, torch.Tensor]:
    """Seeded weights in the layout of pytorch-fid's weight file (torchvision Inception3 keys, plus its fc layer):
    torch.rand plus exact arithmetic.  BatchNorm statistics are placeholders (mean 0, var 1); the fixture stores
    calibrated ones (calibrate_bn)."""
    g = torch.Generator().manual_seed(seed)

    def uni(shape, lo, hi):
        return torch.rand(shape, generator=g) * (hi - lo) + lo

    sd: Dict[str, torch.Tensor] = {}
    for prefix, cin, cout, k, _, _ in convs():
        b = 1.0 / math.sqrt(cin * k[0] * k[1])
        sd[prefix + ".conv.weight"] = uni((cout, cin) + tuple(k), -b, b)
        sd[prefix + ".bn.weight"] = uni((cout,), 0.5, 1.5)
        sd[prefix + ".bn.bias"] = uni((cout,), -0.1, 0.1)
        sd[prefix + ".bn.running_mean"] = torch.zeros(cout)
        sd[prefix + ".bn.running_var"] = torch.ones(cout)
        sd[prefix + ".bn.num_batches_tracked"] = torch.tensor(0, dtype=torch.int64)
    b = 1.0 / math.sqrt(2048)
    sd["fc.weight"] = uni((num_classes, 2048), -b, b)
    sd["fc.bias"] = uni((num_classes,), -b, b)
    return sd


def calibrate_bn(sd: Dict[str, torch.Tensor], x: torch.Tensor) -> None:
    """Set every conv's running statistics from its output y on x (preprocessed images), conv after conv in forward
    order, so that every unit's output is O(1): running_mean = mean(y) / 2 and running_var = mean((y - running_mean)^2)
    per channel.  Centring on half the mean keeps a channel whose values barely vary from being normalised through a
    cancellation (y - mean(y) over a tiny variance), which would amplify every rounding error 94 convs deep.  Rounded
    to 2^-12 so the stored vectors are short exact values."""
    q = lambda t: torch.round(t * 4096) / 4096

    def conv(t, prefix):
        k, s, p = _GEOM[prefix]
        y = F.conv2d(t, sd[prefix + ".conv.weight"], None, stride=s, padding=p)
        m = q(y.mean(dim=(0, 2, 3)) / 2)
        sd[prefix + ".bn.running_mean"] = m
        sd[prefix + ".bn.running_var"] = torch.clamp(q(((y - m.view(1, -1, 1, 1)) ** 2).mean(dim=(0, 2, 3))),
                                                     min=2.0 ** -12)
        return basic_conv(t, sd, prefix)

    with torch.no_grad():
        for p in ("Conv2d_1a_3x3", "Conv2d_2a_3x3", "Conv2d_2b_3x3"):
            x = conv(x, p)
        x = F.max_pool2d(x, 3, 2)
        x = F.max_pool2d(conv(conv(x, "Conv2d_3b_1x1"), "Conv2d_4a_3x3"), 3, 2)
        for name, kind, _, _ in BLOCKS:
            x = _block(x, sd, name, kind, conv)


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


def fold_bn(sd, prefix, eps=1e-3) -> Tuple[torch.Tensor, torch.Tensor]:
    """BatchNorm folded into the conv in float64: W' = W s, b' = beta - mean s with s = gamma / sqrt(var + eps)."""
    w = sd[prefix + ".conv.weight"].double()
    s = sd[prefix + ".bn.weight"].double() / torch.sqrt(sd[prefix + ".bn.running_var"].double() + eps)
    b = sd[prefix + ".bn.bias"].double() - sd[prefix + ".bn.running_mean"].double() * s
    return (w * s.view(-1, 1, 1, 1)).float(), b.float()


def endpoint_summary(x: torch.Tensor, seed: int, n: int = 64) -> Dict[str, torch.Tensor]:
    """Channel means and a seeded sample of elements of an endpoint (B, C, H, W), for localising a fault."""
    flat = x.flatten()
    idx = torch.randint(0, flat.numel(), (n,), generator=torch.Generator().manual_seed(seed))
    return {"channel_mean": x.mean(dim=(0, 2, 3)), "idx": idx, "val": flat[idx]}


def image_bytes(shape, seed) -> torch.Tensor:
    """Seeded uint8 (H, W, 3) test image; seed None: a constant image."""
    if seed is None:
        return torch.full(tuple(shape) + (3,), 200, dtype=torch.uint8)
    return torch.randint(0, 256, tuple(shape) + (3,), generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)
