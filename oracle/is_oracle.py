"""CPU fp32 restatement of the video-metric suite's Inception Score (evaluation/common_metrics_on_video_quality/
calculate_is.py: calculate_is and inception_score with torchvision's inception_v3), written from their spec.  TEST
INFRASTRUCTURE ONLY: the product never imports it.

- preprocess: nn.Upsample(size=(299, 299), mode='bilinear') (align_corners=False), or nothing (inception_score's
  resize=False); no normalisation (transform_input=False).
- network: fid_oracle.forward with torchvision's pool wiring (every branch_pool is avg_pool2d(3, 1, 1) with
  count_include_pad=True, Mixed_7c's too), then AdaptiveAvgPool2d(1), then fc (2048 -> 1000, with bias).
- F.softmax over the classes; the rows go into a float64 array.
- split k = preds[k (N // splits) : (k + 1) (N // splits)]; per row scipy.stats.entropy(p(y|x), p(y)) with p(y) the
  split's column mean: both vectors renormalised to sum 1, then sum x log(x / y) with 0 where x = 0; the split's score
  is exp of the mean; the result is (np.mean, np.std) over the splits.

The keyword arguments of `logits`, `preprocess`, `probabilities` and `split_scores` break one wiring each; tests use
them to show the fixture detects it.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from oracle import fid_oracle as fo

NUM_CLASSES = 1000
# torchvision Inception3's InceptionAux (unused in eval mode, but part of the weight file): key -> shape
AUX_SHAPES = {"AuxLogits.conv0.conv.weight": (128, 768, 1, 1), "AuxLogits.conv1.conv.weight": (768, 128, 5, 5),
              "AuxLogits.fc.weight": (NUM_CLASSES, 768), "AuxLogits.fc.bias": (NUM_CLASSES,)}


def preprocess(x: torch.Tensor, resize: bool = True, align_corners: bool = False) -> torch.Tensor:
    """(N, 3, H, W) fp32 -> the network input."""
    if not resize:
        return x
    return F.interpolate(x, size=(299, 299), mode="bilinear", align_corners=align_corners)


def logits(sd: Dict[str, torch.Tensor], x: torch.Tensor, endpoints: Optional[dict] = None,
           count_include_pad: bool = True, e2_avg: bool = True) -> torch.Tensor:
    """Inception3.forward in eval mode on the preprocessed (N, 3, H, W) batch -> (N, 1000) logits."""
    f = fo.forward(sd, x, endpoints, count_include_pad=count_include_pad, e2_avg=e2_avg)
    return F.linear(f, sd["fc.weight"], sd["fc.bias"])


def probabilities(sd, x: torch.Tensor, resize: bool = True, softmax_dim: int = 1, align_corners: bool = False,
                  **wiring) -> torch.Tensor:
    """get_pred of calculate_is.py on one batch: (N, 3, H, W) fp32 -> (N, 1000) fp32 softmax rows."""
    return F.softmax(logits(sd, preprocess(x, resize, align_corners), **wiring), dim=softmax_dim)


def entropy(pk: np.ndarray, qk: np.ndarray, renormalise: bool = True) -> float:
    """scipy.stats.entropy(pk, qk) in float64: sum of x log(x / y) over the renormalised vectors, 0 where x = 0."""
    if renormalise:
        pk, qk = pk / pk.sum(), qk / qk.sum()
    pos = pk > 0
    return float(np.sum(pk[pos] * np.log(pk[pos] / qk[pos])))


def split_scores(preds: np.ndarray, splits: int, renormalise: bool = True, keep_leftover: bool = False) -> List[float]:
    """exp(mean KL) of every split of the float64 (N, classes) predictions."""
    N = preds.shape[0]
    n = N // splits
    out = []
    for k in range(splits):
        end = N if keep_leftover and k == splits - 1 else (k + 1) * n
        part = preds[k * n:end]
        py = np.mean(part, axis=0)
        out.append(math.exp(np.mean([entropy(part[i], py, renormalise) for i in range(part.shape[0])])))
    return out


def inception_score(preds: np.ndarray, splits: int, **wiring):
    s = split_scores(preds, splits, **wiring)
    return np.mean(s), np.std(s)


def make_state_dict(seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded weights in the layout of torchvision's inception_v3_google-0cc3c7bd.pth: fid_oracle.make_state_dict with
    a 1000-class fc, plus seeded AuxLogits (BatchNorm placeholders as make_state_dict's).  calibrate then sets the
    BatchNorm statistics and fc's scale."""
    sd = fo.make_state_dict(seed, num_classes=NUM_CLASSES)
    g = torch.Generator().manual_seed(seed + 1000)
    for k, shape in AUX_SHAPES.items():
        b = 1.0 / math.sqrt(shape[1] * (shape[2] * shape[3] if len(shape) == 4 else 1)) if len(shape) > 1 else 0.01
        sd[k] = (torch.rand(shape, generator=g) * 2 - 1) * b
        if k.endswith(".conv.weight"):
            p = k[:-len(".conv.weight")]
            c = shape[0]
            sd[p + ".bn.weight"] = torch.rand(c, generator=g) + 0.5
            sd[p + ".bn.bias"] = (torch.rand(c, generator=g) - 0.5) * 0.2
            sd[p + ".bn.running_mean"] = torch.zeros(c)
            sd[p + ".bn.running_var"] = torch.ones(c)
            sd[p + ".bn.num_batches_tracked"] = torch.tensor(0, dtype=torch.int64)
    return sd


def calibrate(sd: Dict[str, torch.Tensor], x: torch.Tensor, logit_spread: float = 4.0) -> float:
    """fid_oracle.calibrate_bn's statistics through torchvision's pool wiring (the averages count the padding, Mixed_7c
    averages), on the preprocessed calibration batch x; then fc scaled by a power of two so that the logits' standard
    deviation over x's frames is about logit_spread, with the bias centring them (rounded to 2^-12); returns the scale.
    Random weights
    give every frame nearly the same features; without this the classes barely differ and the score is 1."""
    q = lambda t: torch.round(t * 4096) / 4096

    def conv(t, prefix):
        k, s, p = fo._GEOM[prefix]
        y = F.conv2d(t, sd[prefix + ".conv.weight"], None, stride=s, padding=p)
        m = q(y.mean(dim=(0, 2, 3)) / 2)
        sd[prefix + ".bn.running_mean"] = m
        sd[prefix + ".bn.running_var"] = torch.clamp(q(((y - m.view(1, -1, 1, 1)) ** 2).mean(dim=(0, 2, 3))),
                                                     min=2.0 ** -12)
        return fo.basic_conv(t, sd, prefix)

    with torch.no_grad():
        h = x
        for p in ("Conv2d_1a_3x3", "Conv2d_2a_3x3", "Conv2d_2b_3x3"):
            h = conv(h, p)
        h = F.max_pool2d(h, 3, 2)
        h = F.max_pool2d(conv(conv(h, "Conv2d_3b_1x1"), "Conv2d_4a_3x3"), 3, 2)
        for name, kind, _, _ in fo.BLOCKS:
            h = fo._block(h, sd, name, kind, conv, True, True)
        f = F.adaptive_avg_pool2d(h, (1, 1)).flatten(1).double()
        w = sd["fc.weight"].double()
        centred = (f - f.mean(0)) @ w.t()
        scale = 2.0 ** round(math.log2(logit_spread / float(centred.std(0).mean())))
        sd["fc.weight"] = (w * scale).float()
        sd["fc.bias"] = q(-(f.mean(0) @ w.t()) * scale + sd["fc.bias"].double()).float()
    return scale


def fixture_state_dict(golden: dict) -> Dict[str, torch.Tensor]:
    """The fixture's weights: make_state_dict(w_seed) with the stored BatchNorm statistics, fc.weight times the stored
    power of two and the stored fc.bias (nothing here depends on the CPU that calibrated them)."""
    sd = make_state_dict(golden["w_seed"])
    sd.update(golden["bn"])
    sd["fc.weight"] = sd["fc.weight"] * golden["fc_scale"]
    sd["fc.bias"] = golden["fc_bias"].clone()
    return sd


def frames(shape: Sequence[int], seed: int, lo: float = 0.0, hi: float = 1.0) -> torch.Tensor:
    """Seeded fp32 (N, 3, H, W) frames in [lo, hi]: smooth random colour fields (a 4 x 4 grid, bilinearly upsampled)
    with per-frame contrast and a little noise, so the frames differ in what the network sees."""
    N, H, W = shape
    g = torch.Generator().manual_seed(seed)
    base = F.interpolate(torch.rand(N, 3, 4, 4, generator=g), size=(H, W), mode="bilinear", align_corners=False)
    gain = torch.rand(N, 1, 1, 1, generator=g) * 1.5 + 0.25
    x = (base - 0.5) * gain + 0.5 + (torch.rand(N, 3, H, W, generator=g) - 0.5) * 0.1
    return x.clamp(0, 1) * (hi - lo) + lo


def endpoint_summary(x: torch.Tensor, seed: int, n: int = 64) -> Dict[str, torch.Tensor]:
    return fo.endpoint_summary(x, seed, n)


# The fixture's cases (oracle/make_golden_is.py): calculate_is on (B, T, 3, H, W) clips, one network batch per clip,
# or inception_score on N (3, H, W) images in batches of batch_size.  u8: the clip is bytes / 255 of uint8 frames.
CASES = {
    "calc_up64": dict(fn="calculate_is", B=2, T=3, H=64, W=64, seed=101, splits=1),
    "calc_down_336x400": dict(fn="calculate_is", B=1, T=4, H=336, W=400, seed=102, splits=1),
    "calc_signed_64x80": dict(fn="calculate_is", B=2, T=2, H=64, W=80, seed=103, lo=-1.0, splits=1),
    "calc_u8_48x64": dict(fn="calculate_is", B=2, T=3, H=48, W=64, seed=104, u8=True, splits=1),
    "calc_n7_splits3": dict(fn="calculate_is", B=1, T=7, H=64, W=64, seed=105, splits=3),
    "score_299": dict(fn="inception_score", N=5, H=299, W=299, seed=106, batch_size=2, resize=False, splits=1),
    # the network at 96 x 128 ends on a 1 x 2 map: its features lie far from the 299 x 299 calibration frames', fc's
    # bias dominates and every frame gets the same class (IS ~1).  The case tests the native-size path's logits.
    "score_96x128": dict(fn="inception_score", N=5, H=96, W=128, seed=107, batch_size=2, resize=False, splits=1,
                         scored=False),
    "score_up32": dict(fn="inception_score", N=5, H=32, W=32, seed=108, batch_size=2, resize=True, splits=2),
}


def case_input(spec: dict):
    """(x, u8): calculate_is's fp32 (B, T, 3, H, W) clips or inception_score's fp32 (N, 3, H, W) images, and for a u8
    case the uint8 (B, T, H, W, 3) frames x stands for (else None)."""
    if spec["fn"] == "calculate_is":
        B, T = spec["B"], spec["T"]
        x = frames((B * T, spec["H"], spec["W"]), spec["seed"], spec.get("lo", 0.0))
        u8 = None
        if spec.get("u8"):
            u8 = torch.round(x * 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()
            x = u8.permute(0, 3, 1, 2).float() / 255
            u8 = u8.view(B, T, spec["H"], spec["W"], 3)
        return x.reshape(B, T, 3, spec["H"], spec["W"]), u8
    return frames((spec["N"], spec["H"], spec["W"]), spec["seed"]), None


def case_batches(spec: dict, x: torch.Tensor) -> List[torch.Tensor]:
    """The batches the reference feeds its network: one per clip, or the DataLoader's batches of batch_size."""
    if spec["fn"] == "calculate_is":
        return list(x)
    return list(torch.split(x, spec["batch_size"]))


def case_probabilities(sd, spec: dict, **wiring) -> torch.Tensor:
    x, _ = case_input(spec)
    resize = spec.get("resize", True)
    with torch.no_grad():
        return torch.cat([probabilities(sd, b, resize, **wiring) for b in case_batches(spec, x)])
