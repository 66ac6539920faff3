"""CPU fp32 restatement of evaluation/common_metrics_on_video_quality's FVD (calculate_fvd.py, fvd/styleganv/fvd.py,
fvd/videogpt/fvd.py and the StyleGAN-V I3D of i3d_torchscript.pt), written from their spec.  TEST INFRASTRUCTURE ONLY:
the product never imports it.

- trans: grey repeated to 3 channels, (B, T, C, H, W) -> (B, C, T, H, W).
- preprocess_styleganv: per clip (C, t, H, W) view, F.interpolate to the shorter side 224 (the longer one
  ceil(n * 224 / min(H, W))), the centre crop, (v - 0.5) * 2.
- preprocess_videogpt: (v * 255) truncated to uint8, then per clip (t, C, H, W) bytes / 255, the same resize and crop,
  -= 0.5, * 2.  torch picks its bilinear kernel for this batch by its thread count; the reference script runs
  multi-threaded, so the interpolate runs here with at least two threads.
- forward_styleganv: the StyleGAN-V I3D = i3d_oracle.forward on its weights under pytorch_i3d's keys with BatchNorm
  eps 1e-3 (its fixed pad tables equal SAME padding at 224 x 224).
"""
from __future__ import annotations

import contextlib
import math
from typing import Dict

import torch
import torch.nn.functional as F

from oracle import i3d_oracle as io

RES = 224
EPS_STYLEGANV = 1e-3


def trans(x: torch.Tensor) -> torch.Tensor:
    if x.shape[-3] == 1:
        x = x.repeat(1, 1, 3, 1, 1)
    return x.permute(0, 2, 1, 3, 4)


def target_size(h: int, w: int):
    scale = RES / min(h, w)
    return (RES, math.ceil(w * scale)) if h < w else (math.ceil(h * scale), RES)


def _crop(v: torch.Tensor) -> torch.Tensor:
    h, w = v.shape[-2:]
    hs, ws = (h - RES) // 2, (w - RES) // 2
    return v[..., hs:hs + RES, ws:ws + RES]


@contextlib.contextmanager
def threads_at_least(n: int):
    old = torch.get_num_threads()
    torch.set_num_threads(max(old, n))
    try:
        yield
    finally:
        torch.set_num_threads(old)


def preprocess_styleganv(videos: torch.Tensor, t: int) -> torch.Tensor:
    """fp32 (B, T, C, H, W) in [0, 1] -> (B, 3, t, 224, 224) network input of the first t frames."""
    v = trans(videos)[:, :, :t]
    out = []
    for clip in v:                                           # (C, t, H, W), a non-contiguous view
        y = F.interpolate(clip, size=target_size(*clip.shape[-2:]), mode="bilinear", align_corners=False)
        out.append(((_crop(y) - 0.5) * 2).contiguous())
    return torch.stack(out)


def preprocess_videogpt(videos: torch.Tensor, t: int) -> torch.Tensor:
    """fp32 (B, T, C, H, W) in [0, 1] -> (B, 3, t, 224, 224) network input of the first t frames."""
    v = trans(videos)[:, :, :t]
    u8 = torch.from_numpy((v.permute(0, 2, 3, 4, 1) * 255).numpy().astype("uint8"))   # b t h w c
    out = []
    with threads_at_least(2):
        for clip in u8:
            x = clip.permute(0, 3, 1, 2).float() / 255.                                  # (t, C, H, W)
            y = F.interpolate(x, size=target_size(*x.shape[-2:]), mode="bilinear", align_corners=False)
            y = _crop(y).permute(1, 0, 2, 3).contiguous()
            y -= 0.5
            out.append(y)
    return torch.stack(out) * 2


def pytorch_i3d_keys(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """The StyleGAN-V I3D's state_dict under pytorch_i3d's key names (num_batches_tracked dropped)."""
    out = {}
    br = {"branch_0.": "b0.", "branch_1.0.": "b1a.", "branch_1.1.": "b1b.", "branch_2.0.": "b2a.",
          "branch_2.1.": "b2b.", "branch_3.1.": "b3b."}
    for k, v in sd.items():
        if k.endswith("num_batches_tracked"):
            continue
        n = k.replace("conv3d_0c_1x1.", "logits.").replace(".batch3d.", ".bn.")
        for a, b in br.items():
            n = n.replace("." + a, "." + b)
        head, rest = n.split(".", 1)
        if head.startswith("conv3d_"):
            head = "Conv3d_" + head[len("conv3d_"):]
        elif head.startswith("mixed_"):
            head = "Mixed_" + head[len("mixed_"):]
        out[f"{head}.{rest}"] = v
    return out


def styleganv_keys(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """pytorch_i3d's layout -> the StyleGAN-V I3D's (the inverse of pytorch_i3d_keys)."""
    out = {}
    br = {"b0": "branch_0", "b1a": "branch_1.0", "b1b": "branch_1.1", "b2a": "branch_2.0", "b2b": "branch_2.1",
          "b3b": "branch_3.1"}
    for k, v in sd.items():
        parts = k.split(".")
        if parts[0] == "logits":
            out["conv3d_0c_1x1." + ".".join(parts[1:])] = v
            continue
        parts[0] = parts[0][0].lower() + parts[0][1:]
        if parts[0].startswith("mixed_"):
            parts[1] = br[parts[1]]
        out[".".join(parts).replace(".bn.", ".batch3d.")] = v
    return out


def forward_styleganv(sd: Dict[str, torch.Tensor], x: torch.Tensor) -> torch.Tensor:
    """The torchscript's forward(x, rescale=False, resize=False, return_features=True) on (b, 3, t, 224, 224)."""
    return io.forward(pytorch_i3d_keys(sd), x, eps=EPS_STYLEGANV)
