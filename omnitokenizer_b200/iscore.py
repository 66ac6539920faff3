"""The video-metric suite's Inception Score on the device: evaluation/common_metrics_on_video_quality/calculate_is.py
(calculate_is and inception_score) with torchvision's inception_v3 classifier, on the sm_90a kernels of csrc/i3d.cu,
csrc/resample.cu and csrc/quality.cu.

Drop-in names: calculate_is(videos, device, splits, model) and inception_score(imgs, cuda, batch_size, resize, splits,
model), with the network given (load_is_model(device, path) reads torchvision's inception_v3_google-0cc3c7bd.pth;
nothing is downloaded).

The network is fid.py's InceptionV3 trunk with torchvision's pool wiring: every branch_pool averages with
count_include_pad=True (omt_pool2d's POOL_AVG_PAD), Mixed_7c's included.  After the trunk, AdaptiveAvgPool2d(1) is
one omt_pool2d window over the whole map, `fc` (2048 -> 1000, with bias) is omt_conv3d as a 1 x 1 conv without ReLU
(3xTF32), and F.softmax over the classes is omt_softmax_rows.  The frames enter through omt_is_preprocess (the
nn.Upsample to 299 x 299 in torch's CPU arithmetic, or the frame as it is), and the split arithmetic of scipy.stats.entropy
runs in fp64 in omt_inception_score; the host takes exp, np.mean and np.std of the per-split values.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import _cabi
from . import fid
from .engine import CLIP_DESC_WORDS, run_graphed
from .metricnet import (FORM_F32, FORM_U8, MAX_WORKSPACES, axis_table, axis_tables, bounded,  # noqa: F401
                        check_state_dict, clip_descs, resolve_device)

NUM_CLASSES = 1000
FEATURES = fid.DIMS
TARGET_RESOLUTION = (299, 299)       # calculate_is.py:30 nn.Upsample(size=(299, 299), mode='bilinear')
MIN_SIZE = 75                        # the least frame Inception3 takes: Mixed_7a's 3 x 3 / 2 conv then sees a 3 x 3 map
BLOCKS = fid.blocks(fid.POOL_AVG_PAD, fid.POOL_AVG_PAD)     # torchvision's InceptionA / C / E: avg_pool2d(3, 1, 1)
FC = fid._c("fc", "x", FEATURES, NUM_CLASSES, 1)
# Frames per launch sequence.  A 299 x 299 frame's buffers take 48.7 MB on the device (every activation of the trunk,
# input to probabilities, as _Workspace allocates them), so 64 frames hold 3.1 GB: Mixed_7's 8 x 8 maps still give
# each conv launch 4096 rows to spread over the SMs, and the few workspaces kept alive stay a small share of the card.
CHUNK_FRAMES = 64


def expected_keys() -> Dict[str, tuple]:
    """The state_dict keys ISInception takes and their shapes: fid.expected_keys' 94 BasicConv2d units, plus fc."""
    keys = fid.expected_keys()
    keys["fc.weight"] = (NUM_CLASSES, FEATURES)
    keys["fc.bias"] = (NUM_CLASSES,)
    return keys


def trunk_size(H: int, W: int) -> Tuple[int, int]:
    """The size of Mixed_7c's map for an H x W input (the window of the global average pool); (0, 0) or less on an
    axis when the input is too small for the network."""
    hw = (H, W)
    for layer in fid.STEM:
        if isinstance(layer, fid.Conv):
            hw = tuple(fid.out_size(n, k, layer.s, p) for n, k, p in zip(hw, layer.k, layer.p))
        else:
            hw = tuple(fid.out_size(n, layer.k, layer.s, layer.p) for n in hw)
        if min(hw) < 1:
            return hw
    for _, _, pool, _ in BLOCKS:
        if pool.col is not None:
            hw = tuple(fid.out_size(n, pool.k, pool.s, pool.p) for n in hw)
    return hw


class _Workspace(fid.Launches):
    """Buffers, launch list and CUDA graph state of the network on n frames of oh x ow: the input x (written by
    omt_is_preprocess outside the graph), the trunk, the pool, fc, and the softmax into probs."""

    def __init__(self, net: "ISInception", n: int, oh: int, ow: int):
        super().__init__(net.device, n)
        self.x = self._act(oh, ow, 3)
        cur, c, hw = self.trunk(net.units, self.x, (oh, ow), BLOCKS)
        pooled = self._act(1, 1, c)
        self._pool(fid.Pool(fid.POOL_AVG, 0, 1, 0, None), cur, c, hw, out=(pooled, 0), k=hw)
        self.logits = torch.empty(n, NUM_CLASSES, device=net.device)
        self._conv(net.fc, pooled, (1, 1), out=(self.logits.view(n, 1, 1, NUM_CLASSES), 0), relu=0)
        self.probs = torch.empty(n, NUM_CLASSES, device=net.device)
        self.ops.append(lambda: _cabi.call("omt_softmax_rows", self.logits, NUM_CLASSES, n, NUM_CLASSES, self.probs,
                                           NUM_CLASSES))


class ISInception:
    """torchvision's Inception3 (transform_input=False, eval mode: no AuxLogits, no dropout) from a state_dict in the
    layout of inception_v3_google-0cc3c7bd.pth: the 94 BasicConv2d units (`Mixed_6b.branch7x7_2.conv.weight`, ...,
    BatchNorm eps 1e-3) and `fc.weight` (1000, 2048), `fc.bias`; `AuxLogits.*` and `num_batches_tracked` are ignored.
    BatchNorm is folded and the weights packed once, on `device` (a CUDA device); every (frames, height, width) of a
    launch sequence gets its own buffers and CUDA graph (the last few are kept)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device="cuda"):
        sd = {k: v for k, v in state_dict.items()
              if not (k.endswith(".num_batches_tracked") or k.startswith("AuxLogits."))}
        check_state_dict(sd, expected_keys(), "IS Inception3")
        self.device = check_device(device)
        sd = {k: v.detach().float().cpu() for k, v in sd.items()}
        self.units = fid.pack_units(sd, self.device)
        self.fc = fid._Unit(FC, sd["fc.weight"].view(NUM_CLASSES, FEATURES, 1, 1), sd["fc.bias"], self.device)
        self._ws = {}
        self._tables = {}

    def _table(self, H: int, W: int, resize: bool):
        """(host, device) int32 axis tables of an H x W frame (metricnet.axis_tables), resized or at its own size."""
        def make():
            host = axis_tables(H, W, *(TARGET_RESOLUTION if resize else (None, None)))
            return host, host.to(self.device)
        return bounded(self._tables, MAX_WORKSPACES, (H, W, resize), make)

    def probabilities(self, frames: torch.Tensor, resize: bool = True) -> torch.Tensor:
        """F.softmax(inception_model(up(x))) of calculate_is.py's get_pred for every frame: fp32 (N, 3, H, W) frames
        taken as they are, or uint8 (N, H, W, 3) frames standing for byte / 255, on this network's device ->
        (N, 1000) fp32 on the device.  resize=False runs the network at the frames' own size (H, W >= 75).  The frames
        run CHUNK_FRAMES at a time, each chunk read in place from `frames`; a frame's row does not depend on the
        frames around it."""
        form, N, H, W = check_frames(frames, resize)
        if frames.device != self.device:
            raise ValueError(f"ISInception: frames on {frames.device}, the network is on {self.device}")
        src = frames.contiguous()
        oh, ow = TARGET_RESOLUTION if resize else (H, W)
        tab_host, tab = self._table(H, W, resize)
        desc = clip_descs(N, 3 * H * W, H, W, oh, ow)
        desc_dev = desc.to(self.device)
        out = torch.empty(N, NUM_CLASSES, device=self.device)
        for f0 in range(0, N, CHUNK_FRAMES):
            n = min(CHUNK_FRAMES, N - f0)
            ws = bounded(self._ws, MAX_WORKSPACES, (n, oh, ow), lambda: _Workspace(self, n, oh, ow))
            _cabi.call("omt_is_preprocess", src, src.numel(), form, desc_dev.data_ptr() + f0 * 4 * CLIP_DESC_WORDS,
                       desc[f0:], tab, tab_host, tab_host.numel(), n, 1, oh, ow, ws.x)
            run_graphed(ws.graphs, self.device, "is", ws.run)
            out[f0:f0 + n] = ws.probs
        return out


def check_device(device) -> torch.device:
    dev = resolve_device(device)
    if dev.type != "cuda":
        raise ValueError(f"the Inception Score runs on a CUDA device, got {dev}")
    return dev


def check_frames(frames, resize: bool) -> Tuple[int, int, int, int]:
    """(form, N, H, W) of fp32 (N, 3, H, W) or uint8 (N, H, W, 3) frames; raises on anything else."""
    if not isinstance(frames, torch.Tensor) or frames.dtype not in (torch.float32, torch.uint8):
        raise TypeError(f"the Inception Score takes fp32 or uint8 frames, got {getattr(frames, 'dtype', type(frames))}")
    if frames.dim() != 4:
        raise ValueError(f"frames must be (N, 3, H, W) fp32 or (N, H, W, 3) uint8, got {tuple(frames.shape)}")
    if frames.dtype == torch.float32:
        form, (N, C, H, W) = FORM_F32, frames.shape
    else:
        form, (N, H, W, C) = FORM_U8, frames.shape
    if C != 3:
        raise ValueError(f"the Inception Score takes 3-channel frames, got {C} channels ({tuple(frames.shape)})")
    if min(N, H, W) < 1:
        raise ValueError(f"empty frame batch {tuple(frames.shape)}")
    if not resize and min(H, W) < MIN_SIZE:
        raise ValueError(f"without resize, Inception3 needs frames of at least {MIN_SIZE} x {MIN_SIZE}, got {H} x {W}")
    return form, int(N), int(H), int(W)


def check_splits(N: int, splits: int):
    if not isinstance(splits, (int, np.integer)) or not 1 <= splits <= N:
        raise ValueError(f"splits must be between 1 and the {N} frames (an empty split has no score), got {splits}")


def split_rows(N: int, splits: int) -> int:
    """Rows per split: preds[k * (N // splits) : (k + 1) * (N // splits)], the N % splits last rows unused."""
    check_splits(N, splits)
    return N // splits


def score(probs: torch.Tensor, splits: int = 1) -> Tuple[np.float64, np.float64]:
    """calculate_is.py:44-57 on (N, 1000) fp32 probabilities on the device: per split, exp of the mean
    scipy.stats.entropy(p(y|x), p(y)), then (np.mean, np.std) over the splits."""
    if not isinstance(probs, torch.Tensor) or probs.dtype != torch.float32 or probs.dim() != 2 or probs.shape[1] < 1:
        raise ValueError(f"score takes (N, classes) fp32 probabilities, got {getattr(probs, 'shape', type(probs))}")
    check_device(probs.device)
    N, C = (int(v) for v in probs.shape)
    n = split_rows(N, splits)
    p = probs.contiguous()
    col_mean = torch.empty(splits, C, dtype=torch.float64, device=p.device)
    kl = torch.empty(splits, dtype=torch.float64, device=p.device)
    with torch.cuda.device(p.device):
        _cabi.call("omt_inception_score", p, C, C, n, splits, col_mean, kl)
    split_scores = np.exp(kl.cpu().numpy())
    return np.mean(split_scores), np.std(split_scores)


def _model(model) -> ISInception:
    if not isinstance(model, ISInception):
        raise TypeError("model= must be an ISInception (load_is_model(device, path)); no weights are downloaded")
    return model


def calculate_is(videos, device, splits: int = 1, model: Optional[ISInception] = None):
    """calculate_is (calculate_is.py:13-57) with the network given: videos fp32 (B, T, 3, H, W) as the reference takes
    them, or uint8 (B, T, H, W, 3) standing for byte / 255, on the host or on the network's device.  Every frame is
    resized to 299 x 299.  Returns (mean, std) of the split scores."""
    model = _model(model)
    if check_device(device) != model.device:
        raise ValueError(f"calculate_is: device {device}, the network is on {model.device}")
    if not isinstance(videos, torch.Tensor) or videos.dim() != 5:
        raise ValueError(f"calculate_is takes a (B, T, 3, H, W) fp32 or (B, T, H, W, 3) uint8 tensor, got "
                         f"{getattr(videos, 'shape', type(videos))}")
    frames = videos.reshape(videos.shape[0] * videos.shape[1], *videos.shape[2:])
    check_frames(frames, True)
    check_splits(frames.shape[0], splits)
    if frames.device.type == "cuda" and frames.device != model.device:
        raise ValueError(f"calculate_is: videos on {frames.device}, the network is on {model.device}")
    return score(model.probabilities(frames.to(model.device), resize=True), splits)


def inception_score(imgs, cuda: bool = True, batch_size: int = 32, resize: bool = False, splits: int = 1,
                    model: Optional[ISInception] = None):
    """inception_score (calculate_is.py:61-116) with the network given: imgs an (N, 3, H, W) fp32 tensor (or uint8
    (N, H, W, 3) standing for byte / 255), or a dataset of (3, H, W) images (torch or numpy, cast to fp32 as the
    reference's batch.type does).  The frames run in the network's own chunks, so batch_size changes nothing but is
    checked as the reference checks it.  Returns (mean, std) of the split scores."""
    model = _model(model)
    if not cuda:
        raise ValueError("inception_score runs on the GPU (cuda=True)")
    if batch_size < 1:
        raise ValueError(f"batch_size must be positive, got {batch_size}")
    if isinstance(imgs, torch.Tensor):
        frames = imgs
    else:
        if len(imgs) < 1:
            raise ValueError("empty image dataset")
        items = [torch.as_tensor(imgs[i]) for i in range(len(imgs))]
        if not all(t.is_floating_point() for t in items):
            raise TypeError("inception_score's datasets hold floating-point (3, H, W) images")
        frames = torch.stack([t.float() for t in items])
    check_frames(frames, resize)
    check_splits(frames.shape[0], splits)
    if frames.device.type == "cuda" and frames.device != model.device:
        raise ValueError(f"inception_score: images on {frames.device}, the network is on {model.device}")
    return score(model.probabilities(frames.to(model.device), resize=resize), splits)


def load_is_model(device, path: str) -> ISInception:
    """inception_v3(pretrained=True, transform_input=False) (calculate_is.py:28) with its weights read from path
    (torchvision's inception_v3_google-0cc3c7bd.pth, not shipped; nothing is downloaded)."""
    return ISInception(torch.load(path, map_location="cpu"), device)
