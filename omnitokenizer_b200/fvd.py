"""The FVD metric's feature network on the device: OmniTokenizer/fvd/fvd.py's preprocess and InceptionI3d
(fvd/pytorch_i3d.py) from device uint8 clips, on the sm_90a kernels of csrc/i3d.cu and csrc/resample.cu.

Drop-in names for vqgan_eval.py:18 (`from OmniTokenizer.fvd.fvd import load_fvd_model, frechet_distance,
get_fvd_logits`): load_fvd_model(device, path), get_fvd_logits(videos, i3d, device), frechet_distance(x1, x2).

The same network also runs evaluation/common_metrics_on_video_quality's StyleGAN-V I3D (fvd/styleganv's
i3d_torchscript.pt, load_i3d_styleganv): the same topology and widths with its own key names, BatchNorm eps 1e-3 and
fixed F.pad tables that equal SAME padding at 224 x 224 (checked per clip length, check_styleganv_pads).  I3D.features
runs either network on one side of quality.calculate_fvd: omt_fvd_suite_preprocess, then the network's CUDA graph.

Activations are channels-last fp32 [B][T][H][W][Cs], Cs the channel count rounded up to a multiple of 32 (4 for the
network input); the pad columns are zero.  Every Unit3D is one omt_conv3d launch (3xTF32, BatchNorm folded into the
weights at pack time), and each Inception branch writes its slice of the block's concat buffer in place.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from . import _cabi
from . import layout as L
from . import metricnet
from .engine import CLIP_DESC_WORDS, run_graphed
# cpad, pack_weight and the FORM_* values stay importable from here: the I3D's channel strides, weight layout and
# SuiteClips forms
from .metricnet import (FORM_F32, FORM_F32_TRUNC, FORM_U8, MAX_WORKSPACES, PackedConv, axis_tables,  # noqa: F401
                        bounded, check_state_dict, clip_descs, cpad, pack_weight, real_byte_table, resolve_device)

TARGET_RESOLUTION = (224, 224)
BN_EPS = 1e-5            # pytorch_i3d.py:91
VARIANT_EPS = {"videogpt": BN_EPS,      # fvd/videogpt/pytorch_i3d.py: the network of OmniTokenizer/fvd
               "styleganv": 1e-3}       # i3d_torchscript.pt: batch_norm(..., 0.1, 0.001)
SUITE_CHUNK_FRAMES = 256  # clip frames per feature launch sequence of I3D.features (about 7 MB of activations each)

# pytorch_i3d.py:247-328: (endpoint, kind, spec); unit: (cin, cout, kernel, stride); pool: (kernel, stride);
# mixed: (cin, branch widths b0, b1a, b1b, b2a, b2b, b3b)
ARCH = [
    ("Conv3d_1a_7x7", "unit", (3, 64, 7, 2)),
    ("MaxPool3d_2a_3x3", "pool", ((1, 3, 3), (1, 2, 2))),
    ("Conv3d_2b_1x1", "unit", (64, 64, 1, 1)),
    ("Conv3d_2c_3x3", "unit", (64, 192, 3, 1)),
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
# branch unit -> (width index, kernel, input: the block input "x", the pooled input "p" or another branch unit)
BRANCHES = {"b0": (0, 1, "x"), "b1a": (1, 1, "x"), "b1b": (2, 3, "b1a"), "b2a": (3, 1, "x"), "b2b": (4, 3, "b2a"),
            "b3b": (5, 1, "p")}


def fold_bn(w: torch.Tensor, gamma, beta, mean, var, eps: float = BN_EPS) -> Tuple[torch.Tensor, torch.Tensor]:
    """metricnet.fold_bn with eps 1e-5 (pytorch_i3d.py:91) unless given."""
    return metricnet.fold_bn(w, gamma, beta, mean, var, eps)


def compute_pad(k: int, s: int, n: int) -> int:
    """pytorch_i3d.py:26-30 / 93-97: the total SAME padding of one axis (pad // 2 goes in front)."""
    return max(k - s, 0) if n % s == 0 else max(k - n % s, 0)


def same_geometry(kernel, stride, dims) -> Tuple[Tuple[int, ...], Tuple[int, ...]]:
    """(front padding, output size) per axis of a SAME-padded conv / pool over dims."""
    front, out = [], []
    for k, s, n in zip(kernel, stride, dims):
        p = compute_pad(k, s, n)
        front.append(p // 2)
        out.append((n + p - k) // s + 1)
    return tuple(front), tuple(out)


def unit_names() -> List[Tuple[str, int, int, int, int]]:
    """Every Unit3D with BatchNorm: (prefix, cin, cout, kernel, stride), in the reference's order."""
    out = []
    for name, kind, spec in ARCH:
        if kind == "unit":
            out.append((name,) + spec)
        elif kind == "mixed":
            cin, w = spec
            for b, (wi, k, src) in BRANCHES.items():
                out.append((f"{name}.{b}", cin if src in ("x", "p") else w[BRANCHES[src][0]], w[wi], k, 1))
    return out


def expected_keys(num_classes: int = 400) -> Dict[str, tuple]:
    keys = {}
    for prefix, cin, cout, k, _ in unit_names():
        keys[prefix + ".conv3d.weight"] = (cout, cin, k, k, k)
        for f in ("weight", "bias", "running_mean", "running_var"):
            keys[f"{prefix}.bn.{f}"] = (cout,)
    keys["logits.conv3d.weight"] = (num_classes, 1024, 1, 1, 1)
    keys["logits.conv3d.bias"] = (num_classes,)
    return keys


class _Workspace:
    """Buffers, launch list and CUDA graph state of one (B, T, H, W)."""

    def __init__(self, net: "I3D", B: int, T: int, H: Optional[int], W: Optional[int],
                 real_norm: Optional[L.U8Norm] = None):
        """H = W = None: the network alone; the caller writes the input self.x (I3D.features)."""
        dev = net.device
        self.graphs = {}
        oh, ow = TARGET_RESOLUTION
        if net.variant == "styleganv":
            check_styleganv_pads(T)
        self.ops = []
        f = dict(device=dev, dtype=torch.float32)

        def act(T_, H_, W_, c):
            return torch.zeros(B, T_, H_, W_, cpad(c), **f)       # pad columns stay zero: no kernel writes them

        x = self.x = act(T, oh, ow, 3)
        self.out = torch.empty(B, net.num_classes, device=dev)
        if H is not None:
            self._preprocess(net, B, T, H, W, real_norm, x)
        self._network(net, B, T, x, act)

    def _preprocess(self, net: "I3D", B: int, T: int, H: int, W: int, real_norm: Optional[L.U8Norm], x):
        dev = net.device
        self.u8 = torch.empty(B, T, H, W, 3, dtype=torch.uint8, device=dev)
        # byte -> value table: float(byte), or the real-byte map of real_norm, picked per clip with VideoNorm's test
        self.lut = net.byte_lut if real_norm is None else real_byte_table(real_norm).float().to(dev)
        self.sel = torch.empty(B, dtype=torch.int32, device=dev) if real_norm is not None and real_norm.max_test else None
        # preprocess tables (fvd.py:24: F.interpolate to 224 x 224 from the multi-threaded script: the separable kernel)
        oh, ow = TARGET_RESOLUTION
        self.tab_host, self.desc_host = axis_tables(H, W, oh, ow), clip_descs(B, T * H * W * 3, H, W, oh, ow)
        self.desc, self.tab = self.desc_host.to(dev), self.tab_host.to(dev)
        if self.sel is not None:
            self.ops.append(lambda: _cabi.call("omt_u8_norm_select", self.u8, B, T * H * W * 3, self.sel))
        self.ops.append(lambda x=x: _cabi.call(
            "omt_fvd_preprocess", self.u8, self.u8.numel(), self.desc, self.desc_host, self.tab, self.tab_host,
            self.tab_host.numel(), self.lut, self.sel, B, T, oh, ow, x))

    def _network(self, net: "I3D", B: int, T: int, x, act):
        shape = (T,) + TARGET_RESOLUTION
        cur, c_cur = x, 3
        for name, kind, spec in ARCH:
            if kind == "unit":
                y, yshape = self._conv(net.units[name], cur, shape, act)
                cur, c_cur, shape = y, spec[1], yshape
            elif kind == "pool":
                cur, shape = self._pool(cur, shape, spec[0], spec[1], act, c_cur)
            else:
                cin, w = spec
                cout = w[0] + w[2] + w[4] + w[5]
                y = act(*shape, cout)
                offs = {"b0": 0, "b1b": w[0], "b2b": w[0] + w[2], "b3b": w[0] + w[2] + w[4]}
                pooled, _ = self._pool(cur, shape, (3, 3, 3), (1, 1, 1), act, cin)
                mids = {}
                for b in ("b0", "b1a", "b1b", "b2a", "b2b", "b3b"):
                    wi, k, src = BRANCHES[b]
                    inp = {"x": cur, "p": pooled}.get(src, mids.get(src))
                    if b in offs:
                        self._conv(net.units[f"{name}.{b}"], inp, shape, act, out=(y, offs[b]))
                    else:
                        mids[b], _ = self._conv(net.units[f"{name}.{b}"], inp, shape, act)
                cur, c_cur = y, cout
        T5 = shape[0]
        if shape[1:] != (7, 7) or T5 < 2:
            raise ValueError(f"the I3D head needs [>= 2, 7, 7] features, got {shape}")
        self.ops.append(lambda cur=cur, T5=T5: _cabi.call(
            "omt_i3d_head", cur, cur.shape[-1], 1024, B, T5, net.head_w, net.head_b, net.num_classes, self.out))

    def _conv(self, u: PackedConv, x, shape, act, out=None):
        front, o = same_geometry(u.k, u.stride, shape)
        y, col = (act(*o, u.cout), 0) if out is None else out
        self.ops.append(u.launch(x, x.shape[0], shape, front, o, y, col))
        return y, o

    def _pool(self, x, shape, k, s, act, c):
        front, o = same_geometry(k, s, shape)
        y = act(*o, c)
        B = x.shape[0]
        self.ops.append(lambda: _cabi.call("omt_maxpool3d", x, x.shape[-1], B, *shape, *k, *s, *front, *o, y))
        return y, o

    def run(self):
        for op in self.ops:
            op()


class I3D:
    """InceptionI3d (pytorch_i3d.py:163-365) in eval mode from a state_dict in the reference's layout
    (`Conv3d_1a_7x7.conv3d.weight`, `Mixed_4e.b1b.bn.running_var`, ..., `logits.conv3d.{weight,bias}`).  BatchNorm is
    folded and the weights packed once, on `device`; every (B, T, H, W) gets its own buffers and CUDA graph (the last
    few are kept).
    variant: "videogpt" (this network, BatchNorm eps 1e-5) or "styleganv" (the StyleGAN-V I3D's weights mapped onto
    these keys by styleganv_state_dict, eps 1e-3; see load_i3d_styleganv)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device="cuda", variant: str = "videogpt"):
        if variant not in VARIANT_EPS:
            raise ValueError(f"unknown I3D variant {variant!r}; expected one of {sorted(VARIANT_EPS)}")
        self.variant = variant
        sd = {k: v for k, v in state_dict.items() if not k.endswith(".num_batches_tracked")}
        lw = sd.get("logits.conv3d.weight")
        self.num_classes = int(lw.shape[0]) if lw is not None and lw.dim() == 5 else 400
        check_state_dict(sd, expected_keys(self.num_classes), "I3D")
        self.device = resolve_device(device)
        sd = {k: v.detach().float().cpu() for k, v in sd.items()}
        self.units = {}
        for prefix, _, _, _, s in unit_names():
            bn = (sd[f"{prefix}.bn.{f}"] for f in ("weight", "bias", "running_mean", "running_var"))
            w, b = fold_bn(sd[prefix + ".conv3d.weight"], *bn, eps=VARIANT_EPS[variant])
            self.units[prefix] = PackedConv(w, b, self.device, stride=(s,) * 3)
        self.head_w = sd["logits.conv3d.weight"].reshape(self.num_classes, 1024).contiguous().to(self.device)
        self.head_b = sd["logits.conv3d.bias"].contiguous().to(self.device)
        self.byte_lut = torch.arange(256, dtype=torch.float32).to(self.device)     # torch.FloatTensor(videos)
        self._ws = {}
        self._suite_ws = {}

    @staticmethod
    def check_frames(frames: torch.Tensor):
        if not isinstance(frames, torch.Tensor) or frames.dtype != torch.uint8:
            raise TypeError(f"I3D.logits takes a uint8 tensor, got {getattr(frames, 'dtype', type(frames))}")
        if frames.dim() != 5 or frames.shape[-1] != 3:
            raise ValueError(f"I3D.logits takes (B, T, H, W, 3) frames, got {tuple(frames.shape)}")
        if frames.shape[1] < 9:
            raise ValueError(f"I3D needs T >= 9 frames (its AvgPool3d spans 2 time steps after 8x temporal "
                             f"downsampling), got T={frames.shape[1]}")
        if min(frames.shape[:4]) < 1:
            raise ValueError(f"empty clip batch {tuple(frames.shape)}")

    def logits(self, frames_u8: torch.Tensor, real_norm: Optional[L.U8Norm] = None) -> torch.Tensor:
        """(B, T, H, W, 3) uint8 on this I3D's device -> logits (B, num_classes) fp32: get_fvd_logits of the reference.
        real_norm: the frames are the loader's bytes, and the network sees the bytes vqgan_eval.py makes of the
        normalised clip, shift_dim((video + 0.5) * 255, 1, -1).byte() (real_byte_table, its branch picked per clip).
        The returned tensor is the workspace's static output: clone it before the next call of the same shape."""
        self.check_frames(frames_u8)
        if self.variant != "videogpt":
            raise ValueError(f"I3D.logits runs OmniTokenizer/fvd's preprocess and network; this is the {self.variant} "
                             f"network (quality.calculate_fvd runs it)")
        if frames_u8.device != self.device:
            raise ValueError(f"I3D.logits: frames on {frames_u8.device}, the network is on {self.device}")
        if real_norm is not None:
            real_byte_table(real_norm)                      # refuses a per-channel normalisation before any launch
        key = tuple(int(v) for v in frames_u8.shape[:4]) + (real_norm,)
        ws = bounded(self._ws, MAX_WORKSPACES, key, lambda: _Workspace(self, *key))
        ws.u8.copy_(frames_u8)
        run_graphed(ws.graphs, self.device, "i3d", ws.run)
        return ws.out

    def features(self, clips: "SuiteClips", t: int) -> torch.Tensor:
        """The network's features (B, num_classes) fp32 on the device of the first t frames of every clip of one
        calculate_fvd side, in chunks of at most SUITE_CHUNK_FRAMES frames: each chunk is one omt_fvd_suite_preprocess
        launch reading the clips in place, then the (chunk, t) workspace's CUDA graph."""
        if clips.src.device != self.device:
            raise ValueError(f"I3D.features: clips on {clips.src.device}, the network is on {self.device}")
        if not 1 <= t <= clips.T:
            raise ValueError(f"I3D.features: prefix of {t} frames of {clips.T}-frame clips")
        B = clips.B
        out = torch.empty(B, self.num_classes, device=self.device)
        chunk = max(1, min(B, SUITE_CHUNK_FRAMES // t))
        oh, ow = TARGET_RESOLUTION
        for b0 in range(0, B, chunk):
            n = min(chunk, B - b0)
            ws = bounded(self._suite_ws, MAX_WORKSPACES, (n, t), lambda: _Workspace(self, n, t, None, None))
            _cabi.call("omt_fvd_suite_preprocess", clips.src, clips.src.numel(), clips.form, clips.C,
                       clips.desc.data_ptr() + b0 * 4 * CLIP_DESC_WORDS, clips.desc_host[b0:], clips.tab, clips.tab_host,
                       clips.tab_host.numel(), n, t, oh, ow, ws.x)
            run_graphed(ws.graphs, self.device, "i3d", ws.run)
            out[b0:b0 + n] = ws.out
        return out


def suite_geometry(H: int, W: int, resolution: int = 224) -> Tuple[int, int, int, int]:
    """preprocess_single's resize and crop (fvd/styleganv/fvd.py:38-64, fvd/videogpt/fvd.py:21-49): the shorter side
    scaled to `resolution` with the longer one's size ceil(n * resolution / min(H, W)) in Python's double, then the
    centre crop at ((rh - resolution) // 2, (rw - resolution) // 2).  Returns (rh, rw, cy, cx)."""
    scale = resolution / min(H, W)
    rh, rw = (resolution, math.ceil(W * scale)) if H < W else (math.ceil(H * scale), resolution)
    return rh, rw, (rh - resolution) // 2, (rw - resolution) // 2


class SuiteClips:
    """One side of quality.calculate_fvd on the device, read in place by omt_fvd_suite_preprocess: src is uint8
    (B, T, H, W, 3) (form FORM_U8) or fp32 (B, T, C, H, W) (FORM_F32, FORM_F32_TRUNC), contiguous; the descriptors
    point at each clip's first frame with the full T stride, so every prefix length reads the same buffer.  Both
    methods' F.interpolate calls take torch's generic bilinear kernel (layout.INTERP_SEPARABLE): styleganv's
    (C, t, H, W) view always, videogpt's contiguous (t, 3, H, W) batch whenever torch runs on more than one thread."""

    def __init__(self, src: torch.Tensor, form: int):
        self.src, self.form = src, form
        if form == FORM_U8:
            self.B, self.T, H, W, self.C = (int(v) for v in src.shape)
            frame = H * W * 3
        else:
            self.B, self.T, self.C, H, W = (int(v) for v in src.shape)
            frame = self.C * H * W
        self.H, self.W = H, W
        rh, rw, cy, cx = suite_geometry(H, W)
        self.tab_host = axis_tables(H, W, rh, rw)
        self.desc_host = clip_descs(self.B, self.T * frame, H, W, rh, rw, cy, cx)
        self.desc, self.tab = self.desc_host.to(src.device), self.tab_host.to(src.device)


# ------------------------------------------------------------------------------------------------ StyleGAN-V I3D
# i3d_torchscript.pt's module names -> this network's
_SGV_UNITS = {"conv3d_1a_7x7": "Conv3d_1a_7x7", "conv3d_2b_1x1": "Conv3d_2b_1x1", "conv3d_2c_3x3": "Conv3d_2c_3x3"}
_SGV_BRANCHES = {"branch_0": "b0", "branch_1.0": "b1a", "branch_1.1": "b1b", "branch_2.0": "b2a", "branch_2.1": "b2b",
                 "branch_3.1": "b3b"}
_SGV_FIELDS = {"conv3d.weight": "conv3d.weight", "batch3d.weight": "bn.weight", "batch3d.bias": "bn.bias",
               "batch3d.running_mean": "bn.running_mean", "batch3d.running_var": "bn.running_var",
               "batch3d.num_batches_tracked": "bn.num_batches_tracked"}

# The torchscript's F.pad tables of every strided layer and of the Inception pool branch, as F.pad's
# (w front, w back, h front, h back, t front, t back): pads[0] when T % stride_t == 0, pads[1] when it is 1.  They are
# fixed for a 224 x 224 input.  Its stride-1 convs pad k // 2 on every side inside conv3d; its max pools run with
# ceil_mode=True after the zero F.pad.
STYLEGANV_PADS = {
    "Conv3d_1a_7x7": ((7, 7, 7), (2, 2, 2), ((2, 3, 2, 3, 2, 3), (2, 3, 2, 3, 3, 3))),
    "MaxPool3d_2a_3x3": ((1, 3, 3), (1, 2, 2), ((0, 1, 0, 1, 0, 0), None)),
    "MaxPool3d_3a_3x3": ((1, 3, 3), (1, 2, 2), ((0, 1, 0, 1, 0, 0), None)),
    "MaxPool3d_4a_3x3": ((3, 3, 3), (2, 2, 2), ((0, 1, 0, 1, 0, 1), (0, 1, 0, 1, 1, 1))),
    "MaxPool3d_5a_2x2": ((2, 2, 2), (2, 2, 2), ((0, 0, 0, 0, 0, 0), (0, 0, 0, 0, 0, 1))),
    "branch_3.0": ((3, 3, 3), (1, 1, 1), ((1, 1, 1, 1, 1, 1), None)),
}


def styleganv_key(key: str) -> str:
    """One i3d_torchscript.pt state_dict key in this network's layout (KeyError for a key the network does not have)."""
    if key.startswith("conv3d_0c_1x1.conv3d."):
        return "logits.conv3d." + key[len("conv3d_0c_1x1.conv3d."):]
    head, _, rest = key.partition(".")
    if head in _SGV_UNITS and rest in _SGV_FIELDS:
        return f"{_SGV_UNITS[head]}.{_SGV_FIELDS[rest]}"
    if head.startswith("mixed_"):
        for b, name in _SGV_BRANCHES.items():
            if rest.startswith(b + ".") and rest[len(b) + 1:] in _SGV_FIELDS:
                return f"Mixed_{head[len('mixed_'):]}.{name}.{_SGV_FIELDS[rest[len(b) + 1:]]}"
    raise KeyError(f"StyleGAN-V I3D state_dict: unexpected key {key}")


def styleganv_state_dict(state_dict: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """i3d_torchscript.pt's state_dict (`conv3d_1a_7x7.batch3d.running_var`, `mixed_4e.branch_1.1.conv3d.weight`,
    `conv3d_0c_1x1.conv3d.bias`, ...) under this network's keys."""
    return {styleganv_key(k): v for k, v in state_dict.items()}


def _scripted_pads(module) -> Dict[str, tuple]:
    """The F.pad tables of a loaded i3d_torchscript.pt, in STYLEGANV_PADS's layout."""
    names = {"Conv3d_1a_7x7": "conv3d_1a_7x7", "MaxPool3d_2a_3x3": "maxPool3d_2a_3x3",
             "MaxPool3d_3a_3x3": "maxPool3d_3a_3x3", "MaxPool3d_4a_3x3": "maxPool3d_4a_3x3",
             "MaxPool3d_5a_2x2": "maxPool3d_5a_2x2"}
    mods = [(k, getattr(module, v)) for k, v in names.items()]
    mods += [("branch_3.0", getattr(getattr(module, name.lower()).branch_3, "0")) for name, kind, _ in ARCH
             if kind == "mixed"]
    out = {}
    for k, m in mods:
        tabs = [getattr(getattr(m.pads, i), "padding", None) for i in ("0", "1")]
        tabs = tuple(tuple(int(v) for v in p) if p is not None else None for p in tabs)
        if out.setdefault(k, tabs) != tabs:
            raise ValueError(f"StyleGAN-V I3D: the Inception pool branches differ in their pad tables ({tabs})")
    return out


def check_styleganv_pads(T: int, H: int = 224, W: int = 224, pads: Optional[Dict[str, tuple]] = None):
    """pads: {layer: (pads[0], pads[1])} to check instead of STYLEGANV_PADS's tables (e.g. a loaded torchscript's).

    The StyleGAN-V I3D on a (T, H, W) input computes what omt_conv3d / omt_maxpool3d compute with SAME padding
    (same_geometry): at every strided layer and Inception pool branch, the F.pad table the torchscript picks for the
    layer's input length equals SAME's front / back padding, ceil_mode adds no window ((n + pad - k) % s == 0 on every
    axis), and the zero padding of a max pool reads post-ReLU values (>= 0), so it never wins where SAME's does not.
    Raises ValueError naming the first layer that differs."""
    pads = {k: v[2] for k, v in STYLEGANV_PADS.items()} if pads is None else pads
    shape = (T, H, W)

    def check(name, dims):
        k, s, _ = STYLEGANV_PADS[name]
        tabs = pads[name]
        r = dims[0] % s[0]
        tab = tabs[r] if r < 2 else None
        if tab is None:
            raise ValueError(f"StyleGAN-V I3D {name}: no pad table for T % {s[0]} == {r}")
        fb = [(tab[4], tab[5]), (tab[2], tab[3]), (tab[0], tab[1])]
        front, out = same_geometry(k, s, dims)
        for ax, (kk, ss, n) in enumerate(zip(k, s, dims)):
            p = compute_pad(kk, ss, n)
            if fb[ax] != (front[ax], p - front[ax]) or (n + p - kk) % ss:
                raise ValueError(f"StyleGAN-V I3D {name} at input {tuple(dims)}: F.pad {tab} is not SAME padding "
                                 f"{front} / {p} on axis {ax} or ceil_mode adds a window")
        return out

    for name, kind, spec in ARCH:
        if kind == "unit":
            if name in STYLEGANV_PADS:
                shape = check(name, shape)
            else:
                shape = same_geometry((spec[2],) * 3, (spec[3],) * 3, shape)[1]
        elif kind == "pool":
            shape = check(name, shape)
        else:
            check("branch_3.0", shape)
    if shape[1:] != (7, 7) or shape[0] < 2:
        raise ValueError(f"the I3D head needs [>= 2, 7, 7] features, got {shape} for a {T} x {H} x {W} input")


def load_i3d_styleganv(device, path) -> I3D:
    """The StyleGAN-V I3D of evaluation/common_metrics_on_video_quality/fvd/styleganv (load_i3d_pretrained) from
    `path`: its i3d_torchscript.pt (read with torch.jit.load; its pad tables are checked against STYLEGANV_PADS), a
    plain state_dict file in either key layout, or a state_dict.  Nothing is downloaded."""
    if isinstance(path, dict):
        sd = path
    else:
        try:
            module = torch.jit.load(path, map_location="cpu")
        except (RuntimeError, ValueError):
            module = None
        if module is not None:
            scripted = _scripted_pads(module)
            if scripted != {k: v[2] for k, v in STYLEGANV_PADS.items()}:
                raise ValueError(f"{path}: pad tables {scripted} are not the StyleGAN-V I3D's")
            sd = module.state_dict()
        else:
            sd = torch.load(path, map_location="cpu")
    if any(k.startswith(("conv3d_", "mixed_")) for k in sd):
        sd = styleganv_state_dict(sd)
    return I3D(sd, device, variant="styleganv")


def load_fvd_model(device, path: str) -> I3D:
    """fvd.py:36-42 with the checkpoint path given (the weights are not shipped): i3d_pretrained_400.pt."""
    return I3D(torch.load(path, map_location="cpu"), device)


def get_fvd_logits(videos, i3d: I3D, device=None) -> torch.Tensor:
    """fvd.py:31-34: numpy or torch uint8 (b, t, h, w, c) on the CPU or the device -> logits (b, num_classes) on the
    device.  Host input is copied as uint8 (a quarter of the bytes of the reference's fp32 copy)."""
    if isinstance(videos, np.ndarray):
        videos = torch.from_numpy(np.ascontiguousarray(videos))
    I3D.check_frames(videos)
    return i3d.logits(videos.to(i3d.device, non_blocking=False)).clone()


def frechet_distance(x1: torch.Tensor, x2: torch.Tensor) -> torch.Tensor:
    """fvd.py:101-112 (with _symmetric_matrix_square_root, trace_sqrt_product and cov, :56-98): the Frechet distance
    between two sets of embeddings.  Runs once per split in torch; it is not a kernel."""
    def sqrtm(mat, eps=1e-10):
        u, s, v = torch.svd(mat)
        return u @ torch.diag(torch.where(s < eps, s, torch.sqrt(s))) @ v.t()

    def cov(m):
        m = m.t()
        c = m - m.mean(dim=1, keepdim=True)
        return (1.0 / (m.size(1) - 1)) * (c @ c.t()).squeeze()

    x1, x2 = x1.flatten(start_dim=1), x2.flatten(start_dim=1)
    sigma, sigma_w = cov(x1), cov(x2)
    r = sqrtm(sigma)
    trace = torch.trace(sigma + sigma_w) - 2.0 * torch.trace(sqrtm(r @ (sigma_w @ r)))
    return trace + torch.sum((x1.mean(dim=0) - x2.mean(dim=0)) ** 2)
