"""Host setup shared by the metric networks (fid.py, fvd.py, quality.py, iscore.py): the state_dict check, device
resolution, BatchNorm folding, conv weights packed for omt_conv3d, bounded workspace caches, the byte tables of the
uint8 inputs, and the axis tables and omt_clip_desc rows of the clip preprocess kernels.  Each network keeps its own
topology, launch walk, workspaces and input checks.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import _cabi
from . import layout as L
from .engine import CLIP_DESC_WORDS

FORM_U8, FORM_F32, FORM_F32_TRUNC = 0, 1, 2      # OMT_FVDS_U8 / OMT_FVDS_F32 / OMT_FVDS_F32_TRUNC
MAX_WORKSPACES = 4       # workspaces (buffers and CUDA graphs) a network keeps per cache; the oldest goes first


def check_state_dict(sd: Dict[str, torch.Tensor], want: Dict[str, tuple], what: str):
    """Refuses a state_dict whose keys differ from want's (KeyError naming every missing and unexpected key) or whose
    first mis-shaped tensor differs from want's shape (ValueError)."""
    missing, unexpected = sorted(set(want) - set(sd)), sorted(set(sd) - set(want))
    if missing or unexpected:
        raise KeyError(f"{what} state_dict: missing keys {missing}, unexpected keys {unexpected}")
    for k, shape in want.items():
        if tuple(sd[k].shape) != shape:
            raise ValueError(f"{what} state_dict: {k} has shape {tuple(sd[k].shape)}, expected {shape}")


def resolve_device(device) -> torch.device:
    """torch.device(device), with a CUDA device without an index (vqgan_eval.py passes torch.device('cuda')) taken as
    the current one."""
    dev = torch.device(device)
    if dev.type == "cuda" and dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    return dev


def fold_bn(w: torch.Tensor, gamma, beta, mean, var, eps: float) -> Tuple[torch.Tensor, torch.Tensor]:
    """BatchNorm (running statistics) folded into a conv weight (cout, cin, ...) of any rank, in float64:
    (W s, beta - mean s) with s = gamma / sqrt(var + eps), rounded to fp32."""
    s = gamma.double() / torch.sqrt(var.double() + eps)
    return (w.double() * s.view(-1, *(1,) * (w.dim() - 1))).float(), (beta.double() - mean.double() * s).float()


def cpad(c: int) -> int:
    """Channel stride of an activation with c channels: 4 for the RGB input, else a multiple of 32."""
    return 4 if c <= 4 else L.round_up(c, 32)


def pack_weight(w: torch.Tensor) -> Tuple[torch.Tensor, int]:
    """A conv weight (cout, cin, kt, kh, kw) as omt_conv3d's W: rows of K = (dt, dh, dw, c) with c padded to cpad(cin)
    (K rounded up to 32 for the RGB input), cout padded to a multiple of 128.  Returns (W [n_pad, K] fp32, K)."""
    cout, cin = int(w.shape[0]), int(w.shape[1])
    wk = torch.zeros(cout, *w.shape[2:], cpad(cin))
    wk[..., :cin] = w.float().permute(0, 2, 3, 4, 1)
    wk = wk.reshape(cout, -1)
    K = L.round_up(wk.shape[1], 32)
    packed = torch.zeros(L.round_up(cout, 128), K)
    packed[:cout, :wk.shape[1]] = wk
    return packed, K


class PackedConv:
    """One conv packed for omt_conv3d on `device`: the tf32 hi / lo planes of W (pack_weight), the bias, the kernel
    (kt, kh, kw) of the (cout, cin, [kt,] kh, kw) weight (kt 1 for a 2-D one), the stride, and the network's own
    geometry record `conv`."""

    def __init__(self, w: torch.Tensor, bias: torch.Tensor, device, conv=None, stride: Tuple[int, int, int] = (1, 1, 1)):
        w = w.float()
        if w.dim() == 4:
            w = w.unsqueeze(2)
        packed, self.K = pack_weight(w)
        hi = L.tf32_round(packed)
        self.w_hi, self.w_lo = hi.to(device), (packed - hi).to(device)
        self.bias = bias.float().contiguous().to(device)
        self.cout, self.k, self.stride, self.conv = int(w.shape[0]), tuple(w.shape[2:]), tuple(stride), conv

    def launch(self, x, B: int, dims, front, out, y, col: int = 0, relu: int = 1):
        """The omt_conv3d launch of this conv over x, channels-last (B, *dims, Cs), with `front` padding per axis, into
        columns col onwards of y, channels-last (B, *out, ldy).  The closure holds x and y themselves, not only their
        addresses, and looks _cabi.call up when it runs, so a wrapper of _cabi.call sees every launch."""
        ypt = y.data_ptr() + 4 * col
        return lambda: _cabi.call(
            "omt_conv3d", x, x.shape[-1], B, *dims, self.w_hi, self.w_lo, self.K, self.bias, self.cout,
            *self.k, *self.stride, *front, *out, ypt, y.shape[-1], relu)


def bounded(cache: dict, cap: int, key, make):
    """cache[key], made by make() when it is missing, after dropping the oldest entries so that at most cap stay."""
    v = cache.get(key)
    if v is None:
        while len(cache) >= cap:
            cache.pop(next(iter(cache)))
        v = cache[key] = make()
    return v


def real_byte_table(norm: L.U8Norm) -> torch.Tensor:
    """uint8 [n_tab, 256]: the byte vqgan_eval.py feeds the metric networks for each loader byte u of a real clip,
    ((v + 0.5) * 255).byte() (:144, :156) of the normalised value v (layout.u8_norm_table, fp32, its own op order).
    Table 1 (VideoNorm's max <= 1 branch) is only used for clips whose bytes are all 0 or 1."""
    tab = L.u8_norm_table(norm, 3)                          # [n_tab, 3, 256]
    if not bool((tab == tab[:, :1]).all()):
        raise ValueError(f"normalisation {norm.name!r} differs per channel; the FVD byte map is one table per branch")
    return ((tab[:, 0] + 0.5) * 255).byte()


def byte_lut(real_norm: Optional[L.U8Norm] = None) -> torch.Tensor:
    """fp32 [n_tab, 256]: the value the network's input takes for each byte before the resize: ToTensor's byte / 255
    (fid_score.py:146), or, for the loader's bytes of a real image, / 255 of the byte vqgan_eval.py saves for it,
    ((v + 0.5) * 255).astype(uint8) of the normalised value v (:205; real_byte_table)."""
    b = torch.arange(256, dtype=torch.float32).view(1, 256) if real_norm is None else real_byte_table(real_norm).float()
    return b / 255


def axis_table(n_in: int, n_out: Optional[int]) -> np.ndarray:
    """int32 [n_out, 4] of one axis: torch's bilinear resize of n_in to n_out (layout.clip_axis_table), or, with n_out
    None (no resize), the identity [n_in, 4] of entries (i, i, 1.0, 0.0), whose fma chain reproduces each value."""
    if n_out is None:
        ident = np.zeros((n_in, 4), dtype=np.int32)
        ident[:, 0] = ident[:, 1] = np.arange(n_in)
        ident[:, 2] = np.float32(1).view(np.int32)
        return ident
    return L.clip_axis_table(n_in, n_out, float(np.float32(n_in) / np.float32(n_out)))


def axis_tables(H: int, W: int, rh: Optional[int], rw: Optional[int]) -> torch.Tensor:
    """int32 host tables of an H x W -> rh x rw resize (None: the axis at its own size): the vertical one at word 0,
    the horizontal one after it, at word 4 rh (clip_descs' th)."""
    return torch.from_numpy(np.concatenate([axis_table(H, rh).reshape(-1), axis_table(W, rw).reshape(-1)]))


def clip_descs(B: int, clip_elems: int, H: int, W: int, rh: int, rw: int, cy: int = 0, cx: int = 0) -> torch.Tensor:
    """int32 host omt_clip_desc rows [B, CLIP_DESC_WORDS] of B clips of H x W frames, clip_elems source elements apart
    (words 0-1: clip b's offset b clip_elems): the whole frame, resized to rh x rw through axis_tables(H, W, rh, rw)
    and cropped at (cy, cx), in torch's separable bilinear form."""
    desc = torch.zeros(B, CLIP_DESC_WORDS, dtype=torch.int32)
    desc[:, :2] = (torch.arange(B, dtype=torch.int64) * clip_elems).view(torch.int32).view(B, 2)
    desc[:, 2:] = torch.tensor([H, W, 0, 0, H, W, rh, rw, cy, cx, 0, 0, 4 * rh, L.INTERP_SEPARABLE], dtype=torch.int32)
    return desc
