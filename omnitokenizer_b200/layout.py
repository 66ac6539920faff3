"""Host-side index maps and one-time weight packing for the omnitok_b200 kernels.

Everything here is tiny integer / table work done once per (shape, checkpoint) and uploaded;
the per-token arithmetic all happens in the CUDA kernels.
"""
from __future__ import annotations

import math
from typing import NamedTuple, Tuple

import torch


class U8Norm(NamedTuple):
    """A data pipeline's uint8 -> fp32 normalisation, (u / 255 - mean_c) / std_c per channel in fp32.
    max_test: VideoNorm's `if max(clip) > 1: div_(255)` (OmniTokenizer/video_utils.py:53-54) -- a clip whose largest
    byte is <= 1 is only shifted and scaled, (u - mean_c) / std_c."""
    name: str
    mean: Tuple[float, ...]
    std: Tuple[float, ...]
    max_test: bool = False


def u8_norm_table(norm: U8Norm, channels: int) -> torch.Tensor:
    """fp32 [n_tab, channels, 256]: the value every byte of every channel stands for, computed on the host CPU with the
    pipelines' own torch expression and op order (ToTensor / to_tensor / VideoNorm: / 255; Normalize / VideoNorm:
    .sub_(mean).div_(std) with fp32 mean / std tensors).  Table 0 is the normal mapping; with max_test, table 1 is
    the undivided one.  Kernels only look values up, so they reproduce the pipeline's bits (CUDA would divide by
    multiplying with the reciprocal, which differs in about half of the byte values)."""
    if len(norm.mean) != channels or len(norm.std) != channels:
        raise ValueError(f"normalisation {norm.name!r} has {len(norm.mean)} channels, the model takes {channels}")
    mean = torch.tensor(norm.mean, dtype=torch.float32).view(channels, 1)
    std = torch.tensor(norm.std, dtype=torch.float32).view(channels, 1)
    u = torch.arange(256, dtype=torch.uint8).float().expand(channels, 256).contiguous()
    tabs = [(u / 255.0).sub_(mean).div_(std)]
    if norm.max_test:
        tabs.append(u.clone().sub_(mean).div_(std))
    return torch.stack(tabs).contiguous()


def u8_normalize(frames: torch.Tensor, norm: U8Norm) -> torch.Tensor:
    """(B, T, H, W, C) uint8 -> the (B, C, T, H, W) fp32 video the pipeline hands the model, by table lookup (exact on
    any device).  With max_test the table is chosen per sample from its largest byte, as VideoNorm sees one clip."""
    B, C = frames.shape[0], frames.shape[-1]
    tab = u8_norm_table(norm, C).to(frames.device)
    sel = torch.zeros(B, dtype=torch.long, device=frames.device)
    if norm.max_test and frames.numel() > 0:
        sel = (frames.reshape(B, -1).amax(dim=1) <= 1).long()
    x = frames.permute(0, 4, 1, 2, 3).long()
    return tab[sel.view(B, 1, 1, 1, 1), torch.arange(C, device=frames.device).view(1, C, 1, 1, 1), x]


def peg_neighbour_table(T: int, h: int, w: int, temporal: bool, causal: bool) -> torch.Tensor:
    """int32 [T*h*w, 27]: canonical neighbour row (inside one batch element) of every tap of the
    PEG depthwise 3x3x3 stencil, -1 where the reference zero-pads.

    Spatial transformers see the true (t,h,w) volume.  Temporal transformers hand PEG a
    '(b h w) t d' tensor that the reference reshapes LITERALLY to (b,t,h,w,d)
    (modules/attention.py:313-319), i.e. flat position f = n*T + tau is unravelled over (T,h,w):
    the stencil runs in that scrambled space and is mapped back to canonical rows tau*N + n.
    Padding: (1,1) on h and w, (2,0) on t when causal else (1,1) (attention.py:323-325).
    """
    N = h * w
    tau = torch.arange(T).view(T, 1).expand(T, N).reshape(-1)
    n = torch.arange(N).view(1, N).expand(T, N).reshape(-1)
    f = (n * T + tau) if temporal else (tau * N + n)
    t2 = f // N
    h2 = (f % N) // w
    w2 = f % w
    out = torch.empty(T * N, 27, dtype=torch.int64)
    k = 0
    for kt in range(3):
        tt = t2 + kt - (2 if causal else 1)
        for kh in range(3):
            hh = h2 + kh - 1
            for kw in range(3):
                ww = w2 + kw - 1
                ok = (tt >= 0) & (tt < T) & (hh >= 0) & (hh < h) & (ww >= 0) & (ww < w)
                f2 = (tt * h + hh) * w + ww
                r2 = (f2 % T) * N + (f2 // T) if temporal else f2
                out[:, k] = torch.where(ok, r2, torch.full_like(r2, -1))
                k += 1
    return out.to(torch.int32)


def rope_tables(N: int, dim_head: int, theta: float = 10000.0) -> Tuple[torch.Tensor, torch.Tensor]:
    """(cos, sin) [N, dim_head/2] of the 2-D axial rope (modules/attention.py:28-44), computed with
    the same torch fp32 ops as the reference so the table is bit-identical to its freqs_cis."""
    H = int(N ** 0.5)
    pos = torch.arange(N)
    x_pos, y_pos = pos % H, pos // H
    freqs = 1.0 / (theta ** (torch.arange(0, dim_head, 4)[: (dim_head // 4)].float() / dim_head))
    xf = torch.outer(x_pos, freqs).float()
    yf = torch.outer(y_pos, freqs).float()
    x_cis = torch.polar(torch.ones_like(xf), xf)
    y_cis = torch.polar(torch.ones_like(yf), yf)
    cis = torch.cat([x_cis.unsqueeze(-1), y_cis.unsqueeze(-1)], dim=-1).reshape(N, -1)
    return cis.real.contiguous().float(), cis.imag.contiguous().float()


def window_bias(table: torch.Tensor, index: torch.Tensor, ws: int) -> torch.Tensor:
    """[heads, ws*ws, ws*ws] gathered relative position bias (modules/attention.py:277-279)."""
    n = ws * ws
    b = table[index.reshape(-1).long()].reshape(n, n, -1)
    return b.permute(2, 0, 1).contiguous().float()


def tf32_round(w: torch.Tensor) -> torch.Tensor:
    """Round fp32 to tf32 (10-bit mantissa), nearest / ties away -- the `cvt.rna.tf32.f32` rule."""
    i = w.contiguous().view(torch.int32)
    return ((i + 0x1000) & -8192).view(torch.float32)


F16X3_LO_SCALE = 2048.0


def split_f16(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Operand planes of the f16x3 tensor-core path (csrc/omt_common.cuh): hi = fp16(w) (round to nearest, saturating)
    and lo = fp16((w - hi) * 2^11); w ~= hi + lo * 2^-11 to 2^-23 |w|.  Same rounding as the device-side split."""
    w = w.float()
    hi = w.clamp(-65504.0, 65504.0).to(torch.float16)
    lo = ((w - hi.float()) * F16X3_LO_SCALE).clamp(-65504.0, 65504.0).to(torch.float16)
    return hi.contiguous(), lo.contiguous()


def split_f16_rs(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, float]:
    """Row-scaled form for a WEIGHT matrix (one scale for the whole matrix): w' = w * 2^e with max |w'| in [2^14, 2^15),
    hi = fp16(w'), lo = fp16(w' - hi) unscaled.  Returns (hi, lo, 2^-e)."""
    w = w.float()
    mx = float(w.abs().max())
    e = 14 - math.floor(math.log2(mx)) if mx > 0 else 0
    e = max(-100, min(100, e))
    ws = w * (2.0 ** e)
    hi = ws.clamp(-65504.0, 65504.0).to(torch.float16)
    lo = (ws - hi.float()).to(torch.float16)
    return hi.contiguous(), lo.contiguous(), 2.0 ** -e


def pow2_scale(bound: float) -> float:
    """The power of two that maps values bounded by `bound` into [2^14, 2^15) (fp16 range with headroom); 1.0 for 0."""
    if not (bound > 0.0) or not math.isfinite(bound):
        return 1.0
    return 2.0 ** max(-100, min(100, 14 - math.floor(math.log2(bound))))


def split_rows_rs(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Row-scaled form of an activation matrix, the host twin of csrc/omt_common.cuh row_scale(): per row the power of two
    that puts the largest magnitude in [2^14, 2^15).  Returns (hi, lo, inverse row scales [rows])."""
    x = x.float()
    eb = ((x.abs().amax(dim=1).contiguous().view(torch.int32) >> 23) & 0xFF).clamp(15, 254)
    scale = ((268 - eb) << 23).view(torch.float32)
    inv = ((eb - 14) << 23).view(torch.float32)
    xs = x * scale[:, None]
    hi = xs.clamp(-65504.0, 65504.0).to(torch.float16)
    lo = (xs - hi.float()).to(torch.float16)
    return hi.contiguous(), lo.contiguous(), inv.contiguous()


def join_f16(hi: torch.Tensor, lo: torch.Tensor) -> torch.Tensor:
    """fp32 value a pair of operand planes stands for (int16 views are reinterpreted as fp16)."""
    return hi.view(torch.float16).float() + lo.view(torch.float16).float() / F16X3_LO_SCALE


def pad_rows(w: torch.Tensor, mult: int) -> torch.Tensor:
    n = w.shape[0]
    n_pad = (n + mult - 1) // mult * mult
    if n_pad == n:
        return w.contiguous()
    out = torch.zeros(n_pad, w.shape[1], dtype=w.dtype, device=w.device)
    out[:n] = w
    return out


def pad_cols(w: torch.Tensor, k_pad: int) -> torch.Tensor:
    if w.shape[1] == k_pad:
        return w.contiguous()
    out = torch.zeros(w.shape[0], k_pad, dtype=w.dtype, device=w.device)
    out[:, : w.shape[1]] = w
    return out


def pack_geglu(w1: torch.Tensor, inner: int, ku: int) -> torch.Tensor:
    """Interleave FeedForward's first Linear (modules/attention.py:164, rows [value | gate]) so that
    packed rows (2j, 2j+1) = (value_j, gate_j); zero rows pad j up to ku."""
    out = torch.zeros(2 * ku, w1.shape[1], dtype=w1.dtype, device=w1.device)
    out[0: 2 * inner: 2] = w1[:inner]
    out[1: 2 * inner: 2] = w1[inner: 2 * inner]
    return out


def round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def isqrt_exact(n: int) -> int:
    r = int(math.sqrt(n))
    return r
