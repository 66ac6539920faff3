"""Kernel orchestration for OmniTokenizer_VQGAN.encode / decode / forward on one H100.

The engine owns (a) the packed device copies of the checkpoint in kernel layouts and (b) the
per-shape workspace; every arithmetic step is a call into libomnitok_b200.so (see
include/omnitok_b200.h).  torch is used for device memory, streams and a handful of
O(codebook)-sized reductions (usage statistics) -- never for the per-token math.

Activations stay in ONE canonical buffer X[B][T'][N][C] for the whole network.  The reference's
four rearrange copies between spatial and temporal blocks (omnitokenizer.py:891,902,907,1072,1081)
do not exist here: spatial kernels read rows contiguously, temporal kernels stride by N, window
attention and both PEG variants go through index maps.
"""
from __future__ import annotations

import gc
import math
import os
from typing import Dict, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _cabi
from . import layout as L

# f16x1 is the opt-in throughput mode: one fp16 product per tensor-core product, NOT reference-exact (INTEGRATION.md)
MATH_MODES = {"fp32": _cabi.MATH_FP32, "3xtf32": _cabi.MATH_3XTF32, "f16x3": _cabi.MATH_F16X3, "f16x1": _cabi.MATH_F16X1}
DEFAULT_MATH = "f16x3"
PLANE_MATHS = (_cabi.MATH_F16X3, _cabi.MATH_F16X1)    # modes whose GEMM operands are fp16 planes (shared weight packing)
# largest codebook of the VQ search kernel (csrc/vq.cu): an eighth of the table (36 B per code) and the z rows of a 512-row
# block (16 KB) share 200 KB of shared memory.  Launches of few rows take 256-row blocks and would fit 43 648 codes, but a
# codebook must not work for small batches and fail for large ones.
VQ_MAX_CODES = 41856
# longest latent sequence of the temporal attention core (csrc/attention_fp32.cu attn_temporal_kernel keeps the K / V of
# one pixel's T' frames in registers, one template instance per T'): 17 latent frames, 65 frames at temporal patch 4
TEMPORAL_MAX_FRAMES = 17
# longest patch vector (C * pt * p * p features) of the patch gather + LayerNorm (csrc/rowwise.cu omt_patchify_ln, _u8)
PATCH_MAX_K = 1024
# k-block of each math mode's GEMM (csrc/gemm_fp32.cu, gemm_tc2.cu, gemm_f16.cu): a patch vector is a whole number of them
PATCH_K_BLOCK = {_cabi.MATH_FP32: 8, _cabi.MATH_3XTF32: 32, _cabi.MATH_F16X3: 64, _cabi.MATH_F16X1: 64}
# window side of the window attention kernel (csrc/attention_fp32.cu omt_attn_window: 64-token windows)
WINDOW_SIZE = 8
# model widths C (--embedding_dim) the kernels take: LayerNorm holds a row of at most 1024 channels in one warp's registers,
# post_vq / pre_vq / the VQ lookup take C <= 1024, and every width here is a whole number of 256-column GEMM tiles
MODEL_WIDTHS = (256, 512, 768, 1024)
# head dimension of every attention core (AD = 64, the wgmma tiles)
HEAD_DIM = 64
# attention width A = 64 * heads: the fused QKV GEMM switches from the normalised to the raw input at column A, which must
# start a 128-column output tile, so heads is even; 2..16 heads give A = 128..1024
MAX_HEADS = 16
# int32 words of one omt_resample_desc (include/omnitok_b200.h): the int64 source offset, then 16 int32 fields
DESC_WORDS = 18
# int32 words of one omt_clip_desc: the int64 source offset, then 14 int32 fields
CLIP_DESC_WORDS = 16


def default_math() -> str:
    return os.environ.get("OMT_MATH", DEFAULT_MATH).lower()


class Planes:
    """fp16 hi / lo operand planes of an [M, ld] fp32 matrix (the A operands of the f16x3 GEMMs; layout.split_f16)."""

    def __init__(self, device, M: int, ld: int, row_scaled: bool = False):
        self.buf = torch.empty(2, M, ld, device=device, dtype=torch.int16)
        self.hi, self.lo, self.ld = self.buf[0], self.buf[1], ld
        # row-scaled form (written by producers that see whole rows): inverse per-row scales; None = the 2^11-scaled lo form
        self.rs = torch.empty(M, device=device, dtype=torch.float32) if row_scaled else None


class PackedLinear:
    """nn.Linear weight in GEMM layout: rows padded to 128, K padded, optional tf32 hi/lo split.  f16x1 packs the f16x3
    planes and scales and keeps only the hi plane."""

    def __init__(self, weight: torch.Tensor, bias: Optional[torch.Tensor], device, math: int,
                 k_pad: Optional[int] = None, geglu: Optional[Tuple[int, int]] = None, row_scaled: bool = False):
        w = weight.detach().to(device=device, dtype=torch.float32)
        if geglu is not None:
            inner, ku = geglu
            w = L.pack_geglu(w, inner, ku)
        self.n = w.shape[0]
        if k_pad is not None:
            w = L.pad_cols(w, k_pad)
        self.k = w.shape[1]
        w = L.pad_rows(w, 256 if math in PLANE_MATHS else 128)
        if math == _cabi.MATH_3XTF32:
            hi = L.tf32_round(w)
            self.w, self.w_lo = hi, (w - hi).contiguous()
        elif math in PLANE_MATHS and row_scaled:
            self.w, self.w_lo, self.w_scale = L.split_f16_rs(w)      # fp16 planes, one scale per matrix (single-accumulator GEMM)
        elif math in PLANE_MATHS:
            self.w, self.w_lo = L.split_f16(w)          # fp16 operand planes, lo scaled by 2^11 (two-accumulator GEMM)
        else:
            self.w, self.w_lo = w, None
        if math == _cabi.MATH_F16X1:
            self.w_lo = None                            # the single-product GEMM reads the hi plane only
        self.bias = None if bias is None else bias.detach().to(device=device, dtype=torch.float32).contiguous()
        self.math = math
        self.row_scaled = row_scaled and math in PLANE_MATHS


def run_graphed(graphs: dict, device, key, body):
    """Run ``body`` (a fixed launch sequence over static buffers): the first call of a shape runs eagerly
    (sets function attributes, builds tables), the second captures a CUDA graph, later calls replay it --
    ~170 launches per encode+decode collapse into one submission.  ``graphs``: the workspace's key -> graph state."""
    if not Engine.graphs_enabled():
        return body()
    g = graphs.get(key)
    if g is None:
        body()
        graphs[key] = "warm"
    elif g == "warm":
        graph = torch.cuda.CUDAGraph()
        torch.cuda.synchronize(device)
        n0 = _cabi.launch_count
        # An evicted workspace lives on in a reference cycle (its launch closures hold it) until the cyclic collector
        # frees it; freeing its captured graph inside this capture would reset that graph and invalidate the capture.
        collecting = gc.isenabled()
        gc.disable()
        try:
            with torch.cuda.graph(graph):
                body()
        finally:
            if collecting:
                gc.enable()
        graphs[key] = (graph, _cabi.launch_count - n0)
        graph.replay()
    else:
        g[0].replay()
        _cabi.launch_count += g[1]        # kernels inside the replayed graph (bench.py accounting)


class Workspace:
    """Per-shape buffers.  C: model width; A: attention width (q | k | v and the attention output; a window layer, whose
    width is C, runs only in models with C == A)."""

    def __init__(self, device, M: int, C: int, A: int, ku: int, kmax: int, cd: int, planes: bool):
        f = dict(device=device, dtype=torch.float32)
        self.M = M
        self.buf0 = torch.empty(M, C, **f)
        self.buf1 = torch.empty(M, C, **f)
        self.X, self.Y = self.buf0, self.buf1
        self.QKV = torch.empty(M, 3 * A, **f)
        self.P = torch.empty(M, kmax, **f)       # patch matrix (pixels side), rows x K
        if planes:     # f16x3: every GEMM A operand lives as fp16 hi / lo planes written by its producer
            self.XNp, self.XSp = Planes(device, M, C, True), Planes(device, M, C, True)     # LayerNorm sees whole rows
            self.Op, self.Up = Planes(device, M, A), Planes(device, M, ku)                  # attention heads / GEGLU tiles do not
            self.Pp = Planes(device, M, kmax, True)
            self.QKVp = Planes(device, M, 3 * A)     # q | k | v operand planes for the f16 attention core (QKV GEMM epilogue)
            self.vinv = torch.empty(A // 64, M, device=device, dtype=torch.float32)   # inverse (row, head) scales of the v planes
        else:
            self.XN = torch.empty(M, C, **f)
            self.O = torch.empty(M, A, **f)
            self.U = torch.empty(M, ku, **f)
        self.z = torch.empty(M, cd, **f)
        self.idx = torch.empty(M, device=device, dtype=torch.int64)
        self.counts = torch.zeros(8192, device=device, dtype=torch.int32)
        self.idx_in = torch.empty(M, device=device, dtype=torch.int64)
        self.zc_in = torch.empty(M, cd, **f)
        self.zq = torch.empty(M, cd, **f)
        # static I/O buffers per slot {slot: (layout key, buffers)} (static()), the layout tables of the layouts they hold
        # (Engine._layout_tables), and the captured CUDA graphs {(slot, layout key, mode, extra): graph state}
        self.sets, self.layout_tables, self.graphs = {}, {}, {}

    def reset(self):
        self.X, self.Y = self.buf0, self.buf1

    def static(self, slot: str, lay_key, make):
        """The static buffers of `slot` for the layout lay_key.  A slot holds one set: a set of another layout replaces
        it (make() builds the new one), which drops exactly the graphs captured over the slot and the layout tables no
        held set uses any more."""
        held = self.sets.get(slot)
        if held is not None and held[0] == lay_key:
            return held[1]
        bufs = make()
        self.sets[slot] = (lay_key, bufs)
        for k in self.graphs_of(slot):
            del self.graphs[k]
        live = {k for k, _ in self.sets.values()}
        self.layout_tables = {k: v for k, v in self.layout_tables.items() if k in live}
        return bufs

    def graphs_of(self, slot: str) -> dict:
        """The graph states captured over the static buffers of `slot`, by graph key."""
        return {k: v for k, v in self.graphs.items() if k[0] == slot}


class Group(NamedTuple):
    """Equal-length samples of a packed batch: n samples of tp latent frames from latent frame f0 on (sorted order s0..)."""
    tp: int
    s0: int
    n: int
    f0: int


class BatchLayout:
    """Where the samples of one pass lie in the canonical buffer X[frames][N][C].  Samples are sorted stably by their
    number of latent frames T', so equal lengths are contiguous (one group each); sample i of the caller's order sits at
    slot[i] = (group, index in the group) and owns latent frames [f_in[i], f_in[i] + tps[i]).  Row-wise kernels never
    see the layout; PEG and temporal attention take the per-sample offsets t_off (device table, a single launch for every
    length); the patch gather / un-patchify and the patch GEMMs run once per group.  A uniform batch is the one-group
    case and runs the uniform kernels (no table)."""

    def __init__(self, tps: Sequence[int], h: int, w: int):
        self.tps = tuple(int(t) for t in tps)
        self.B, self.h, self.w, self.N = len(self.tps), h, w, h * w
        self.order = sorted(range(self.B), key=self.tps.__getitem__)       # stable: equal lengths keep the caller's order
        self.pos = [0] * self.B                                              # caller's sample i -> its sorted position
        for s_, i in enumerate(self.order):
            self.pos[i] = s_
        sorted_tp = [self.tps[i] for i in self.order]
        self.t_off = [0]
        for t in sorted_tp:
            self.t_off.append(self.t_off[-1] + t)
        self.groups: List[Group] = []
        s0 = 0
        while s0 < self.B:
            n = 1
            while s0 + n < self.B and sorted_tp[s0 + n] == sorted_tp[s0]:
                n += 1
            self.groups.append(Group(sorted_tp[s0], s0, n, self.t_off[s0]))
            s0 += n
        self.frames = self.t_off[-1]
        self.M = self.frames * self.N
        self.uniform = len(self.groups) <= 1
        # caller's sample i -> (group, index inside the group) and its first latent frame
        self.slot = [None] * self.B
        self.f_in = [0] * self.B
        for gi, g in enumerate(self.groups):
            for k in range(g.n):
                i = self.order[g.s0 + k]
                self.slot[i] = (gi, k)
                self.f_in[i] = g.f0 + k * g.tp
        # graphs and static I/O buffers are keyed on this (with cin, p, pt it fixes every input and output shape): two
        # layouts with the same M differ here
        self.key = (tuple(sorted_tp), h, w)

    def rows(self, i: int) -> slice:
        """Canonical rows of sample i (caller's order)."""
        return slice(self.f_in[i] * self.N, (self.f_in[i] + self.tps[i]) * self.N)


class Engine:
    def __init__(self, model, device: torch.device, math: Optional[str] = None):
        _cabi.load()
        _cabi.set_option("pdl", int(os.environ.get("OMT_PDL", "0")))     # programmatic dependent launch between kernels
        # process-wide kernel selectors (tuning knobs; see omt_set_option): the environment or the library default
        for env, opt in (("OMT_PEG_KERNEL", "peg_kernel"),        # 4 (cp.async gather, default) | 3
                         ("OMT_ATTN_CTAS", "attn_f16_ctas"),      # CTAs per SM of the f16 attention core
                         ("OMT_F16_BN", "f16_bn")):               # 0 (by shape) | 128 | 256: tile N of the two-accumulator GEMM form
            _cabi.set_option(opt, int(os.environ.get(env) or _cabi.DEFAULT_OPTIONS[opt]))
        self.device = device
        self.math_name = (math or default_math()).lower()
        if self.math_name not in MATH_MODES:
            raise ValueError(f"unknown OMT_MATH mode {self.math_name!r}; choose from {sorted(MATH_MODES)}")
        self.math = MATH_MODES[self.math_name]
        a = model.args
        # C: the model width (LayerNorm, PEG, FF, residual stream); A: the attention width of the temporal / spatial
        # attention blocks, heads x dim_head, independent of C (to_q C -> A, to_kv C -> 2A, to_out A -> C, attention.py:395-486)
        self.C = a.embedding_dim
        self.heads, self.dh = a.heads, a.dim_head
        self.A = self.heads * self.dh
        if self.dh != HEAD_DIM:
            raise NotImplementedError(f"--dim_head {self.dh}: every attention core is built on {HEAD_DIM}-wide heads")
        if self.heads % 2 or not 2 <= self.heads <= MAX_HEADS:
            raise NotImplementedError(f"--heads {self.heads}: the kernels take an even number of heads from 2 to {MAX_HEADS} "
                                      f"(the fused QKV GEMM switches its input at column {HEAD_DIM} x heads, which must start "
                                      "a 128-column output tile)")
        if self.C not in MODEL_WIDTHS:
            raise NotImplementedError(f"--embedding_dim {self.C}: the kernels take model widths {', '.join(map(str, MODEL_WIDTHS))}")
        self.p, self.pt, self.cin = a.patch_size, a.temporal_patch_size, a.image_channels
        self.ws = a.twod_window_size
        self.has_window = "w" in (a.enc_block + a.dec_block)
        if self.has_window and self.ws != WINDOW_SIZE:
            raise NotImplementedError(f"--twod_window_size {self.ws}: omt_attn_window is specialised for "
                                      f"{WINDOW_SIZE}x{WINDOW_SIZE} windows (enc_block {a.enc_block!r}, dec_block {a.dec_block!r})")
        # window attention splits the model width itself into heads of C / heads (attention.py:254-293)
        if self.has_window and self.C != HEAD_DIM * self.heads:
            raise NotImplementedError(f"--heads {self.heads} with --embedding_dim {self.C}: window blocks (enc_block "
                                      f"{a.enc_block!r}, dec_block {a.dec_block!r}) take heads of C / heads = "
                                      f"{self.C / self.heads:g} channels; omt_attn_window takes {HEAD_DIM}")
        self.causal_attn = bool(a.causal_in_temporal_transformer)
        self.causal_peg = bool(a.causal_in_peg)
        self.rope = a.spatial_pos == "rope"
        self.use_vae = bool(model.use_vae)
        self.cd = a.codebook_dim
        self.l2 = bool(a.l2_code)
        if not self.use_vae and self.cd != 8:
            raise NotImplementedError(f"--codebook_dim {self.cd}: the VQ search / post_vq kernels are specialised for "
                                      "codebook_dim 8 (every shipped config); VAE mode takes 8 latent channels as well")
        self.planes = self.math in PLANE_MATHS
        # a first-frame patch vector is K of the encoder's patch GEMM and N of the decoder's to_pixels GEMM (the other
        # frames' vectors are whole multiples of it): it must be a whole k-block of the mode's GEMM
        k_block = PATCH_K_BLOCK[self.math]
        if (self.cin * self.p * self.p) % k_block:
            raise NotImplementedError(f"--patch_size {self.p}: a patch vector of {self.cin * self.p * self.p} features is not "
                                      f"a whole {k_block}-wide k-block of the {self.math_name} GEMM")
        # f16x1: every GEMM and the f16 spatial core take their single-product forms (omt_linear_h1, omt_attn_spatial_h1)
        self.h1 = self.math == _cabi.MATH_F16X1
        # spatial attention core on fp16 operand planes (attention_f16.cu, default); OMT_ATTN_F16=0 = the 3xTF32 core on the fp32 QKV buffer
        self.attn_f16 = self.planes and os.environ.get("OMT_ATTN_F16", "1") == "1"
        # GEGLU output planes with a static (pack-time) scale -> the second FF GEMM takes the single-accumulator form (default).
        # The bound |U| <= (|LN(x)|_2 max|W1_n|_2)^2 is structural (|LN(x)|_2 <= max|gamma| sqrt(C) + |beta|_2), at most ~2^10
        # above typical values, so the planes keep 22 significant bits; OMT_STATIC_U=0 = per-element 2^11 form, two accumulators
        self.static_u = self.planes and os.environ.get("OMT_STATIC_U", "1") == "1"
        if a.attn_dropout != 0 or a.ff_dropout != 0:
            raise NotImplementedError("non-zero dropout reaches SDPA even in eval in the reference (attention.py:451); rejected")
        self._ws: Dict[Tuple, Workspace] = {}
        self._tables: Dict[Tuple, torch.Tensor] = {}
        # omt_resample_u8 input: grow-only pinned staging buffer, its device copy, and the event of the last copy out of it
        self._stage = self._stage_dev = self._stage_done = None
        sd = {k: v for k, v in model.state_dict().items()}
        self._pack(sd, a)

    # ------------------------------------------------------------------ packing
    def _pack(self, sd, a):
        dev, m = self.device, self.math
        f32 = lambda t: t.detach().to(device=dev, dtype=torch.float32).contiguous()
        self.inner = sd["encoder.enc_spatial_transformer.layers.0.3.4.weight"].shape[1]
        self.ku = L.round_up(self.inner, 64 if self.planes else 32)     # K of the second FF GEMM: whole k-blocks

        def PL(weight, bias, **kw):
            return PackedLinear(weight, bias, dev, m, **kw)

        def lin(name, bias=True, **kw):
            return PL(sd[name + ".weight"], sd.get(name + ".bias") if bias else None, **kw)

        def t_layer(lp):
            d = {"kind": "t"}
            d["peg_w"] = f32(sd[lp + ".0.dsconv.weight"].reshape(self.C, 27).t())      # [27, C]
            d["peg_b"] = f32(sd[lp + ".0.dsconv.bias"])
            ap = lp + ".1"
            d["norm_g"], d["norm_b"] = f32(sd[ap + ".norm.gamma"]), f32(sd[ap + ".norm.beta"])
            d["q_scale"], d["k_scale"] = f32(sd[ap + ".q_scale"]), f32(sd[ap + ".k_scale"])
            # after l2norm every |q_d| <= |q_scale_d|: one exact power of two per layer puts the q / k planes in fp16 range
            d["q_ps"], d["k_ps"] = L.pow2_scale(float(d["q_scale"].abs().max())), L.pow2_scale(float(d["k_scale"].abs().max()))
            # [Wq; Wkv] stacked: one dual-A GEMM writes q | k | v into the QKV buffer
            d["to_qkv"] = PL(torch.cat([sd[ap + ".to_q.weight"], sd[ap + ".to_kv.weight"]], dim=0), None, row_scaled=True)
            d["to_out"] = lin(ap + ".to_out", bias=False)
            ff(d, lp + ".3")
            return d

        def w_layer(lp):
            d = {"kind": "w"}
            ap = lp + ".1"
            d["norm_g"], d["norm_b"] = f32(sd[ap + ".norm.gamma"]), f32(sd[ap + ".norm.beta"])
            d["bias"] = L.window_bias(sd[ap + ".relative_position_bias_table"].detach().float().cpu(),
                                      sd[ap + ".relative_position_index"].cpu(), self.ws).to(dev)
            d["qkv"] = lin(ap + ".qkv", bias=False, row_scaled=True)
            d["proj"] = lin(ap + ".proj")
            ff(d, lp + ".3")
            return d

        def ff(d, fp):
            d["ff_g"], d["ff_b"] = f32(sd[fp + ".0.weight"]), f32(sd[fp + ".0.bias"])
            d["ff1"] = PL(sd[fp + ".1.weight"], None, geglu=(self.inner, self.ku), row_scaled=True)
            # |U| = |gelu(g) a| <= |g| |a| <= (|LN(x)|_2 max_n |W1_n|_2)^2 with |LN(x)|_2 <= max|gamma| sqrt(C) + |beta|_2: a bound
            # known at pack time, so the U planes take ONE static power-of-two scale (single-accumulator FF2, no overflow possible)
            w1 = sd[fp + ".1.weight"].detach().float()
            ln_bound = float(d["ff_g"].abs().max()) * math.sqrt(self.C) + float(d["ff_b"].norm())
            u_bound = (ln_bound * float(w1[:self.inner].norm(dim=1).max())) * (ln_bound * float(w1[self.inner:].norm(dim=1).max()))
            d["u_scale"] = L.pow2_scale(u_bound) if self.static_u else 0.0
            d["ff2"] = PL(sd[fp + ".4.weight"], None, k_pad=self.ku, row_scaled=self.static_u)

        def transformer(pre, block):
            layers = []
            for i, blk in enumerate(block):
                if blk == "t":
                    layers.append(t_layer(f"{pre}.layers.{i}"))
                elif blk == "w":
                    layers.append(w_layer(f"{pre}.layers.{i}"))
                else:
                    raise NotImplementedError(f"block type {blk!r}: pooling/upsampling blocks are outside the shipped configs")
            return {"layers": layers, "out_g": f32(sd[pre + ".norm_out.gamma"]), "out_b": f32(sd[pre + ".norm_out.beta"])}

        tb = "t" * a.temporal_depth
        self.enc_spatial = transformer("encoder.enc_spatial_transformer", a.enc_block)
        self.enc_temporal = transformer("encoder.enc_temporal_transformer", tb)
        self.dec_temporal = transformer("decoder.dec_temporal_transformer", tb)
        self.dec_spatial = transformer("decoder.dec_spatial_transformer", a.dec_block)

        self.pe = {}
        self.cnn = getattr(a, "patch_embed", "linear") == "cnn"
        if self.cnn:
            # patch_embed='cnn' (omnitokenizer.py:823-838, 1019-1035): a Conv3d with kernel == stride is a GEMM over
            # the same (c, pt, p1, p2) patch vectors as the linear variant, and eval-mode (Sync)BatchNorm is a
            # per-channel affine -> both fold into ONE packed weight/bias; no LayerNorms in this variant.
            def bn_affine(pre):
                g, b = sd[pre + ".weight"].float(), sd[pre + ".bias"].float()
                rm, rv = sd[pre + ".running_mean"].float(), sd[pre + ".running_var"].float()
                s_ = g / torch.sqrt(rv + 1e-5)
                return s_, b - rm * s_
            for key, pre in (("first", "encoder.to_patch_emb_first_frame"), ("rest", "encoder.to_patch_emb")):
                w = sd[pre + ".0.weight"].float().reshape(self.C, -1)                 # (dim, c*pt*p*p)
                s_, t_ = bn_affine(pre + ".1")
                self.pe[key] = dict(ln1_g=None, ln1_b=None, ln2_g=None, ln2_b=None,
                                    lin=PL(w * s_[:, None], sd[pre + ".0.bias"].float() * s_ + t_, row_scaled=True))
            self.px = {}
            for key, pre in (("first", "decoder.to_pixels_first_frame"), ("rest", "decoder.to_pixels")):
                wt = sd[pre + ".1.weight"].float()                                    # (dim, channels, pt, p, p)
                per_c = wt[0, 0].numel()
                s_, t_ = bn_affine(pre + ".2")
                w = wt.reshape(self.C, -1).t() * s_.repeat_interleave(per_c)[:, None]  # (channels*pt*p*p, dim)
                bias = (sd[pre + ".1.bias"].float() * s_ + t_).repeat_interleave(per_c)
                self.px[key] = PL(w.contiguous(), bias, row_scaled=True)
        else:
            for key, pre in (("first", "encoder.to_patch_emb_first_frame"), ("rest", "encoder.to_patch_emb")):
                self.pe[key] = dict(ln1_g=f32(sd[pre + ".1.weight"]), ln1_b=f32(sd[pre + ".1.bias"]), lin=lin(pre + ".2", row_scaled=True),
                                    ln2_g=f32(sd[pre + ".3.weight"]), ln2_b=f32(sd[pre + ".3.bias"]))
            self.px = {"first": lin("decoder.to_pixels_first_frame.0", row_scaled=True),
                       "rest": lin("decoder.to_pixels.0", row_scaled=True)}
        self.pre_w, self.pre_b = f32(sd["pre_vq_conv.1.weight"]), f32(sd["pre_vq_conv.1.bias"])
        self.post_w, self.post_b = f32(sd["post_vq_conv.1.weight"]), f32(sd["post_vq_conv.1.bias"])
        E = sd["codebook.embeddings"].detach().float().cpu()
        self.n_codes = E.shape[0]
        # the search kernel takes whole groups of 8 codes in each of its 8 slices: zero rows pad the table to a multiple
        # of 64, and their sum E^2 of +inf makes every distance to them +inf, so they never win and the first-minimum
        # rule over the real codes is unchanged
        self.n_codes_padded = L.round_up(self.n_codes, 64)
        if not self.use_vae and self.n_codes_padded > VQ_MAX_CODES:
            raise NotImplementedError(f"--n_codes {self.n_codes}: the VQ search kernel holds an eighth of the codebook in "
                                      f"shared memory and takes at most {VQ_MAX_CODES} codes")
        # sum E^2 with the reference's own expression (modules/codebook.py:84), evaluated on the host
        e2 = (E.t() ** 2).sum(dim=0)
        pad = self.n_codes_padded - self.n_codes
        self.E = torch.cat([E, E.new_zeros(pad, E.shape[1])]).to(dev).contiguous()
        self.e2 = torch.cat([e2, e2.new_full((pad,), math.inf)]).to(dev).contiguous()

    # ------------------------------------------------------------------ helpers
    @staticmethod
    def fuse_qkprep(M: int) -> bool:
        """rope + l2norm + scale ride in the QKV GEMM epilogue.  The choice must NOT depend on the batch size: the
        fused epilogue and the stand-alone kernel round differently (x * (1/|x|) vs x / |x|, different reduction
        trees), and a shard of a batch has to reproduce the full batch bit for bit (tests/test_gpu_fullsize.py)."""
        return os.environ.get("OMT_FUSE_QKPREP", "1") != "0"

    def _workspace(self, M: int) -> Workspace:
        ws = self._ws.get(M)
        if ws is None:
            kmax = self.cin * self.pt * self.p * self.p
            ws = Workspace(self.device, M, self.C, self.A, self.ku, kmax, max(self.cd, 16), self.planes)
            if ws.counts.numel() < self.n_codes:
                ws.counts = torch.zeros(self.n_codes, device=self.device, dtype=torch.int32)
            while len(self._ws) >= 3:  # keep a few shapes (and their graphs) resident
                self._ws.pop(next(iter(self._ws)))
            self._ws[M] = ws
        return ws

    def _table(self, key, fn):
        t = self._tables.get(key)
        if t is None:
            t = fn()
            t = tuple(x.to(self.device) for x in t) if isinstance(t, tuple) else t.to(self.device)
            self._tables[key] = t
        return t

    def _linear(self, A, lda, lin: PackedLinear, C, ldc, M, *, a_map=(0, 0, 0), c_map=(0, 0, 0), residual=None,
                ldr=0, epi=_cabi.EPI_NONE, bias=True):
        """nn.Linear on the fp32-operand paths (CUDA-core fp32 / wgmma 3xTF32)."""
        _cabi.call("omt_linear", A, lda, a_map[0], a_map[1], a_map[2], lin.w, lin.w_lo, C, ldc, c_map[0], c_map[1],
                   c_map[2], M, lin.n, lin.k, lin.bias if bias else None, residual, ldr, epi, lin.math)

    def _linear_h(self, A: Planes, lin: PackedLinear, M, *, C=None, ldc=0, U: Optional[Planes] = None, A2: Optional[Planes] = None,
                  n_split=0, a_map=(0, 0, 0), c_map=(0, 0, 0), residual=None, ldr=0, epi=_cabi.EPI_NONE, qk=None,
                  planes=None, a_uniform=0.0, u_scale=0.0):
        """nn.Linear on operand planes (wgmma f16x3, or f16x1: hi planes only).  U: GEGLU output planes;
        qk: (q_scale, k_scale, cos, sin, qk_cols, tokens)."""
        if ((A.rs is not None) or a_uniform > 0.0) != lin.row_scaled:
            raise RuntimeError("operand planes and weight planes are in different f16x3 forms (row-scaled vs 2^11-scaled lo)")
        kw = dict(a_hi=A.hi, a_lo=A.lo, lda=A.ld, a_seg=a_map[0], a_seg_stride=a_map[1], a_seg_off=a_map[2],
                  w_hi=lin.w, w_lo=lin.w_lo, c=C, ldc=ldc, c_seg=c_map[0], c_seg_stride=c_map[1], c_seg_off=c_map[2],
                  M=M, N=lin.n, K=lin.k, bias=lin.bias, residual=residual, ldr=ldr, epilogue=epi)
        if A.rs is not None:
            kw.update(a_rs=A.rs, w_scale=lin.w_scale)
        elif a_uniform > 0.0:
            kw.update(a_rs_uniform=a_uniform, w_scale=lin.w_scale)
        if u_scale > 0.0:
            kw.update(u_scale=u_scale)
        if A2 is not None:
            kw.update(a2_hi=A2.hi, a2_lo=A2.lo, a2_rs=A2.rs, n_split=n_split)
        if U is not None:
            kw.update(u_hi=U.hi, u_lo=U.lo, ldu=U.ld)
        if qk is not None:
            kw.update(q_scale=qk[0], k_scale=qk[1], rope_cos=qk[2], rope_sin=qk[3], qk_cols=qk[4], tokens=qk[5])
        if planes is not None:      # EPI_QKV_PLANES: U = the q | k | v planes, (q plane scale, k plane scale, vinv)
            kw.update(q_plane_scale=planes[0], k_plane_scale=planes[1], vinv=planes[2])
        if self.h1:
            kw.update(a_lo=None, a2_lo=None, w_lo=None, u_lo=None)
            _cabi.linear_h("omt_linear_h1", **kw)
        else:
            _cabi.linear_h(**kw)

    def _ln(self, x, y, g, b, M, C=None, seg=(0, 0, 0)):
        C = C or self.C
        _cabi.call("omt_layernorm", x, C, y, C, g, b, M, C, 1e-5, seg[0], seg[1], seg[2])

    def _ln_h(self, x, yp: Planes, g, b, M, xp: Optional[Planes] = None):
        """LayerNorm straight into the operand planes of the consuming GEMM (+ planes of the raw row for to_kv)."""
        C = self.C
        _cabi.call("omt_layernorm_h", x, C, None, 0, yp.hi, yp.lo, yp.rs, None if xp is None else xp.hi,
                   None if xp is None else xp.lo, None if xp is None else xp.rs, yp.ld, g, b, M, C, 1e-5, 0, 0, 0)

    # ------------------------------------------------------------------ transformer
    def _layout_tables(self, ws: Workspace, lay: BatchLayout):
        """(t_off host copy, t_off device copy, int64 [M] sorted position of the sample each row belongs to) of a packed
        layout.  They live in the workspace for as long as a static buffer set of that layout does (Workspace.static),
        and with it every graph that reads them; the copy to the device is asynchronous (pinned host memory)."""
        t = ws.layout_tables.get(lay.key)
        if t is None:
            host = torch.tensor(lay.t_off, dtype=torch.int32).pin_memory()
            dev = host.to(self.device, non_blocking=True)
            frame = torch.arange(lay.M, device=self.device, dtype=torch.int32) // lay.N
            t = ws.layout_tables[lay.key] = (host, dev, torch.searchsorted(dev, frame, right=True) - 1)
        return t

    def row_sample(self, ws: Workspace, lay: BatchLayout) -> torch.Tensor:
        """int64 [M] on the device: sorted position (lay.pos) of the sample each canonical row of the layout belongs to."""
        return self._layout_tables(ws, lay)[2]

    def _check_packed(self, tps: Sequence[int]):
        """A batch of different lengths runs PEG and temporal attention through the layout-table entry points, which take
        1..17 latent frames per sample -- also in a model without temporal blocks, where encode() takes longer clips."""
        if len(set(tps)) > 1 and max(tps) > TEMPORAL_MAX_FRAMES:
            raise NotImplementedError(f"{max(tps)} latent frames: an element of a batch of different lengths takes at most "
                                      f"{TEMPORAL_MAX_FRAMES} latent frames ({1 + (TEMPORAL_MAX_FRAMES - 1) * self.pt} frames)")

    def _transformer(self, tr, ws: Workspace, lay: BatchLayout, temporal: bool, out_planes: Optional[Planes] = None):
        """modules/attention.py:655-689.  out_planes: norm_out goes to operand planes (decoder -> to_pixels GEMMs)."""
        C, A, N, M = self.C, self.A, lay.N, ws.M
        h, w, F = lay.h, lay.w, lay.frames
        B, T = lay.B, lay.groups[0].tp
        H = self.planes
        # q | k | v [M, 3A] and the attention output [M, A]; a window layer's are 3C / C wide, and C == A in a model with one
        q_ptr = ws.QKV.data_ptr()
        k_ptr, v_ptr = q_ptr + A * 4, q_ptr + 2 * A * 4
        ld3 = 3 * A
        o, o_hi, o_lo = (None, ws.Op.hi, ws.Op.lo) if H else (ws.O, None, None)
        t_off = None if lay.uniform else self._layout_tables(ws, lay)[:2]
        for lyr in tr["layers"]:
            if lyr["kind"] == "t":
                if lay.uniform:
                    _cabi.call("omt_peg_volume", ws.X, ws.Y, lyr["peg_w"], lyr["peg_b"], B, T, h, w, C, int(temporal),
                               int(self.causal_peg))
                else:
                    _cabi.call("omt_peg_volume_varlen", ws.X, ws.Y, lyr["peg_w"], lyr["peg_b"], *t_off, B, M, h, w, C,
                               int(temporal), int(self.causal_peg))
                ws.X, ws.Y = ws.Y, ws.X
                # q from the normalised input, k / v from the RAW input (attention.py:407-412), one launch;
                # rope (spatial blocks) + l2norm + q/k scale ride in the same launch (fused GEMM epilogue)
                wq = lyr["to_qkv"]
                cos = sin = None
                if (not temporal) and self.rope:
                    cos, sin = self._table(("rope", N), lambda: L.rope_tables(N, self.dh))
                f16_core = H and self.attn_f16 and (not temporal) and N % 128 == 0
                if f16_core:
                    self._ln_h(ws.X, ws.XNp, lyr["norm_g"], lyr["norm_b"], M, xp=ws.XSp)
                    self._linear_h(ws.XNp, wq, M, U=ws.QKVp, A2=ws.XSp, n_split=A, epi=_cabi.EPI_QKV_PLANES,
                                   qk=(lyr["q_scale"], lyr["k_scale"], cos, sin, 2 * A, N),
                                   planes=(lyr["q_ps"], lyr["k_ps"], ws.vinv))
                elif H:
                    self._ln_h(ws.X, ws.XNp, lyr["norm_g"], lyr["norm_b"], M, xp=ws.XSp)
                    self._linear_h(ws.XNp, wq, M, C=q_ptr, ldc=ld3, A2=ws.XSp, n_split=A, epi=_cabi.EPI_QKV,
                                   qk=(lyr["q_scale"], lyr["k_scale"], cos, sin, 2 * A, N))
                else:
                    self._ln(ws.X, ws.XN, lyr["norm_g"], lyr["norm_b"], M)
                    if self.fuse_qkprep(M):
                        _cabi.call("omt_linear2", ws.XN, ws.X, A, C, wq.w, wq.w_lo, q_ptr, ld3, M, wq.n, wq.k, wq.math,
                                   lyr["q_scale"], lyr["k_scale"], cos, sin, 2 * A, N)
                    else:
                        _cabi.call("omt_linear2", ws.XN, ws.X, A, C, wq.w, wq.w_lo, q_ptr, ld3, M, wq.n, wq.k, wq.math,
                                   None, None, None, None, 0, 0)
                        _cabi.call("omt_qk_prep", q_ptr, ld3, k_ptr, ld3, lyr["q_scale"], lyr["k_scale"], cos, sin, M, N,
                                   self.heads)
                if f16_core and self.h1:
                    ph = ws.QKVp.hi.data_ptr()
                    _cabi.call("omt_attn_spatial_h1", ph, ld3, ph + 2 * A, ld3, ph + 4 * A, ld3, ws.vinv, lyr["q_ps"] * lyr["k_ps"],
                               None, o_hi, A, F, N, self.heads, 8.0)
                elif f16_core:
                    ph, pl = ws.QKVp.hi.data_ptr(), ws.QKVp.lo.data_ptr()
                    _cabi.call("omt_attn_spatial_h", ph, pl, ld3, ph + 2 * A, pl + 2 * A, ld3, ph + 4 * A, pl + 4 * A, ld3,
                               ws.vinv, lyr["q_ps"] * lyr["k_ps"], None, o_hi, o_lo, A, F, N, self.heads, 8.0)
                elif temporal and lay.uniform:
                    _cabi.call("omt_attn_temporal", q_ptr, ld3, k_ptr, ld3, v_ptr, ld3, o, o_hi, o_lo, A, B, T, N,
                               self.heads, 8.0, int(self.causal_attn))
                elif temporal:
                    _cabi.call("omt_attn_temporal_varlen", q_ptr, ld3, k_ptr, ld3, v_ptr, ld3, o, o_hi, o_lo, A, *t_off, B,
                               M, N, self.heads, 8.0, int(self.causal_attn))
                else:
                    _cabi.call("omt_attn_spatial", q_ptr, ld3, k_ptr, ld3, v_ptr, ld3, o, o_hi, o_lo, A, F, N,
                               self.heads, 8.0)
                proj = lyr["to_out"]
            else:
                if H:
                    self._ln_h(ws.X, ws.XNp, lyr["norm_g"], lyr["norm_b"], M)
                    self._linear_h(ws.XNp, lyr["qkv"], M, C=q_ptr, ldc=ld3)
                else:
                    self._ln(ws.X, ws.XN, lyr["norm_g"], lyr["norm_b"], M)
                    self._linear(ws.XN, C, lyr["qkv"], q_ptr, ld3, M)
                # C == A here (Engine.__init__): the window qkv is 3C wide with heads of C / heads = 64; scale (C / heads)^-0.5
                _cabi.call("omt_attn_window", q_ptr, ld3, k_ptr, ld3, v_ptr, ld3, o, o_hi, o_lo, A, lyr["bias"], F, h,
                           w, self.ws, self.heads, float(C // self.heads) ** -0.5)
                proj = lyr["proj"]
            if H:
                self._linear_h(ws.Op, proj, M, C=ws.X, ldc=C, residual=ws.X, ldr=C)
                self._ln_h(ws.X, ws.XNp, lyr["ff_g"], lyr["ff_b"], M)
                us = lyr["u_scale"]
                self._linear_h(ws.XNp, lyr["ff1"], M, U=ws.Up, epi=_cabi.EPI_GEGLU, u_scale=us)
                self._linear_h(ws.Up, lyr["ff2"], M, C=ws.X, ldc=C, residual=ws.X, ldr=C, a_uniform=(1.0 / us if us > 0 else 0.0))
            else:
                self._linear(ws.O, A, proj, ws.X, C, M, residual=ws.X, ldr=C)
                self._ln(ws.X, ws.XN, lyr["ff_g"], lyr["ff_b"], M)
                self._linear(ws.XN, C, lyr["ff1"], ws.U, self.ku, M, epi=_cabi.EPI_GEGLU)
                self._linear(ws.U, self.ku, lyr["ff2"], ws.X, C, M, residual=ws.X, ldr=C)
        if out_planes is not None:
            self._ln_h(ws.X, out_planes, tr["out_g"], tr["out_b"], M)
        else:
            self._ln(ws.X, ws.X, tr["out_g"], tr["out_b"], M)

    # ------------------------------------------------------------------ shapes / graphs
    def _shape(self, shape):
        B, Cin, T, H, W = shape
        if Cin != self.cin:
            raise ValueError(f"expected {self.cin} channels, got {Cin}")
        assert (T - 1) % self.pt == 0, (f"number of frames ({T}) minus one ({T - 1}) must be divisible by temporal "
                                        f"patch size ({self.pt})")
        if H != W or H % self.p != 0:
            raise ValueError(f"frames must be square with side a multiple of the patch size {self.p} (got {H}x{W})")
        if self.has_window and (H // self.p) % self.ws != 0:
            raise ValueError(f"window blocks need a token grid divisible by the window (got window {self.ws}, grid "
                             f"{H // self.p}x{W // self.p})")
        k = self.cin * (self.pt if T > 1 else 1) * self.p * self.p
        if k > PATCH_MAX_K:
            raise NotImplementedError(f"--patch_size {self.p} with --temporal_patch_size {self.pt}: a patch vector of {k} "
                                      f"features is longer than the {PATCH_MAX_K} the patch gather takes")
        if ((H // self.p) * (W // self.p)) % 64 != 0:
            raise ValueError(f"tokens per frame ({(H // self.p) * (W // self.p)}) must be a multiple of 64 (attention tiles)")
        Tp = 1 + (T - 1) // self.pt
        self._check_latent_frames(Tp)
        return B, T, H, W, Tp, H // self.p, W // self.p

    def _check_latent_frames(self, Tp):
        """Reject what the temporal attention core cannot run before the first launch, not in the middle of a pass."""
        if Tp > TEMPORAL_MAX_FRAMES and self.enc_temporal["layers"]:
            raise NotImplementedError(f"{Tp} latent frames: the temporal attention kernel takes at most "
                                      f"{TEMPORAL_MAX_FRAMES} latent frames ({1 + (TEMPORAL_MAX_FRAMES - 1) * self.pt} "
                                      f"frames)")

    @staticmethod
    def graphs_enabled() -> bool:
        return os.environ.get("OMT_CUDA_GRAPH", "1") != "0"

    def _run(self, ws: Workspace, key, body):
        run_graphed(ws.graphs, self.device, key, body)

    # ------------------------------------------------------------------ encoder side
    def _encode_body(self, ws: Workspace, gather, lay: BatchLayout, mode: str):
        """patch embed -> spatial -> temporal -> pre_vq [-> VQ search].  omnitokenizer.py:881-947, 247-258.
        gather(group, first, A, A_hi, A_lo, A_rs, ln_w, ln_b) launches the patch gather + LayerNorm of one group's videos."""
        N, C = lay.N, self.C
        ws.reset()
        k1 = self.cin * self.p * self.p

        def embed(pe, gi, first, rows, K, cmap):
            if self.planes:
                Pp = Planes.__new__(Planes)          # dense [rows, K] view at the start of the patch planes
                Pp.hi, Pp.lo, Pp.ld, Pp.rs = ws.Pp.hi, ws.Pp.lo, K, ws.Pp.rs
                gather(gi, first, None, Pp.hi, Pp.lo, Pp.rs, pe["ln1_g"], pe["ln1_b"])
                self._linear_h(Pp, pe["lin"], rows, C=ws.X, ldc=C, c_map=cmap)
            else:
                gather(gi, first, ws.P, None, None, None, pe["ln1_g"], pe["ln1_b"])
                self._linear(ws.P, K, pe["lin"], ws.X, C, rows, c_map=cmap)
            if not self.cnn:
                self._ln(ws.X, ws.X, pe["ln2_g"], pe["ln2_b"], rows, seg=cmap)

        for gi, g in enumerate(lay.groups):      # each group's frames start at canonical row g.f0 * N
            embed(self.pe["first"], gi, 1, g.n * N, k1, (N, g.tp * N, g.f0 * N))
            if g.tp > 1:
                embed(self.pe["rest"], gi, 0, g.n * (g.tp - 1) * N, k1 * self.pt, ((g.tp - 1) * N, g.tp * N, g.f0 * N + N))
        self._transformer(self.enc_spatial, ws, lay, temporal=False)
        self._transformer(self.enc_temporal, ws, lay, temporal=True)
        cd = self.pre_w.shape[0]
        z = ws.z.view(-1)[: ws.M * cd].view(ws.M, cd)
        if mode == "vq":      # pre_vq + l2norm + modules/codebook.py:82-86 in one cluster kernel
            ws.counts.zero_()
            _cabi.call("omt_vq_fused", ws.X, C, self.pre_w, self.pre_b, C, int(self.l2), z, self.E, self.e2, ws.M,
                       self.n_codes_padded, ws.idx, ws.counts)
        else:
            _cabi.call("omt_pre_vq", ws.X, C, self.pre_w, self.pre_b, z, ws.M, C, cd, 0)

    def encode(self, x: torch.Tensor, mode: str):
        """x (B,C,T,H,W) fp32 on the device.  mode 'vq': returns (ws, dims) with ws.z (l2-normalised z),
        ws.idx, ws.counts filled; mode 'raw': ws.z = pre_vq output (VAE moments).  Results live in the
        workspace until the next call of the same shape."""
        return self._encode_input(tuple(x.shape), mode, lambda bufs: bufs[0].copy_(x))

    def encode_clips_u8(self, clips: Sequence[torch.Tensor], resize: L.ClipResize, flips, mode: str, norm: L.U8Norm):
        """encode() of the (B, 3, F, oh, ow) fp32 clips the Latte loader's transform `resize` (flips[i]: clip i mirrored)
        and Normalize `norm` make of a ragged list of (F, H_i, W_i, 3) uint8 clips in host memory: omt_resample_clips
        writes encode's input buffer (eagerly: the source geometry changes every batch), then encode's body or graph of
        that shape runs -- the same graph a later encode() of that shape replays."""
        F, H, W = (int(v) for v in clips[0].shape[:3])
        shape = (len(clips), self.cin, F) + L.clip_out_size(H, W, resize)
        return self._encode_input(shape, mode, lambda bufs: self.resample_clips(clips, resize, flips, norm, bufs[0]))

    def _encode_input(self, shape, mode: str, fill):
        """encode of the (B,C,T,H,W) fp32 video fill(bufs) writes into bufs[0], encode's static input buffer."""
        B, T, H, W, Tp, h, w = self._shape(shape)
        return self._encode_pass("encode", BatchLayout((Tp,) * B, h, w), mode, fill), (B, Tp, h, w)

    def _encode_pass(self, slot: str, lay: BatchLayout, mode: str, fill) -> Workspace:
        """One encode of the layout lay from the static fp32 input buffers of `slot`, one (n,C,T,H,W) video per group,
        which fill(bufs) writes."""
        ws = self._workspace(lay.M)
        bufs = ws.static(slot, lay.key, lambda: [
            torch.empty(self._video_shape(g.n, g.tp, lay.h, lay.w, False), device=self.device, dtype=torch.float32)
            for g in lay.groups])
        fill(bufs)
        H, W = lay.h * self.p, lay.w * self.p

        def gather(gi, first, *out):
            g, x = lay.groups[gi], bufs[gi]
            _cabi.call("omt_patchify_ln", x, *out, g.n, self.cin, x.shape[2], H, W, self.p, self.pt, first, 1e-5)

        self._run(ws, (slot, lay.key, mode, None), lambda: self._encode_body(ws, gather, lay, mode))
        return ws

    def encode_batch(self, xs: Sequence[torch.Tensor], mode: str):
        """encode() of a list of single videos xs[i] (C, T_i, H, W) fp32 on the device, all with the same C, H, W, in ONE pass:
        the samples are packed by length (BatchLayout).  Returns (ws, lay): sample i's results are the rows lay.rows(i)
        of ws.z / ws.idx, equal bit for bit to what encode(xs[i][None]) leaves there.  ws.counts is not filled."""
        dims = [self._shape((1,) + tuple(x.shape)) for x in xs]
        H, W = dims[0][2], dims[0][3]
        for d in dims:
            if (d[2], d[3]) != (H, W):
                raise ValueError(f"every element of a batch must have the same frame size: {H}x{W} and {d[2]}x{d[3]}")
        self._check_packed([d[4] for d in dims])
        lay = BatchLayout([d[4] for d in dims], dims[0][5], dims[0][6])

        def fill(bufs):
            for g, buf in zip(lay.groups, bufs):
                torch.stack([xs[i].to(device=self.device, dtype=torch.float32) for i in lay.order[g.s0:g.s0 + g.n]], out=buf)

        return self._encode_pass("encode_batch", lay, mode, fill), lay

    def encode_u8(self, frames: torch.Tensor, mode: str, norm: L.U8Norm):
        """encode() from uint8 frames (B,T,H,W,C) on the device: the patch gather maps every byte through the host-built
        table of `norm` (layout.u8_norm_table), so the result equals encode() of the pipeline's fp32 video bit for bit.
        With norm.max_test the table is picked per sample on the device (omt_u8_norm_select), inside the graph."""
        if frames.dtype != torch.uint8 or frames.ndim != 5:
            raise TypeError(f"encode_u8 takes (B, T, H, W, C) uint8 frames, got {tuple(frames.shape)} {frames.dtype}")
        return self._encode_u8_input(tuple(frames.shape), mode, norm, lambda buf: buf.copy_(frames))

    def encode_images_u8(self, images: Sequence[torch.Tensor], resize: L.U8Resize, params, mode: str, norm: L.U8Norm,
                         jpegs=None):
        """encode_u8() of the images the loader's transform `resize` (with params[i] = (top, left, flip)) makes of a ragged
        list of (H_i, W_i, 3) uint8 images in host memory: omt_resample_u8 writes the transformed bytes into encode_u8's
        input buffer (eagerly: the source geometry changes every batch), then encode_u8's body or graph of that shape runs."""
        oh, ow = resize.out_size
        return self._encode_u8_input((len(images), 1, oh, ow, self.cin), mode, norm,
                                     lambda buf: self.resample_u8(images, resize, params, buf, jpegs))

    def encode_u8_frames(self, shape) -> torch.Tensor:
        """The encode_u8 slot's static uint8 input buffer for frames of `shape` (B, T, H, W, C): the bytes the last
        encode_u8 / encode_images_u8 of that shape encoded (for images, the loader's transform as omt_resample_u8 made
        it).  Valid until the next call of either; raises LookupError if the slot holds another shape."""
        Bf, Tf, Hf, Wf, Cf = shape
        B, T, H, W, Tp, h, w = self._shape((Bf, Cf, Tf, Hf, Wf))
        lay = BatchLayout((Tp,) * B, h, w)
        ws = self._ws.get(lay.M)
        held = None if ws is None else ws.sets.get("encode_u8")
        if held is None or held[0] != lay.key or tuple(held[1][0].shape) != tuple(shape):
            raise LookupError(f"the encode_u8 slot holds no {tuple(shape)} frames")
        return held[1][0]

    def _encode_u8_input(self, shape, mode: str, norm: L.U8Norm, fill):
        """encode_u8 of the (B,T,H,W,C) uint8 frames fill(buf) writes into the static input buffer buf."""
        Bf, Tf, Hf, Wf, Cf = shape
        B, T, H, W, Tp, h, w = self._shape((Bf, Cf, Tf, Hf, Wf))
        lay = BatchLayout((Tp,) * B, h, w)
        ws = self._workspace(lay.M)
        frames, sel = ws.static("encode_u8", lay.key, lambda: (
            torch.empty(shape, device=self.device, dtype=torch.uint8),
            torch.empty(B, device=self.device, dtype=torch.int32)))      # per-sample table index (omt_u8_norm_select)
        fill(frames)
        lut = self._table(("u8norm", norm), lambda: L.u8_norm_table(norm, self.cin))
        sel = sel if norm.max_test else None

        def gather(gi, first, *out):
            _cabi.call("omt_patchify_ln_u8", frames, lut, sel, *out, B, self.cin, T, H, W, self.p, self.pt, first, 1e-5)

        def body():
            if sel is not None:
                _cabi.call("omt_u8_norm_select", frames, B, T * H * W * self.cin, sel)
            self._encode_body(ws, gather, lay, mode)

        self._run(ws, ("encode_u8", lay.key, mode, norm), body)
        return ws, (B, Tp, h, w)

    def resample_descs(self, shapes, resize: L.U8Resize, params) -> tuple:
        """omt_resample_u8's descriptors and the batch's distinct coefficient tables (layout.resample_coeffs) for images of
        sizes shapes[i] = (H_i, W_i): (desc int32 [B, DESC_WORDS] without the source offsets, table parts, tab_len).
        Needs no source bytes, so an image decoded on the device can be laid out like a host one."""
        rh, rw = resize.size
        B = len(shapes)
        desc = torch.zeros(B, DESC_WORDS, dtype=torch.int32)
        tables, parts, tab_len = {}, [], 0

        def axis(n_in, n_out):
            nonlocal tab_len
            key = (n_in, n_out)
            if key not in tables:
                bounds, coeffs = L.resample_coeffs(n_in, n_out, resize.filter)
                tables[key] = (tab_len, tab_len + bounds.size, coeffs.shape[1])
                parts.extend((bounds.reshape(-1), coeffs.reshape(-1)))
                tab_len += bounds.size + coeffs.size
            return tables[key]

        for b, ((H, W), (i, j, flip)) in enumerate(zip(shapes, params)):
            need_h, need_v = W != rw, H != rh
            hb, hc, hk = axis(W, rw) if need_h else (0, 0, 0)
            vb, vc, vk = axis(H, rh) if need_v else (0, 0, 0)
            desc[b, 2:] = torch.tensor([H, W, rh, rw, i, j, int(flip), int(need_h), int(need_v), hb, hc, hk, vb, vc, vk,
                                        int(L.vertical_first(H, W, rh, rw))], dtype=torch.int32)
        return desc, parts, tab_len

    def stage_images_u8(self, images: Sequence[torch.Tensor], resize: L.U8Resize, params, jpegs=None) -> tuple:
        """Packs a ragged list of (H_i, W_i, 3) uint8 host images for omt_resample_u8 -- descriptors, the batch's distinct
        coefficient tables (resample_descs), source bytes -- into the grow-only pinned staging buffer and copies it
        to the device asynchronously on the current stream.  Returns the entry point's arguments up to the output.
        jpegs: (staged batch, names) of jpeg.split_sources, whose files stand as jpeg.Pending entries in images; their
        sources are laid out after the host images' and decoded there on the device (jpeg.decode_into), so only the host
        images' bytes cross to the device and a corrupt scan raises before the resize launches."""
        if self.cin != 3:
            raise NotImplementedError(f"omt_resample_u8 resizes RGB images; the model takes {self.cin} channels")
        desc, parts, tab_len = self.resample_descs([(int(im.shape[0]), int(im.shape[1])) for im in images], resize,
                                                   params)
        offsets, srcs, src_len = [0] * len(images), [], 0
        for host_side in (True, False):
            for b, im in enumerate(images):
                if isinstance(im, torch.Tensor) == host_side:
                    offsets[b] = src_len
                    if host_side:
                        srcs.append((src_len, im))
                    src_len += int(im.shape[0]) * int(im.shape[1]) * 3
        host_len = sum(t.numel() for _, t in srcs)
        dev, host, o_tab, o_src = self._stage_upload(desc, parts, srcs, src_len, offsets, host_len)
        if jpegs is not None:
            from . import jpeg
            staged, names = jpegs
            pending = sorted((im.index, offsets[b]) for b, im in enumerate(images) if isinstance(im, jpeg.Pending))
            jpeg.decode_into(staged, names, self._stage_dev[o_src:o_src + src_len], [o for _, o in pending])
        return (dev + o_src, src_len, dev, host, dev + o_tab if tab_len else None, host + o_tab if tab_len else None,
                tab_len, len(images)) + tuple(resize.out_size)

    def _stage_upload(self, desc: torch.Tensor, parts, srcs, src_len: int, offsets=None, copy_len=None):
        """Packs descriptors (int32 [B, words], the int64 source offset in words 0-1), int32 table parts and the source
        tensors (srcs: (byte offset, uint8 tensor)) into the grow-only pinned staging buffer, 16-byte aligned sections,
        and copies it to the device asynchronously on the current stream.  An event guards the pinned buffer's reuse.
        offsets: every sample's source offset (default: those of srcs); copy_len: source bytes to copy (default src_len;
        the rest is filled on the device).  Returns (device base, host base, table offset, source offset) in bytes."""
        B = desc.shape[0]
        offsets = [s for s, _ in srcs] if offsets is None else offsets
        desc[:, :2] = torch.tensor(offsets, dtype=torch.int64).view(torch.int32).view(B, 2)
        tab_len = sum(p.size for p in parts)
        o_tab = L.round_up(desc.numel() * 4, 16)
        o_src = L.round_up(o_tab + tab_len * 4, 16)
        total = o_src + src_len
        if self._stage is None or self._stage.numel() < total:
            if self._stage_done is not None:
                self._stage_done.synchronize()
            cap = max(total, 3 * (0 if self._stage is None else self._stage.numel()) // 2)
            self._stage = torch.empty(cap, dtype=torch.uint8, pin_memory=True)
            self._stage_dev = torch.empty(cap, dtype=torch.uint8, device=self.device)
        elif self._stage_done is not None:
            self._stage_done.synchronize()       # the previous batch's copy has read the staging buffer
        st = self._stage
        st[:o_tab].view(torch.int32)[: desc.numel()].copy_(desc.view(-1))
        if tab_len:
            st[o_tab:o_tab + tab_len * 4].view(torch.int32).copy_(torch.from_numpy(np.concatenate(parts)))
        for off, t in srcs:
            st[o_src + off:o_src + off + t.numel()].view(t.shape).copy_(t)
        n = o_src + (src_len if copy_len is None else copy_len)
        self._stage_dev[:n].copy_(st[:n], non_blocking=True)
        if self._stage_done is None:
            self._stage_done = torch.cuda.Event()
        self._stage_done.record()
        return self._stage_dev.data_ptr(), st.data_ptr(), o_tab, o_src

    def stage_clips_u8(self, clips: Sequence[torch.Tensor], resize: L.ClipResize, flips) -> tuple:
        """Packs a ragged list of (F, H_i, W_i, 3) uint8 host clips for omt_resample_clips -- descriptors, the batch's
        distinct axis tables (layout.clip_axis_table), source bytes -- through the staging buffer (_stage_upload).
        Returns the entry point's arguments up to the normalisation table, then (B, F, oh, ow)."""
        if self.cin != 3:
            raise NotImplementedError(f"omt_resample_clips resizes RGB clips; the model takes {self.cin} channels")
        B = len(clips)
        F = int(clips[0].shape[0])
        desc = torch.zeros(B, CLIP_DESC_WORDS, dtype=torch.int32)
        tables, parts, tab_len, src_len, srcs = {}, [], 0, 0, []

        def axis(n_in, n_out, scale):
            nonlocal tab_len
            key = (n_in, n_out, scale)
            if key not in tables:
                tables[key] = tab_len
                parts.append(L.clip_axis_table(n_in, n_out, scale).reshape(-1))
                tab_len += 4 * n_out
            return tables[key]

        for b, (clip, flip) in enumerate(zip(clips, flips)):
            H, W = int(clip.shape[1]), int(clip.shape[2])
            g = L.clip_geometry(H, W, resize)
            tv, th = axis(g.wh, g.rh, g.scale_h), axis(g.ww, g.rw, g.scale_w)
            desc[b, 2:] = torch.tensor([H, W, g.y0, g.x0, g.wh, g.ww, g.rh, g.rw, g.cy, g.cx, int(flip), tv, th,
                                        L.clip_interp_form(g, resize.in_workers)], dtype=torch.int32)
            srcs.append((src_len, clip))
            src_len += clip.numel()
        oh, ow = L.clip_out_size(int(clips[0].shape[1]), int(clips[0].shape[2]), resize)
        dev, host, o_tab, o_src = self._stage_upload(desc, parts, srcs, src_len)
        return (dev + o_src, src_len, dev, host, dev + o_tab, host + o_tab, tab_len), (B, F, oh, ow)

    def resample_clips(self, clips: Sequence[torch.Tensor], resize: L.ClipResize, flips, norm: L.U8Norm,
                       out: torch.Tensor) -> torch.Tensor:
        """The Latte loader's transform `resize` (flips[i]: clip i mirrored) and Normalize `norm` of a ragged list of
        (F, H_i, W_i, 3) uint8 host clips, on the device in one launch: out (B, 3, F, oh, ow) fp32 contiguous, equal bit
        for bit to layout.resize_clip / the loader's torch CPU pipeline."""
        B, (F, H, W) = len(clips), tuple(int(v) for v in clips[0].shape[:3])
        shape = (B, 3, F) + L.clip_out_size(H, W, resize)
        if out.dtype != torch.float32 or out.device != self.device or not out.is_contiguous() or tuple(out.shape) != shape:
            raise ValueError(f"resample_clips writes a contiguous fp32 {shape} tensor on {self.device}, "
                             f"got {tuple(out.shape)} {out.dtype} on {out.device}")
        lut = self._table(("clipnorm", norm), lambda: L.clip_norm_table(norm))
        args, (B, F, oh, ow) = self.stage_clips_u8(clips, resize, flips)
        _cabi.call("omt_resample_clips", *args, lut, B, F, oh, ow, out)
        return out

    def resample_u8(self, images: Sequence[torch.Tensor], resize: L.U8Resize, params, out: torch.Tensor,
                    jpegs=None) -> torch.Tensor:
        """The loader's transform `resize` (params[i] = (top, left, flip)) of a ragged list of (H_i, W_i, 3) uint8 host images,
        on the device: out (B, oh, ow, 3) uint8 (any shape of that size), equal byte for byte to layout.resize_u8 / Pillow."""
        oh, ow = resize.out_size
        if out.dtype != torch.uint8 or out.device != self.device or not out.is_contiguous() or out.numel() != len(images) * oh * ow * 3:
            raise ValueError(f"resample_u8 writes {len(images)} x {oh} x {ow} x 3 contiguous uint8 bytes on {self.device}, "
                             f"got {tuple(out.shape)} {out.dtype} on {out.device}")
        _cabi.call("omt_resample_u8", *self.stage_images_u8(images, resize, params, jpegs), out)
        return out

    def z_view(self, ws: Workspace) -> torch.Tensor:
        return self._dense(ws.z, ws.M, self.pre_w.shape[0])

    @staticmethod
    def _dense(buf: torch.Tensor, M: int, cols: int) -> torch.Tensor:
        """Dense [M, cols] view at the start of a wider scratch buffer (kernels take packed rows)."""
        return buf.view(-1)[: M * cols].view(M, cols)

    def zq_view(self, ws: Workspace) -> torch.Tensor:
        return self._dense(ws.zq, ws.M, self.post_w.shape[1])

    # ------------------------------------------------------------------ decoder side
    def _decode_body(self, ws: Workspace, lay: BatchLayout, mode: str, outs, u8=None):
        """[gather +] post_vq -> temporal -> spatial -> to_pixels.  omnitokenizer.py:268-317, 1059-1118.
        outs[g]: the output videos of group g, (n,C,T,H,W) fp32, or with u8 = (mul, add, lo, hi, post) uint8 (n,T,H,W,C)
        = trunc(clamp(x*mul+add, lo, hi)*post)."""
        N, M, C = lay.N, ws.M, self.C
        ws.reset()
        cdp = self.post_w.shape[1]
        if mode == "idx":
            _cabi.call("omt_post_vq", ws.idx_in, self.E, None, None, None, self.post_w, self.post_b, ws.X, M, C, cdp)
        elif mode == "idx_st":    # forward(): decoder sees (E[idx] - z) + z, codebook.py:120
            _cabi.call("omt_post_vq", ws.idx_in, self.E, None, self.z_view(ws), self.zq_view(ws), self.post_w,
                       self.post_b, ws.X, M, C, cdp)
        else:
            _cabi.call("omt_post_vq", None, None, self._dense(ws.zc_in, M, cdp), None, None, self.post_w, self.post_b,
                       ws.X, M, C, cdp)
        self._transformer(self.dec_temporal, ws, lay, temporal=True)
        self._transformer(self.dec_spatial, ws, lay, temporal=False, out_planes=ws.XNp if self.planes else None)
        H, W = lay.h * self.p, lay.w * self.p
        k1 = self.cin * self.p * self.p

        def pixels(px, g, out, first, rows, K, amap):
            if self.planes:
                self._linear_h(ws.XNp, px, rows, C=ws.P, ldc=K, a_map=amap)
            else:
                self._linear(ws.X, C, px, ws.P, K, rows, a_map=amap)
            T = 1 + (g.tp - 1) * self.pt
            if u8 is None:
                _cabi.call("omt_unpatchify", ws.P, out, g.n, self.cin, T, H, W, self.p, self.pt, first)
            else:
                _cabi.call("omt_unpatchify_u8", ws.P, out, g.n, self.cin, T, H, W, self.p, self.pt, first, *u8)

        for g, out in zip(lay.groups, outs):     # each group's frames start at canonical row g.f0 * N
            pixels(self.px["first"], g, out, 1, g.n * N, k1, (N, g.tp * N, g.f0 * N))
            if g.tp > 1:
                pixels(self.px["rest"], g, out, 0, g.n * (g.tp - 1) * N, k1 * self.pt, ((g.tp - 1) * N, g.tp * N, g.f0 * N + N))

    def _video_shape(self, n, tp, h, w, u8: bool):
        T, H, W = 1 + (tp - 1) * self.pt, h * self.p, w * self.p
        return (n, T, H, W, self.cin) if u8 else (n, self.cin, T, H, W)

    def decode(self, dims, *, idx=None, zc=None, straight_through=False, u8=None) -> torch.Tensor:
        """dims (B,T',h,w).  idx: int64 [M] codes | zc: fp32 [M, cd] latents (VAE).  With straight_through
        the rows are (E[idx] - z) + z using the z left in the workspace by encode(); ws.zq receives them.
        Returns a fresh (B,C,T,H,W) tensor (the reference's decoder ends in .clone(), omnitokenizer.py:1116);
        with u8 = (mul, add, lo, hi, post) a fresh uint8 (B,T,H,W,C) tensor (fused consumer conversion)."""
        B, Tp, h, w = dims
        self._check_latent_frames(Tp)
        outs = self._decode_pass("decode", BatchLayout((Tp,) * B, h, w), None if idx is None else idx.reshape(-1), zc, u8,
                                 straight_through)
        return outs[0].clone()

    def decode_batch(self, tps: Sequence[int], h: int, w: int, *, idx=None, zc=None, u8=None) -> List[torch.Tensor]:
        """decode() of a list of single samples in ONE pass.  tps[i]: latent frames of sample i; idx: list of int64 codes
        (tps[i]*h*w each) | zc: list of fp32 [tps[i]*h*w, cd] latents.  Returns, in the caller's order, what
        decode((1, tps[i], h, w), ...) returns for each sample, bit for bit."""
        for tp in tps:
            self._check_latent_frames(tp)
        self._check_packed(tps)
        lay = BatchLayout(tps, h, w)
        if idx is not None:
            idx = torch.cat([idx[i].reshape(-1) for i in lay.order])
        else:
            zc = torch.cat([zc[i].reshape(-1, zc[0].shape[-1]) for i in lay.order])
        outs = self._decode_pass("decode_batch", lay, idx, zc, u8)
        return [outs[gi][k].clone() for gi, k in lay.slot]

    def _decode_pass(self, slot: str, lay: BatchLayout, idx, zc, u8, straight_through=False) -> List[torch.Tensor]:
        """One decode of the layout lay from the codes idx (int64 [M]) or latents zc (fp32 [M, cd]) in its row order, into
        the static output videos of `slot` (fp32), or of slot + "_u8" with u8 = (mul, add, lo, hi, post): one per group."""
        ws = self._workspace(lay.M)
        if u8 is not None:
            u8, slot = tuple(float(v) for v in u8), slot + "_u8"
        dt = torch.float32 if u8 is None else torch.uint8
        outs = ws.static(slot, lay.key, lambda: [
            torch.empty(self._video_shape(g.n, g.tp, lay.h, lay.w, u8 is not None), device=self.device, dtype=dt)
            for g in lay.groups])
        if idx is not None:
            ws.idx_in.copy_(idx)
            mode = "idx_st" if straight_through else "idx"
        else:
            self._dense(ws.zc_in, ws.M, zc.shape[1]).copy_(zc)
            mode = "zc"
        self._run(ws, (slot, lay.key, mode, u8), lambda: self._decode_body(ws, lay, mode, outs, u8))
        return outs
