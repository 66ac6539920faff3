"""Operands for the fp32-operand attention-core tests (test_attn_cases_cpu.py checks the construction on the CPU,
test_gpu_attn_cores.py launches csrc/attention_tc3.cu and csrc/attention_fp32.cu on it).

A case is a set of attention sequences over the rows of q, k, v ([M, H * 64] each), in one of three topologies:

* spatial  : n_seq sequences of N consecutive rows (omt_attn_spatial);
* window   : the 8x8 windows of each frame's h x w token grid, in oo.window_rows order, with a [H, 64, 64] bias added to
             the scores (omt_attn_window);
* temporal : the T' rows (b T' + t) N + n of pixel n of video b, causal or not (omt_attn_temporal).

Topology.sets lists the rows of every sequence ([n_sets, L]); the fp64 reference and the planted answers work on it
alone, so one reference serves all three cores.  Operand families:

* model   : q and k unit-norm rows times a per-dimension scale in [0.5, 1.5] (what the QKV epilogue leaves), score scale
            8; v rows with magnitudes spread over 1e-2 .. 1e2 (test_gpu_attn_walk.Problem's construction).
* ramp    : model, with key norms growing along each sequence (x 0.1 at its first key, up to x 2.5 at its last), so
            every row's maximum rises from key tile to key tile and the online-softmax rescale runs on every tile.
* hot     : q, k uniform in [-1, 1], not normalised: |scale q.k| reaches about 60 (test_temporal_attention's regime).
* planted : random unit keys, and q_i = lam_i k_t(i) for a target key t(i) inside row i's attention set, with lam_i
            chosen so that the fp32 logit of the target beats every other key of the row (bias included) by at least
            100.  Every other softmax weight is below e^-100, so the exact output is v_t(i) (target_plan places the
            targets on the tiling edges of the cores).

q, k and v live in separate buffers with distinct leading dimensions (64 H + 4, + 12, + 20: multiples of 4, so rows stay
16-byte aligned); the columns past 64 H hold NaN, so a kernel that read them would put NaN into its output.

The builders are plain torch and run on any device; the GPU tests build on the device to keep the large cases fast.
"""
import torch

from oracle import omni_oracle as oo

D = 64
EXTRA = (4, 12, 20)          # columns of q, k, v past the heads
SCALE = 8.0                  # the model's score scale for l2-normalised q, k (and the one these tests use throughout)
PLANT_GAP = 100.0            # least fp32 logit gap between a planted target and any other key of its row
PLANT_MARGIN = 20.0          # lam is chosen for PLANT_GAP + PLANT_MARGIN in fp64: room for the fp32 rounding of q, k, bias
FAMILIES = ("model", "ramp", "hot", "planted")
CHUNK = 1 << 20              # rows generated per step: bounds the temporaries of the grid-limit cases


class Topology:
    """Attention sequences over M rows: sets [n_sets, L] (row indices), causal mask, and the launch geometry: `units`
    (sequences, frames or videos) of `unit_rows` consecutive rows each, the unit of the entry point's count argument."""

    def __init__(self, kind, sets, units, unit_rows, causal=False, **dims):
        self.kind, self.sets, self.units, self.unit_rows, self.causal = kind, sets, units, unit_rows, causal
        self.M = units * unit_rows
        self.L = sets.shape[1]
        self.dims = dims

    @staticmethod
    def spatial(n_seq, N):
        return Topology("spatial", torch.arange(n_seq * N).view(n_seq, N), n_seq, N, N=N)

    @staticmethod
    def window(frames, h, w):
        rows = oo.window_rows(h, w, 8)                                        # (nW, 64) token of each window slot
        sets = (torch.arange(frames)[:, None, None] * (h * w) + rows).reshape(-1, 64)
        return Topology("window", sets, frames, h * w, h=h, w=w)

    @staticmethod
    def temporal(B, T, N, causal):
        b, n, t = torch.arange(B)[:, None, None], torch.arange(N)[None, :, None], torch.arange(T)[None, None, :]
        return Topology("temporal", ((b * T + t) * N + n).reshape(B * N, T), B, T * N, causal=bool(causal), T=T, N=N)

    def __repr__(self):
        d = ",".join(f"{k}={v}" for k, v in self.dims.items())
        return f"{self.kind}[units={self.units},{d}{',causal' if self.causal else ''}]"


def target_plan(topo, H):
    """Target slot t(i) within its sequence for every (sequence, query slot, head): [n_sets, L, H].

    spatial : keys 0, 63, 64, 127, 128, N - 1 and one key in every 64-key tile, dealt round-robin to the queries, so
              every query (every query tile, both 64-row halves of a 128-row tile) has a target and every listed key
              is the target of some query;
    window  : the four window corners and two inner slots, in every window;
    temporal: causal - frame 0, the query's own frame (j = i) or an earlier one; non-causal - the first frame, the last
              frame, the query's own frame or any other one."""
    n, L = topo.sets.shape
    s = torch.arange(n)[:, None, None]
    i = torch.arange(L)[None, :, None]
    h = torch.arange(H)[None, None, :]
    if topo.kind == "spatial":
        keys = {k for k in (0, 63, 64, 127, 128, L - 1) if k < L}
        keys |= {64 * j + (37 * j + 11) % 64 for j in range(L // 64)}
        keys = torch.tensor(sorted(keys))
        return keys[(i + 5 * s + 3 * h) % len(keys)].expand(n, L, H).contiguous()
    if topo.kind == "window":
        keys = torch.tensor([0, 7, 56, 63, 27, 36])
        return keys[(i + s + h) % len(keys)].expand(n, L, H).contiguous()
    other = (7 * i + s + h) % (i + 1 if topo.causal else L)
    if topo.causal:
        choice = torch.stack(torch.broadcast_tensors(torch.zeros_like(other), i.expand_as(other), other))
        sel = (i + s + h) % 3
    else:
        choice = torch.stack(torch.broadcast_tensors(torch.zeros_like(other), torch.full_like(other, L - 1),
                                                     i.expand_as(other), other))
        sel = (i + s + h) % 4
    return choice.gather(0, sel.expand(n, L, H)[None]).squeeze(0).contiguous()


class Case:
    """q, k, v of one topology and family, in NaN-padded buffers qb, kb, vb ([M, ld]); q, k, v are the [M, 64 H] views."""

    def __init__(self, topo, H, family, seed, device="cpu", bias=None):
        assert family in FAMILIES, family
        self.topo, self.H, self.family, self.scale = topo, H, family, SCALE
        self.device = torch.device(device)
        self.bias = None if bias is None else bias.to(self.device, torch.float32).contiguous()
        M, C = topo.M, H * D
        self.ldq, self.ldk, self.ldv = (C + e for e in EXTRA)
        self.qb, self.kb, self.vb = (torch.full((M, ld), float("nan"), device=self.device)
                                     for ld in (self.ldq, self.ldk, self.ldv))
        self.q, self.k, self.v = self.qb[:, :C], self.kb[:, :C], self.vb[:, :C]
        g = torch.Generator(device=self.device).manual_seed(seed)

        def rand(*shape):
            return torch.rand(*shape, generator=g, device=self.device)

        def unit(c):
            return torch.nn.functional.normalize(torch.randn(c, H, D, generator=g, device=self.device), dim=-1)

        qs, ks = rand(D) + 0.5, rand(D) + 0.5
        if family == "ramp":
            pos = torch.empty(M, dtype=torch.float32)
            pos[topo.sets.reshape(-1)] = torch.arange(topo.L, dtype=torch.float32).repeat(topo.sets.shape[0])
            ramp = (0.1 + 2.4 * pos / topo.L).to(self.device)
        for r0 in range(0, M, CHUNK):
            r1 = min(M, r0 + CHUNK)
            c = r1 - r0
            mag = 10.0 ** (rand(c, 1, 1) * 4.0 - 2.0)
            self.v[r0:r1] = (torch.randn(c, H, D, generator=g, device=self.device) * mag).view(c, C)
            if family == "hot":
                q, k = rand(c, H, D) * 2.0 - 1.0, rand(c, H, D) * 2.0 - 1.0
            elif family == "planted":
                q, k = torch.zeros(c, H, D, device=self.device), unit(c)
            else:
                q, k = unit(c) * qs, unit(c) * ks
                if family == "ramp":
                    k = k * ramp[r0:r1, None, None]
            self.q[r0:r1] = q.view(c, C)
            self.k[r0:r1] = k.view(c, C)
        self.target = target_plan(topo, H) if family == "planted" else None
        if family == "planted":
            self._plant()

    def _chunks(self, set_ids):
        """Groups of sequences whose [c, L, L] fp64 score blocks stay near 128 MB."""
        L = self.topo.L
        step = max(1, (1 << 24) // (L * L))
        for s0 in range(0, len(set_ids), step):
            yield set_ids[s0:s0 + step]

    def _scores(self, ids, h, q, k):
        """fp64 scale q k^T (+ bias) of head h over sequences ids: [c, L, L], with rows and the causal mask applied
        as -inf.  q, k: [M, 64 H] views (any dtype; the products are formed in fp64)."""
        rows = self.topo.sets[ids].to(self.device)
        cols = slice(h * D, (h + 1) * D)
        qq, kk = q[rows][..., cols].double(), k[rows][..., cols].double()
        s = (qq @ kk.transpose(-1, -2)) * self.scale
        if self.bias is not None:
            s = s + self.bias[h].double()
        if self.topo.causal:
            L = self.topo.L
            s = s.masked_fill(torch.ones(L, L, dtype=torch.bool, device=self.device).triu(1), float("-inf"))
        return rows, s

    def _plant(self):
        """q_i = lam_i k_t(i) with scale lam_i (k_t.k_t - k_t.k_j) + b_it - b_ij >= PLANT_GAP + PLANT_MARGIN for every
        other key j the row attends to, in fp64."""
        L, H = self.topo.L, self.H
        for ids in self._chunks(torch.arange(self.topo.sets.shape[0])):
            rows = self.topo.sets[ids].to(self.device)
            c = rows.shape[0]
            for h in range(H):
                cols = slice(h * D, (h + 1) * D)
                kk = self.k[rows][..., cols].double()                                   # [c, L, D]
                t = self.target[ids, :, h].to(self.device)                              # [c, L]
                kt = kk.gather(1, t[..., None].expand(c, L, D))                         # k_t(i) for every query i
                dot = kt @ kk.transpose(-1, -2)                                         # [c, i, j]
                drop = dot.gather(2, t[..., None]) - dot                                # k_t.k_t - k_t.k_j
                need = torch.full_like(dot, PLANT_GAP + PLANT_MARGIN)
                if self.bias is not None:
                    b = self.bias[h].double().expand(c, L, L)
                    need = need - (b.gather(2, t[..., None]) - b)
                other = torch.arange(L, device=self.device)[None, None, :] != t[..., None]
                if self.topo.causal:
                    other = other & torch.ones(L, L, dtype=torch.bool, device=self.device).tril()[None]
                lam = (need / (self.scale * drop)).masked_fill(~other, 0.0).amax(dim=2).clamp_min(1.0)
                assert bool(torch.isfinite(lam).all()), "two keys of a sequence coincide"
                self.q[rows.reshape(-1), cols] = (kt * lam[..., None]).reshape(c * L, D).float()

    def gap(self, dtype=torch.float64):
        """Least logit gap between a planted target and any other key its row attends to, over the whole case.  float64:
        the exact gap of the stored fp32 q, k and bias; float32: the scores formed and rounded in fp32."""
        L, H = self.topo.L, self.H
        least = float("inf")
        for ids in self._chunks(torch.arange(self.topo.sets.shape[0])):
            for h in range(H):
                if dtype == torch.float64:
                    _, s = self._scores(ids, h, self.q, self.k)
                else:
                    rows = self.topo.sets[ids].to(self.device)
                    cols = slice(h * D, (h + 1) * D)
                    s = (self.q[rows][..., cols] * self.scale) @ self.k[rows][..., cols].transpose(-1, -2)
                    if self.bias is not None:
                        s = s + self.bias[h]
                    if self.topo.causal:
                        s = s.masked_fill(torch.ones(L, L, dtype=torch.bool, device=self.device).triu(1), float("-inf"))
                t = self.target[ids, :, h].to(self.device)[..., None]
                st = s.gather(2, t)
                rest = s.scatter(2, t, float("-inf")).amax(dim=2, keepdim=True)
                if L > 1 and not bool(torch.isinf(rest).all()):
                    least = min(least, float((st - rest).min()))
        return least

    def answer(self, set_ids=None):
        """Planted case: v_t(i) for every row of the listed sequences, [n L, 64 H] in the order of sets[set_ids]."""
        set_ids = torch.arange(self.topo.sets.shape[0]) if set_ids is None else set_ids
        sets = self.topo.sets[set_ids]
        target = self.target[set_ids]
        trow = sets[..., None].expand_as(target).gather(1, target).to(self.device)            # [n, L, H] target rows
        v = self.v.reshape(self.topo.M, self.H, D)
        return v[trow, torch.arange(self.H, device=self.device)].reshape(-1, self.H * D)

    def reference(self, set_ids=None, magnitude=False):
        """fp64 softmax(scale q k^T + bias, causal mask) v for every row of the listed sequences (all by default):
        [n L, 64 H] in the order of sets[set_ids].  magnitude=True also returns softmax(...) |v|, the size of the terms
        each output element is summed from."""
        set_ids = torch.arange(self.topo.sets.shape[0]) if set_ids is None else set_ids
        L, H = self.topo.L, self.H
        out = torch.empty(len(set_ids), L, H * D, dtype=torch.float64, device=self.device)
        mag = torch.empty_like(out) if magnitude else None
        n0 = 0
        for ids in self._chunks(set_ids):
            for h in range(H):
                rows, s = self._scores(ids, h, self.q, self.k)
                vv = self.v[rows][..., h * D:(h + 1) * D].double()
                p = torch.softmax(s, dim=-1)
                out[n0:n0 + len(ids), :, h * D:(h + 1) * D] = p @ vv
                if magnitude:
                    mag[n0:n0 + len(ids), :, h * D:(h + 1) * D] = p @ vv.abs()
            n0 += len(ids)
        if magnitude:
            return out.reshape(-1, H * D), mag.reshape(-1, H * D)
        return out.reshape(-1, H * D)

    def rows(self, set_ids=None):
        """Row indices of the listed sequences, in the order reference() and answer() use."""
        set_ids = torch.arange(self.topo.sets.shape[0]) if set_ids is None else set_ids
        return self.topo.sets[set_ids].reshape(-1).to(self.device)


def real_window_bias(H, seed):
    """[H, 64, 64] bias gathered from a random [225, H] table through the window block's own relative_position_index
    (vqgan._WindowAttention), by layout.window_bias as the engine does."""
    from omnitokenizer_b200 import layout as L
    from omnitokenizer_b200.vqgan import _WindowAttention
    index = _WindowAttention(64, 8, H).relative_position_index
    table = torch.rand(225, H, generator=torch.Generator().manual_seed(seed)) * 4.0 - 2.0
    return L.window_bias(table, index, 8)


def random_window_bias(H, seed):
    """[H, 64, 64] bias with no structure at all."""
    return torch.rand(H, 64, 64, generator=torch.Generator().manual_seed(seed)) * 4.0 - 2.0
