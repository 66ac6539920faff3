"""Cases, a host model of the kernel's arithmetic and a derived error bound for the f16 spatial attention cores
(csrc/attention_f16.cu: omt_attn_spatial_h, "x3", and omt_attn_spatial_h1, "x1").

test_attn_f16_cases_cpu.py checks the cases, the model and the bound on the CPU; test_gpu_attn_f16_edges.py runs both
entry points on them.

* The host model restates one (sequence, head) of the kernel: S from the q / k planes (Q_lo.K_hi + Q_hi.K_lo + Q_hi.K_hi,
  or Q_hi.K_hi alone in x1; lo.lo is never formed), the online softmax per 64-key tile in fp32 (running max, alpha and
  ex2 of (s - m) * scale * log2(e), ex2 exact and flushed below 2^-126), p_scale / p_inv from row_scale() of the
  sequence's largest vinv, P'' = e * (vinv_j * p_scale) rounded to fp16 hi / lo as split2u / pack_f16x2_sat do
  (saturating, subnormals kept), O += P''.V on the row-scaled V planes of layout.split_rows_rs, then O * (p_inv / l).
  Sums of exact products are taken in fp64; their fp32 rounding is part of the bound instead.
* Mutants restate the model with one fault each (MUTANTS).
* bound(): a per-output bound of |O - O64| (O64 = fp64 softmax attention of the unsplit operands), derived term by term
  from the model's arithmetic below.  It is normalised by softmax(...) |v| of the output, never by the output itself, so
  a large-v key cannot hide the error of a small-v one.
* Planted cases give every query row one key whose logit beats every other by more than 128 / (scale log2(e)), so ex2 of
  the rest is 0 in fp32: where the target's P'' is a power of two the kernel's result is exact and the model gives its
  bits.  Every key position of every (sequence, head) is a target.  Some targets carry a vinv that is not a power of
  two (P'' then has a lo plane), and every 16th row is a pair row whose two best keys tie in the hi planes and are told
  apart only by Q_lo.K_hi.
"""
import math
from typing import NamedTuple

import torch

from omnitokenizer_b200 import layout as L

KT = 64                          # keys per tile
SCALE = 8.0                      # the engine's softmax scale
LOG2E32 = float(torch.tensor(1.4426950408889634, dtype=torch.float32))
U32 = 2.0 ** -24                 # fp32 unit roundoff (round to nearest)
U_TC = 2.0 ** -23                # one wgmma accumulation step: fp32 result truncated, at most 1 ulp
# ex2.approx.ftz.f32 is modelled as exact.  Its approximation allowance, a relative error of each e and alpha, enters
# the bound here (PTX ISA: ex2.approx.f32 has a maximum relative error of 2^-22 over its range; twice that is allowed).
# ex2(0) = 1 exactly, which the exact planted outputs rely on.
U_EX2 = 2.0 ** -21
MODES = ("x3", "x1")
# One fault each: vinv of the neighbouring qd pair (keys 2 qd ^ 2), vinv of the previous ring stage (the key 64 before),
# the P'' words of rows h = 0 / 1 swapped, the lo plane of P'' dropped (x3), the Q_lo.K_hi product dropped (x3), and
# p_scale from the first key tile's vinv instead of the sequence's.
MUTANTS = ("vinv_qd", "vinv_stage", "swap_h", "no_p_lo", "no_qlo_khi", "pscale_tile0")
X3_ONLY = ("no_p_lo", "no_qlo_khi")


def mutants(mode):
    return [m for m in MUTANTS if mode == "x3" or m not in X3_ONLY]


class Case(NamedTuple):
    name: str
    family: str                  # planted | spread | logit
    nseq: int
    N: int
    H: int
    q: torch.Tensor              # [M, H, 64] float64: the unsplit operands the fp64 reference uses
    k: torch.Tensor
    v: torch.Tensor
    qs: float                    # static pow2 plane scales of q and k (layout.pow2_scale)
    ks: float
    qh: torch.Tensor             # [M, H * 64] float16 planes: q * qs split into hi / lo (lo unscaled)
    ql: torch.Tensor
    kh: torch.Tensor
    kl: torch.Tensor
    vh: torch.Tensor             # row-scaled v planes (layout.split_rows_rs)
    vl: torch.Tensor
    vinv: torch.Tensor           # [H, M] float32

    @property
    def M(self):
        return self.nseq * self.N


def _planes_static(x, ps):
    xs = (x * ps).float()
    hi = xs.clamp(-65504, 65504).half()
    return hi, (xs - hi.float()).half()


def _make(name, family, nseq, N, H, q, k, v, vinv_factor=None, qs=None, ks=None):
    """Planes of (q, k, v) [M, H, 64].  vinv_factor [M, H] (planted): vinv *= factor, v := vinv (V_hi + V_lo) exactly.
    qs / ks: the static plane scales, as the engine takes them from max |q_scale| / max |k_scale| (engine.py); by
    default from the operands' own largest element."""
    M = nseq * N
    qs = L.pow2_scale(float(q.abs().max())) if qs is None else qs
    ks = L.pow2_scale(float(k.abs().max())) if ks is None else ks
    qh, ql = _planes_static(q.reshape(M, H * 64), qs)
    kh, kl = _planes_static(k.reshape(M, H * 64), ks)
    vh, vl, vinv = L.split_rows_rs(v.reshape(M * H, 64).float())
    vinv = vinv.view(M, H)
    if vinv_factor is not None:
        vinv = (vinv * vinv_factor.float()).float()
        v = (vinv.double()[:, :, None] * (vh.double() + vl.double()).view(M, H, 64))
    return Case(name, family, nseq, N, H, q.double(), k.double(), v.double(), qs, ks, qh.reshape(M, H * 64),
                ql.reshape(M, H * 64), kh.reshape(M, H * 64), kl.reshape(M, H * 64), vh.reshape(M, H * 64),
                vl.reshape(M, H * 64), vinv.t().contiguous())


# ------------------------------------------------------------------------------------------------------ planted cases
# Keys are codewords of a 12-dimensional subcode of the Reed-Muller code RM(2, 6): 64 signs, any two distinct codewords
# differ in at least 16, so a query equal to one codeword (times 6 / 8 per component, l2 norm 6 = |q_scale| for q and k)
# has logit 8 * 36 with its own key and at most 8 * 18 with any other: a margin of 144 * log2(e) = 207 > 128 in ex2's
# argument.  Generator 0 is x1 x2 (weight 16): codeword m ^ 1 is m's pair partner.
_RM_GEN = [(0, 1), (0,), (1,), (2,), (3,), (4,), (5,), (2, 3), (4, 5), (0, 2), (1, 3), ()]
PLANT_C = 0.75                   # |q_d| = |k_d| of a planted operand
PLANT_LO = 7.5 / 24576.0         # relative lo part of a planted q: 7.5 of the plane's 24576 (half ulp is 8)


def rm_codewords(n):
    pts = torch.arange(64)
    x = [(pts >> b) & 1 for b in range(6)]
    gens = []
    for mono in _RM_GEN:
        g = torch.ones(64, dtype=torch.long)
        for b in mono:
            g = g * x[b]
        gens.append(g)
    msgs = torch.arange(n)
    bits = torch.stack([(msgs >> i) & 1 for i in range(12)], dim=1)          # [n, 12]
    cw = (bits @ torch.stack(gens)) % 2                                      # [n, 64]
    return 1.0 - 2.0 * cw.double()                                           # signs


def key_exponent(j):
    """log2 of the magnitude of key j's v row in a planted case (vinv grows with it): neighbours 2 apart differ by 3,
    keys 64 apart by 5, and the first key tile's rows are 2^16 smaller, so its largest vinv is at least 2^8 below the
    sequence's and a p_scale taken from it saturates both P'' planes."""
    return 3 * ((j >> 1) & 1) + 5 * ((j >> 6) & 1) - 16 * (j < KT)


def planted(nseq, N, H, seed):
    g = torch.Generator().manual_seed(seed)
    M = nseq * N
    cw = rm_codewords(N)
    q = torch.empty(M, H, 64, dtype=torch.float64)
    k = torch.empty(M, H, 64, dtype=torch.float64)
    v = torch.empty(M, H, 64, dtype=torch.float64)
    target = torch.empty(M, H, dtype=torch.long)       # key position (inside the sequence) of each row's best key
    partner = torch.full((M, H), -1, dtype=torch.long)
    fac = torch.ones(M, H, dtype=torch.float64)
    jpos = torch.arange(N)
    for s in range(nseq):
        for h in range(H):
            r0 = s * N
            word = torch.randperm(N, generator=g)                  # key position -> codeword
            pos = torch.empty(N, dtype=torch.long)
            pos[word] = jpos                                        # codeword -> key position
            k[r0:r0 + N, h] = cw[word] * PLANT_C
            tgt = torch.randperm(N, generator=g)                    # query row -> target key position
            target[r0:r0 + N, h] = tgt
            sgn = torch.where(torch.rand(N, 64, generator=g) < 0.5, -1.0, 1.0).double()
            qh = cw[word[tgt]].clone()
            pair = (torch.arange(N) % 16) == 3
            for i in torch.nonzero(pair).flatten().tolist():
                a = cw[word[tgt[i]]]
                u = int(pos[int(word[tgt[i]]) ^ 1])
                b = cw[word[u]]
                diff = torch.nonzero(a != b).flatten()
                mixed = a.clone()
                mixed[diff[len(diff) // 2:]] = b[diff[len(diff) // 2:]]     # ties with a and b in the hi planes
                qh[i] = mixed
                sgn[i, diff] = mixed[diff] * (a[diff] - b[diff]).sign()      # lo favours a on every differing dim
                partner[r0 + i, h] = u
            q[r0:r0 + N, h] = qh * PLANT_C * (1.0 + sgn * PLANT_LO)
            mag = 2.0 ** torch.tensor([float(key_exponent(j)) for j in range(N)], dtype=torch.float64)
            v[r0:r0 + N, h] = torch.randn(N, 64, generator=g, dtype=torch.float64) * mag[:, None]
            odd = (jpos % 3) == 1                                   # targets whose vinv is not a power of two
            fac[r0:r0 + N, h] = torch.where(odd, 1.0 + torch.randint(1, 2 ** 20, (N,), generator=g).double() / 2 ** 20, 1.0)
    c = _make(f"planted_s{nseq}_n{N}_h{H}", "planted", nseq, N, H, q, k, v, vinv_factor=fac)
    return c, target, partner


# ------------------------------------------------------------------------------------------------- spread and logits
def _unit_scaled(g, shape, scale):
    return torch.nn.functional.normalize(torch.randn(*shape, generator=g, dtype=torch.float64), dim=-1) * scale


def spread(R, nseq, N, H, seed):
    """v row magnitudes 2^0 ... 2^R inside every (sequence, head).  Seven keys in eight are 2^0 rows and hold the
    attention; the eighth are 2^(R u) rows, u uniform (one of them 2^R), whose k points away from the queries' shared
    direction so that their p, about 2^-(R + 4) / (N / 8) each, leaves them a sixteenth of the output's magnitude."""
    g = torch.Generator().manual_seed(seed)
    M = nseq * N
    z = torch.randn(64, generator=g, dtype=torch.float64)
    big = (torch.rand(M, H, generator=g) < 0.125)
    big[0::N, :] = True                                            # every (sequence, head) spans the full 2^R
    u = torch.where(big, torch.rand(M, H, generator=g, dtype=torch.float64), torch.zeros(M, H, dtype=torch.float64))
    u[0::N, :] = 1.0
    gap = (R + 4 + math.log2(N / 8)) * math.log(2)                 # logit gap, natural units, small over big keys
    ab = max(0.5, gap / (SCALE * 1.6))                             # |q| |k| so that 8 |q| |k| (0.8 + 0.8) = gap
    sgn = torch.where(big, -1.0, 1.0).double()[:, :, None]
    q = torch.nn.functional.normalize(z + 0.5 * torch.randn(M, H, 64, generator=g, dtype=torch.float64), dim=-1)
    k = torch.nn.functional.normalize(sgn * z + 0.5 * torch.randn(M, H, 64, generator=g, dtype=torch.float64), dim=-1)
    q, k = q * math.sqrt(ab), k * math.sqrt(ab)
    v = torch.randn(M, H, 64, generator=g, dtype=torch.float64) * (2.0 ** (R * u))[:, :, None]
    return _make(f"spread_r{R}_n{N}_h{H}", "spread", nseq, N, H, q, k, v)


def logits(qmax, kmax, nseq, N, H, seed, ramp=False):
    """Per-dim q / k scales in [qmax / 2, qmax], dim 7 exactly qmax / kmax, and the plane scales the engine would take
    from them: pow2_scale(qmax), pow2_scale(kmax).  Every 37th query row and every 41st key point along dim 7, so those
    pairs reach the logit bound 8 qmax kmax and the planes hold qmax / kmax themselves.  ramp: q and k share a direction
    and the key norms grow along the sequence, so every row's maximum sits in the last key tile, after 63 tiles of
    smaller maxima when N = 4096."""
    g = torch.Generator().manual_seed(seed)
    M = nseq * N
    qsc = qmax * (0.5 + 0.5 * torch.rand(64, generator=g, dtype=torch.float64))
    ksc = kmax * (0.5 + 0.5 * torch.rand(64, generator=g, dtype=torch.float64))
    qsc[7], ksc[7] = qmax, kmax
    if ramp:
        z = torch.randn(64, generator=g, dtype=torch.float64)
        qd = torch.nn.functional.normalize(z + 0.5 * torch.randn(M, H, 64, generator=g, dtype=torch.float64), dim=-1)
        kd = torch.nn.functional.normalize(z + 0.02 * torch.randn(M, H, 64, generator=g, dtype=torch.float64), dim=-1)
        ramp_w = 0.25 + 0.75 * (torch.arange(M) % N).double() / (N - 1)
        q, k = qd * qsc, kd * ksc * ramp_w[:, None, None]
    else:
        q, k = _unit_scaled(g, (M, H, 64), qsc), _unit_scaled(g, (M, H, 64), ksc)
        rows, keys = torch.arange(M) % 37 == 5, torch.arange(M) % 41 == 9
        sq = torch.where(torch.rand(int(rows.sum()), H, generator=g) < 0.5, -1.0, 1.0).double()
        sk = torch.where(torch.rand(int(keys.sum()), H, generator=g) < 0.5, -1.0, 1.0).double()
        q[rows] = 0.0
        q[rows, :, 7] = sq * qmax
        k[keys] = 0.0
        k[keys, :, 7] = sk * kmax
    v = torch.randn(M, H, 64, generator=g, dtype=torch.float64) * torch.logspace(-2, 2, M, dtype=torch.float64)[
        torch.randperm(M, generator=g)][:, None, None]
    tag = f"logit_q{qmax:g}_k{kmax:g}" + ("_ramp" if ramp else "")
    return _make(f"{tag}_n{N}_h{H}", "logit", nseq, N, H, q, k, v, qs=L.pow2_scale(qmax), ks=L.pow2_scale(kmax))


SPREADS = (0, 6, 12, 18, 24, 30)
# (q scale max, k scale max): logit bounds 8 qmax kmax of 32 to 2048, each reached by the dim-7 rows and keys.  With the
# engine's plane scales 1, 4, 8 and 16 put their largest component at the bottom of the planes' binade (exactly 2^14),
# 8 - 2^-9 and 16 - 2^-8 just below its top (2^15 - 8 and 2^15 - 16).  In x1 the hi-only logits are off by up to
# 2^-10 of 8 qmax kmax, several natural units from 8 x 16 on: there the bound falls back to the hull of the v rows
# (bound_head), so those x1 cases check that the output is finite and inside the hull, not its accuracy.
LOGIT_SCALES = ((1.0, 4.0), (4.0, 8.0), (8.0 - 2.0 ** -9, 16.0 - 2.0 ** -8), (16.0, 16.0))


def planted_cases():
    return [planted(2, 128, 8, 11), planted(1, 256, 1, 12), planted(1, 4096, 1, 13)]


def spread_cases():
    return [spread(R, 2, 256, 8, 100 + R) for R in SPREADS] + [spread(30, 1, 4096, 1, 140)]


def logit_cases():
    out = [logits(qm, km, 2, 128, 8, 200 + i) for i, (qm, km) in enumerate(LOGIT_SCALES)]
    out.append(logits(4.0, 4.0, 1, 4096, 1, 210, ramp=True))
    return out


def max_logit(c):
    """largest |8 q.k| of the case, and the largest vinv spread log2(max / min) of any (sequence, head)."""
    qq = c.q.view(c.nseq, c.N, c.H, 64).permute(0, 2, 1, 3)
    kk = c.k.view(c.nseq, c.N, c.H, 64).permute(0, 2, 1, 3)
    lg = max(float((qq[s] @ kk[s].transpose(-1, -2)).abs().max()) for s in range(c.nseq)) * SCALE
    vi = c.vinv.view(c.H, c.nseq, c.N)
    sp = float(torch.log2(vi.amax(-1) / vi.amin(-1)).max())
    return lg, sp


# ------------------------------------------------------------------------------------------------------- host model
def f32(x):
    return x.float().double() if x.dtype == torch.float64 else x.float()


def ex2(x):
    """ex2 of fp32 arguments, exact, rounded to fp32, flushed to 0 below 2^-126 (ex2.approx.ftz)."""
    y = torch.exp2(x.double()).float()
    return torch.where(y < 2.0 ** -126, torch.zeros_like(y), y)


def row_scale(mx):
    eb = (torch.tensor([mx], dtype=torch.float32).view(torch.int32) >> 23) & 0xFF
    eb = int(eb.clamp(15, 254))
    return 2.0 ** (141 - eb), 2.0 ** (eb - 141)


def f16_sat(x):
    return x.float().clamp(-65504.0, 65504.0).half().float()


def _head(c, s, h, rows=None):
    r0 = s * c.N
    sl = slice(r0, r0 + c.N)
    cols = slice(64 * h, 64 * h + 64)
    g = lambda t: t[sl, cols].double()
    qr = slice(r0, r0 + c.N) if rows is None else rows
    gq = lambda t: t[qr, cols].double()
    return gq(c.qh), gq(c.ql), g(c.kh), g(c.kl), g(c.vh), g(c.vl), c.vinv[h, sl].float()


def model_head(c, s, h, mode, mutant=None, rows=None, detail=False):
    """The kernel's output for query rows `rows` (absolute; default the whole sequence) of (sequence s, head h)."""
    qh, ql, kh, kl, vh, vl, vinv = _head(c, s, h, rows)
    x1 = mode == "x1"
    N = c.N
    sc = ql @ kh.t() if not x1 and mutant != "no_qlo_khi" else 0.0
    S = f32(qh @ kh.t() + (0.0 if x1 else qh @ kl.t()) + sc)                        # fp32 accumulator, [rows, N]
    sl32 = float(torch.tensor(SCALE, dtype=torch.float32) * torch.tensor(LOG2E32, dtype=torch.float32)) / (c.qs * c.ks)
    sl32 = float(torch.tensor(sl32, dtype=torch.float32))
    vmx = float(vinv[:KT].max()) if mutant == "pscale_tile0" else float(vinv.max())
    p_scale, p_inv = row_scale(vmx)
    jj = torch.arange(N)
    if mutant == "vinv_qd":
        w = vinv[jj ^ 2]
    elif mutant == "vinv_stage":
        w = vinv[(jj - KT) % N]
    else:
        w = vinv
    wp = (w * p_scale).float()
    R = S.shape[0]
    m = torch.full((R,), -math.inf, dtype=torch.float32)
    o = torch.zeros(R, 64, dtype=torch.float64)
    l = torch.zeros(R, dtype=torch.float64)
    e_all = torch.zeros(R, N, dtype=torch.float32) if detail else None
    keep = torch.ones(R, N, dtype=torch.float64) if detail else None
    for t in range(N // KT):
        ks = slice(t * KT, (t + 1) * KT)
        st = S[:, ks]
        m_new = torch.maximum(m, st.max(dim=1).values)
        alpha = ex2((m - m_new) * sl32).double()
        m = m_new
        e = ex2(((st + (-m_new)[:, None]).float() * sl32).float())
        P = (e * wp[ks]).float()
        if mutant == "swap_h":
            idx = torch.arange(R) ^ 8
            P = P[idx]
        hi = f16_sat(P)
        lo = f16_sat(P - hi) if not x1 and mutant != "no_p_lo" else torch.zeros_like(P)
        hi, lo = hi.double(), lo.double()
        vt_h, vt_l = vh[ks], vl[ks]
        pv = hi @ vt_h + (0.0 if x1 else hi @ vt_l + lo @ vt_h)
        o = o * alpha[:, None] + pv
        l = l * alpha + e.double().sum(dim=1)
        if detail:
            keep[:, :t * KT] *= alpha[:, None]
            e_all[:, ks] = e
    inv = f32(torch.tensor(p_inv, dtype=torch.float64) / f32(l))
    out = f32(o * inv[:, None])
    if not detail:
        return out
    return out, dict(S=S, e=e_all.double() * keep, l=l, p_scale=p_scale, p_inv=p_inv, sl32=sl32, m=m)


def reference_head(c, s, h, rows=None):
    """fp64 softmax(8 q k^T) of the unsplit operands: (probabilities [rows, N], output [rows, 64])."""
    r0 = s * c.N
    qr = slice(r0, r0 + c.N) if rows is None else rows
    qq, kk, vv = c.q[qr, h], c.k[r0:r0 + c.N, h], c.v[r0:r0 + c.N, h]
    p = torch.softmax((qq @ kk.t()) * SCALE, dim=-1)
    return p, p @ vv


def bound_head(c, s, h, mode, rows=None):
    """Per-output bound of |O_kernel - O64| for the query rows of (s, h), with the model's output and O64.

    Write O = sum_j w_j v_j / sum_j w_j.  Each source of error becomes a relative error eps_j of a key's weight w_j,
    |eps_j| <= E_j, or an absolute error of a product.  With p_j the exact softmax, mag_d = sum_j p_j |v_jd| and
    Ebar = sum_j p_j E_j, the weights move by p_j (eps_j - sum_k p_k eps_k) / (1 + sum_k p_k eps_k), and
    |eps_j - sum_k p_k eps_k| <= (1 - p_j) E_j + Ebar - p_j E_j, so
        |dO_d| <= sum_j p_j (E_j + Ebar - 2 p_j E_j) |v_jd| / (1 - Ebar)  +  the absolute terms
    (a key that holds all the weight moves nothing: the row sum carries the same error).
    Weight errors E_j:
      * the logit: q / k planes (2^-22 of each component for x3, 2^-11 for x1, plus a subnormal 2^-25 / plane scale),
        the dropped lo.lo product (x3, 2^-22), and the fp32 accumulator (12 wgmma steps for x3, 4 for x1, 2^-23 of the
        sum of |products| each), all times scale sum_d |q_d k_jd|; exp of that minus 1.
      * ex2's argument (s - m) * scale_log2: the fp32 subtraction, the product and scale_log2's own rounding, 3 2^-24
        |x| ln 2; ex2 itself U_EX2.  alpha's error cancels (o and l are scaled by the same alpha) except the fp32 products
        o * alpha and l * alpha: 2 2^-24 per key tile.
    Product / sum errors:
      * P'' = e * (vinv p_scale): one fp32 rounding; its fp16 split: 2^-22 relative for x3 (hi / lo, 11 bits each),
        2^-11 for x1.  The row sum adds the unrounded e, so these do not cancel.
      * V planes: 2^-22 of |v_jd| for x3 (2^-11 for x1, and P''_lo.V_lo as above), 2^-25 vinv_j in subnormals.
      * P'' below fp16's normal range: 2^-25 absolute in P'' units, i.e. 2^-25 p_inv |V_jd| / l per key with e_j > 0.
        This is the precision floor of the shared p_scale: a key whose vinv is 2^-r of the sequence's largest (its v
        row 2^r larger than the smallest) gets P'' = p 2^(14 - r).
      * keys whose e flushed to 0 (ex2 below 2^-126): their whole share p_j |v_jd|.
      * the fp32 P''.V accumulator: 2^-23 per wgmma step (12 per key tile for x3, 4 for x1) of sum_j e_j |V'_jd| / l.
      * the row sum (16 lane adds, one fma per key tile, 2 shuffle adds) and the final p_inv / l and O * inv: 2^-24
        each, relative to |O_d| <= mag_d.
    """
    x1 = mode == "x1"
    N, nt = c.N, c.N // KT
    out, d = model_head(c, s, h, mode, rows=rows, detail=True)
    p, ref = reference_head(c, s, h, rows)
    qh, ql, kh, kl, vh, vl, vinv = _head(c, s, h, rows)
    r0 = s * c.N
    qr = slice(r0, r0 + c.N) if rows is None else rows
    qa, ka = c.q[qr, h].abs(), c.k[r0:r0 + N, h].abs()
    vv = c.v[r0:r0 + N, h]
    u_pl = 2.0 ** -11 if x1 else 2.0 ** -22
    n_s = 4 if x1 else 12
    eps_s = 2 * u_pl + (0.0 if x1 else 2.0 ** -22) + n_s * U_TC * (1 + 2.0 ** -20)
    qk = qa @ ka.t()
    dS = SCALE * (eps_s * qk + 2.0 ** -25 * ((qa.sum(1, keepdim=True) / c.ks) + ka.sum(1)[None, :] / c.qs))
    x = d["S"] * d["sl32"] - d["m"].double()[:, None] * d["sl32"]
    tile = torch.arange(N) // KT
    E = (torch.expm1(dS) + 3 * U32 * x.abs() * math.log(2) + U_EX2 + 2 * U32 * (nt - 1 - tile).double()[None, :]
)
    E = E * (1 + 1e-6)
    pE = p * E
    Ebar = pE.sum(1, keepdim=True)
    va = vv.abs()
    mag = p @ va
    b = (pE @ va + Ebar * mag - 2 * (p * pE) @ va).clamp_min(0) / (1 - Ebar)
    # V planes
    b = b + (2.0 ** -11 if x1 else 2.0 ** -22) * mag + 2.0 ** -25 * (p @ vinv.double())[:, None]
    # P'' subnormal floor and flushed keys
    lk = d["l"][:, None]
    vfull = vh.abs() + (0.0 if x1 else vl.abs())
    alive = (d["e"] > 0).double()
    b = b + 2.0 ** -25 * d["p_inv"] * (alive @ vfull) / lk + ((1 - alive) * p) @ va
    # P''.V accumulator, the row sum and the final scaling
    vplane = vinv.double()[:, None] * vfull
    # P'' (its fp32 rounding and fp16 split; l sums the unrounded e), the P''.V accumulator, the row sum, the scaling
    b = b + (U32 + u_pl + n_s * nt * U_TC) * (d["e"] @ vplane) / lk + (16 + nt + 2 + 2) * U32 * 1.01 * mag
    # where the logit error is too large for the expansion (x1 at large logits): O is a convex combination of the plane
    # v rows, so |dO_d| <= max_j |v'_jd| + |O64_d|
    triv = (1 + 2.0 ** -10) * vplane.amax(0)[None, :] + ref.abs()
    b = torch.where(Ebar < 0.5, torch.minimum(b, triv), triv)
    return out, ref, b, mag


def exact_rows(c, s, h, mode, target):
    """Planted rows whose kernel result is exact: one-hot in the model, and the target's P'' a power of two that fp16
    holds, so P''.V = P'' (V_hi + V_lo) and the final scaling are exact in fp32."""
    r0 = s * c.N
    _, d = model_head(c, s, h, mode, detail=True)
    onehot = (d["e"] > 0).sum(1) == 1
    t = target[r0:r0 + c.N, h]
    vi = c.vinv[h, r0:r0 + c.N].double()
    P = vi[t] * d["p_scale"]
    pow2 = (torch.frexp(P).mantissa == 0.5) & (P >= 2.0 ** -24)
    return onehot & pow2


ROW_BLOCK = 512


def evaluate(c, mode, mutant=None, out=None, target=None):
    """Run the model (or a mutant) on every (sequence, head) and compare it, or a kernel's output `out` [M, H * 64], with
    the check the GPU test makes: bit-exact against the model on the planted rows the model predicts exactly, within
    bound_head() of fp64 elsewhere.  Returns (ok, worst |err| / bound, worst |err| / mag, worst bound / mag, bad)."""
    worst_r, worst_e, worst_b, bad = 0.0, 0.0, 0.0, 0
    ok = True
    for s in range(c.nseq):
        for h in range(c.H):
            r0 = s * c.N
            ex = exact_rows(c, s, h, mode, target) if c.family == "planted" else torch.zeros(c.N, dtype=torch.bool)
            for b0 in range(0, c.N, ROW_BLOCK):
                rows = slice(r0 + b0, r0 + min(c.N, b0 + ROW_BLOCK))
                mout, ref, bnd, mag = bound_head(c, s, h, mode, rows=rows)
                if out is not None:
                    got = out[rows, 64 * h:64 * h + 64].double()
                elif mutant is not None:
                    got = model_head(c, s, h, mode, mutant=mutant, rows=rows).double()
                else:
                    got = mout.double()
                exb = ex[b0:b0 + ROW_BLOCK]
                if bool(exb.any()):
                    diff = (got[exb].float().view(torch.int32) != mout[exb].float().view(torch.int32)).any(1)
                    bad += int(diff.sum())
                    ok &= not bool(diff.any())
                err = (got - ref).abs()
                fin = torch.isfinite(got).all(1)
                bad += int((~fin).sum())
                ok &= bool(fin.all())
                nx = ~exb & fin
                if bool(nx.any()):
                    r = err[nx] / bnd[nx]
                    worst_r = max(worst_r, float(r.max()))
                    bad += int((r > 1).any(1).sum())
                    ok &= bool((r <= 1).all())
                mg = mag.amax(1, keepdim=True).clamp_min(1e-300)
                worst_e = max(worst_e, float((err[fin] / mg[fin]).max()) if bool(fin.any()) else math.inf)
                worst_b = max(worst_b, float((bnd / mg).max()))
    return ok, worst_r, worst_e, worst_b, bad
