"""Cases, host models and float64 references for the evaluation reductions of csrc/quality.cu: omt_psnr_ssim,
omt_lpips_head, omt_softmax_rows and omt_inception_score.

test_quality_cases_cpu.py checks the builders, the references and the bars on the CPU; test_gpu_quality_reductions.py
launches the kernels on the same builders and checks them with the same check functions.

* Cases put the sizes where these kernels go wrong into every sweep: the valid SSIM crop on both sides of the 32 x 32
  output tile, feature maps with fewer pixels than the head's 16 warps and channel counts below a warp, softmax rows
  below one warp and across the 256-thread stride, KL rows across the 16-warp row stride and past 512 classes, and
  padding columns (NaN) that no kernel may read.
* References are float64: oracle.quality_oracle for PSNR / SSIM / the LPIPS head, torch.softmax of the fp64 logits,
  scipy.stats.entropy with numpy column means for the Inception Score.
* Models restate each kernel's arithmetic on the host; MUTANTS give each one fault.  The CPU test shows the unmutated
  model passes each check and every mutant fails it, so the GPU checks would catch a kernel with that fault.
* Every check returns (ok, worst measured error in the units of its bar, a message naming the first failure).
"""
import math
from typing import List, NamedTuple, Optional

import numpy as np
import torch

from oracle import quality_oracle as qo

U32 = 2.0 ** -24                  # fp32 unit roundoff (round to nearest)
TINY32 = 2.0 ** -149              # fp32's smallest subnormal
TAPS = qo.gaussian(11, 1.5)       # the 11 Gaussian taps every SSIM case runs with (fp64)

MUTANTS = {
    "ssim": ("halo_shift", "ignore_sel_b"),        # last tile column's halo one column right; table 0 for image b
    "head": ("drop_last", "pad_read"),             # last pixel skipped when hw % 16 != 0; the Cs - C padding summed
    "softmax": ("sum_short", "max_early"),         # sum over N - 1 columns; max before the last 256-column stride
    "is": ("mean_short", "zero_nan"),              # column sum over n - 1 rows; x log(x / q) also where x == 0
}


def padded(x, ld):
    """x [rows, C] in a [rows, ld] buffer on x's device whose columns past C are NaN."""
    buf = torch.full((x.shape[0], ld), float("nan"), dtype=x.dtype, device=x.device)
    buf[:, :x.shape[1]] = x
    return buf


# ============================================================================================================ PSNR / SSIM
SSIM_SIZES = (11, 12, 42, 43, 53, 74, 75)    # H, W; the valid crop Ho = H - 10 is 1, 2, 32, 33, 43, 64, 65
SS_T = 32                                    # outputs per tile side
SSIM_BAR = 1e-12                             # sse relative, SSIM absolute: both are fp64 throughout


def byte_tables():
    """fp32 [2, 256]: table 0 is byte / 255, table 1 a gamma curve (byte / 255)^(1 / 2.2), so a wrong pick shows."""
    v = torch.arange(256, dtype=torch.float64) / 255
    return torch.stack([torch.arange(256, dtype=torch.float32) / 255, (v ** (1 / 2.2)).float()])


def axis_marks(n):
    """Coordinates along an axis of n pixels where a one-pixel difference sits on a tile edge: each tile's first input
    column, its last output column, its last halo column and the column past its halo, and the frame's last column."""
    marks = {n - 1}
    for x0 in range(0, n - 10, SS_T):
        marks |= {x0, x0 + SS_T - 1, x0 + SS_T + 9, x0 + SS_T + 10}
    return sorted(m for m in marks if m < n)


class SsimCase(NamedTuple):
    name: str
    form: str                    # "u8" | "f32"
    H: int
    W: int
    a: torch.Tensor              # [P, H, W, 3] uint8 or float32
    b: torch.Tensor
    sel_a: Optional[torch.Tensor]    # [P] int32 table index per pair (u8 form)
    sel_b: Optional[torch.Tensor]
    kinds: List[str]             # per pair: noise | same | const | pixel | wide

    @property
    def P(self):
        return self.a.shape[0]


def _ssim_case(H, W, form):
    g = torch.Generator().manual_seed(1000 * H + W + (0 if form == "u8" else 7))
    A, B, sa, sb, kinds = [], [], [], [], []

    def add(a, b, kind, s=(0, 0)):
        A.append(a)
        B.append(b)
        sa.append(s[0])
        sb.append(s[1])
        kinds.append(kind)

    if form == "u8":
        for s in ((0, 0), (1, 0), (0, 1), (1, 1)):
            a = torch.randint(0, 256, (H, W, 3), generator=g, dtype=torch.uint8)
            n = torch.randint(-20, 21, (H, W, 3), generator=g, dtype=torch.int16)
            add(a, (a.to(torch.int16) + n).clamp(0, 255).to(torch.uint8), "noise", s)
        for s in ((0, 0), (1, 1)):
            a = torch.randint(0, 256, (H, W, 3), generator=g, dtype=torch.uint8)
            add(a, a.clone(), "same", s)
        add(torch.full((H, W, 3), 200, dtype=torch.uint8), torch.full((H, W, 3), 190, dtype=torch.uint8), "const")
        add(torch.full((H, W, 3), 37, dtype=torch.uint8), torch.full((H, W, 3), 250, dtype=torch.uint8), "const", (1, 0))
        i = 0
        for r in axis_marks(H):
            for c in axis_marks(W):
                a = torch.randint(0, 255, (H, W, 3), generator=g, dtype=torch.uint8)
                b = a.clone()
                b[r, c, i % 3] += 1
                add(a, b, "pixel", (i % 2, i % 2))
                i += 1
        sel = lambda s: torch.tensor(s, dtype=torch.int32)
        return SsimCase(f"u8_{H}x{W}", form, H, W, torch.stack(A), torch.stack(B), sel(sa), sel(sb), kinds)
    for _ in range(3):                       # values outside [0, 1], negative ones among them
        a = torch.randn(H, W, 3, generator=g) * 1.5
        add(a, a + 0.1 * torch.randn(H, W, 3, generator=g), "wide")
    a = torch.randn(H, W, 3, generator=g) * 1.5
    add(a, a.clone(), "same")
    add(torch.full((H, W, 3), -0.75), torch.full((H, W, 3), 1.5), "const")
    for r, c in ((H - 1, W - 1), (min(H - 1, SS_T + 9), min(W - 1, SS_T + 9))):
        a = torch.rand(H, W, 3, generator=g)
        b = a.clone()
        b[r, c, 1] += 0.25
        add(a, b, "pixel")
    return SsimCase(f"f32_{H}x{W}", form, H, W, torch.stack(A), torch.stack(B), None, None, kinds)


def ssim_cases(form):
    """One case per (H, W) in SSIM_SIZES x SSIM_SIZES.  u8: noisy pairs in all four table selections, identical pairs,
    two constant pairs, and a one-pixel difference at every (row, column) of axis_marks, each in one pair.  f32: noisy
    pairs of values around +-1.5, an identical pair, a constant pair and two one-pixel differences."""
    return [_ssim_case(H, W, form) for H in SSIM_SIZES for W in SSIM_SIZES]


def ssim_values(case, ignore_sel_b=False):
    """The fp64 values the kernel loads: [P, H, W, 3] for image a and image b."""
    if case.form == "f32":
        return case.a.double(), case.b.double()
    t = byte_tables().double()
    sb = torch.zeros_like(case.sel_b) if ignore_sel_b else case.sel_b
    va = t[case.sel_a.long()[:, None, None, None], case.a.long()]
    vb = t[sb.long()[:, None, None, None], case.b.long()]
    return va, vb


def ssim_reference(case):
    """(sse, ssim) float64 [P]: the sum of squared differences and oracle.quality_oracle.ssim of every pair."""
    va, vb = ssim_values(case)
    sse = ((va - vb) ** 2).sum((1, 2, 3))
    ssim = torch.tensor([qo.ssim(va[p].permute(2, 0, 1).numpy(), vb[p].permute(2, 0, 1).numpy(), TAPS)
                         for p in range(case.P)], dtype=torch.float64)
    return sse, ssim


def ssim_constant(alpha, beta):
    """SSIM of two constant frames of values alpha and beta: every variance is 0, so each map term is
    (2 alpha beta + C1) C2 / ((alpha^2 + beta^2 + C1) C2)."""
    C1 = 0.01 ** 2
    return (2 * alpha * beta + C1) / (alpha * alpha + beta * beta + C1)


def ssim_constant_slack(alpha, beta):
    """How far a computed SSIM of constant frames may sit from the closed form, and so two computations from each
    other.  The variances s = E[x y] - mu_x mu_y are 0 only up to rounding: each filtered map carries 22 roundings of
    2^-53 (11 taps each way) of v^2 = max(alpha^2, beta^2), so |ds| <= 44 2^-53 v^2 for each of s1, s2, s12.  The map
    term moves by at most (2 |ds12| + |ds1| + |ds2|) / C2, and two computations each by that much."""
    return 2 * 4 * 44 * 2.0 ** -53 * max(alpha * alpha, beta * beta) / 0.03 ** 2


def ssim_model(case, mutant=None):
    """psnr_ssim_kernel on the host in fp64: per channel and per 32-column tile, the tile's 42-column input halo (0 past
    the frame), the 11-tap filter along w, then along h, the SSIM map over the valid crop, the channel means."""
    va, vb = ssim_values(case, ignore_sel_b=mutant == "ignore_sel_b")
    P, H, W = case.P, case.H, case.W
    Ho, Wo = H - 10, W - 10
    ty, tx = -(-Ho // SS_T), -(-Wo // SS_T)
    k = torch.as_tensor(TAPS, dtype=torch.float64)
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    sse = ((va - vb) ** 2).sum((1, 2, 3))
    total = torch.zeros(P, dtype=torch.float64)
    rows = ty * SS_T + 10
    for c in range(3):
        acc = torch.zeros(P, dtype=torch.float64)
        for t in range(tx):
            x0 = t * SS_T
            shift = 1 if mutant == "halo_shift" and t == tx - 1 else 0
            cols = torch.arange(SS_T + 10) + x0 + shift
            inside = cols < W
            x = torch.zeros(P, rows, SS_T + 10, dtype=torch.float64)
            y = torch.zeros_like(x)
            x[:, :H, inside] = va[:, :, cols[inside], c]
            y[:, :H, inside] = vb[:, :, cols[inside], c]
            maps = []
            for z in (x, y, x * x, y * y, x * y):
                h = sum(k[j] * z[:, :, j:j + SS_T] for j in range(11))
                maps.append(sum(k[j] * h[:, j:j + ty * SS_T, :] for j in range(11)))
            m1, m2, e11, e22, e12 = maps
            m1s, m2s, m12 = m1 * m1, m2 * m2, m1 * m2
            num = (2 * m12 + C1) * (2 * (e12 - m12) + C2)
            den = (m1s + m2s + C1) * ((e11 - m1s) + (e22 - m2s) + C2)
            valid = (torch.arange(ty * SS_T)[:, None] < Ho) & (torch.arange(SS_T)[None, :] + x0 < Wo)
            acc = acc + torch.where(valid, num / den, torch.zeros_like(num)).sum((1, 2))
        total = total + acc / (Ho * Wo)
    return sse, total / 3


def ssim_bars(case):
    """Per pair, the SSIM bar: SSIM_BAR, plus ssim_constant_slack for constant pairs."""
    va, vb = ssim_values(case)
    return torch.tensor([SSIM_BAR + (ssim_constant_slack(float(va[p, 0, 0, 0]), float(vb[p, 0, 0, 0]))
                                     if k == "const" else 0.0) for p, k in enumerate(case.kinds)], dtype=torch.float64)


def ssim_check(case, sse, ssim, ref=None):
    """sse within SSIM_BAR relative of fp64 and SSIM within ssim_bars absolute; identical frames give sse == 0 and
    SSIM == 1 exactly.  Returns (ok, worst sse rel, worst ssim abs of the other pairs, worst ssim abs / bar of the
    constant pairs, message)."""
    r_sse, r_ssim = ssim_reference(case) if ref is None else ref
    sse, ssim = sse.double().cpu(), ssim.double().cpu()
    e_sse = ((sse - r_sse).abs() / r_sse.clamp_min(1e-300)).nan_to_num(math.inf)
    e_sse = torch.where(sse == r_sse, torch.zeros_like(e_sse), e_sse)
    e_ssim = (ssim - r_ssim).abs().nan_to_num(math.inf)
    bars = ssim_bars(case)
    bad = (e_sse > SSIM_BAR) | (e_ssim > bars)
    const = torch.tensor([k == "const" for k in case.kinds])
    e_const = float((e_ssim / bars)[const].max()) if bool(const.any()) else 0.0
    e_ssim = torch.where(const, torch.zeros_like(e_ssim), e_ssim)
    same = torch.tensor([k == "same" for k in case.kinds])
    bad |= same & ((sse != 0.0) | (ssim != 1.0))
    msg = ""
    if bool(bad.any()):
        p = int(bad.nonzero()[0])
        msg = (f"{case.name} pair {p} ({case.kinds[p]}): sse {float(sse[p])!r} vs {float(r_sse[p])!r}, "
               f"ssim {float(ssim[p])!r} vs {float(r_ssim[p])!r}")
    return not bool(bad.any()), float(e_sse.max()), float(e_ssim.max()), e_const, msg


# ============================================================================================================ LPIPS head
HEAD_C = (1, 3, 31, 32, 33, 64, 512)
HEAD_HW = ((1, 1), (3, 5), (4, 4), (17, 1), (37, 29))      # h w = 1, 15, 16, 17, 1073 around the kernel's 16 warps
HEAD_P = (1, 7)
HEAD_WARPS = 16
HEAD_CEIL = 2e-6              # the bar test_gpu_quality.py's head test holds; no derived bar here exceeds it


def head_k(C):
    """Roundings of the head's fp32 arithmetic, relative to mag = mean over pixels of sum_c |w_c| (|na_c| + |nb_c|)^2
    (na, nb the exactly normalised vectors).  With m = ceil(C / 32) terms per lane:
      * |x|^2: m fmas per lane and 5 butterfly adds, (m + 5) u; its sqrt halves that and adds u, the + 1e-10 adds u;
        the division adds u: each normalised entry is off by e_n = ((m + 5) / 2 + 3) u of itself;
      * d = na - nb: (e_n + u)(|na| + |nb|); d * d: twice that, plus u, so (2 e_n + 3 u)(|na| + |nb|)^2;
      * the weighted sum: m fmas per lane and 5 butterfly adds over positive terms, (m + 5) u;
      * the fp64 pixel sum and division are exact to fp32's eye; the final rounding to fp32, u.
    Total (2 m + 20) u."""
    return 2 * (-(-C // 32)) + 20


def head_bar(C):
    return min(head_k(C) * U32, HEAD_CEIL)


class HeadCase(NamedTuple):
    name: str
    C: int
    Cs: int
    P: int
    h: int
    w: int
    x: torch.Tensor              # [2P, h, w, Cs] float32, NaN in the Cs - C padding columns
    lin: torch.Tensor            # [C] float32
    tap: int
    prev: torch.Tensor           # [5, P] float32: the earlier taps' values the total adds
    equal: torch.Tensor          # [P] bool: pairs whose two images are equal (the head is exactly 0)

    @property
    def hw(self):
        return self.h * self.w


def head_cases():
    """Every C of HEAD_C, Cs = C and C + 4 k, every map size of HEAD_HW and P of HEAD_P.  Features are ReLU'd normal
    values, channel 0 raised by 0.5, scaled per pixel by 10^u, u in [-3, 3].  With C = 1 every such vector normalises
    to 1, so the planted zero vectors are what the head measures.  Image a of pair 0 has an all-zero vector at pixel 0, image b of the
    last pair one at the last pixel (unless that is the same pixel of the same pair); pair 3 of P = 7 has equal
    images.  Taps rotate through 0 .. 4."""
    out = []
    i = 0
    for C in HEAD_C:
        for Cs in (C, C + 4 * (1 + C % 3)):
            for h, w in HEAD_HW:
                for P in HEAD_P:
                    g = torch.Generator().manual_seed(7919 * i + C)
                    x = torch.relu(torch.randn(2 * P, h, w, C, generator=g))
                    x[..., 0] = x[..., 0] + 0.5          # no vector is zero but the planted ones
                    x = x * 10.0 ** (torch.rand(2 * P, h, w, 1, generator=g) * 6 - 3)
                    x[0, 0, 0] = 0
                    if P > 1 or h * w > 1:       # else it is pair 0's only pixel too, and the head would be 0
                        x[2 * P - 1, h - 1, w - 1] = 0
                    equal = torch.zeros(P, dtype=torch.bool)
                    if P > 3:
                        x[P + 3] = x[3]
                        equal[3] = True
                    xs = torch.full((2 * P, h, w, Cs), float("nan"))
                    xs[..., :C] = x
                    out.append(HeadCase(f"C{C}_Cs{Cs}_{h}x{w}_P{P}", C, Cs, P, h, w, xs, torch.rand(C, generator=g),
                                        i % 5, torch.rand(5, P, generator=g), equal))
                    i += 1
    return out


def head_reference(case):
    """(head, mag) float64 [P]: oracle.quality_oracle.lpips_head64, and the scale head_k's roundings are relative to."""
    f = case.x[..., :case.C].double().permute(0, 3, 1, 2)
    fa, fb = f[:case.P], f[case.P:]
    ref = qo.lpips_head64(fa, fb, case.lin)
    na = fa / (torch.sqrt((fa ** 2).sum(1, keepdim=True)) + 1e-10)
    nb = fb / (torch.sqrt((fb ** 2).sum(1, keepdim=True)) + 1e-10)
    mag = ((na.abs() + nb.abs()) ** 2 * case.lin.double().abs().view(1, -1, 1, 1)).sum(1).mean((1, 2))
    return ref, mag


def _fma32(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def _lanes(t, m):
    """[..., n] -> [..., m, 32]: element c to (c // 32, c % 32), zero-filled."""
    z = torch.zeros(*t.shape[:-1], m * 32, dtype=t.dtype)
    z[..., :t.shape[-1]] = t
    return z.view(*t.shape[:-1], m, 32)


def _butterfly(v):
    """warp_sum: the xor butterfly over the last dimension (32 lanes) in fp32; every lane ends with the same value."""
    lane = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., lane ^ o]
    return v[..., 0]


def head_model(case, mutant=None):
    """lpips_head_kernel on the host: per pixel, lane partials of the squared norms (fma chains over c = lane + 32 i),
    the butterfly, sqrt + 1e-10, fp32 divisions, the lin-weighted fma chain and the butterfly; the pixels summed in
    fp64 and divided by h w, rounded to fp32.  Returns [P] float32."""
    P, hw = case.P, case.hw
    cols = case.Cs if mutant == "pad_read" else case.C
    used = hw - 1 if mutant == "drop_last" and hw % HEAD_WARPS else hw
    x = case.x.reshape(2 * P, hw, case.Cs)[:, :used, :cols]
    m = -(-cols // 32)
    lin = torch.zeros(cols)
    lin[:case.C] = case.lin
    xa, xb, wl = _lanes(x[:P], m), _lanes(x[P:], m), _lanes(lin, m)
    na = torch.zeros(P, used, 32)
    nb = torch.zeros(P, used, 32)
    for i in range(m):
        na = _fma32(xa[:, :, i], xa[:, :, i], na)
        nb = _fma32(xb[:, :, i], xb[:, :, i], nb)
    eps = torch.tensor(1e-10, dtype=torch.float32)
    da = (torch.sqrt(_butterfly(na)) + eps)[..., None]
    db = (torch.sqrt(_butterfly(nb)) + eps)[..., None]
    s = torch.zeros(P, used, 32)
    for i in range(m):
        d = xa[:, :, i] / da - xb[:, :, i] / db
        s = _fma32(wl[i], d * d, s)
    s = _butterfly(s).double()
    return (s.sum(1) / hw).float()


def head_check(case, got, ref=None):
    """|head - fp64| <= head_bar(C) mag, and exactly 0 for equal pairs.  Returns (ok, worst err / mag, message)."""
    r, mag = head_reference(case) if ref is None else ref
    got = got.double().cpu()
    err = (got - r).abs().nan_to_num(math.inf)
    bad = err > head_bar(case.C) * mag
    bad |= case.equal & (got != 0.0)
    rel = err / mag.clamp_min(1e-300)
    msg = ""
    if bool(bad.any()):
        p = int(bad.nonzero()[0])
        msg = f"{case.name} pair {p}: {float(got[p])!r} vs {float(r[p])!r} (mag {float(mag[p]):.3e})"
    return not bool(bad.any()), float(rel.max()), msg


def head_total(prev, tap, r):
    """lpips.py's val = res[0]; val += res[1] ... in fp32 up to `tap`, whose value is r: ((t0 + t1) + t2) + ..."""
    v = r if tap == 0 else prev[0]
    for i in range(1, tap + 1):
        v = v + (r if i == tap else prev[i])
    return v


# ============================================================================================================ softmax
SM_N = (1, 2, 31, 32, 255, 256, 257, 1000, 1008, 4097, 6144)
SM_THREADS = 256
SM_FAMILIES = ("logits", "spread", "ties", "inf", "equal", "dominant")
SM_ROWS = (1, 333)
SM_PADS = ((0, 0), (3, 0), (0, 3), (3, 3))     # (ldx - N, ldy - N)


def softmax_k(N):
    """Roundings of an entry y = e / s relative to y: e's rounding to fp32 in the numerator, and the same rounding of
    every term inside s; ceil(N / 256) per-thread adds, 5 butterfly levels and 7 warp adds in s; the division.
    Subnormal e and y add at most 2^-150 each in absolute terms (the bar's 2^-149)."""
    return -(-N // SM_THREADS) + 15


class SoftmaxCase(NamedTuple):
    name: str
    N: int
    ldx: int
    ldy: int
    xbuf: torch.Tensor           # [rows, ldx] float32, NaN past N
    family: torch.Tensor         # [rows] index into SM_FAMILIES

    @property
    def x(self):
        return self.xbuf[:, :self.N]

    @property
    def rows(self):
        return self.xbuf.shape[0]


def softmax_rows(rows, N, seed, device="cpu", first=0):
    """float32 [rows, N]; row r belongs to SM_FAMILIES[(r + first) % 6]:
    logits    normal values times 3;
    spread    an offset minus a permutation of linspace(0, 120, N): e = exp(-t) is an fp32 subnormal for t in
              (87.3, 103.3] and rounds to 0 past 103.98, so such rows hold subnormal and zero probabilities;
    ties      every fifth column and the last one equal to the row's maximum;
    inf       by (r // 6) % 3: -inf in every seventh column from column 1; one +inf at column N // 2; all -inf;
    equal     one value across the row: y = fl(1 / N);
    dominant  the last column 100 above the rest: the maximum sits in the last 256-column stride."""
    g = torch.Generator(device=device).manual_seed(seed)
    x = torch.randn(rows, N, generator=g, device=device) * 3
    fam = (torch.arange(rows, device=device) + first) % 6
    t = torch.linspace(0, 120, N, dtype=torch.float64, device=device)
    perm = torch.rand(rows, N, generator=g, device=device).argsort(1)
    off = torch.randn(rows, 1, generator=g, device=device, dtype=torch.float64) * 5
    x = torch.where((fam == 1)[:, None], (off - t[perm]).float(), x)
    mx = x.max(1, keepdim=True).values + 1
    tie = (torch.arange(N, device=device) % 5 == 0) | (torch.arange(N, device=device) == N - 1)
    x = torch.where((fam == 2)[:, None] & tie[None, :], mx.expand(rows, N), x)
    var = (torch.arange(rows, device=device) // 6) % 3
    col = torch.arange(N, device=device)[None, :]
    inf = fam[:, None] == 3
    x = torch.where(inf & (var[:, None] == 0) & (col % 7 == 1), torch.full_like(x, -math.inf), x)
    x = torch.where(inf & (var[:, None] == 1) & (col == N // 2), torch.full_like(x, math.inf), x)
    x = torch.where(inf & (var[:, None] == 2), torch.full_like(x, -math.inf), x)
    x = torch.where((fam == 4)[:, None], x[:, :1].expand(rows, N), x)
    dom = (fam == 5)[:, None] & (col == N - 1)
    x = torch.where(dom, x.max(1, keepdim=True).values + 100, x)
    return x.contiguous(), fam


def softmax_cases(device="cpu"):
    out = []
    for i, N in enumerate(SM_N):
        for j, (px, py) in enumerate(SM_PADS):
            for rows in SM_ROWS:
                x, fam = softmax_rows(rows, N, 31 * i + 7 * j + rows, device, first=i + j)
                out.append(SoftmaxCase(f"N{N}_ldx{N + px}_ldy{N + py}_rows{rows}", N, N + px, N + py,
                                       padded(x, N + px), fam))
    return out


def softmax_model(x, mutant=None):
    """softmax_rows_kernel on the host, x float32 [rows, N] (CPU): the fp32 max (fmaxf over the row, or over all but
    the last 256-column stride), e = fp32(exp(x - m)) in fp64, each thread's partial over its columns in order, the
    warp butterfly, the eight warps in order, one fp32 division per entry."""
    rows, N = x.shape
    K = -(-N // SM_THREADS)
    if mutant == "max_early":
        m = x[:, :(K - 1) * SM_THREADS].amax(1) if K > 1 else torch.full((rows,), -math.inf)
    else:
        m = x.amax(1)
    e = torch.exp(x.double() - m.double()[:, None]).float()
    terms = torch.zeros(rows, K * SM_THREADS)
    n = N - 1 if mutant == "sum_short" else N
    terms[:, :n] = e[:, :n]
    s = torch.zeros(rows, SM_THREADS)
    for k in range(K):
        s = s + terms[:, k * SM_THREADS:(k + 1) * SM_THREADS]
    s = _butterfly(s.view(rows, 8, 32))
    tot = s[:, 0]
    for w in range(1, 8):
        tot = tot + s[:, w]
    return e / tot[:, None]


def softmax_check(x, y):
    """x [rows, N] float32 logits, y [rows, N] float32 probabilities (CPU).  Every entry: |y - y64| <= k_N 2^-24 y64
    + 2^-149, or NaN where y64 is NaN; rows with an infinite logit also match torch.softmax(x.double()) zero for zero.
    Returns (ok, worst (|y - y64| - 2^-149) / (2^-24 y64), message)."""
    ref = torch.softmax(x.double(), 1)
    y = y.double()
    N = x.shape[1]
    err = (y - ref).abs()
    both_nan = torch.isnan(y) & torch.isnan(ref)
    good = both_nan | (err <= softmax_k(N) * U32 * ref + TINY32)
    inf_rows = torch.isinf(x).any(1, keepdim=True)
    good &= ~inf_rows | ((y == 0) == (ref == 0))
    units = ((err - TINY32).clamp_min(0) / (U32 * ref)).nan_to_num(math.inf)
    units = torch.where(both_nan | (err <= TINY32), torch.zeros_like(err), units)
    msg = ""
    if not bool(good.all()):
        r, c = (int(v) for v in (~good).nonzero()[0])
        msg = f"N={N} row {r} col {c}: {float(y[r, c])!r} vs {float(ref[r, c])!r}"
    return bool(good.all()), float(units.max()), msg


# ============================================================================================================ IS reduction
IS_N = (1, 7, 512, 513, 1000, 6144)
IS_ROWS = (1, 15, 16, 17, 250)        # n, rows per split, around the KL kernel's 16-warp row stride
IS_SPLITS = (1, 3, 10)
IS_REL = 1e-12


def is_floor(N):
    """Absolute floor of the KL check.  A one-row split's KL is sum_j x_j log(x_j / q_j) with q = x up to rounding: the
    row sum (ceil(N / 32) lane adds, 5 butterfly adds), the marginal's sum (ceil(N / 512) adds, 5 + 15 tree adds), two
    divisions and log's ulp put each ratio within (ceil(N / 32) + ceil(N / 512) + 30) 2^-53 of 1 on each side; scipy's
    normalisations add as much again."""
    return 2 * (-(-N // 32) + -(-N // 512) + 30) * 2.0 ** -53


class IsCase(NamedTuple):
    name: str
    N: int
    n: int
    splits: int
    ldp: int
    pbuf: torch.Tensor           # [splits n, ldp] float32, NaN past N

    @property
    def p(self):
        return self.pbuf[:, :self.N]


def is_probs(rows, N, seed, device="cpu"):
    """float32 [rows, N]; row r by r % 4: a softmax of normal logits times 2; the same with exact zeros in every third
    column (never all of the row); one-hot; a softmax times 0.5 .. 1.5, so the row does not sum to 1."""
    g = torch.Generator(device=device).manual_seed(seed)
    p = torch.softmax(torch.randn(rows, N, generator=g, device=device) * 2, 1)
    fam = torch.arange(rows, device=device) % 4
    r = torch.arange(rows, device=device)[:, None]
    col = torch.arange(N, device=device)[None, :]
    zero = (fam[:, None] == 1) & (col % 3 == r % 3) & (col != r % N)
    p = torch.where(zero, torch.zeros_like(p), p)
    hot = torch.randint(0, N, (rows, 1), generator=g, device=device)
    p = torch.where((fam == 2)[:, None], (col == hot).float(), p)
    scale = 0.5 + torch.rand(rows, 1, generator=g, device=device)
    return torch.where((fam == 3)[:, None], p * scale, p).contiguous()


def is_cases(device="cpu"):
    """Every (N, n) of IS_N x IS_ROWS; the split count rotates so each N meets all three, ldp alternates N and N + 5."""
    out = []
    for i, N in enumerate(IS_N):
        for j, n in enumerate(IS_ROWS):
            splits = IS_SPLITS[(i + j) % 3]
            ldp = N + 5 * (j % 2)
            p = is_probs(splits * n, N, 100 * i + j, device)
            out.append(IsCase(f"N{N}_n{n}_splits{splits}_ldp{ldp}", N, n, splits, ldp, padded(p, ldp)))
    return out


def is_reference(case):
    """(column means float64 [splits, N], KL float64 [splits]): numpy means in fp64 and the mean over the split's rows
    of scipy.stats.entropy(row, column mean)."""
    from scipy.stats import entropy
    p = case.p.double().cpu().numpy().reshape(case.splits, case.n, case.N)
    cm = p.mean(1)
    kl = np.array([np.mean(entropy(p[k], cm[k][None, :], axis=1)) for k in range(case.splits)])
    return torch.from_numpy(cm), torch.from_numpy(kl)


def is_model(case, mutant=None):
    """is_col_mean_kernel and is_kl_kernel on the host in fp64: the column sums over the split's rows, / n; q = the
    means over their sum; each row over its sum; sum_j x_j log(x_j / q_j) where x_j > 0; the mean over the rows."""
    p = case.p.double().cpu().view(case.splits, case.n, case.N)
    rows = case.n - 1 if mutant == "mean_short" else case.n
    cm = p[:, :rows].sum(1) / case.n
    q = cm / cm.sum(1, keepdim=True)
    x = p / p.sum(2, keepdim=True)
    t = x * torch.log(x / q[:, None, :])
    if mutant != "zero_nan":
        t = torch.where(x > 0, t, torch.zeros_like(t))
    return cm, t.sum(2).mean(1)


def is_check(case, col_mean, kl, ref=None):
    """Column means within IS_REL of numpy's, KL within IS_REL relative plus is_floor(N) of scipy's.  Returns (ok,
    worst column-mean rel, worst KL err / (|KL| + floor / IS_REL), message)."""
    r_cm, r_kl = is_reference(case) if ref is None else ref
    col_mean, kl = col_mean.double().cpu().view(case.splits, case.N), kl.double().cpu()
    e_cm = ((col_mean - r_cm).abs() / r_cm.abs().clamp_min(1e-300)).nan_to_num(math.inf)
    e_cm = torch.where(col_mean == r_cm, torch.zeros_like(e_cm), e_cm)
    e_kl = (kl - r_kl).abs().nan_to_num(math.inf)
    fl = is_floor(case.N)
    ok_cm = bool((e_cm <= IS_REL).all())
    ok_kl = bool((e_kl <= IS_REL * r_kl.abs() + fl).all())
    msg = ""
    if not ok_cm:
        k, j = (int(v) for v in (e_cm > IS_REL).nonzero()[0])
        msg = f"{case.name} column mean [{k}, {j}]: {float(col_mean[k, j])!r} vs {float(r_cm[k, j])!r}"
    elif not ok_kl:
        k = int((e_kl > IS_REL * r_kl.abs() + fl).nonzero()[0])
        msg = f"{case.name} KL [{k}]: {float(kl[k])!r} vs {float(r_kl[k])!r}"
    return ok_cm and ok_kl, float(e_cm.max()), float((e_kl / (r_kl.abs() + fl / IS_REL)).max()), msg
