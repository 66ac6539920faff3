"""Cases, exact operands and fp64 references for the fp32-operand GEMMs: the 3xTF32 path of the persistent wgmma GEMM
(csrc/gemm_tc2.cu -> gemm_wgmma.cuh with TF32 = true) and the CUDA-core fp32 GEMM (csrc/gemm_fp32.cu).

test_gemm_fp32_cases_cpu.py checks the construction and that every mutant reference breaks every case on the CPU;
test_gpu_gemm_fp32_operands.py runs the kernels on the same operands.  Operands are drawn on the CPU from fixed seeds,
so both files see the same values.

* Split-grid A (3xTF32).  A = hi + lo with hi in {-1, 0, 1} and lo in {-1, 0, 1} * 2^-12, lo non-zero only where hi
  is.  2^-12 is at most half a tf32 ulp of 1, so the kernel's tf32_rn (ties away) gives hi and leaves lo = A - hi exactly:
  its shared-memory split writes a non-zero A_lo slot and the A_lo.W_hi wgmma adds a non-zero product.  The reference
  splits A with layout.tf32_round (the kernel's rule) rather than assuming hi.  W is a (w_hi, w_lo) pair on the same
  grid.  No output column keeps more than MAX_PRODUCTS non-zero weight taps, so every partial sum of the three products
  the scheme forms (A_hi.W_hi, A_lo.W_hi, A_hi.W_lo; lo.lo is not formed and not in the reference) is a multiple of 2^-12
  below 2^8: 20 significant bits.  Neither the tensor core's internal alignment nor the accumulation order can round,
  so fp64 gives the one value a correct kernel produces.  Bias and residual are multiples of 2^-12 in [-4, 4], so the
  epilogue's fp32 additions are exact too.
* CUDA-core operands.  The same split-grid A against weights that are integers in [-2, 2] times 2^-4 (at most
  MAX_PRODUCTS taps a column): every fma product is a multiple of 2^-16 and every partial sum stays below 2^5, 21
  significant bits, so the full fp32 product A.W is exact in any order.
* Mutants.  tf32_y(..., mutant=) restates the reference with one fault a kernel could have: a dropped correction
  product, A_lo of the other 64-row half of the tile or of the next 32-column k-block (zero past M or K, as the TMA fill
  gives), the first A matrix for dual-A columns >= n_split; qkv_ref(..., shift_rope=True) rotates every row at the next
  row's rope position.  The CPU test shows each one moves some output of every case past the GPU test's check.
"""
from typing import NamedTuple, Optional, Tuple

import torch

from omnitokenizer_b200 import layout as L
from tests.test_gpu_gemm_walk import T_KEYS, _qk_ref, _qkv_layout, _shape, map_rows

H100_SMS = 132              # SMs of an H100 SXM; the GPU test passes the device's own count
KB = 32                     # K per k-block of the 3xTF32 kernel (one 128-byte fp32 row of a stage)
LO_STEP = 2.0 ** -12        # split-grid lo quantum: below tf32's half ulp at 1, so tf32_rn(hi + lo) = hi
W_STEP = 2.0 ** -4          # CUDA-core weight quantum
MAX_PRODUCTS = 240          # non-zero weight taps per output column
BUDGET = 2.0 ** 8           # every partial sum stays below this: 20 significant bits on the 2^-12 grid
QK_TOL = 2.0 ** -18         # q / k after rope + l2norm + scale: |error| <= QK_TOL |scale_d| (test_gpu_gemm_walk._case_qkv)
MUTANTS = ("drop_lo_hi", "drop_hi_lo", "lo_other_half", "lo_next_kblock", "dual_first")


def walk_seed(i: int) -> int:
    return 1000 + 10 * i


def qkv_seed(i: int) -> int:
    return 2000 + 10 * i


def fp32_seed(i: int) -> int:
    return 3000 + 10 * i


def _gen(seed: int) -> torch.Generator:
    return torch.Generator().manual_seed(seed)


def split_grid(shape, g, lo_zero: bool = True) -> Tuple[torch.Tensor, torch.Tensor]:
    """(hi, lo): hi in {-1, 0, 1}, lo in {-1, 0, 1} * 2^-12 and non-zero only where hi is (lo_zero False: lo in
    {-1, 1} * 2^-12 wherever hi is non-zero)."""
    hi = torch.randint(-1, 2, shape, generator=g).float()
    if lo_zero:
        lo = torch.randint(-1, 2, shape, generator=g).float()
    else:
        lo = torch.randint(0, 2, shape, generator=g).float() * 2 - 1
    return hi, lo * LO_STEP * (hi != 0)


def grid_a(rows: int, K: int, seed: int) -> torch.Tensor:
    """Split-grid A.  Its lo part is non-zero wherever hi is, in about 2/3 of the entries, so that even the 32 entries
    of a one-row tail in a k-block hold many non-zero A_lo values."""
    hi, lo = split_grid((rows, K), _gen(seed), lo_zero=False)
    return hi + lo


def _taps(n: int, K: int, g) -> torch.Tensor:
    """0 / 1 mask keeping MAX_PRODUCTS random taps of each of n rows (all of them if K is no longer)."""
    if K <= MAX_PRODUCTS:
        return torch.ones(n, K)
    keep = torch.rand(n, K, generator=g).argsort(dim=1)[:, :MAX_PRODUCTS]
    return torch.zeros(n, K).scatter_(1, keep, 1.0)


def tf32_weight(n: int, K: int, seed: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """(w_hi, w_lo) [n, K] of a 3xTF32 weight on the split grid."""
    g = _gen(seed)
    hi, lo = split_grid((n, K), g)
    keep = _taps(n, K, g)
    return hi * keep, lo * keep


def fp32_weight(n: int, K: int, seed: int) -> torch.Tensor:
    """[n, K] integers in [-2, 2] times 2^-4."""
    g = _gen(seed)
    w = torch.randint(-2, 3, (n, K), generator=g).float() * W_STEP
    return w * _taps(n, K, g)


def grid_vec(shape, seed: int) -> torch.Tensor:
    """Bias / residual values: multiples of 2^-12 in [-4, 4]."""
    return torch.randint(-(1 << 14), (1 << 14) + 1, shape, generator=_gen(seed)).float() * LO_STEP


def split_a(A: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """The kernel's split of A: hi = tf32_rn(A) (layout.tf32_round, ties away), lo = A - hi."""
    hi = L.tf32_round(A.float())
    return hi, A.float() - hi


def _other_half(t: torch.Tensor) -> torch.Tensor:
    """Rows of t (starting on a 128-row tile) moved to the other 64-row half of their tile; zero past the last row."""
    M = t.shape[0]
    p = torch.zeros(-(-M // 128) * 128, t.shape[1], dtype=t.dtype, device=t.device)
    p[:M] = t
    return p.view(-1, 2, 64, t.shape[1]).flip(1).reshape(-1, t.shape[1])[:M]


def _next_kblock(t: torch.Tensor) -> torch.Tensor:
    """Columns of k-block kb taken from k-block kb + 1; zero for the last one."""
    out = torch.zeros_like(t)
    out[:, : t.shape[1] - KB] = t[:, KB:]
    return out


def tf32_y(A: torch.Tensor, wh: torch.Tensor, wl: torch.Tensor, A2: Optional[torch.Tensor] = None, n_split: int = 0,
           mutant: Optional[str] = None) -> torch.Tensor:
    """fp64 A_hi.W_hi + A_lo.W_hi + A_hi.W_lo over the logical rows of A (the first one at a tile's first row), with
    columns >= n_split from A2 when given.  mutant: one of MUTANTS."""
    def y_of(a):
        ah, al = (t.double() for t in split_a(a))
        if mutant == "lo_other_half":
            al = _other_half(al)
        elif mutant == "lo_next_kblock":
            al = _next_kblock(al)
        whd, wld = wh.double().to(a.device), wl.double().to(a.device)
        y = ah @ whd.t()
        if mutant != "drop_lo_hi":
            y = y + al @ whd.t()
        if mutant != "drop_hi_lo":
            y = y + ah @ wld.t()
        return y

    y = y_of(A)
    if A2 is not None and mutant != "dual_first":
        y[:, n_split:] = y_of(A2)[:, n_split:]
    return y


def fp32_y(A: torch.Tensor, W: torch.Tensor, A2: Optional[torch.Tensor] = None, n_split: int = 0,
           mutant: Optional[str] = None) -> torch.Tensor:
    """fp64 A . W^T (columns >= n_split from A2); mutant "dual_first" uses A for every column."""
    Wd = W.double().to(A.device)
    y = A.double() @ Wd.t()
    if A2 is not None and mutant != "dual_first":
        y[:, n_split:] = (A2.double() @ Wd.t())[:, n_split:]
    return y


def plain_want(y: torch.Tensor, bias, res) -> torch.Tensor:
    """fp32 result of the plain epilogue: y (exact in fp32), + bias, + residual (both additions exact)."""
    out = y.float()
    if bias is not None:
        out = out + bias.to(out.device)
    if res is not None:
        out = out + res.to(out.device)
    return out


def gelu64(x: torch.Tensor) -> torch.Tensor:
    return 0.5 * x * (1.0 + torch.erf(x / 2.0 ** 0.5))


def geglu_ref(y: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(fp64 gelu(gate) * value, bound) of packed y (bias included).  fp32 gelu_erf(gate) * value errs by at most
    2^-22 |gate| |value| (test_gpu_gemm_walk._case_geglu); the bound leaves a factor 4."""
    val, gate = y[:, 0::2], y[:, 1::2]
    return gelu64(gate) * val, 2.0 ** -20 * val.abs() * gate.abs()


# ---------------------------------------------------------------- row maps

class RowMap(NamedTuple):
    seg: int
    stride: int
    off: int
    rows: int                   # physical rows the buffer needs

    def index(self, M: int, dev="cpu") -> torch.Tensor:
        return map_rows(M, self.seg, self.stride, self.off, dev)

    @property
    def args(self) -> Tuple[int, int, int]:
        return self.seg, self.stride, self.off


def segments(M: int, mult: int, extra: int, off: int) -> RowMap:
    """A map of up to four segments over M logical rows, each a multiple of `mult`, `extra` physical rows between
    them, starting `off` rows in."""
    for d in (4, 3, 2, 1):
        if M % (mult * d) == 0:
            seg = M // d
            return RowMap(seg, seg + extra, off, off + d * (seg + extra))
    raise AssertionError(f"M={M} has no row-map segment that is a multiple of {mult}")


def video_map(tokens: int, tp: int, f0: int, first: bool, n: int) -> Tuple[int, RowMap]:
    """(M, map) of the patch-embed c_map / to_pixels a_map of a group of n videos with tp latent frames of `tokens`
    rows each, starting at frame f0 (engine._encode_body / _decode_body): the first frame of every video, or the rest."""
    seg = tokens if first else (tp - 1) * tokens
    off = f0 * tokens + (0 if first else tokens)
    return n * seg, RowMap(seg, tp * tokens, off, (f0 + n * tp) * tokens)


# ---------------------------------------------------------------- the 3xTF32 tile walk

class WalkCase(NamedTuple):
    epi: str                    # "plain" or "geglu"
    t: str                      # tile-count key of T_KEYS
    K: int
    n_list: Tuple[int, ...]     # candidate N: the first whose 128-column block count divides T
    tail: int                   # rows in the last m block
    bias: bool = False
    res: str = ""               # "", "sep" or "inplace"
    amap: bool = False          # A row map, segments a multiple of 64 (to_pixels)
    cmap: bool = False          # C / residual row map, segments a multiple of 32
    n_split: int = 0            # dual-A (omt_linear2, which takes no bias, residual or row map): columns >= n_split
                                # read the second matrix

    @property
    def id(self) -> str:
        opts = [o for o, on in (("bias", self.bias), (f"res{self.res}", self.res), ("amap", self.amap),
                                ("cmap", self.cmap), (f"dual{self.n_split}", self.n_split)) if on]
        return "-".join([self.epi, f"T{self.t}", f"K{self.K}", f"tail{self.tail}"] + opts)


# T covers 1, S - 1 .. 3S + 1 (the CTAs walk 1 to 4 tiles), K covers 32 (one k-block, shorter than the stage ring),
# 64 and 1408 (FF2; 44 k-blocks, 14 passes of the ring), tails 1, 64 and 127.  N lists start with the model's widths
# (512, 768, 1536 QKV, 2816 packed GEGLU) and fall back to ones whose block count divides T; 96, 640 - 32 end in a
# partial 128-column block.
TF32_WALK = [
    WalkCase("plain", "1", 32, (96,), 1, bias=True),
    WalkCase("plain", "S-1", 64, (128,), 127, bias=True, res="sep"),
    WalkCase("plain", "S", 1408, (512, 128), 64, bias=True, res="inplace"),
    WalkCase("plain", "S+1", 64, (896, 128), 64, res="sep", cmap=True),
    WalkCase("plain", "2S", 64, (768, 1536, 128), 64, bias=True, res="inplace", amap=True, cmap=True),
    WalkCase("plain", "S", 64, (512, 128), 127, n_split=128),
    WalkCase("plain", "2S", 32, (1536, 768, 128), 127, n_split=512),
    WalkCase("plain", "2S+1", 32, (640, 128), 127, n_split=256),
    WalkCase("plain", "S+1", 1408, (896, 128), 1, n_split=384),
    WalkCase("plain", "S", 64, (512, 128), 64, bias=True, res="sep", amap=True),
    WalkCase("plain", "3S+1", 32, (128,), 64, bias=True, res="sep"),
    WalkCase("geglu", "2S", 1408, (2816, 128), 64, bias=True, cmap=True),
    WalkCase("geglu", "S-1", 64, (128,), 1),
    WalkCase("geglu", "3S+1", 32, (128,), 127, bias=True),
]


class WalkProblem(NamedTuple):
    M: int
    N: int
    K: int
    A: torch.Tensor             # physical rows of A
    A2: Optional[torch.Tensor]
    amap: Optional[RowMap]
    cmap: Optional[RowMap]
    w_hi: torch.Tensor          # [N, K] (GEGLU: packed value / gate rows)
    w_lo: torch.Tensor
    bias: Optional[torch.Tensor]
    res: Optional[torch.Tensor]  # [M, N] logical rows
    n_split: int
    inner: int                  # GEGLU: real value / gate pairs (the rest of the N / 2 outputs are padding)

    def aidx(self, dev="cpu") -> torch.Tensor:
        return self.amap.index(self.M, dev) if self.amap else torch.arange(self.M, device=dev)

    def cidx(self, dev="cpu") -> torch.Tensor:
        return self.cmap.index(self.M, dev) if self.cmap else torch.arange(self.M, device=dev)

    def logical(self, rows: Optional[slice] = None, dev="cpu"):
        """(A, A2) at logical rows (all of them, or a slice starting on a tile's first row), on dev."""
        idx = self.aidx()
        if rows is not None:
            idx = idx[rows]
        return self.A[idx].to(dev), None if self.A2 is None else self.A2[idx].to(dev)


def walk_problem(c: WalkCase, sms: int, seed: int) -> WalkProblem:
    M, N = _shape(T_KEYS[c.t](sms), list(c.n_list), c.tail)
    amap = segments(M, 64, 192, 128) if c.amap else None
    cmap = segments(M, 32, 96, 32) if c.cmap else None
    arows = amap.rows if amap else M
    A = grid_a(arows, c.K, seed)
    A2 = grid_a(arows, c.K, seed + 1) if c.n_split else None
    inner = 0
    if c.epi == "geglu":
        ku = N // 2
        inner = 1365 if ku == 1408 else ku - 11
        wh, wl = (L.pack_geglu(t, inner, ku) for t in tf32_weight(2 * inner, c.K, seed + 2))
    else:
        wh, wl = tf32_weight(N, c.K, seed + 2)
    bias = None
    if c.bias:
        bias = grid_vec((N,), seed + 3)
        if c.epi == "geglu":
            bias[2 * inner:] = 0.0
    res = grid_vec((M, N), seed + 4) if c.res else None
    return WalkProblem(M, N, c.K, A, A2, amap, cmap, wh, wl, bias, res, c.n_split, inner)


def walk_y(p: WalkProblem, rows: Optional[slice] = None, dev="cpu", mutant: Optional[str] = None) -> torch.Tensor:
    """fp64 pre-epilogue result of the logical rows (GEGLU: bias included)."""
    A, A2 = p.logical(rows, dev)
    y = tf32_y(A, p.w_hi, p.w_lo, A2, p.n_split, mutant)
    if p.inner and p.bias is not None:
        y = y + p.bias.double().to(dev)
    return y


def walk_fails(p: WalkProblem, got: torch.Tensor, y: torch.Tensor, rows: Optional[slice] = None) -> bool:
    """Would the GPU test reject `got` (the GEGLU outputs in fp64, else the fp32 outputs) of the logical rows, given the
    true y of those rows?"""
    if p.inner:
        want, tol = geglu_ref(y)
        return bool(((got[:, : p.inner] - want[:, : p.inner]).abs() > tol[:, : p.inner]).any())
    res = None if p.res is None else (p.res if rows is None else p.res[rows])
    return not torch.equal(got, plain_want(y, p.bias, res))


def mutant_output(p: WalkProblem, y_mut: torch.Tensor, rows: Optional[slice] = None) -> torch.Tensor:
    """What a kernel with the mutant's fault would write: GEGLU in fp64, else the plain epilogue in fp32."""
    if p.inner:
        return geglu_ref(y_mut)[0]
    res = None if p.res is None else (p.res if rows is None else p.res[rows])
    return plain_want(y_mut, p.bias, res)


# ---------------------------------------------------------------- the 3xTF32 fused QKV epilogue

class QkvCase(NamedTuple):
    t: str                      # tile-count key (or "" for a width case: three m blocks of N = 3A)
    K: int
    n_list: Tuple[int, ...]
    tail: int
    tokens: int
    rope: bool
    width: Optional[Tuple[int, int]] = None   # (attention width A, model width C): N = 3A, K = C, n_split = A

    @property
    def id(self) -> str:
        shape = f"A{self.width[0]}-C{self.width[1]}" if self.width else f"T{self.t}-K{self.K}"
        return f"{shape}-tail{self.tail}-tok{self.tokens}-{'rope' if self.rope else 'norope'}"


# QKV_WIDTHS of test_gpu_width_kernels.py: attention widths apart from the model's
QKV_WIDTHS = [(512, 256), (256, 512), (768, 768), (384, 512), (128, 1024)]

TF32_QKV = [
    QkvCase("2S", 64, (1536, 640, 128), 64, 96, True),
    QkvCase("S", 1408, (1536, 640, 128), 127, 128, False),
    QkvCase("2S+1", 32, (640, 1536, 128), 1, 64, True),
    QkvCase("S+1", 64, (896, 1536, 128), 127, 1024, True),
    QkvCase("S-1", 32, (1536, 128), 64, 1024, False),
] + [QkvCase("", C, (3 * A,), 77, 96, rope, (A, C)) for A, C in QKV_WIDTHS for rope in (True, False)]


class QkvProblem(NamedTuple):
    M: int
    N: int
    K: int
    A: torch.Tensor
    A2: Optional[torch.Tensor]
    n_split: int
    qk: int
    tokens: int
    w_hi: torch.Tensor
    w_lo: torch.Tensor
    qs: torch.Tensor
    ks: torch.Tensor
    cos: Optional[torch.Tensor]
    sin: Optional[torch.Tensor]


def qkv_problem(c: QkvCase, sms: int, seed: int) -> QkvProblem:
    if c.width:
        Aw, _ = c.width
        N, qk, n_split = 3 * Aw, 2 * Aw, Aw
        M = 2 * 128 + c.tail
    else:
        M, N = _shape(T_KEYS[c.t](sms), list(c.n_list), c.tail)
        qk, n_split = _qkv_layout(N)
    A = grid_a(M, c.K, seed)
    A2 = grid_a(M, c.K, seed + 1) if n_split else None
    wh, wl = tf32_weight(N, c.K, seed + 2)
    g = _gen(seed + 3)
    qs, ks = 0.5 + torch.rand(64, generator=g), 0.5 + torch.rand(64, generator=g)
    cos, sin = L.rope_tables(c.tokens, 64) if c.rope else (None, None)
    return QkvProblem(M, N, c.K, A, A2, n_split, qk, c.tokens, wh, wl, qs, ks, cos, sin)


def qkv_ref(p: QkvProblem, z: torch.Tensor, shift_rope: bool = False):
    """(fp64 q | k after rope + l2norm + scale, bound) of exact z whose first row is logical row 0.  shift_rope: the
    rope position of every row off by one (row m rotated as row m + 1)."""
    dev = z.device
    cos, sin = p.cos, p.sin
    if cos is not None:
        cos, sin = cos.to(dev), sin.to(dev)
        if shift_rope:
            cos, sin = cos.roll(-1, 0), sin.roll(-1, 0)
    want, sc = _qk_ref(z, p.qk, p.qs.to(dev), p.ks.to(dev), cos, sin, p.tokens)
    return want, QK_TOL * sc


def qkv_fails(p: QkvProblem, got: torch.Tensor, z: torch.Tensor) -> bool:
    """Would the GPU test reject fp64 `got` [rows, N] (q | k | v, rows from logical row 0) given the true exact z?"""
    want, tol = qkv_ref(p, z)
    return bool(((got[:, : p.qk] - want).abs() > tol).any()) or not torch.equal(got[:, p.qk:], z[:, p.qk:])


# ---------------------------------------------------------------- the CUDA-core fp32 GEMM

class Fp32Case(NamedTuple):
    name: str
    M: int
    N: int
    K: int
    bias: bool = False
    res: str = ""               # "", "sep" or "inplace"
    n_split: int = 0            # dual-A (omt_linear2: no bias, residual or row map)
    geglu: bool = False
    amap: Optional[RowMap] = None
    cmap: Optional[RowMap] = None
    ldc_extra: int = 12         # ldc = (GEGLU: N / 2, else N) rounded up to 4, + ldc_extra
    lda_extra: int = 0

    @property
    def out_cols(self) -> int:
        return self.N // 2 if self.geglu else self.N

    @property
    def ldc(self) -> int:
        return L.round_up(self.out_cols, 4) + self.ldc_extra

    @property
    def id(self) -> str:
        return f"{self.name}-M{self.M}-N{self.N}-K{self.K}"


def _video_cases():
    """Patch embed (C row map, K = cin p^2 (pt) -> 512) and to_pixels (A row map, 512 -> cin p^2 (pt)) of a group of
    three videos at 5 and 17 latent frames; the token grids of 6 x 6 and 7 x 7 make segments that are not multiples
    of 64, so 128-row tiles span segment boundaries."""
    out = []
    for tokens, tp, f0 in ((36, 5, 0), (49, 17, 2)):
        for first in (True, False):
            M, m = video_map(tokens, tp, f0, first, 3)
            k = 192 if first else 768
            part = "first" if first else "rest"
            out.append(Fp32Case(f"embed{tp}-{part}", M, 512, k, bias=True, cmap=m,
                                res="inplace" if tp == 17 and not first else ""))
            out.append(Fp32Case(f"pixels{tp}-{part}", M, k, 512, bias=True, amap=m))
    return out


FP32_CASES = [
    Fp32Case("mtail", 1, 4, 8, bias=True),
    Fp32Case("mtail", 127, 124, 24, res="sep", ldc_extra=4),
    Fp32Case("full", 128, 132, 512, bias=True, res="inplace"),
    Fp32Case("dual", 129, 260, 1376, n_split=128),
    Fp32Case("dual", 4097, 1536, 512, n_split=512, lda_extra=8),
    Fp32Case("mtail", 4097, 132, 8, bias=True, res="inplace"),
    Fp32Case("mtail", 129, 1536, 24, ldc_extra=4),
    Fp32Case("mtail", 1, 260, 1376, res="sep"),
    Fp32Case("geglu", 127, 260, 24, bias=True, geglu=True),
    Fp32Case("geglu", 129, 2816, 512, geglu=True, ldc_extra=4),
] + _video_cases()


class Fp32Problem(NamedTuple):
    c: Fp32Case
    A: torch.Tensor             # physical rows, lda = K + lda_extra (the columns past K hold other values)
    A2: Optional[torch.Tensor]
    W: torch.Tensor             # [N, K] (GEGLU: packed)
    bias: Optional[torch.Tensor]
    res: Optional[torch.Tensor]  # [M, N] logical rows
    inner: int

    def aidx(self, dev="cpu") -> torch.Tensor:
        return self.c.amap.index(self.c.M, dev) if self.c.amap else torch.arange(self.c.M, device=dev)

    def cidx(self, dev="cpu") -> torch.Tensor:
        return self.c.cmap.index(self.c.M, dev) if self.c.cmap else torch.arange(self.c.M, device=dev)


def fp32_problem(c: Fp32Case, seed: int) -> Fp32Problem:
    rows = c.amap.rows if c.amap else c.M
    lda = c.K + c.lda_extra
    A = grid_a(rows, lda, seed)
    A2 = grid_a(rows, lda, seed + 1) if c.n_split else None
    inner = 0
    if c.geglu:
        ku = c.N // 2
        inner = 1365 if ku == 1408 else ku - 11
        W = L.pack_geglu(fp32_weight(2 * inner, c.K, seed + 2), inner, ku)
    else:
        W = fp32_weight(c.N, c.K, seed + 2)
    bias = None
    if c.bias:
        bias = grid_vec((c.N,), seed + 3)
        if c.geglu:
            bias[2 * inner:] = 0.0
    res = grid_vec((c.M, c.N), seed + 4) if c.res else None
    return Fp32Problem(c, A, A2, W, bias, res, inner)


def fp32_case_y(p: Fp32Problem, dev="cpu", mutant: Optional[str] = None) -> torch.Tensor:
    """fp64 pre-epilogue result (GEGLU: bias included) of every logical row."""
    idx = p.aidx()
    K = p.c.K
    A = p.A[idx, :K].to(dev)
    A2 = None if p.A2 is None else p.A2[idx, :K].to(dev)
    y = fp32_y(A, p.W, A2, p.c.n_split, mutant)
    if p.inner and p.bias is not None:
        y = y + p.bias.double().to(dev)
    return y
