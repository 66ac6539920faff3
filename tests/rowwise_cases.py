"""Cases, host-selection mirrors and float64 references for the row-wise kernels (csrc/rowwise.cu, csrc/vq.cu).

test_rowwise_cases_cpu.py checks the mirrors and the references on the CPU; test_gpu_rowwise.py runs the kernels.

* Mirrors restate, in Python, how the host picks a compiled kernel or a tile geometry from the shape: LayerNorm's
  (NV, PAIR), the patch gather's NV and PEG's (TT, HB, zero row, v3 | v4).  Every case records what it must reach, so a
  change to the host heuristics fails the CPU test here rather than silently moving a GPU case off its kernel.
* References compute the same operation in float64, independently of the kernels' loop structure.
* Input families put rows where row-wise kernels go wrong into every launch: magnitudes from 1e-3 to 1e3, a common
  offset up to 100x the spread, constant and all-zero rows, a row maximum that is an exact power of two, and elements
  small enough to land in fp16's subnormal range after the row scaling of the operand planes.
"""
import torch

# ---------------------------------------------------------------- host-selection mirrors


def ln_instantiation(C, lds=0, plane_align=16):
    """(NV, PAIR) of layernorm_kernel, as layernorm_impl (csrc/rowwise.cu) picks it from its kernel tables for every
    call but the paired ones at C = 768 and 1024: NV = float4 chunks per lane (1, 2, 3, 4, or 8 for anything larger),
    PAIR when C is a multiple of 256, NV is 2 or 4, the plane leading dimension is a multiple of 8 and every plane
    pointer is 16-byte aligned.  A call without planes has lds = 0 and NULL planes.  At C = 768 and 1024 this mirror
    keeps <8, false>, the form of their unpaired calls; test_gpu_width_kernels.ln_instantiation_wide mirrors the paired
    <6, true> and <8, true> there."""
    nv = (C // 4 + 31) // 32
    pair = C % 256 == 0 and lds % 8 == 0 and plane_align % 16 == 0
    if nv in (2, 4):
        return nv, pair
    return (nv, False) if nv in (1, 3) else (8, False)


def patch_nv(K):
    """NV of patchify_ln_kernel and patchify_ln_u8_kernel for a patch vector of K features, as gather_nv_index
    (csrc/rowwise.cu) picks it for both gathers: 2, 6 or 8 float4 chunks per lane."""
    nv = (K // 4 + 31) // 32
    return 2 if nv <= 2 else (6 if nv <= 6 else 8)


PEG_CC = 16


def peg_geometry(T, w, causal, peg_kernel=4):
    """Tile geometry of omt_peg_volume (peg_volume_launch, csrc/rowwise.cu): dict with TT (planes per CTA), HB (token
    rows per CTA), RS (floats per tile row), kernel ('v4' | 'v3'), smem (v3 bytes), and for v4 zrow (index of the shared
    zero row = tile planes inside the volume x (HB + 2)) and smem4 (v4 bytes)."""
    RS = (w + 2) * PEG_CC
    RS += ((16 - RS % 32) + 32) % 32

    def smem_of(tt, hb):
        return (tt + 2) * (hb + 2) * (RS * 4 + (w + 2) * 8)

    TT, HB = min(T, 5), 4
    while HB > 1 and (smem_of(TT, HB) > 112 * 1024 or TT * HB * 8 > 256):
        HB -= 1
    while TT > 1 and (smem_of(TT, HB) > 112 * 1024 or TT * HB * 8 > 256):
        TT -= 1
    g = dict(TT=TT, HB=HB, RS=RS, smem=smem_of(TT, HB), kernel="v3")
    if peg_kernel == 4 and T <= 64 and w <= 254:
        pad_lo = 2 if causal else 1
        vp = 1
        for t0 in range(0, T, TT):
            lo, hi = max(0, t0 - pad_lo), min(T, t0 - pad_lo + TT + 2)
            vp = max(vp, hi - lo)
        g.update(kernel="v4", zrow=vp * (HB + 2), smem4=(vp * (HB + 2) + 1) * RS * 4)
    return g


# ---------------------------------------------------------------- input families

FAMILIES = ("spread", "offset", "constant", "zero", "pow2", "tiny")


def family_rows(M, C, seed):
    """float32 [M, C]; row r belongs to FAMILIES[r % 6]:
    spread    uniform(-1, 1) times 10^u, u uniform in [-3, 3];
    offset    a common offset of up to 100 spreads (|mean| / std up to ~1e2);
    constant  m * 2^k for a small integer m: the row sum and mean are exact, so the variance is exactly 0;
    zero      all zeros (row_scale clamps the exponent to 15);
    pow2      the largest magnitude is an exact power of two;
    tiny      every third element is 2^-30 .. 2^-36 of the row maximum: fp16 subnormals (or zeros) after row scaling."""
    g = torch.Generator().manual_seed(seed)
    u = torch.rand(M, C, generator=g, dtype=torch.float64) * 2 - 1
    fam = torch.arange(M) % 6
    mag = 10.0 ** (torch.rand(M, 1, generator=g, dtype=torch.float64) * 6 - 3)
    x = u * mag
    off = (torch.rand(M, 1, generator=g, dtype=torch.float64) * 2 - 1) * 100
    x = torch.where((fam == 1)[:, None], (u + off) * mag, x)
    m = torch.randint(-3, 4, (M, 1), generator=g).double() * 2.0 ** torch.randint(-6, 6, (M, 1), generator=g).double()
    x = torch.where((fam == 2)[:, None], m.expand(M, C), x)
    x = torch.where((fam == 3)[:, None], torch.zeros_like(x), x)
    p2 = 2.0 ** torch.randint(-8, 9, (M, 1), generator=g).double()
    pw = u * p2
    col = torch.randint(0, C, (M,), generator=g)
    pw[torch.arange(M), col] = p2[:, 0] * torch.where(torch.rand(M, generator=g) < 0.5, -1.0, 1.0).double()
    x = torch.where((fam == 4)[:, None], pw, x)
    tiny = u.clone()
    tiny[:, ::3] *= 2.0 ** -torch.randint(30, 37, (1, (C + 2) // 3), generator=g).double()
    x = torch.where((fam == 5)[:, None], tiny * mag, x)
    return x.float().contiguous()


def ln_params(C, seed):
    """(gamma, beta) float32 [C]: gamma in [0.5, 1.5] with every 7th entry 2^-30 (its output columns carry fp16
    subnormals after row scaling), beta in [-0.25, 0.25] with beta[0] = 0.5, so the rows whose output is beta (constant
    and zero rows) have an exact power of two as their largest magnitude."""
    g = torch.Generator().manual_seed(seed)
    w = torch.rand(C, generator=g) + 0.5
    w[3::7] = 2.0 ** -30
    b = (torch.rand(C, generator=g) - 0.5) * 0.5
    b[0] = 0.5
    return w, b


# ---------------------------------------------------------------- float64 references


def ln_ref(x, w, b, eps=1e-5):
    """LayerNorm over the last dimension in float64 (biased variance, eps inside the square root).  Also returns the
    per-row scale of the arithmetic: max |gamma| * (1 + |mean| / std) + max |beta|, the size of the terms whose fp32
    rounding any kernel's error is proportional to."""
    x = x.double()
    mu = x.mean(dim=-1, keepdim=True)
    xc = x - mu
    sd = torch.sqrt((xc * xc).mean(dim=-1, keepdim=True) + eps)
    y = xc / sd * w.double()
    mag = w.double().abs().max() * (1 + mu.abs() / sd)
    if b is not None:
        y = y + b.double()
        mag = mag + b.double().abs().max()
    return y, mag


def patch_index(B, Cin, T, H, W, p, pt, first):
    """int64 [rows, K]: flat index into the (B, Cin, T, H, W) video of feature f of patch row r, with the row order of
    patchify_ln_kernel (b, [t-block,] h-block, w-block) and the feature order f = ((c * PT + dt) * p + p1) * p + p2."""
    PT = 1 if first else pt
    hh, ww = H // p, W // p
    tn = 1 if first else (T - 1) // pt
    b = torch.arange(B).view(B, 1, 1, 1, 1, 1, 1, 1)
    ti = torch.arange(tn).view(1, tn, 1, 1, 1, 1, 1, 1)
    hi = torch.arange(hh).view(1, 1, hh, 1, 1, 1, 1, 1)
    wi = torch.arange(ww).view(1, 1, 1, ww, 1, 1, 1, 1)
    c = torch.arange(Cin).view(1, 1, 1, 1, Cin, 1, 1, 1)
    dt = torch.arange(PT).view(1, 1, 1, 1, 1, PT, 1, 1)
    p1 = torch.arange(p).view(1, 1, 1, 1, 1, 1, p, 1)
    p2 = torch.arange(p).view(1, 1, 1, 1, 1, 1, 1, p)
    t = dt if first else 1 + ti * pt + dt
    idx = (((b * Cin + c) * T + t) * H + hi * p + p1) * W + wi * p + p2
    return idx.reshape(B * tn * hh * ww, Cin * PT * p * p)


def patchify_ref(video, p, pt, first):
    """[rows, K] patch vectors (the im2col form) gathered by patch_index; exact, in the video's dtype."""
    B, Cin, T, H, W = video.shape
    return video.reshape(-1)[patch_index(B, Cin, T, H, W, p, pt, first)]


def unpatchify_ref(P, shape, p, pt, first, out=None):
    """The inverse permutation: scatter [rows, K] patch vectors into a (B, Cin, T, H, W) video (zeros, or `out`)."""
    out = torch.zeros(shape, dtype=P.dtype) if out is None else out
    out.view(-1)[patch_index(*shape, p, pt, first)] = P
    return out


def peg_ref(X, wt, bias, h, w, temporal, causal):
    """PEG with its residual, X + bias + depthwise 3x3x3 cross-correlation, in float64 through the reference's own
    conv3d formulation (oracle.omni_oracle.peg with library ops).  X [B, T', N, C] (any device); wt [C, 1, 3, 3, 3].
    Also returns the magnitude |X| + |bias| + sum |w| |x| of the same stencil, for relative error bars."""
    from oracle import omni_oracle as oo
    old = oo.USE_LIBRARY_OPS
    oo.USE_LIBRARY_OPS = True
    try:
        Xd, wd, bd = X.double(), wt.double().to(X.device), bias.double().to(X.device)
        y = oo.peg(Xd, wd, bd, (h, w), temporal, causal) + Xd
        mag = oo.peg(Xd.abs(), wd.abs(), bd.abs(), (h, w), temporal, causal) + Xd.abs()
    finally:
        oo.USE_LIBRARY_OPS = old
    return y, mag


def qk_prep_ref(t, scale, cos=None, sin=None):
    """rope (optional) + l2 normalise (norm clamped below at 1e-12) + per-dim scale of every 64-wide head, float64.
    t [M, heads * 64], cos / sin [M, 32] (already indexed by each row's position)."""
    M = t.shape[0]
    v = t.double().view(M, -1, 32, 2)
    if cos is not None:
        c, s = cos.double().view(M, 1, 32), sin.double().view(M, 1, 32)
        v = torch.stack([v[..., 0] * c - v[..., 1] * s, v[..., 0] * s + v[..., 1] * c], dim=-1)
    v = v.reshape(M, -1, 64)
    v = v / v.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    return (v * scale.double()).reshape(M, -1)


def pre_vq_ref(x, Wt, b, l2):
    """z = x Wt^T + b (then l2 normalised, norm clamped at 1e-12), float64; and the magnitude |x| |Wt|^T + |b|."""
    z = x.double() @ Wt.double().t() + b.double()
    mag = x.double().abs() @ Wt.double().abs().t() + b.double().abs()
    if l2:
        n = z.norm(dim=1, keepdim=True).clamp_min(1e-12)
        z, mag = z / n, mag / n
    return z, mag


def post_vq_ref(rows, Wt, b):
    """X = rows Wt^T + b in float64 (rows [M, 8], Wt [C, 8]); and the magnitude |rows| |Wt|^T + |b|."""
    X = rows.double() @ Wt.double().t() + b.double()
    return X, rows.double().abs() @ Wt.double().abs().t() + b.double().abs()


# ---------------------------------------------------------------- case tables

# LayerNorm: (C, M, ldx, lds, plane byte offset) -> (NV, PAIR) of the fp32-only call and of the plane-writing calls
LN_CASES = [
    (4, 37, 8, 8, 0, (1, False), (1, False)),
    (100, 301, 100, 104, 0, (1, False), (1, False)),
    (128, 64, 132, 128, 0, (1, False), (1, False)),
    (256, 301, 256, 256, 0, (2, True), (2, True)),
    (256, 77, 260, 260, 0, (2, True), (2, False)),            # lds % 8 != 0
    (256, 50, 256, 256, 8, (2, True), (2, False)),            # planes only 8-byte aligned
    (384, 129, 388, 384, 0, (3, False), (3, False)),
    (512, 300, 512, 512, 0, (4, True), (4, True)),
    (512, 257, 516, 516, 0, (4, True), (4, False)),            # lds = 516
    (512, 131, 512, 512, 8, (4, True), (4, False)),            # plane base 8 bytes past 16-byte alignment
    (640, 99, 640, 648, 0, (8, False), (8, False)),
    (768, 65, 772, 768, 0, (8, False), (8, False)),
    (1020, 33, 1020, 1024, 0, (8, False), (8, False)),
    (1024, 203, 1028, 1024, 0, (8, False), (8, False)),
]


def ln_case_id(c):
    return f"C{c[0]}-M{c[1]}-ldx{c[2]}-lds{c[3]}-off{c[4]}"


# patch gather / un-patchify: (Cin, p, pt, first) with K = Cin * (1 | pt) * p * p, and the NV it reaches
PATCH_CASES = [
    (3, 4, 1, 1, 48, 2), (1, 4, 2, 0, 32, 2), (3, 8, 4, 1, 192, 2), (1, 16, 1, 1, 256, 2), (4, 8, 1, 0, 256, 2),
    (3, 8, 2, 0, 384, 6), (3, 4, 4, 0, 192, 2), (1, 8, 4, 0, 256, 2), (3, 8, 4, 0, 768, 6), (4, 16, 1, 1, 1024, 8),
    (4, 8, 4, 0, 1024, 8), (1, 16, 4, 0, 1024, 8), (3, 16, 1, 1, 768, 6),
]


def patch_video_shape(Cin, p, pt):
    """A small (B, Cin, T, H, W) video with two temporal blocks and non-square, several-patch frames."""
    return (2, Cin, 1 + 2 * pt, 3 * p, 2 * p)


# PEG: the geometry table of (TT, HB) at T' = 1 / 2 / >= 5 for each token row w, and its kernel
PEG_TABLE = {
    40: ((1, 4), (2, 4), (5, 3), "v4"),
    48: ((1, 4), (2, 4), (5, 2), "v4"),
    64: ((1, 4), (2, 3), (5, 1), "v4"),
    80: ((1, 4), (2, 2), (4, 1), "v4"),
    96: ((1, 3), (2, 2), (3, 1), "v4"),
    128: ((1, 2), (2, 1), (2, 1), "v4"),
    192: ((1, 1), (1, 1), (1, 1), "v4"),
    256: ((1, 1), (1, 1), (1, 1), "v3"),
}
PEG_T = (1, 2, 4, 5, 6, 9, 17)


def peg_cases():
    """(w, T', C, h): every row of PEG_TABLE at every T' of PEG_T (w = 256 only at T' <= 2) with C = 16, and C = 512 at
    w <= 64.  h = w makes square frames up to w = 128; wider rows and the 512-channel cases use a few token rows (the tile
    geometry depends on T' and w only) with a partial last row block."""
    out = []
    for w in PEG_TABLE:
        for T in PEG_T:
            if w == 256 and T > 2:
                continue
            out.append((w, T, 16, w if w <= 128 else 2 * peg_geometry(T, w, True)["HB"] + 1))
            if w <= 64:
                out.append((w, T, 512, 2 * peg_geometry(T, w, True)["HB"] + 1))
    return out


def peg_params(C, seed):
    """Depthwise weights [C, 1, 3, 3, 3] and bias [C] of the magnitude of a trained PEG."""
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(C, 1, 3, 3, 3, generator=g) - 0.5) * 0.6, (torch.rand(C, generator=g) - 0.5) * 0.2


def peg_input(B, T, N, C, seed, device=None):
    """X [B, T', N, C]: uniform(-1, 1) per row times 10^u, u in [-2, 2] (rows of very different magnitude)."""
    g = torch.Generator(device=device or "cpu").manual_seed(seed)
    x = torch.rand(B, T, N, C, generator=g, device=device) * 2 - 1
    return (x * 10.0 ** (torch.rand(B, T, N, 1, generator=g, device=device) * 4 - 2)).contiguous()

