"""The row-wise kernels at every instantiation, row map and tile geometry the host can pick (cases and float64 references
in tests/rowwise_cases.py):

* layernorm_kernel<NV, PAIR> (all seven), in fp32, 2^11-scaled planes and row-scaled planes of both the normalised and
  the raw row, planes only, with a row map and in place;
* patchify_ln_kernel<2 | 6 | 8> with LayerNorm and as im2col, in each output form; unpatchify_kernel;
* peg_tile4_kernel (v4) at every (TT, HB) of the geometry table and peg_tile_kernel (v3), bit-identical, and the packed
  (varlen) entry point;
* qk_prep_kernel, pre_vq_kernel<8 | 16> past its grid cap and post_vq_kernel in its three source forms.

Every output lands in a sentinel-filled buffer with guard rows before and after it, and guard columns past C / K where the
entry point takes a leading dimension; the guards must survive.  Inputs of out-of-place launches stay bit-identical, two
launches agree bit for bit, and every accuracy check prints its largest error and its bar.  Finally every entry point
refuses a pointer off the alignment of its vector accesses, naming itself, before anything is launched, and every patch
entry point refuses a patch geometry it cannot walk.
"""
import itertools

import pytest
import torch

from omnitokenizer_b200 import layout as L
from tests import rowwise_cases as R

pytestmark = pytest.mark.gpu

SENT32 = 0x7FBADBAD          # fp32 NaN pattern of the fp32 output buffers
SENT16 = 0x7E5B              # fp16 NaN pattern of the plane buffers
PRE, POST = 3, 5             # guard rows before and after every output
EPS = 1e-5

# Error bars.  Each is relative to the size of the terms the fp32 arithmetic rounds, so one bar covers rows from 1e-3
# to 1e3 (rowwise_cases.family_rows).  Largest errors observed on an H100 80GB HBM3 (400 W power limit) in brackets.
#  * LayerNorm and the patch gather's LN, relative to max|gamma| (1 + |mean| / std) + max|beta| (rowwise_cases.ln_ref):
#    the fp32 row sum carries ~log2(C) roundings of up to 2^-24 of |mean| C, which the mean hands on to every centred
#    element; the centred sum of squares and rstd add a few more: ~16 x 2^-24 ~ 1e-6 at C = 1024 [3.9e-7, C = 1020].
LN_BAR = 2e-6
#  * PEG, relative to |x| + |bias| + sum |w||x| over the 27 taps: one rounding per fma and the residual add, 28 x 2^-24
#    ~ 1.7e-6 at worst; rounding errors of a chain of fmas mostly cancel [6.6e-7].
PEG_BAR = 1e-6
#  * qk_prep, relative to max|scale|: rope (two products and a sum), a 64-term sum of squares, sqrt, a division and the
#    scale: ~8 roundings of 2^-24 ~ 5e-7 on a unit vector, at worst [5.6e-8].
QK_BAR = 3e-7
#  * pre_vq, relative to the row's largest |x| |W|^T + |b|: C / 32 = 16 fmas per lane and a 5-level warp tree, ~21
#    roundings, that mostly cancel [4.0e-8]; the l2 normalisation adds the norm's sum of squares, sqrt and division,
#    each relative to the normalised row [1.4e-7].
PREVQ_BAR = {0: 3e-7, 1: 1e-6}
#  * post_vq, relative to |z| |W|^T + |b|: an 8-fma chain and the bias add, 9 x 2^-24 ~ 5e-7 at worst [2.3e-7].
POSTVQ_BAR = 5e-7


def _cabi():
    from omnitokenizer_b200 import _cabi
    _cabi.load()
    return _cabi


class Buf:
    """A [rows, cols] output with leading dimension ld at row PRE of a sentinel-filled flat buffer, `off` elements past
    the buffer's start (an fp32 buffer, or an fp16 plane with planes=True)."""

    def __init__(self, rows, cols, ld, dev, planes=False, off=0):
        self.rows, self.cols, self.ld = rows, cols, ld
        self.sent = SENT16 if planes else SENT32
        self.dtype = torch.float16 if planes else torch.float32
        n = off + (PRE + rows + POST) * ld
        self.flat = torch.full((n,), self.sent, dtype=torch.int16 if planes else torch.int32, device=dev)
        self.start = off + PRE * ld
        self.ptr = self.flat.data_ptr() + self.start * self.flat.element_size()

    def bits(self, flat=None):
        return (self.flat if flat is None else flat).as_strided((self.rows, self.cols), (self.ld, 1), self.start)

    def val(self):
        return self.bits().view(self.dtype)

    def check(self, what, written=None):
        """Everything outside the output (rows `written` of it, or all) still holds the sentinel."""
        c = self.flat.clone()
        if written is None:
            self.bits(c).fill_(self.sent)
        else:
            self.bits(c)[written] = self.sent
        assert bool((c == self.sent).all()), f"{what}: guard elements were written"


def _same(a, b):
    """Bit equality of two tensors of the same element size."""
    ib = {2: torch.int16, 4: torch.int32, 8: torch.int64}[a.element_size()]
    return torch.equal(a.contiguous().view(ib), b.contiguous().view(ib))


def _report(what, err, bar):
    print(f"[rowwise] {what}: max rel err {err:.2e} (bar {bar:.0e})")
    assert err < bar, f"{what}: max error {err:.2e} >= {bar:.0e}"


def _planes_equal(what, got_hi, got_lo, want_hi, want_lo):
    for name, g, w in (("hi", got_hi, want_hi), ("lo", got_lo, want_lo)):
        bad = int((g.view(torch.int16) != w.view(torch.int16)).sum())
        assert bad == 0, f"{what}: {bad} {name} plane elements differ from the host split"


def _padded(x, ld, dev):
    """x [M, C] in an [M, ld] device buffer whose columns past C are NaN (a kernel that reads them returns NaN)."""
    buf = torch.full((x.shape[0], ld), float("nan"), device=dev)
    buf[:, : x.shape[1]] = x.to(dev)
    return buf


# ---------------------------------------------------------------- LayerNorm

def _ln(x_ptr, ldx, y_ptr, ldy, w, b, M, C, seg=(0, 0, 0), yp=None, xp=None, lds=0):
    """omt_layernorm, or omt_layernorm_h when planes are given: yp / xp = (hi, lo, rs or None) Buf triples."""
    if yp is None and xp is None:
        _cabi().call("omt_layernorm", x_ptr, ldx, y_ptr, ldy, w, b, M, C, EPS, *seg)
        return
    yh, yl, yr = yp if yp is not None else (None, None, None)
    xh, xl, xr = xp if xp is not None else (None, None, None)
    p = [None if t is None else t.ptr for t in (yh, yl, yr, xh, xl, xr)]
    _cabi().call("omt_layernorm_h", x_ptr, ldx, y_ptr, ldy, *p, lds, w, b, M, C, EPS, *seg)


def _plane_set(M, C, lds, off, dev, rs):
    return (Buf(M, C, lds, dev, True, off // 2), Buf(M, C, lds, dev, True, off // 2), Buf(M, 1, 1, dev) if rs else None)


@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("case", R.LN_CASES, ids=R.ln_case_id)
def test_layernorm(cuda, case, bias):
    C, M, ldx, lds, off, inst32, inst_pl = case
    assert R.ln_instantiation(C) == inst32 and R.ln_instantiation(C, lds, 8 if off % 16 else 16) == inst_pl
    what = f"layernorm C={C} M={M} ldx={ldx} lds={lds} off={off} {'bias' if bias else 'no bias'} {inst32}/{inst_pl}"
    x = R.family_rows(M, C, 100 + C + M)
    g, b = R.ln_params(C, 200 + C)
    ref, mag = R.ln_ref(x, g, b if bias else None)
    xd = _padded(x, ldx, cuda)
    x0 = xd.clone()
    gd, bd = g.to(cuda), (b.to(cuda) if bias else None)
    ldy = C + 4
    # fp32: two launches, bit for bit; the input is left alone
    ys = []
    for _ in range(2):
        y = Buf(M, C, ldy, cuda)
        _ln(xd, ldx, y.ptr, ldy, gd, bd, M, C)
        torch.cuda.synchronize()
        y.check(what)
        ys.append(y)
    assert _same(ys[0].val(), ys[1].val()), f"{what}: launches differ"
    assert _same(xd, x0), f"{what}: the input was modified"
    got = ys[0].val().double().cpu()
    assert not bool(torch.isnan(got).any()), f"{what}: NaN in the output"
    _report(what, float(((got - ref).abs() / mag).max()), LN_BAR)
    # 2^11 planes of y and of the raw row, next to the fp32 output of the same launch (the plane instantiation)
    y = Buf(M, C, ldy, cuda)
    yp, xp = _plane_set(M, C, lds, off, cuda, False), _plane_set(M, C, lds, off, cuda, False)
    _ln(xd, ldx, y.ptr, ldy, gd, bd, M, C, yp=yp, xp=xp, lds=lds)
    torch.cuda.synchronize()
    for t in (y,) + yp[:2] + xp[:2]:
        t.check(what + " 2^11 planes")
    y11 = y.val()
    _report(what + " (plane launch)", float(((y11.double().cpu() - ref).abs() / mag).max()), LN_BAR)
    _planes_equal(what + " y 2^11", yp[0].val(), yp[1].val(), *L.split_f16(y11))
    _planes_equal(what + " x 2^11", xp[0].val(), xp[1].val(), *L.split_f16(x.to(cuda)))
    # row-scaled planes + inverse row scales; the fp32 output is the same arithmetic as the 2^11 launch
    y = Buf(M, C, ldy, cuda)
    yr, xr = _plane_set(M, C, lds, off, cuda, True), _plane_set(M, C, lds, off, cuda, True)
    _ln(xd, ldx, y.ptr, ldy, gd, bd, M, C, yp=yr, xp=xr, lds=lds)
    torch.cuda.synchronize()
    for t in (y,) + yr + xr:
        t.check(what + " row-scaled planes")
    assert _same(y.val(), y11), f"{what}: the row-scaled launch computed a different y"
    for name, planes, src in (("y", yr, y11), ("x", xr, x.to(cuda))):
        hi, lo, inv = L.split_rows_rs(src)
        _planes_equal(f"{what} {name} row-scaled", planes[0].val(), planes[1].val(), hi, lo)
        assert _same(planes[2].val()[:, 0], inv), f"{what}: {name} row scales differ from split_rows_rs"
    # planes only (y = NULL): the same planes
    for rs, ref_set in ((False, yp), (True, yr)):
        po = _plane_set(M, C, lds, off, cuda, rs)
        _ln(xd, ldx, None, 0, gd, bd, M, C, yp=po, lds=lds)
        torch.cuda.synchronize()
        for t, want in zip(po, ref_set):
            if t is not None:
                t.check(what + " planes only")
                assert _same(t.val(), want.val()), f"{what}: planes-only launch (row-scaled={rs}) differs"


def _row_map(M, seg, stride, soff):
    r = torch.arange(M)
    return (r // seg) * stride + soff + r % seg


@pytest.mark.parametrize("case", R.LN_CASES, ids=R.ln_case_id)
def test_layernorm_row_map_and_in_place(cuda, case):
    """y at the physical rows of the row map (the others untouched), planes and row scales at the logical rows, and in
    place (y == x, as the patch embed's second LayerNorm and the transformers' last one run) with and without the map,
    equal to the out-of-place launch bit for bit."""
    C, M, ldx, lds, off, _, _ = case
    what = f"layernorm row map C={C} M={M} lds={lds} off={off}"
    seg = (5, 8, 2)
    phys = _row_map(M, *seg)
    Mp = int(phys.max()) + 4
    xp = R.family_rows(Mp, C, 300 + C)
    g, b = R.ln_params(C, 400 + C)
    gd, bd = g.to(cuda), b.to(cuda)
    xd = _padded(xp, ldx, cuda)
    x0 = xd.clone()
    ref, mag = R.ln_ref(xp[phys], g, b)
    # the unmapped launch on the gathered rows: the map moves addresses only, so the bits are the same
    xg = _padded(xp[phys], ldx, cuda)
    yg = Buf(M, C, ldx, cuda)
    _ln(xg, ldx, yg.ptr, ldx, gd, bd, M, C)
    yg_pl = Buf(M, C, ldx, cuda)           # with planes: the instantiation of the mapped launch below
    _ln(xg, ldx, yg_pl.ptr, ldx, gd, bd, M, C, yp=_plane_set(M, C, lds, off, cuda, True), lds=lds)
    y = Buf(Mp, C, ldx, cuda)
    yr = _plane_set(M, C, lds, off, cuda, True)
    _ln(xd, ldx, y.ptr, ldx, gd, bd, M, C, seg=seg, yp=yr, lds=lds)
    torch.cuda.synchronize()
    y.check(what, written=phys.to(cuda))
    for t in yr:
        t.check(what + " planes")
    assert _same(xd, x0), f"{what}: the input was modified"
    got = y.val()[phys.to(cuda)]
    assert _same(got, yg_pl.val()), f"{what}: mapped rows differ from the unmapped launch"
    _report(what, float(((got.double().cpu() - ref).abs() / mag).max()), LN_BAR)
    hi, lo, inv = L.split_rows_rs(got)
    _planes_equal(what, yr[0].val(), yr[1].val(), hi, lo)
    assert _same(yr[2].val()[:, 0], inv), f"{what}: row scales are not at the logical rows"
    # in place without a map, then with it
    xi = xg.clone()
    _ln(xi, ldx, xi, ldx, gd, bd, M, C)
    xm = xd.clone()
    _ln(xm, ldx, xm, ldx, gd, bd, M, C, seg=seg)
    torch.cuda.synchronize()
    assert _same(xi[:, :C], yg.val()), f"{what}: in-place launch differs from out-of-place"
    assert bool(torch.isnan(xi[:, C:]).all()), f"{what}: in-place launch wrote past C"
    assert _same(xm[phys.to(cuda), :C], yg.val()), f"{what}: in-place mapped launch differs"
    keep = torch.ones(Mp, dtype=torch.bool)
    keep[phys] = False
    assert _same(xm[keep.to(cuda)], x0[keep.to(cuda)]), f"{what}: in-place mapped launch touched unmapped rows"


# ---------------------------------------------------------------- patch gather and un-patchify

def _case_id(c):
    return f"Cin{c[0]}-p{c[1]}-pt{c[2]}-first{c[3]}-K{c[4]}"


def _patch_video(case, seed):
    """(video, rows): a video whose patch rows of this case are family_rows (the other frames random)."""
    Cin, p, pt, first, K, _ = case
    shape = R.patch_video_shape(Cin, p, pt)
    v = torch.randn(shape, generator=torch.Generator().manual_seed(seed))
    rows = R.family_rows(R.patch_index(*shape, p, pt, first).shape[0], K, seed + 1)
    return R.unpatchify_ref(rows, shape, p, pt, first, out=v), rows


@pytest.mark.parametrize("ln", [True, False], ids=["ln", "im2col"])
@pytest.mark.parametrize("case", R.PATCH_CASES, ids=_case_id)
def test_patch_gather(cuda, case, ln):
    Cin, p, pt, first, K, nv = case
    assert R.patch_nv(K) == nv
    what = f"patch gather {_case_id(case)} NV={nv} {'LN' if ln else 'im2col'}"
    v, rows = _patch_video(case, 500 + K + first)
    B, _, T, H, W = v.shape
    M = rows.shape[0]
    vd = v.to(cuda)
    v0 = vd.clone()
    lw, lb = R.ln_params(K, 600 + K)
    lwd, lbd = (lw.to(cuda), lb.to(cuda)) if ln else (None, None)

    def gather(A=None, hi=None, lo=None, rs=None):
        _cabi().call("omt_patchify_ln", vd, A, hi, lo, rs, lwd, lbd, B, Cin, T, H, W, p, pt, first, EPS)

    outs = []
    for _ in range(2):
        A = Buf(M, K, K, cuda)
        gather(A=A.ptr)
        torch.cuda.synchronize()
        A.check(what)
        outs.append(A)
    assert _same(outs[0].val(), outs[1].val()), f"{what}: launches differ"
    assert _same(vd, v0), f"{what}: the video was modified"
    a = outs[0].val()
    if ln:
        ref, mag = R.ln_ref(rows, lw, lb)
        _report(what, float(((a.double().cpu() - ref).abs() / mag).max()), LN_BAR)
    else:
        assert _same(a.cpu(), rows), f"{what}: im2col is not an exact copy"
    hi, lo = Buf(M, K, K, cuda, True), Buf(M, K, K, cuda, True)
    gather(hi=hi.ptr, lo=lo.ptr)
    hr, lr, rr = Buf(M, K, K, cuda, True), Buf(M, K, K, cuda, True), Buf(M, 1, 1, cuda)
    gather(hi=hr.ptr, lo=lr.ptr, rs=rr.ptr)
    torch.cuda.synchronize()
    for t in (hi, lo, hr, lr, rr):
        t.check(what + " planes")
    _planes_equal(what + " 2^11", hi.val(), lo.val(), *L.split_f16(a))
    h2, l2, inv = L.split_rows_rs(a)
    _planes_equal(what + " row-scaled", hr.val(), lr.val(), h2, l2)
    assert _same(rr.val()[:, 0], inv), f"{what}: row scales differ from split_rows_rs"


@pytest.mark.parametrize("case", R.PATCH_CASES, ids=_case_id)
def test_unpatchify(cuda, case):
    """The exact inverse permutation, writing only its own frames; and gather (im2col) -> un-patchify of the first frame
    and of the rest returns the whole video bit for bit."""
    Cin, p, pt, first, K, _ = case
    what = f"unpatchify {_case_id(case)}"
    shape = R.patch_video_shape(Cin, p, pt)
    B, _, T, H, W = shape
    rows = R.patch_index(*shape, p, pt, first).shape[0]
    P = R.family_rows(rows, K, 700 + K).to(cuda)
    P0 = P.clone()
    vid = Buf(B * Cin * T * H, W, W, cuda)
    _cabi().call("omt_unpatchify", P, vid.ptr, B, Cin, T, H, W, p, pt, first)
    torch.cuda.synchronize()
    assert _same(P, P0), f"{what}: the input was modified"
    want = torch.full((B * Cin * T * H * W,), SENT32, dtype=torch.int32)
    want[R.patch_index(*shape, p, pt, first).reshape(-1)] = P.cpu().view(torch.int32).reshape(-1)
    got = vid.flat.cpu()
    assert bool((got[: vid.start] == SENT32).all() and (got[vid.start + want.numel():] == SENT32).all()), \
        f"{what}: guard elements were written"
    assert torch.equal(got[vid.start: vid.start + want.numel()], want), \
        f"{what}: not the inverse permutation, or frames of the other call were written"
    # round trip over both calls
    v = torch.randn(shape, generator=torch.Generator().manual_seed(800 + K)).to(cuda)
    back = Buf(B * Cin * T * H, W, W, cuda)
    for fst in (1, 0):
        A = torch.empty(R.patch_index(*shape, p, pt, fst).shape[0], Cin * (1 if fst else pt) * p * p, device=cuda)
        _cabi().call("omt_patchify_ln", v, A, None, None, None, None, None, B, Cin, T, H, W, p, pt, fst, EPS)
        _cabi().call("omt_unpatchify", A, back.ptr, B, Cin, T, H, W, p, pt, fst)
    torch.cuda.synchronize()
    back.check(what + " round trip")
    assert _same(back.val().reshape(shape), v), f"{what}: gather -> un-patchify is not the identity"


# ---------------------------------------------------------------- PEG

def _peg_id(c):
    return f"w{c[0]}-T{c[1]}-C{c[2]}-h{c[3]}"


@pytest.mark.parametrize("case", R.peg_cases(), ids=_peg_id)
def test_peg_geometry(cuda, case):
    """Each geometry against the float64 conv3d formulation, spatial and temporal, causal and not, B = 2 samples on
    blockIdx.z; v4 (the default) and v3 agree bit for bit."""
    w, T, C, h = case
    B, N = 2, h * w
    M = B * T * N
    cabi = _cabi()
    X = R.peg_input(B, T, N, C, 900 + w + T + C, device=cuda)
    X0 = X.clone()
    wt, bias = R.peg_params(C, 1000 + C)
    w27, bd = wt.reshape(C, 27).t().contiguous().to(cuda), bias.to(cuda)
    worst = 0.0
    for temporal in (0, 1):
        for causal in (0, 1):
            geo = R.peg_geometry(T, w, causal)
            assert geo["kernel"] == R.PEG_TABLE[w][3]
            what = f"peg {_peg_id(case)} temporal={temporal} causal={causal} {geo['kernel']} TT={geo['TT']} HB={geo['HB']}"
            ref, mag = R.peg_ref(X, wt, bias, h, w, bool(temporal), bool(causal))
            ys = {}
            for pk in (4, 3, 4):
                cabi.set_option("peg_kernel", pk)
                y = Buf(M, C, C, cuda)
                cabi.call("omt_peg_volume", X, y.ptr, w27, bd, B, T, h, w, C, temporal, causal)
                torch.cuda.synchronize()
                y.check(what)
                if pk in ys:
                    assert _same(y.val(), ys[pk]), f"{what}: launches differ"
                ys[pk] = y.val()
            cabi.set_option("peg_kernel", 4)
            assert _same(ys[3], ys[4]), f"{what}: v3 and v4 differ"
            err = float(((ys[4].view(B, T, N, C).double() - ref).abs() / mag).max())
            print(f"[rowwise] {what}: max rel err {err:.2e} (bar {PEG_BAR:.0e})")
            worst = max(worst, err)
            assert err < PEG_BAR, f"{what}: max error {err:.2e} >= {PEG_BAR:.0e}"
            del ref, mag
    assert _same(X, X0), "the input was modified"


@pytest.mark.parametrize("temporal,causal", [(1, 1), (0, 1), (1, 0)])
def test_peg_varlen_equals_per_sample(cuda, temporal, causal):
    """A packed batch of clips of 5, 2, 9 and 1 latent frames at w = 128 (the T = 9 geometry for all) equals per-sample
    launches (each at its own geometry) bit for bit."""
    tps, h, w, C = (5, 2, 9, 1), 16, 128, 32
    N = h * w
    t_off = torch.tensor([0] + list(itertools.accumulate(tps)), dtype=torch.int32)
    M = int(t_off[-1]) * N
    X = R.peg_input(1, int(t_off[-1]), N, C, 77, device=cuda).reshape(M, C)
    wt, bias = R.peg_params(C, 78)
    w27, bd = wt.reshape(C, 27).t().contiguous().to(cuda), bias.to(cuda)
    y = Buf(M, C, C, cuda)
    _cabi().call("omt_peg_volume_varlen", X, y.ptr, w27, bd, t_off, t_off.to(cuda), len(tps), M, h, w, C, temporal, causal)
    ys = Buf(M, C, C, cuda)
    for b, tp in enumerate(tps):
        r0 = int(t_off[b]) * N
        _cabi().call("omt_peg_volume", X[r0:], ys.ptr + r0 * C * 4, w27, bd, 1, tp, h, w, C, temporal, causal)
    torch.cuda.synchronize()
    y.check("peg varlen")
    ys.check("peg per sample")
    assert _same(y.val(), ys.val()), "packed PEG differs from per-sample launches"
    for b, tp in enumerate(tps):
        r0, r1 = int(t_off[b]) * N, int(t_off[b + 1]) * N
        ref, mag = R.peg_ref(X[r0:r1].view(1, tp, N, C), wt, bias, h, w, bool(temporal), bool(causal))
        _report(f"peg varlen sample {b} T'={tp} temporal={temporal} causal={causal}",
                float(((y.val()[r0:r1].view(1, tp, N, C).double() - ref).abs() / mag).max()), PEG_BAR)


# ---------------------------------------------------------------- qk_prep

@pytest.mark.parametrize("rope", [True, False])
@pytest.mark.parametrize("heads", [1, 3, 8])
def test_qk_prep(cuda, heads, rope):
    """In place on q and k of a buffer wider than 3C (ld = 3C + 6); v and the padding stay bit-identical; zero head
    vectors give exact zeros (the 1e-12 clamp), not NaN."""
    N = 64
    M, C = 2 * N + 37, 64 * heads
    ld = 3 * C + 6
    what = f"qk_prep heads={heads} rope={rope}"
    g = torch.Generator().manual_seed(1100 + heads)
    data = torch.randn(M, ld, generator=g) * 10.0 ** (torch.rand(M, 1, generator=g) * 6 - 3)
    qv = data[:, :C].view(M, heads, 64)
    kv = data[:, C:2 * C].view(M, heads, 64)
    qv[::7, 0] = 0.0
    kv[::5, heads - 1] = 0.0
    qv[3, :] = 0.0
    qs, ks = torch.rand(64, generator=g) + 0.5, torch.rand(64, generator=g) + 0.5
    cos, sin = L.rope_tables(N, 64)
    pos = torch.arange(M) % N
    buf = torch.full((PRE + M + POST, ld), float("nan"), device=cuda)
    buf[PRE:PRE + M] = data.to(cuda)
    b0 = buf.clone()
    q_ptr = buf.data_ptr() + PRE * ld * 4
    args = (q_ptr, ld, q_ptr + C * 4, ld, qs.to(cuda), ks.to(cuda), cos.to(cuda) if rope else None,
            sin.to(cuda) if rope else None, M, N, heads)
    _cabi().call("omt_qk_prep", *args)
    torch.cuda.synchronize()
    once = buf.clone()
    buf.copy_(b0)
    _cabi().call("omt_qk_prep", *args)
    torch.cuda.synchronize()
    assert _same(buf, once), f"{what}: launches differ"
    got = once[PRE:PRE + M].cpu()
    assert _same(once[:PRE], b0[:PRE]) and _same(once[PRE + M:], b0[PRE + M:]), f"{what}: guard rows were written"
    assert _same(got[:, 2 * C:], data[:, 2 * C:]), f"{what}: v or the padding columns were written"
    assert not bool(torch.isnan(got[:, :2 * C]).any()), f"{what}: NaN"
    for name, sl, sc, zero in (("q", slice(0, C), qs, (slice(None, None, 7), 0)), ("k", slice(C, 2 * C), ks,
                                                                                    (slice(None, None, 5), heads - 1))):
        ref = R.qk_prep_ref(data[:, sl], sc, cos[pos] if rope else None, sin[pos] if rope else None)
        _report(f"{what} {name}", float((got[:, sl].double() - ref).abs().max() / sc.abs().max()), QK_BAR)
        assert bool((got[:, sl].view(M, heads, 64)[zero] == 0).all()), f"{what}: zero {name} heads are not exact zeros"
    assert bool((got[3, :C] == 0).all())


# ---------------------------------------------------------------- pre_vq / post_vq

@pytest.mark.parametrize("l2", [0, 1])
@pytest.mark.parametrize("cd", [8, 16])
def test_pre_vq(cuda, cd, l2):
    """9 000 rows: more than 4 CTAs per SM x 8 warps, so warps walk rows with the grid stride; ldx > C."""
    M, C, ldx = 9000, 512, 516
    what = f"pre_vq cd={cd} l2={l2}"
    x = R.family_rows(M, C, 1200 + cd)
    g = torch.Generator().manual_seed(1300 + cd)
    Wt, b = (torch.rand(cd, C, generator=g) - 0.5) * 0.1, (torch.rand(cd, generator=g) - 0.5) * 0.2
    xd = _padded(x, ldx, cuda)
    x0 = xd.clone()
    zs = []
    for _ in range(2):
        z = Buf(M, cd, cd, cuda)
        _cabi().call("omt_pre_vq", xd, ldx, Wt.to(cuda), b.to(cuda), z.ptr, M, C, cd, l2)
        torch.cuda.synchronize()
        z.check(what)
        zs.append(z.val())
    assert _same(zs[0], zs[1]), f"{what}: launches differ"
    assert _same(xd, x0), f"{what}: the input was modified"
    ref, mag = R.pre_vq_ref(x, Wt, b, l2)
    _report(what, float(((zs[0].double().cpu() - ref).abs() / mag.amax(1, keepdim=True)).max()), PREVQ_BAR[l2])


@pytest.mark.parametrize("C", [256, 512])
@pytest.mark.parametrize("M", [1, 31, 32, 33, 1000])
def test_post_vq(cuda, M, C):
    """Codes 0 and n_codes - 1 included; rows from E[idx], from (E[idx] - z) + z (straight-through, zq bit-exact) and
    from given latents; C = 256 leaves threads past C idle."""
    n = 1024
    g = torch.Generator().manual_seed(1400 + M + C)
    E = torch.randn(n, 8, generator=g)
    idx = torch.randint(0, n, (M,), generator=g)
    idx[0] = n - 1 if M == 1 else 0
    idx[-1] = n - 1
    z = torch.randn(M, 8, generator=g) * 0.3
    zc = torch.randn(M, 8, generator=g)
    Wq, bq = (torch.rand(C, 8, generator=g) - 0.5) * 0.6, (torch.rand(C, generator=g) - 0.5) * 0.2
    Ed, Wd, bd, idd, zd, zcd = (t.to(cuda) for t in (E, Wq, bq, idx, z, zc))
    st = (E[idx] - z) + z
    for form, rows in (("idx", E[idx]), ("idx+st", st), ("zc", zc)):
        what = f"post_vq M={M} C={C} {form}"
        outs = []
        for _ in range(2):
            X = Buf(M, C, C, cuda)
            zq = Buf(M, 8, 8, cuda) if form == "idx+st" else None
            if form == "zc":
                _cabi().call("omt_post_vq", None, None, zcd, None, None, Wd, bd, X.ptr, M, C, 8)
            else:
                _cabi().call("omt_post_vq", idd, Ed, None, zd if zq is not None else None, None if zq is None else zq.ptr,
                             Wd, bd, X.ptr, M, C, 8)
            torch.cuda.synchronize()
            X.check(what)
            if zq is not None:
                zq.check(what + " zq")
                assert _same(zq.val().cpu(), st), f"{what}: straight-through rows are not bit-exact"
            outs.append(X.val())
        assert _same(outs[0], outs[1]), f"{what}: launches differ"
        ref, mag = R.post_vq_ref(rows, Wq, bq)
        _report(what, float(((outs[0].double().cpu() - ref).abs() / mag).max()), POSTVQ_BAR)


# ---------------------------------------------------------------- misaligned pointers

def test_misaligned_pointers_raise(cuda):
    """Every row-wise and VQ entry point refuses a pointer 4 bytes off the alignment of its vector accesses with a
    RuntimeError naming itself, and launches nothing; the same call with aligned pointers runs."""
    f = torch.zeros(1 << 16, device=cuda)
    o = torch.zeros(1 << 16, device=cuda)
    p, q = f.data_ptr(), o.data_ptr()
    h16 = torch.zeros(1 << 16, dtype=torch.int16, device=cuda)
    hp = h16.data_ptr()
    i64 = torch.zeros(64, dtype=torch.int64, device=cuda)
    u8 = torch.zeros(1 << 14, dtype=torch.uint8, device=cuda)
    lut = L.u8_norm_table(L.U8Norm("t", (0.5,) * 3, (0.5,) * 3), 3).to(cuda)
    nbr = L.peg_neighbour_table(1, 4, 4, False, True).to(cuda)
    t_off = torch.tensor([0, 1], dtype=torch.int32)
    t_offd = t_off.to(cuda)
    E = torch.zeros(64, 8, device=cuda)
    e2 = torch.zeros(64, device=cuda)
    # entry point -> (argument builder over the pointers it checks, {pointer name: aligned value})
    calls = {
        "omt_layernorm": (lambda a: (a["x"], 64, a["y"], 64, a["w"], a["b"], 8, 64, EPS, 0, 0, 0),
                          dict(x=p, y=q, w=p, b=p)),
        "omt_layernorm_h": (lambda a: (a["x"], 64, a["y"], 64, hp, hp + 2048, None, None, None, None, 64, a["w"], a["b"], 8,
                                       64, EPS, 0, 0, 0), dict(x=p, y=q, w=p, b=p)),
        "omt_patchify_ln": (lambda a: (a["video"], a["A"], None, None, None, a["ln_w"], a["ln_b"], 1, 3, 1, 8, 8, 4, 1, 1,
                                       EPS), dict(video=p, A=q, ln_w=p, ln_b=p)),
        "omt_patchify_ln_u8": (lambda a: (u8, lut, None, a["A"], None, None, None, a["ln_w"], a["ln_b"], 1, 3, 1, 8, 8, 4, 1,
                                          1, EPS), dict(A=q, ln_w=p, ln_b=p)),
        "omt_unpatchify": (lambda a: (a["P"], a["video"], 1, 3, 1, 8, 8, 4, 1, 1), dict(P=p, video=q)),
        "omt_unpatchify_u8": (lambda a: (a["P"], u8, 1, 3, 1, 8, 8, 4, 1, 1, 1.0, 0.0, 0.0, 1.0, 255.0), dict(P=p)),
        "omt_peg": (lambda a: (a["x"], a["y"], a["w27"], a["bias"], nbr, 1, 16, 16), dict(x=p, y=q, w27=p, bias=p)),
        "omt_peg_volume": (lambda a: (a["x"], a["y"], a["w27"], a["bias"], 1, 1, 4, 4, 16, 0, 1),
                           dict(x=p, y=q, w27=p, bias=p)),
        "omt_peg_volume_varlen": (lambda a: (a["x"], a["y"], a["w27"], a["bias"], t_off, t_offd, 1, 16, 4, 4, 16, 0, 1),
                                  dict(x=p, y=q, w27=p, bias=p)),
        "omt_qk_prep": (lambda a: (a["q"], 192, a["k"], 192, a["q_scale"], a["k_scale"], None, None, 8, 8, 1),
                        dict(q=q, k=q + 256, q_scale=p, k_scale=p)),
        "omt_pre_vq": (lambda a: (a["x"], 64, a["Wt"], p, q, 8, 64, 8, 1), dict(x=p, Wt=p)),
        "omt_vq_fused": (lambda a: (a["x"], 64, a["Wt"], p, 64, 1, a["z"], a["E"], e2, 8, 64, i64, None),
                         dict(x=p, Wt=p, z=q, E=E.data_ptr())),
        "omt_vq_search": (lambda a: (a["z"], a["E"], e2, 8, 64, i64, None), dict(z=p, E=E.data_ptr())),
        "omt_post_vq": (lambda a: (i64, E, None, None, None, p, a["b"], a["X"], 8, 64, 8), dict(X=q, b=p)),
    }
    # the 8-byte pointers of the PEG tile kernels and qk_prep are tested 4 bytes off; every other one needs 16
    cabi = _cabi()
    for name, (build, good) in calls.items():
        cabi.call(name, *build(good))
        torch.cuda.synchronize()
        for arg in good:
            bad = dict(good, **{arg: good[arg] + 4})
            o.fill_(7.0)
            h16.fill_(7)
            with pytest.raises(RuntimeError, match=f"{name}: .*aligned"):
                cabi.call(name, *build(bad))
            torch.cuda.synchronize()
            assert bool((o == 7.0).all()) and bool((h16 == 7).all()), f"{name}: a call with misaligned {arg} wrote"


# ---------------------------------------------------------------- patch geometry

def test_patch_geometry_refused(cuda):
    """Every patch entry point refuses a geometry it cannot walk -- p = 0 or not a multiple of 4, H not a multiple of p,
    rest frames with pt = 0 or (T - 1) % pt != 0, Cin = 0, B < 0 and, for the gathers, a patch vector of more than 1024
    features -- with a RuntimeError naming itself, and writes nothing; the same call with the valid geometry runs."""
    f = torch.zeros(1 << 16, device=cuda)
    u8 = torch.zeros(1 << 16, dtype=torch.uint8, device=cuda)
    lut = L.u8_norm_table(L.U8Norm("t", (0.5,) * 3, (0.5,) * 3), 3).to(cuda)
    o = torch.empty(1 << 16, dtype=torch.int32, device=cuda)
    good = dict(B=1, Cin=3, T=5, H=8, W=8, p=4, pt=2, first=0)

    def geo(g):
        return tuple(g[k] for k in ("B", "Cin", "T", "H", "W", "p", "pt", "first"))

    # entry point -> argument builder over the geometry
    calls = {
        "omt_patchify_ln": lambda g: (f, o, None, None, None, None, None, *geo(g), EPS),
        "omt_patchify_ln_u8": lambda g: (u8, lut, None, o, None, None, None, None, None, *geo(g), EPS),
        "omt_unpatchify": lambda g: (f, o, *geo(g)),
        "omt_unpatchify_u8": lambda g: (f, o, *geo(g), 1.0, 0.5, 0.0, 1.0, 255.0),
    }
    bad = {"p = 0": dict(p=0), "p = 6": dict(p=6), "H % p != 0": dict(H=10), "rest frames, pt = 0": dict(pt=0),
           "(T - 1) % pt != 0": dict(T=4), "Cin = 0": dict(Cin=0), "B = -1": dict(B=-1)}
    gathers = {"K = 1536 > 1024": dict(p=16, H=16, W=16)}
    cabi = _cabi()
    for name, build in calls.items():
        cabi.call(name, *build(good))
        torch.cuda.synchronize()
        for what, change in {**bad, **(gathers if name.startswith("omt_patchify") else {})}.items():
            o.fill_(SENT32)
            with pytest.raises(RuntimeError, match=f"{name}: "):
                cabi.call(name, *build(dict(good, **change)))
            torch.cuda.synchronize()
            assert bool((o == SENT32).all()), f"{name}: a call with {what} wrote"
