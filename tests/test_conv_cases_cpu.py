"""The omt_conv3d cases, operand families and error bound of conv_cases.py, checked on the CPU: the case list covers the
paths the GPU test claims, the split-grid operands split as the test assumes within the bit budget, and the host model of
the 3xTF32 scheme sits under L2_BOUND while every two-product variant exceeds it at least tenfold."""
import pytest
import torch

from omnitokenizer_b200 import fid, fvd, quality
from omnitokenizer_b200 import layout as L
from tests import conv_cases as cc

CASES = cc.all_cases()


def test_tf32_round_is_the_kernels_rule():
    """layout.tf32_round is tc_ptx.cuh's tf32_rn: (bits + 0x1000) & ~0x1fff, ties away from zero."""
    v = torch.tensor([1 + 2 ** -11, 1 + 3 * 2 ** -11, -(1 + 2 ** -11), 1 - 2 ** -12, 1 + 2 ** -12, 2 ** -130, 3.0],
                     dtype=torch.float32)
    want = torch.tensor([1 + 2 ** -10, 1 + 2 ** -9, -(1 + 2 ** -10), 1.0, 1.0, 2 ** -130, 3.0], dtype=torch.float32)
    assert torch.equal(L.tf32_round(v), want)
    r = torch.randn(1 << 16, generator=torch.Generator().manual_seed(0))
    bits = ((r.view(torch.int32).long() + 0x1000) & ~0x1FFF).to(torch.int32)
    assert torch.equal(L.tf32_round(r).view(torch.int32), bits)


def test_cases_come_from_every_network_table():
    names = {c.name.split("-")[0] for c in cc.i3d_cases()}
    assert {p for p, *_ in fvd.unit_names()} == names
    assert {c.name for c in cc.fid_cases()} == {c.name for c in fid.conv_list()}
    assert len(cc.vgg_cases()) == sum(len(s) for s in quality.SLICES) == 13
    keys = [c.key for c in cc.network_cases()]
    assert len(keys) == len(set(keys))
    every = {c.key for c in cc.i3d_cases() + cc.fid_cases() + cc.vgg_cases()}
    assert set(keys) == every


def test_stylegan_v_pad_tables_are_cases():
    """Both F.pad tables of the StyleGAN-V stem (even and odd T) are cases; the even-T table pads 2 in front, which
    SAME at the odd sizes of the plain stem case does not."""
    stem = {c.front for c in cc.network_cases() if c.k == (7, 7, 7)}
    assert stem == {(3, 3, 3), (2, 2, 2), (3, 2, 2)}


def test_cases_cover_the_kernel_paths():
    net = cc.network_cases()
    assert {c.bn for c in net} == {64, 128}
    assert {16, 24, 64} <= {c.cout for c in net if c.bn == 64}
    assert any(c.bn == 128 and c.cout % 128 for c in net)                      # a partial last column tile
    assert any(c.Cs == 4 and c.taps % 8 for c in net)                           # RGB gather, a part-empty k-block
    kbs = {c.num_kb for c in net}
    assert any(n % cc.PROMOTE for n in kbs) and any(n % cc.PROMOTE == 0 for n in kbs)     # a last chunk of 1 and of 2
    assert any(c.s[1] > 1 for c in net) and any(c.k[0] == 1 for c in net) and any(c.k[0] == 3 for c in net)
    assert any(c.k[1] != c.k[2] for c in net)                                   # 1x7 / 7x1
    assert any(c.col > 0 for c in net) and any(c.col == 0 and c.ldy > c.cout for c in net)
    assert any(c.M % 128 for c in net)
    for sms in (132, 114):
        walk = cc.walk_cases(sms)
        assert [c.tiles for c in walk] == [sms - 1, sms + 1, 2 * sms + 1, 3 * sms + 1]
        assert {c.bn for c in walk} == {64, 128} and all(c.M % 128 for c in walk)


@pytest.mark.parametrize("c", CASES, ids=[c.id for c in CASES])
def test_case_is_a_valid_launch(c):
    """The geometry omt_conv3d checks: padding below the kernel, no output reads past the input, K as packed."""
    assert all(0 <= f < k for f, k in zip(c.front, c.k))
    assert all((o - 1) * s - f < n for o, s, f, n in zip(c.out, c.s, c.front, c.dims))
    assert c.col % 2 == 0 and c.ldy >= c.col + c.cout and c.cout % 2 == 0
    w = torch.zeros((c.cout, c.cin) + c.k)
    assert fvd.pack_weight(w)[1] == c.K


@pytest.mark.parametrize("c", CASES, ids=[c.id for c in CASES])
def test_split_grid_operands(c):
    """tf32_rn(x) is hi and x - hi is lo (non-zero somewhere) in x and in the packed W; lo.hi and hi.lo products are
    present; no output sums more than 3 * MAX_PRODUCTS non-zero products, so every partial sum is a multiple of 2^-12
    below 2^8: within 20 significant bits.  The fp64 reference is then exact, and equals the fp32 sum."""
    x, w, b = cc.split_grid_operands(c, 1)
    for t in (x, w):
        hi, lo = cc.split_tf32(t)
        assert bool((hi.abs() <= 1).all()) and torch.equal(hi, hi.round())
        assert bool(((lo / cc.LO_STEP).abs() <= 1).all()) and torch.equal(lo / cc.LO_STEP, (lo / cc.LO_STEP).round())
        assert bool((lo[hi == 0] == 0).all()) and bool((lo != 0).any())
        assert torch.equal(cc.tf32_read(lo), lo)                        # lo is read as tf32 without loss
    w_hi, w_lo = cc.pack(w, c)
    wp, _ = fvd.pack_weight(w)
    assert torch.equal(w_hi + w_lo, wp) and bool((w_lo != 0).any())
    taps = (w != 0).reshape(c.cout, -1).sum(1)
    assert int(taps.max()) <= cc.MAX_PRODUCTS
    rc = cc.reduced(c, cout=min(c.cout, 64)) if c.M > 2048 else c
    if rc is not c:
        x, w, b = cc.split_grid_operands(rc, 1)
    count = cc.conv64((x != 0).double(), (w != 0).double(), rc)
    assert float(count.max()) <= cc.MAX_PRODUCTS
    # each non-zero position adds hi.hi (|.| <= 1) + lo.hi + hi.lo (|.| <= 2^-12 each): |partial sum| < 2^8
    assert cc.MAX_PRODUCTS * (1 + 2 * cc.LO_STEP) < 2 ** 8
    ref = cc.split_grid_reference(x, w, b, rc, False).double()
    assert torch.equal(ref, ((ref / cc.LO_STEP).round() * cc.LO_STEP))
    assert bool((ref.abs() < 2 ** 8 + 4).all())


def _variant_errors(c):
    r = cc.reduced(c)
    x, w, b = cc.realistic_operands(r, 5)
    ref = cc.conv64(x, w, r, b)
    scale = cc.l2_scale(x, w, b, r)
    full = cc.l2_error(cc.emulate(x, w, b, r), ref, scale)
    drops = {p: cc.l2_error(cc.emulate(x, w, b, r, drop=p), ref, scale) for p in ("lo_hi", "hi_lo")}
    return full, drops


@pytest.mark.parametrize("c", CASES, ids=[c.id for c in CASES])
def test_bound_separates_the_scheme_from_a_dropped_product(c):
    """On realistic operands the three-product scheme sits well under L2_BOUND (the GPU's fp32 accumulation needs the
    room), and dropping A_lo.W_hi or A_hi.W_lo puts the error at least 10x above it."""
    full, drops = _variant_errors(c)
    print(f"{c.id}: scheme {full:.2e}, without lo.hi {drops['lo_hi']:.2e}, without hi.lo {drops['hi_lo']:.2e}")
    assert full <= cc.L2_BOUND / 10, full
    for p, e in drops.items():
        assert e >= 10 * cc.L2_BOUND, (p, e)
