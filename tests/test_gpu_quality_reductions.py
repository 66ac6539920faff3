"""The evaluation reductions of csrc/quality.cu on their raw entry points, at every block geometry and value edge of
tests/quality_cases.py:

* omt_psnr_ssim in both forms, the valid crop on both sides of the 32 x 32 output tile in both directions, per-pair
  tables for both images, identical, constant and one-pixel-apart frames;
* omt_lpips_head with padded feature rows, maps of fewer pixels than its 16 warps, C below a warp, every tap's total;
* omt_softmax_rows below a warp and across its 256-column stride, padded rows, subnormal and zero probabilities,
  infinite logits and ties;
* omt_inception_score past 512 classes and at the 6144-class cap, rows around the 16-warp stride, one-row splits,
  padded rows, exact zeros.

Every output sits inside a sentinel-filled buffer with guard rows (and guard columns where the entry point takes a
leading dimension); the guards keep their bits, inputs are unchanged, two launches give the same bits, and each check
prints its largest error next to its bar.  Finally each entry point refuses arguments just past its limits, naming
itself, without launching anything.
"""
import pytest
import torch

from omnitokenizer_b200 import _cabi
from omnitokenizer_b200 import quality
from tests import quality_cases as Q

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SENT = {torch.float32: 0x7FBADBAD, torch.float64: 0x7FF4BADBADBADBAD}     # NaN patterns
INT = {torch.float32: torch.int32, torch.float64: torch.int64}
PRE, POST = 3, 5

# Bars (tests/quality_cases.py derives each).  Largest errors measured on an H100 80GB HBM3 (700 W power limit) in
# brackets.
#  * sse, relative, and SSIM, absolute: fp64 throughout, Q.SSIM_BAR = 1e-12 [sse 3.6e-16, SSIM 1.8e-15].  Identical
#    frames: sse 0 and SSIM 1 exactly.  Constant frames: Q.ssim_constant_slack on top, the variances' cancellation
#    [0.018 of the bar, f32 form].
#  * LPIPS head, relative to Q.head_reference's mag: (2 ceil(C / 32) + 20) 2^-24, at most 2e-6 [0.14 of the bar, C = 3;
#    0.054 at C = 512].  The fp32 total of taps 0 .. 4 bit for bit.
#  * softmax, per entry: (ceil(N / 256) + 15) 2^-24 y64 + 2^-149, 16 to 39 roundings [5.9 roundings, N = 1008]; NaN
#    for NaN and 0 for 0 on rows with an infinite logit.
#  * IS: column means 1e-12 relative [0: numpy's bits]; KL 1e-12 relative plus Q.is_floor(N) [4.3e-16 relative].


@pytest.fixture(autouse=True, scope="module")
def _device(cuda):
    """Skip, rather than fail, where there is no CUDA device (before the module's fixtures build on it)."""


class Out:
    """A [rows, cols] output with leading dimension ld inside a sentinel-filled buffer, PRE guard rows before it and
    POST after it."""

    def __init__(self, rows, cols, ld, dtype):
        self.rows, self.cols, self.ld, self.dtype = rows, cols, ld, dtype
        self.flat = torch.full(((PRE + rows + POST) * ld,), SENT[dtype], dtype=INT[dtype], device=DEV)
        self.ptr = self.flat.data_ptr() + PRE * ld * self.flat.element_size()

    def bits(self, flat=None):
        return (self.flat if flat is None else flat).as_strided((self.rows, self.cols), (self.ld, 1), PRE * self.ld)

    def val(self):
        return self.bits().clone().view(self.dtype).cpu()

    def guards_ok(self):
        """Every element outside the [rows, cols] output, guard columns included, holds the sentinel."""
        c = self.flat.clone()
        self.bits(c).fill_(SENT[self.dtype])
        return bool((c == SENT[self.dtype]).all())

    def untouched(self):
        return bool((self.flat == SENT[self.dtype]).all())


def _bits(t):
    return t.contiguous().view({1: torch.uint8, 4: torch.int32, 8: torch.int64}[t.element_size()]).clone()


def _launch_twice(launch, outs, inputs):
    """Run the launch twice; the outputs' bits of the two runs agree, the guards and the inputs keep theirs.  Returns
    the first run's outputs on the host."""
    before = [_bits(t) for t in inputs]
    launch()
    torch.cuda.synchronize()
    first = [o.val() for o in outs]
    launch()
    torch.cuda.synchronize()
    for o, f in zip(outs, first):
        assert torch.equal(_bits(o.val()), _bits(f)), "two launches differ"
        assert o.guards_ok(), "a guard element was written"
    for t, b in zip(inputs, before):
        assert torch.equal(_bits(t), b), "an input was written"
    return first


def _report(what, err, bar):
    print(f"[quality] {what}: worst {err:.2e} (bar {bar:.2e})")


# ------------------------------------------------------------------------------------------------------- PSNR / SSIM
@pytest.mark.parametrize("form", ["u8", "f32"])
def test_psnr_ssim(form):
    lut = Q.byte_tables().reshape(-1).to(DEV)
    taps = torch.from_numpy(Q.TAPS).to(DEV)
    worst = [0.0, 0.0, 0.0]
    for c in Q.ssim_cases(form):
        a, b = c.a.to(DEV), c.b.to(DEV)
        u8 = form == "u8"
        sa, sb = (c.sel_a.to(DEV), c.sel_b.to(DEV)) if u8 else (None, None)
        sse, ssim = Out(1, c.P, c.P, torch.float64), Out(1, c.P, c.P, torch.float64)
        code = quality.FORM_U8 if u8 else quality.FORM_F32
        launch = lambda: _cabi.call("omt_psnr_ssim", a, lut if u8 else None, sa, b, lut if u8 else None, sb, code,
                                    c.P, c.H, c.W, taps, sse.ptr, ssim.ptr)
        got_sse, got_ssim = _launch_twice(launch, (sse, ssim), [t for t in (a, b, sa, sb, lut, taps) if t is not None])
        ok, e_sse, e_ssim, e_const, msg = Q.ssim_check(c, got_sse[0], got_ssim[0])
        assert ok, msg
        worst = [max(worst[0], e_sse), max(worst[1], e_ssim), max(worst[2], e_const)]
    _report(f"{form} sse rel", worst[0], Q.SSIM_BAR)
    _report(f"{form} ssim abs", worst[1], Q.SSIM_BAR)
    _report(f"{form} constant pairs' ssim / bar", worst[2], 1.0)


# ------------------------------------------------------------------------------------------------------- LPIPS head
@pytest.mark.parametrize("C", Q.HEAD_C)
def test_lpips_head(C):
    worst = 0.0
    for c in Q.head_cases():
        if c.C != C:
            continue
        x, lin = c.x.to(DEV), c.lin.to(DEV)
        taps, total = Out(5, c.P, c.P, torch.float32), Out(1, c.P, c.P, torch.float32)
        taps.bits()[:c.tap].copy_(c.prev[:c.tap].to(DEV).view(torch.int32))
        launch = lambda: _cabi.call("omt_lpips_head", x, c.Cs, c.C, c.P, c.h, c.w, lin, c.tap, taps.ptr, total.ptr)
        got, tot = _launch_twice(launch, (taps, total), (x, lin))
        assert torch.equal(_bits(got[:c.tap]), _bits(c.prev[:c.tap])), f"{c.name}: earlier taps changed"
        assert bool((got[c.tap + 1:].view(torch.int32) == SENT[torch.float32]).all()), f"{c.name}: later taps written"
        ok, w, msg = Q.head_check(c, got[c.tap])
        assert ok, msg
        worst = max(worst, w / Q.head_bar(C))
        want = Q.head_total(c.prev, c.tap, got[c.tap])
        assert torch.equal(_bits(tot[0]), _bits(want)), f"{c.name}: total of taps 0 .. {c.tap}"
    _report(f"head C={C} err / mag, over the bar", worst, 1.0)


# ------------------------------------------------------------------------------------------------------- softmax
@pytest.fixture(scope="module")
def softmaxes():
    return Q.softmax_cases(DEV)


@pytest.mark.parametrize("N", Q.SM_N)
def test_softmax_rows(softmaxes, N):
    worst = 0.0
    for c in softmaxes:
        if c.N != N:
            continue
        y = Out(c.rows, N, c.ldy, torch.float32)
        launch = lambda: _cabi.call("omt_softmax_rows", c.xbuf, c.ldx, c.rows, N, y.ptr, c.ldy)
        got, = _launch_twice(launch, (y,), (c.xbuf,))
        ok, w, msg = Q.softmax_check(c.x.cpu(), got)
        assert ok, f"{c.name}: {msg}"
        worst = max(worst, w)
    _report(f"softmax N={N} err / (2^-24 y64)", worst, Q.softmax_k(N))


# ------------------------------------------------------------------------------------------------------- IS reduction
@pytest.fixture(scope="module")
def iss():
    return Q.is_cases(DEV)


@pytest.mark.parametrize("N", Q.IS_N)
def test_inception_score(iss, N):
    worst = [0.0, 0.0]
    for c in iss:
        if c.N != N:
            continue
        cm, kl = Out(c.splits, N, N, torch.float64), Out(1, c.splits, c.splits, torch.float64)
        launch = lambda: _cabi.call("omt_inception_score", c.pbuf, c.ldp, N, c.n, c.splits, cm.ptr, kl.ptr)
        got_cm, got_kl = _launch_twice(launch, (cm, kl), (c.pbuf,))
        ok, e_cm, e_kl, msg = Q.is_check(c, got_cm, got_kl[0])
        assert ok, msg
        worst = [max(worst[0], e_cm), max(worst[1], e_kl)]
    _report(f"IS N={N} column means rel", worst[0], Q.IS_REL)
    _report(f"IS N={N} KL err / (|KL| + floor / 1e-12)", worst[1], Q.IS_REL)


@pytest.mark.parametrize("N", [6129, 6144])
def test_kl_shared_memory_past_48k_with_static_red(N):
    """Regression: the KL kernel's q[N] fp64 marginal plus its static red[16] exceed 48 KiB from N = 6129 on, which
    the launch refused ("invalid argument") until the kernel opted in to its dynamic shared memory."""
    p = Q.is_probs(3 * 17, N, N, DEV)
    c = Q.IsCase(f"N{N}", N, 17, 3, N, p)
    cm, kl = Out(3, N, N, torch.float64), Out(1, 3, 3, torch.float64)
    got_cm, got_kl = _launch_twice(lambda: _cabi.call("omt_inception_score", p, N, N, 17, 3, cm.ptr, kl.ptr),
                                   (cm, kl), (p,))
    ok, _, _, msg = Q.is_check(c, got_cm, got_kl[0])
    assert ok, msg


# ------------------------------------------------------------------------------------------------------- refusals
def _refused(name, outs, *args):
    n0 = _cabi.launch_count
    with pytest.raises(RuntimeError, match=f"{name}: "):
        _cabi.call(name, *args)
    torch.cuda.synchronize()
    assert _cabi.launch_count == n0, f"{name}: a refused call counted a launch"
    assert all(o.untouched() for o in outs), f"{name}: a refused call wrote its output"


def test_refusals_past_each_limit():
    """H or W of 10 (SSIM needs 11); N = 6145 (past the 48 KiB of fp64 marginal) and 65536 splits; ldy < N; Cs < C and
    tap 5.  Every buffer is large enough for the call as if it were accepted."""
    a = torch.zeros(1, 11, 11, 3, dtype=torch.uint8, device=DEV)
    lut = Q.byte_tables()[0].to(DEV)
    taps = torch.from_numpy(Q.TAPS).to(DEV)
    sse, ssim = Out(1, 1, 1, torch.float64), Out(1, 1, 1, torch.float64)
    for H, W in ((10, 11), (11, 10)):
        _refused("omt_psnr_ssim", (sse, ssim), a, lut, None, a, lut, None, quality.FORM_U8, 1, H, W, taps, sse.ptr,
                 ssim.ptr)
    for N, splits in ((6145, 1), (7, 65536)):
        p = torch.full((splits, N), 1.0 / N, device=DEV)
        cm, kl = Out(splits, N, N, torch.float64), Out(1, splits, splits, torch.float64)
        _refused("omt_inception_score", (cm, kl), p, N, N, 1, splits, cm.ptr, kl.ptr)
    x = torch.zeros(2, 32, device=DEV)
    y = Out(2, 32, 32, torch.float32)
    _refused("omt_softmax_rows", (y,), x, 32, 2, 32, y.ptr, 31)
    x = torch.ones(2, 3, 3, 8, device=DEV)
    lin = torch.ones(8, device=DEV)
    t, tot = Out(6, 1, 1, torch.float32), Out(1, 1, 1, torch.float32)
    _refused("omt_lpips_head", (t, tot), x, 7, 8, 1, 3, 3, lin, 0, t.ptr, tot.ptr)
    _refused("omt_lpips_head", (t, tot), x, 8, 8, 1, 3, 3, lin, 5, t.ptr, tot.ptr)
