"""The fp32-operand GEMMs on exact operands (tests/gemm_fp32_cases.py), checked bit for bit.

* The 3xTF32 path of the persistent wgmma GEMM (omt_linear / omt_linear2 with MATH_3XTF32) on split-grid A: A carries a
  non-zero lo part, so each consumer warpgroup's shared-memory split writes non-zero A_lo values and the A_lo.W_hi wgmma
  adds non-zero products in every (64-row half, k-block) of every tile.  A wrong lo slot, the other warpgroup's half, a
  stale stage or a dropped correction product changes some output by at least 2^-12 (test_gemm_fp32_cases_cpu.py shows
  it for every case).  The walk covers T = 1 .. 3S + 1 tiles (S from the device), K = 32, 64 and 1408, tails of 1, 64
  and 127 rows, bias, residual (separate and in place), C and A row maps, dual-A and GEGLU; then the fused QKV epilogue.
* The CUDA-core fp32 GEMM (MATH_FP32) on operands whose full fp32 product is exact: M tails, N not a multiple of 128
  inside a wider ldc, small K, row maps whose segments are not multiples of 64, dual-A, residual and GEGLU; then the
  fp32 QKV path (the GEMM, then omt_qk_prep).

Every output sits in a sentinel-filled buffer with guard rows before and after it and guard columns past N; every guard
bit must survive, and three launches must give identical bits.  The GEGLU and q / k outputs go through fp32 gelu, rope
and l2norm and are held to the bounds of test_gpu_gemm_walk.py; each test prints its worst case against its bound.
"""
import pytest
import torch

from omnitokenizer_b200 import layout as L
from tests import gemm_fp32_cases as FC
from tests.test_gpu_gemm_walk import POST, PRE, SENT32, _check_guard, _f32_buf, _launch3


def _cabi():
    from omnitokenizer_b200 import _cabi
    _cabi.load()
    return _cabi


def _sms():
    return _cabi().device_info()[0]


def _args(m):
    return m.args if m is not None else (0, 0, 0)


def _out_buffer(cmap, cidx, M, cols, ldc, dev):
    """(sentinel buffer with PRE / POST guard rows, C view, mask of the written elements)."""
    crows = cmap.rows if cmap is not None else M
    cb = _f32_buf(PRE + crows + POST, ldc, dev)
    mask = torch.zeros(cb.shape, dtype=torch.bool, device=dev)
    mask[PRE + cidx, :cols] = True
    return cb, cb[PRE:], mask


def _check_plain(cb, C, cidx, mask, N, want, what):
    got = C[cidx, :N]
    assert not torch.isnan(got).any(), f"{what}: NaN left inside the output"
    bad = got != want
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.numel()} outputs differ from the exact result, first at "
                           f"{bad.nonzero()[0].tolist()}, max |diff| {(got - want).abs().max().item():.3e}")
    _check_guard(cb, mask, SENT32, what)


def _check_geglu(cb, C, cidx, mask, y, inner, ku, what):
    got = C[cidx, :ku].double()
    assert not torch.isnan(got).any(), f"{what}: NaN left inside the output"
    want, tol = FC.geglu_ref(y)
    ratio = ((got[:, :inner] - want[:, :inner]).abs() / tol[:, :inner].clamp_min(1e-300)).max().item()
    print(f"{what}: GEGLU max |err| / bound = {ratio:.3f}")
    assert ((got[:, :inner] - want[:, :inner]).abs() <= tol[:, :inner]).all(), f"{what}: GEGLU off by {ratio:.2f} x its bound"
    assert torch.count_nonzero(got[:, inner:]).item() == 0, f"{what}: padding columns are not exact zeros"
    _check_guard(cb, mask, SENT32, what)


# ---- 1. the 3xTF32 tile walk ----------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(FC.TF32_WALK)), ids=[c.id for c in FC.TF32_WALK])
def test_tf32_walk(cuda, i):
    cabi = _cabi()
    c = FC.TF32_WALK[i]
    S = _sms()
    p = FC.walk_problem(c, S, FC.walk_seed(i))
    M, N, K = p.M, p.N, p.K
    assert ((M + 127) // 128) * ((N + 127) // 128) == FC.T_KEYS[c.t](S)
    A = p.A.to(cuda)
    A2 = None if p.A2 is None else p.A2.to(cuda)
    wh, wl = (L.pad_rows(t, 128).to(cuda) for t in (p.w_hi, p.w_lo))
    bias = None if p.bias is None else p.bias.to(cuda)
    cidx = p.cidx(cuda)
    y = FC.walk_y(p, dev=cuda)
    aseg, astr, aoff = _args(p.amap)
    cseg, cstr, coff = _args(p.cmap)
    epi = cabi.EPI_GEGLU if p.inner else cabi.EPI_NONE
    cols = N // 2 if p.inner else N
    ldc = cols + 12
    cb, C, mask = _out_buffer(p.cmap, cidx, M, cols, ldc, cuda)
    res_vals = None if p.res is None else p.res.to(cuda)
    res, ldr = None, 0
    if c.res == "sep":
        res = torch.zeros(p.cmap.rows if p.cmap else M, N, device=cuda)
        res[cidx] = res_vals
        ldr = N
    elif c.res == "inplace":
        res, ldr = C, ldc

    def reset():
        cb.view(torch.int32).fill_(SENT32)
        if c.res == "inplace":
            C[cidx, :N] = res_vals

    if p.n_split:
        def launch():
            cabi.call("omt_linear2", A, A2, p.n_split, K, wh, wl, C, ldc, M, N, K, cabi.MATH_3XTF32, None, None, None,
                      None, 0, 0)
    else:
        def launch():
            cabi.call("omt_linear", A, K, aseg, astr, aoff, wh, wl, C, ldc, cseg, cstr, coff, M, N, K, bias, res, ldr,
                      epi, cabi.MATH_3XTF32)

    _launch3(launch, [cb], reset)
    if p.inner:
        _check_geglu(cb, C, cidx, mask, y, p.inner, cols, c.id)
    else:
        _check_plain(cb, C, cidx, mask, N, FC.plain_want(y, bias, res_vals), c.id)


# ---- 2. the 3xTF32 fused QKV epilogue -------------------------------------------------------------------------------

def _qkv_launch(cabi, p, A, A2, W, Wlo, C, ldc, M, math, qk=True):
    dev = C.device
    cos = None if p.cos is None else p.cos.to(dev)
    sin = None if p.sin is None else p.sin.to(dev)
    if qk:
        cabi.call("omt_linear2", A, A2, p.n_split, p.K, W, Wlo, C, ldc, M, p.N, p.K, math, p.qs.to(dev), p.ks.to(dev),
                  cos, sin, p.qk, p.tokens)
    else:
        cabi.call("omt_linear2", A, A2, p.n_split, p.K, W, Wlo, C, ldc, M, p.N, p.K, math, None, None, None, None, 0, 0)


def _check_qkv(p, got, z, what):
    """q / k within QK_TOL |scale_d| of fp64, v bit-exact; returns the worst q / k error over its bound."""
    assert not torch.isnan(got).any(), f"{what}: NaN left inside the output"
    want, tol = FC.qkv_ref(p, z)
    ratio = ((got[:, : p.qk].double() - want).abs() / tol).max().item()
    assert ratio <= 1.0, f"{what}: q / k off by {ratio:.2f} x the bound"
    v = z[:, p.qk:].float()
    bad = got[:, p.qk:] != v
    assert not bad.any(), f"{what}: {int(bad.sum())} v outputs are not exact, first at {bad.nonzero()[0].tolist()}"
    return ratio


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(FC.TF32_QKV)), ids=[c.id for c in FC.TF32_QKV])
def test_tf32_qkv(cuda, i):
    cabi = _cabi()
    c = FC.TF32_QKV[i]
    p = FC.qkv_problem(c, _sms(), FC.qkv_seed(i))
    M, N = p.M, p.N
    A = p.A.to(cuda)
    A2 = None if p.A2 is None else p.A2.to(cuda)
    wh, wl = (L.pad_rows(t, 128).to(cuda) for t in (p.w_hi, p.w_lo))
    z = FC.tf32_y(A, wh[:N], wl[:N], A2, p.n_split)
    ldc = N + 12
    cb = _f32_buf(PRE + M + POST, ldc, cuda)
    _launch3(lambda: _qkv_launch(cabi, p, A, A2, wh, wl, cb[PRE:], ldc, M, cabi.MATH_3XTF32), [cb],
             lambda: cb.view(torch.int32).fill_(SENT32))
    ratio = _check_qkv(p, cb[PRE: PRE + M, :N], z, c.id)
    print(f"{c.id}: 3xTF32 q / k max |err| / bound = {ratio:.3f}")
    mask = torch.zeros(cb.shape, dtype=torch.bool, device=cuda)
    mask[PRE: PRE + M, :N] = True
    _check_guard(cb, mask, SENT32, c.id)


@pytest.mark.gpu
@pytest.mark.parametrize("i", [0, 3, len(FC.TF32_QKV) - 2], ids=lambda i: FC.TF32_QKV[i].id)
def test_tf32_qkv_placement(cuda, i):
    """Rows shifted by a multiple of `tokens` (the rope position of row m is m % tokens) give identical bits: a row's
    result does not depend on which tile, half or warpgroup computes it."""
    cabi = _cabi()
    c = FC.TF32_QKV[i]
    p = FC.qkv_problem(c, _sms(), FC.qkv_seed(i))
    M, N = p.M, p.N
    A = p.A.to(cuda)
    A2 = None if p.A2 is None else p.A2.to(cuda)
    wh, wl = (L.pad_rows(t, 128).to(cuda) for t in (p.w_hi, p.w_lo))
    big = torch.full((M, N), float("nan"), device=cuda)
    _qkv_launch(cabi, p, A, A2, wh, wl, big, N, M, cabi.MATH_3XTF32)
    Mw = min(320, M // 2)
    shifts = sorted({p.tokens * j for j in (1, 2, (M - Mw) // p.tokens) if p.tokens * j + Mw <= M})
    assert shifts, "no shift fits"
    for r in shifts:
        small = torch.full((Mw, N), float("nan"), device=cuda)
        _qkv_launch(cabi, p, A[r: r + Mw], None if A2 is None else A2[r: r + Mw], wh, wl, small, N, Mw,
                    cabi.MATH_3XTF32)
        assert torch.equal(small, big[r: r + Mw]), f"rows shifted by {r}: max |diff| {(small - big[r: r + Mw]).abs().max():.3e}"


# ---- 3. the CUDA-core fp32 GEMM -------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(FC.FP32_CASES)), ids=[c.id for c in FC.FP32_CASES])
def test_fp32_exact(cuda, i):
    cabi = _cabi()
    c = FC.FP32_CASES[i]
    p = FC.fp32_problem(c, FC.fp32_seed(i))
    M, N, K = c.M, c.N, c.K
    lda = K + c.lda_extra
    A = p.A.to(cuda)
    A2 = None if p.A2 is None else p.A2.to(cuda)
    W = L.pad_rows(p.W, 128).to(cuda)
    bias = None if p.bias is None else p.bias.to(cuda)
    cidx = p.cidx(cuda)
    y = FC.fp32_case_y(p, dev=cuda)
    cols, ldc = c.out_cols, c.ldc
    cb, C, mask = _out_buffer(c.cmap, cidx, M, cols, ldc, cuda)
    res_vals = None if p.res is None else p.res.to(cuda)
    res, ldr = None, 0
    if c.res == "sep":
        ldr = N + 8
        res = torch.zeros(c.cmap.rows if c.cmap else M, ldr, device=cuda)
        res[cidx, :N] = res_vals
    elif c.res == "inplace":
        res, ldr = C, ldc

    def reset():
        cb.view(torch.int32).fill_(SENT32)
        if c.res == "inplace":
            C[cidx, :N] = res_vals

    if c.n_split:
        def launch():
            cabi.call("omt_linear2", A, A2, c.n_split, lda, W, None, C, ldc, M, N, K, cabi.MATH_FP32, None, None, None,
                      None, 0, 0)
    else:
        aseg, astr, aoff = _args(c.amap)
        cseg, cstr, coff = _args(c.cmap)
        epi = cabi.EPI_GEGLU if c.geglu else cabi.EPI_NONE

        def launch():
            cabi.call("omt_linear", A, lda, aseg, astr, aoff, W, None, C, ldc, cseg, cstr, coff, M, N, K, bias, res, ldr,
                      epi, cabi.MATH_FP32)

    _launch3(launch, [cb], reset)
    if c.geglu:
        _check_geglu(cb, C, cidx, mask, y, p.inner, cols, c.id)
    else:
        _check_plain(cb, C, cidx, mask, N, FC.plain_want(y, bias, res_vals), c.id)


# ---- 4. the fp32 QKV path -------------------------------------------------------------------------------------------

FP32_QKV = [FC.QkvCase("", 512, (1536,), 37, 96, True, (512, 512)),
            FC.QkvCase("", 512, (1536,), 100, 128, False, (512, 512)),
            FC.QkvCase("", 512, (768,), 1, 64, True, (256, 512)),
            FC.QkvCase("", 1024, (384,), 77, 1024, True, (128, 1024))]


@pytest.mark.gpu
@pytest.mark.parametrize("c", FP32_QKV, ids=[c.id for c in FP32_QKV])
def test_fp32_qkv(cuda, c):
    """omt_linear2 with q_scale under MATH_FP32 is the plain GEMM followed by omt_qk_prep, bit for bit, and within the
    q / k bound of fp64 (v exact)."""
    cabi = _cabi()
    p = FC.qkv_problem(c, _sms(), 4000 + FP32_QKV.index(c))
    M, N = p.M, p.N
    A = p.A.to(cuda)
    A2 = None if p.A2 is None else p.A2.to(cuda)
    Wt = FC.fp32_weight(N, p.K, 4100 + FP32_QKV.index(c))
    W = L.pad_rows(Wt, 128).to(cuda)
    z = FC.fp32_y(A, Wt.to(cuda), A2, p.n_split)
    ldc = N + 12
    cb = _f32_buf(PRE + M + POST, ldc, cuda)
    _launch3(lambda: _qkv_launch(cabi, p, A, A2, W, None, cb[PRE:], ldc, M, cabi.MATH_FP32), [cb],
             lambda: cb.view(torch.int32).fill_(SENT32))
    two = _f32_buf(PRE + M + POST, ldc, cuda)
    C2 = two[PRE:]
    _qkv_launch(cabi, p, A, A2, W, None, C2, ldc, M, cabi.MATH_FP32, qk=False)
    assert torch.equal(C2[:M, :N], z.float()), "the fp32 GEMM of the q | k | v columns is not exact"
    dev_tab = [None if t is None else t.to(cuda) for t in (p.cos, p.sin)]
    cabi.call("omt_qk_prep", C2, ldc, C2[:, p.qk // 2:], ldc, p.qs.to(cuda), p.ks.to(cuda), *dev_tab, M, p.tokens,
              p.qk // 128)
    torch.cuda.synchronize()
    assert torch.equal(cb.view(torch.int32), two.view(torch.int32)), "omt_linear2 differs from the GEMM + omt_qk_prep"
    ratio = _check_qkv(p, cb[PRE: PRE + M, :N], z, c.id)
    print(f"{c.id}: fp32 q / k max |err| / bound = {ratio:.3f}")
    mask = torch.zeros(cb.shape, dtype=torch.bool, device=cuda)
    mask[PRE: PRE + M, :N] = True
    _check_guard(cb, mask, SENT32, c.id)


# ---- 5. argument checks ---------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_tf32_rejects_bad_arguments(cuda):
    """Each call raises before any launch: valid buffers, and the output keeps its sentinel bits."""
    cabi = _cabi()
    M, N, K = 192, 256, 96
    A = FC.grid_a(M, K, 5000).to(cuda)
    wh, wl = (t.to(cuda) for t in FC.tf32_weight(N, K, 5001))
    cb = _f32_buf(M, N, cuda)
    T3 = cabi.MATH_3XTF32
    bad = [
        ("K=40", "multiple of 32", lambda: cabi.call("omt_linear", A, K, 0, 0, 0, wh, wl, cb, N, 0, 0, 0, M, N, 40,
                                                       None, None, 0, cabi.EPI_NONE, T3)),
        ("a_seg=96", "segment", lambda: cabi.call("omt_linear", A, K, 96, 96, 0, wh, wl, cb, N, 0, 0, 0, M, N, K, None,
                                                  None, 0, cabi.EPI_NONE, T3)),
        ("a_seg=128, M=192", "segment", lambda: cabi.call("omt_linear", A, K, 128, 128, 0, wh, wl, cb, N, 0, 0, 0, M, N,
                                                          K, None, None, 0, cabi.EPI_NONE, T3)),
        ("n_split=64", "n_split", lambda: cabi.call("omt_linear2", A, A, 64, K, wh, wl, cb, N, M, N, K, T3, None, None,
                                                    None, None, 0, 0)),
    ]
    for what, msg, call in bad:
        with pytest.raises(RuntimeError, match=msg):
            call()
        torch.cuda.synchronize()
        assert (cb.view(torch.int32) == SENT32).all(), f"{what}: the output was written"
