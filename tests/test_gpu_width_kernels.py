"""The kernel instantiations and shapes that model widths other than 512 reach, against float64 references in sentinel-filled
buffers with guards (the helpers of test_gpu_rowwise.py and test_gpu_gemm_walk.py, unchanged):

* layernorm_kernel<6, true> (C = 768) and <8, true> (C = 1024), the 16-byte plane-store forms, in fp32, 2^11-scaled and
  row-scaled planes, with a row map and in place; where the planes are only 8-byte aligned, <8, false> as before;
* post_vq_wide_kernel (C in (512, 1024]) in its three source forms;
* PEG (v4 and v3, bit-identical) at C = 256, 768 and 1024;
* the QKV GEMM with the attention width A apart from the model width C: q | k | v = [0, A) | [A, 2A) | [2A, 3A), the
  dual-A switch at n = A (a multiple of 128, not always of 256), rope + l2norm + scale head by head, in the fp32 and the
  operand-plane epilogue, on exact-grid operands.

Which kernel ran is read from the profiler, so a host that picked another instantiation fails here.
"""
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import tests.test_gpu_gemm_walk as GW
import tests.test_gpu_rowwise as G
from tests import rowwise_cases as R

pytestmark = pytest.mark.gpu


def _kernels(fn):
    """Names of the CUDA kernels fn launches (the second of two profiled calls: the first session of a process can miss
    kernels while the profiler starts up)."""
    for _ in range(2):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
    return {e.name for e in prof.events() if e.device_type.name == "CUDA" and "omt::" in e.name}


def _ran(names, what):
    hits = [n for n in names if what in n]
    assert hits, f"{what} did not run; launched: {sorted(names)}"


def ln_instantiation_wide(C, lds=0, plane_align=16):
    """(NV, PAIR) of layernorm_kernel as layernorm_impl picks it with the paired forms of C = 768 and 1024: PAIR when C is
    a multiple of 256 (NV = C / 128), the plane leading dimension a multiple of 8 and every plane pointer 16-byte aligned;
    otherwise NV 1, 2, 3, 4, or 8 for anything larger, as before."""
    nv = (C // 4 + 31) // 32
    pair = C % 256 == 0 and lds % 8 == 0 and plane_align % 16 == 0
    if nv in (2, 4) or (nv in (6, 8) and pair):
        return nv, pair
    return (nv, False) if nv in (1, 3) else (8, False)


# (C, M, ldx, lds, plane byte offset, (NV, PAIR) of the fp32-only call, of the plane-writing calls)
LN_WIDE = [
    (768, 65, 768, 768, 0, (6, True), (6, True)),
    (768, 131, 772, 776, 0, (6, True), (6, True)),
    (768, 50, 768, 768, 8, (6, True), (8, False)),             # planes only 8-byte aligned
    (1024, 203, 1028, 1024, 0, (8, True), (8, True)),
    (1024, 77, 1024, 1032, 8, (8, True), (8, False)),
]


@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("case", LN_WIDE, ids=R.ln_case_id)
def test_layernorm_paired_wide(cuda, case, bias, monkeypatch):
    monkeypatch.setattr(R, "ln_instantiation", ln_instantiation_wide)
    G.test_layernorm(cuda, case, bias)
    C, M, ldx, lds, off, inst32, inst_pl = case
    x = G._padded(R.family_rows(M, C, 7 + C), ldx, cuda)
    g, b = (t.to(cuda) for t in R.ln_params(C, 8 + C))
    y = G.Buf(M, C, C, cuda)
    _ran(_kernels(lambda: G._ln(x, ldx, y.ptr, C, g, b, M, C)), f"layernorm_kernel<{inst32[0]}, {str(inst32[1]).lower()}>")
    yp = G._plane_set(M, C, lds, off, cuda, True)
    _ran(_kernels(lambda: G._ln(x, ldx, None, 0, g, b, M, C, yp=yp, lds=lds)),
         f"layernorm_kernel<{inst_pl[0]}, {str(inst_pl[1]).lower()}>")


@pytest.mark.parametrize("case", LN_WIDE, ids=R.ln_case_id)
def test_layernorm_paired_wide_row_map_and_in_place(cuda, case):
    G.test_layernorm_row_map_and_in_place(cuda, case)


@pytest.mark.parametrize("C", [768, 1024])
@pytest.mark.parametrize("M", [1, 33, 1000])
def test_post_vq_wide(cuda, M, C):
    G.test_post_vq(cuda, M, C)


@pytest.mark.parametrize("C,kernel", [(512, "post_vq_kernel<8>"), (516, "post_vq_wide_kernel<8>"),
                                      (768, "post_vq_wide_kernel<8>"), (1024, "post_vq_wide_kernel<8>")])
def test_post_vq_kernel_choice(cuda, C, kernel):
    M = 40
    E, W, b = torch.randn(64, 8, device=cuda), torch.randn(C, 8, device=cuda), torch.randn(C, device=cuda)
    idx = torch.arange(M, device=cuda) % 64
    X = torch.empty(M, C, device=cuda)
    names = _kernels(lambda: G._cabi().call("omt_post_vq", idx, E, None, None, None, W, b, X, M, C, 8))
    _ran(names, kernel)
    if kernel.startswith("post_vq_kernel"):
        assert not [n for n in names if "post_vq_wide" in n]
    torch.testing.assert_close(X, E[idx] @ W.t() + b, rtol=1e-5, atol=1e-5)


def test_post_vq_rejects_past_1024(cuda):
    X = torch.empty(4, 1028, device=cuda)
    W, b = torch.zeros(1028, 8, device=cuda), torch.zeros(1028, device=cuda)
    zc = torch.zeros(4, 8, device=cuda)
    with pytest.raises(RuntimeError, match="omt_post_vq: C=1028"):
        G._cabi().call("omt_post_vq", None, None, zc, None, None, W, b, X, 4, 1028, 8)


# (w, T', C, h): token rows of the geometry table at the model widths; a few token rows, a partial last row block
PEG_WIDE = [(w, T, C, h) for C in (256, 768, 1024) for (w, T, h) in ((64, 5, 3), (40, 9, 5), (128, 2, 3))]


@pytest.mark.parametrize("case", PEG_WIDE, ids=G._peg_id)
def test_peg_wide(cuda, case):
    G.test_peg_geometry(cuda, case)


# (A, C): attention width apart from the model width -- A > C, A < C, A = C = 768 (switch at a multiple of 128 only),
# 6 heads (A = 384) and 2 heads (A = 128) at C = 1024
QKV_WIDTHS = [(512, 256), (256, 512), (768, 768), (384, 512), (128, 1024)]


@pytest.mark.parametrize("planes", [False, True], ids=["qkv", "planes"])
@pytest.mark.parametrize("rope", [True, False], ids=["rope", "norope"])
@pytest.mark.parametrize("A,C", QKV_WIDTHS, ids=[f"A{a}-C{c}" for a, c in QKV_WIDTHS])
def test_qkv_epilogue_attention_width(cuda, A, C, rope, planes, monkeypatch):
    """N = 3A output columns over K = C: q from the first A matrix, k | v from the second from column A on."""
    monkeypatch.setattr(GW, "_qkv_layout", lambda N: (2 * A, A))
    N = 3 * A
    T = 3 * (N // 128)          # three 128-row blocks, the last one partial
    M, n = GW._case_qkv(GW._cabi(), cuda, T, C, [N], 77, dict(tokens=96), rope, planes)
    assert (M, n) == (2 * 128 + 77, N)
