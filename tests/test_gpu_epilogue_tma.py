"""The plane-writing f16 GEMM epilogues (GEGLU -> U planes, QKV -> q | k | v planes), which stage their planes in shared
memory and write them by TMA stores, checked bit for bit against kernels that do not go through that path.

* QKV planes: the fp32-output QKV epilogue runs the same rope / l2 norm / scale arithmetic on the same fragments and
  stores fp32 with per-thread stores, so the q / k planes must be exactly the host split of its output times the plane
  scale, and the v planes and vinv exactly the host row-scaled split of its v columns.  Cases: the dual-A split at
  A = 384 and 768, M not a multiple of 128, and rope positions that wrap past `tokens` inside a tile.
* GEGLU: a row-mapped C (32-row segments, so the 64-row halves straddle segments) must hold, row for row, the bits of
  the same launch without a row map.
Every output sits in a larger sentinel-filled buffer whose guard bands must keep their bits.
"""
import pytest
import torch

from omnitokenizer_b200 import layout as L

SENT16 = 0x7E5B
PRE, POST = 3, 5


def _cabi():
    from omnitokenizer_b200 import _cabi
    _cabi.load()
    return _cabi


def _rand(shape, seed, dev):
    return torch.rand(shape, generator=torch.Generator(device=dev).manual_seed(seed), device=dev) - 0.5


def _split_pow2(x):
    """fp16 hi / lo planes of x (already multiplied by its power-of-two scale), as the kernel's split2u forms them."""
    hi = x.half()
    lo = (x - hi.float()).half()
    return hi.view(torch.int16), lo.view(torch.int16)


@pytest.mark.gpu
@pytest.mark.parametrize("A,M,tokens", [(384, 1000, 64), (768, 680, 96), (512, 1088, 1024)])
def test_qkv_planes_match_fp32_epilogue(cuda, A, M, tokens):
    cabi = _cabi()
    dev, K, N = cuda, 512, 3 * A
    ah, al, ars = L.split_rows_rs(_rand((M, K), 1, dev))
    a2h, a2l, a2rs = L.split_rows_rs(_rand((M, K), 2, dev))
    wh, wl, wsc = L.split_f16_rs(L.pad_rows(_rand((N, K), 3, dev) * 0.1, 256))
    g = torch.Generator(device=dev).manual_seed(4)
    qs, ks = 0.5 + torch.rand(64, generator=g, device=dev), 0.5 + torch.rand(64, generator=g, device=dev)
    cos, sin = (t.to(dev).contiguous() for t in L.rope_tables(tokens, 64))
    kw = dict(a_hi=ah, a_lo=al, a_rs=ars, a2_hi=a2h, a2_lo=a2l, a2_rs=a2rs, n_split=A, w_hi=wh, w_lo=wl, w_scale=wsc,
              lda=K, M=M, N=N, K=K, q_scale=qs, k_scale=ks, rope_cos=cos, rope_sin=sin, qk_cols=2 * A, tokens=tokens)
    C = torch.empty(M, N, device=dev)
    cabi.linear_h(c=C, ldc=N, epilogue=cabi.EPI_QKV, **kw)
    qps, kps = L.pow2_scale(float(qs.max())), L.pow2_scale(float(ks.max()))
    ldu, hv = N + 40, A // 64
    pb = torch.full((2, PRE + M + POST, ldu), SENT16, dtype=torch.int16, device=dev)
    vinv = torch.full((hv * M + 7,), float("nan"), device=dev)
    cabi.linear_h(u_hi=pb[0, PRE:], u_lo=pb[1, PRE:], ldu=ldu, epilogue=cabi.EPI_QKV_PLANES, q_plane_scale=qps,
                  k_plane_scale=kps, vinv=vinv, **kw)
    torch.cuda.synchronize()
    hi, lo = pb[0, PRE: PRE + M, :N], pb[1, PRE: PRE + M, :N]
    ps = torch.tensor([qps] * A + [kps] * A, device=dev)
    qh, ql = _split_pow2(C[:, : 2 * A] * ps)
    assert torch.equal(hi[:, : 2 * A], qh), "q / k hi plane differs from the fp32 epilogue's split"
    assert torch.equal(lo[:, : 2 * A], ql), "q / k lo plane differs from the fp32 epilogue's split"
    vh, vl, vi = L.split_rows_rs(C[:, 2 * A:].reshape(M * hv, 64))
    assert torch.equal(hi[:, 2 * A:], vh.view(torch.int16).reshape(M, A)), "v hi plane differs"
    assert torch.equal(lo[:, 2 * A:], vl.view(torch.int16).reshape(M, A)), "v lo plane differs"
    assert torch.equal(vinv[: hv * M].view(hv, M), vi.view(M, hv).t()), "vinv differs"
    assert vinv[hv * M:].isnan().all(), "vinv written past its end"
    mask = torch.zeros(pb.shape, dtype=torch.bool, device=dev)
    mask[:, PRE: PRE + M, :N] = True
    assert (pb[~mask] == SENT16).all(), "planes written outside [M, N]"


@pytest.mark.gpu
@pytest.mark.parametrize("h1", [False, True])
@pytest.mark.parametrize("M,seg,stride,off", [(40 * 32 + 0, 32, 48, 7), (1000, 0, 0, 0), (25 * 96, 96, 160, 3)])
def test_geglu_row_map(cuda, h1, M, seg, stride, off):
    cabi = _cabi()
    dev, K, inner = cuda, 256, 1365
    ku = L.round_up(inner, 64)
    N = 2 * ku
    ah, al, ars = L.split_rows_rs(_rand((M, K), 11, dev))
    W = L.pack_geglu(_rand((2 * inner, K), 12, dev) * 0.2, inner, ku)
    wh, wl, wsc = L.split_f16_rs(L.pad_rows(W, 256))
    kw = dict(a_hi=ah, a_rs=ars, w_hi=wh, w_scale=wsc, lda=K, M=M, N=N, K=K, epilogue=cabi.EPI_GEGLU)
    name = "omt_linear_h1" if h1 else "omt_linear_h"
    if not h1:
        kw.update(a_lo=al, w_lo=wl)
    ldu = ku + 24
    planes = 1 if h1 else 2

    def run(rows, **rm):
        ub = torch.full((2, PRE + rows + POST, ldu), SENT16, dtype=torch.int16, device=dev)
        cabi.linear_h(name, u_hi=ub[0, PRE:], u_lo=None if h1 else ub[1, PRE:], ldu=ldu, **rm, **kw)
        return ub

    ref = run(M)
    if seg > 0:
        rows = (M // seg - 1) * stride + off + seg
        ub = run(rows, c_seg=seg, c_seg_stride=stride, c_seg_off=off)
        r = torch.arange(M, device=dev)
        phys = (r // seg) * stride + off + r % seg
    else:
        ub, phys = ref, torch.arange(M, device=dev)
    torch.cuda.synchronize()
    assert not (ref[:planes, PRE: PRE + M, :ku].view(torch.float16).isnan().any()), "NaN left inside the U planes"
    assert torch.equal(ub[:planes, PRE + phys, :ku], ref[:planes, PRE: PRE + M, :ku]), "row-mapped U differs"
    mask = torch.zeros(ub.shape, dtype=torch.bool, device=dev)
    mask[:planes, PRE + phys, :ku] = True
    assert (ub[~mask] == SENT16).all(), "U planes written outside the mapped rows"
