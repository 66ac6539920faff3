"""GPU op-level parity of the f16x3 path: the kind::f16 GEMM on fp16 hi / lo operand planes (omt_linear_h) and
every producer that writes planes (LayerNorm, patch gather, the three attention cores, the GEGLU epilogue), against
fp64 torch on the same inputs.  Tolerance: fp32 round-off class (2e-5 on |A.W| ~ 1), the same bar as 3xTF32."""

import pytest
import torch

from oracle import omni_oracle as oo

pytestmark = pytest.mark.gpu

def _cabi():
    from omnitokenizer_b200 import _cabi
    _cabi.load()
    return _cabi


def _rand(shape, seed, scale=1.0):
    return (torch.rand(shape, generator=torch.Generator().manual_seed(seed)) - 0.5) * 2 * scale


def _planes(t, dev, pad_rows=0):
    from omnitokenizer_b200 import layout as L
    if pad_rows:
        t = L.pad_rows(t, pad_rows)
    hi, lo = L.split_f16(t)
    return hi.to(dev), lo.to(dev)


def _join(hi, lo):
    """fp32 value the planes stand for."""
    from omnitokenizer_b200 import layout as L
    return L.join_f16(hi.cpu(), lo.cpu())


# the last five: partial last m / n blocks, and 133 to 268 tiles so the persistent CTAs walk two or three tiles each
@pytest.mark.parametrize("M,N,K", [(64, 512, 512), (320, 192, 512), (1024, 1024, 768), (4160, 2816, 512), (192, 512, 192),
                                   (127, 96, 64), (200, 544, 192), (2305, 896, 1408), (8449, 512, 128),
                                   (16896, 192, 256)])
def test_linear_h_plain_bias_residual(cuda, M, N, K):
    cabi = _cabi()
    A, Wt, b, R = _rand((M, K), 1), _rand((N, K), 2, 0.05), _rand((N,), 3), _rand((M, N), 4)
    ref = (A.double() @ Wt.double().t() + b.double() + R.double()).float()
    ah, al = _planes(A, cuda)
    wh, wl = _planes(Wt, cuda, 256)
    out = torch.full((M, N), float("nan"), device=cuda)
    cabi.linear_h(a_hi=ah, a_lo=al, lda=K, w_hi=wh, w_lo=wl, c=out, ldc=N, M=M, N=N, K=K, bias=b.to(cuda),
                  residual=R.to(cuda), ldr=N, epilogue=cabi.EPI_NONE)
    torch.cuda.synchronize()
    err = (out.cpu() - ref).abs().max().item()
    assert err < 2e-5, f"f16x3 M{M} N{N} K{K}: max err {err:.3e}"
    # in-place residual (C aliases the residual, as every out-projection / FF2 call does)
    X = R.to(cuda).clone()
    cabi.linear_h(a_hi=ah, a_lo=al, lda=K, w_hi=wh, w_lo=wl, c=X, ldc=N, M=M, N=N, K=K, bias=b.to(cuda), residual=X,
                  ldr=N, epilogue=cabi.EPI_NONE)
    assert torch.equal(X, out)


@pytest.mark.parametrize("part", ["geglu_ff2", "rowmaps"])
def test_linear_h_geglu_and_rowmaps(cuda, part):
    cabi = _cabi()
    from omnitokenizer_b200 import layout as L
    if part == "rowmaps":
        _rowmaps(cabi, cuda)
        return
    M, K, inner = 320, 512, 1365
    ku = L.round_up(inner, 64)
    A, W1 = _rand((M, K), 5), _rand((2 * inner, K), 6, 0.05)
    y = A.double() @ W1.double().t()
    ref = (oo.gelu_erf(y[:, inner:]) * y[:, :inner]).float()
    ah, al = _planes(A, cuda)
    wh, wl = _planes(L.pack_geglu(W1, inner, ku), cuda, 256)
    U = torch.full((2, M, ku), -1, dtype=torch.int16, device=cuda)
    cabi.linear_h(a_hi=ah, a_lo=al, lda=K, w_hi=wh, w_lo=wl, u_hi=U[0], u_lo=U[1], ldu=ku, M=M, N=2 * ku, K=K,
                  epilogue=cabi.EPI_GEGLU)
    torch.cuda.synchronize()
    got = _join(U[0], U[1])
    assert (got[:, :inner] - ref).abs().max().item() < 2e-5
    assert torch.count_nonzero(U[:, :, inner:]).item() == 0          # zero padding columns are exact zeros in both planes
    # second FF GEMM straight from the planes (K = ku, zero-padded)
    W2 = _rand((512, inner), 16, 0.05)
    w2h, w2l = _planes(L.pad_cols(W2, ku), cuda, 256)
    X = torch.empty(M, 512, device=cuda)
    cabi.linear_h(a_hi=U[0], a_lo=U[1], lda=ku, w_hi=w2h, w_lo=w2l, c=X, ldc=512, M=M, N=512, K=ku, epilogue=cabi.EPI_NONE)
    assert (X.cpu() - (ref.double() @ W2.double().t()).float()).abs().max().item() < 2e-5


def _rowmaps(cabi, cuda):
    """Row maps: logical rows gather from / scatter into the canonical buffer (first-frame / rest-frames)."""
    B, T, N, Kp = 2, 3, 64, 192
    Xc = _rand((B * T * N, 512), 7)
    xh, xl = _planes(Xc, cuda)
    Wt = _rand((Kp, 512), 8, 0.05)
    wqh, wql = _planes(Wt, cuda, 256)
    rows = B * (T - 1) * N
    P = torch.full((rows, Kp), float("nan"), device=cuda)
    cabi.linear_h(a_hi=xh, a_lo=xl, lda=512, a_seg=(T - 1) * N, a_seg_stride=T * N, a_seg_off=N, w_hi=wqh, w_lo=wql,
                  c=P, ldc=Kp, M=rows, N=Kp, K=512, epilogue=cabi.EPI_NONE)
    sel = Xc.view(B, T, N, 512)[:, 1:].reshape(rows, 512)
    assert (P.cpu() - (sel.double() @ Wt.double().t()).float()).abs().max().item() < 2e-5
    Xo = torch.zeros(B * T * N, 512, device=cuda)
    Wb = _rand((512, Kp), 9, 0.05)
    wbh, wbl = _planes(Wb, cuda, 256)
    ph, pl = _planes(P.cpu(), cuda)
    cabi.linear_h(a_hi=ph, a_lo=pl, lda=Kp, w_hi=wbh, w_lo=wbl, c=Xo, ldc=512, c_seg=(T - 1) * N, c_seg_stride=T * N,
                  c_seg_off=N, M=rows, N=512, K=Kp, epilogue=cabi.EPI_NONE)
    want = torch.zeros(B, T, N, 512)
    want[:, 1:] = (P.cpu().double() @ Wb.double().t()).float().view(B, T - 1, N, 512)
    assert (Xo.cpu().view(B, T, N, 512) - want).abs().max().item() < 2e-5


@pytest.mark.parametrize("epilogue", ["qkv_rope", "qkv", "plain"])
def test_linear_h_dual_a_qkv(cuda, epilogue):
    """q from LN(x), k/v from raw x in one launch (attention.py:407-412), rope + l2norm + scale in the epilogue."""
    cabi = _cabi()
    from omnitokenizer_b200 import layout as L
    M, K, N = 640, 512, 128
    A1, A2, Wt = _rand((M, K), 70), _rand((M, K), 71), _rand((1536, K), 72, 0.05)
    ref = torch.cat([A1.double() @ Wt[:512].double().t(), A2.double() @ Wt[512:].double().t()], dim=1).float()
    a1h, a1l = _planes(A1, cuda)
    a2h, a2l = _planes(A2, cuda)
    wh, wl = _planes(Wt, cuda, 256)
    qs, ks = _rand((64,), 73, 0.5) + 1.0, _rand((64,), 74, 0.5) + 1.0
    cos, sin = L.rope_tables(N, 64)
    out = torch.empty(M, 1536, device=cuda)
    if epilogue != "plain":
        tables = (cos, sin) if epilogue == "qkv_rope" else (None, None)
        out.fill_(float("nan"))
        cabi.linear_h(a_hi=a1h, a_lo=a1l, a2_hi=a2h, a2_lo=a2l, n_split=512, lda=K, w_hi=wh, w_lo=wl, c=out, ldc=1536,
                      M=M, N=1536, K=K, epilogue=cabi.EPI_QKV, q_scale=qs.to(cuda), k_scale=ks.to(cuda),
                      rope_cos=None if tables[0] is None else tables[0].to(cuda),
                      rope_sin=None if tables[1] is None else tables[1].to(cuda), qk_cols=1024, tokens=N)
        got = out.cpu()
        for sl, sc in ((slice(0, 512), qs), (slice(512, 1024), ks)):
            t = ref[:, sl].reshape(M // N, N, 8, 64)
            if tables[0] is not None:
                t = oo.apply_rope(t, cos, sin)
            want = (oo.l2norm(t) * sc).reshape(M, 512)
            assert (got[:, sl] - want).abs().max().item() < 2e-5
        assert (got[:, 1024:] - ref[:, 1024:]).abs().max().item() < 2e-5
        return
    # plain dual-A form (window qkv uses the plain epilogue)
    out.fill_(float("nan"))
    cabi.linear_h(a_hi=a1h, a_lo=a1l, a2_hi=a2h, a2_lo=a2l, n_split=512, lda=K, w_hi=wh, w_lo=wl, c=out, ldc=1536,
                  M=M, N=1536, K=K, epilogue=cabi.EPI_NONE)
    assert (out.cpu() - ref).abs().max().item() < 2e-5


@pytest.mark.parametrize("form", ["two_acc", "row_scaled"])
@pytest.mark.parametrize("M,N,K", [(20480, 1024, 1408), (5120, 512, 512), (40960, 512, 512)])
def test_linear_h_multiwave_deterministic(cuda, M, N, K, form):
    """Many tiles per persistent CTA (up to 10 on 132 SMs), in the two-accumulator (cooperative) and the row-scaled
    (ping-pong) forms: the same bits run after run, and the first / last rows are right."""
    cabi = _cabi()
    from omnitokenizer_b200 import layout as L
    A = (torch.rand((M, K), device=cuda, generator=torch.Generator(device=cuda).manual_seed(31)) - 0.5)
    W = (torch.rand((N, K), device=cuda, generator=torch.Generator(device=cuda).manual_seed(32)) - 0.5) * 0.05
    R = (torch.rand((M, N), device=cuda, generator=torch.Generator(device=cuda).manual_seed(33)) - 0.5)
    if form == "row_scaled":
        ah, al, ars = L.split_rows_rs(A)
        wh, wl, wsc = L.split_f16_rs(L.pad_rows(W, 256))
        scales = dict(a_rs=ars, w_scale=wsc)
    else:
        ah, al = L.split_f16(A)
        wh, wl = L.split_f16(L.pad_rows(W, 256))
        scales = {}
    outs = []
    for _ in range(4):
        out = torch.full((M, N), float("nan"), device=cuda)
        cabi.linear_h(a_hi=ah, a_lo=al, lda=K, w_hi=wh, w_lo=wl, c=out, ldc=N, M=M, N=N, K=K, residual=R, ldr=N,
                      epilogue=cabi.EPI_NONE, **scales)
        outs.append(out)
    torch.cuda.synchronize()
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    for sl in (slice(0, 256), slice(M - 256, M)):
        ref = (A[sl].double() @ W.double().t() + R[sl].double()).float()
        assert (outs[0][sl] - ref).abs().max().item() < 2e-5
    assert not torch.isnan(outs[0]).any()


def test_plane_producers(cuda):
    """LayerNorm (+ raw-row planes), patch gather and the attention cores write planes that stand for the same fp32 values
    their fp32 forms produce (within the split's 2^-22 relative representation error)."""
    cabi = _cabi()
    from omnitokenizer_b200 import layout as L
    M = 320
    x = _rand((M, 512), 10, 3.0)
    g, b = _rand((512,), 11) + 1.0, _rand((512,), 12)
    y = torch.empty(M, 512, device=cuda)
    cabi.call("omt_layernorm", x.to(cuda), 512, y, 512, g.to(cuda), b.to(cuda), M, 512, 1e-5, 0, 0, 0)
    yp = torch.zeros(2, M, 512, dtype=torch.int16, device=cuda)
    xp = torch.zeros(2, M, 512, dtype=torch.int16, device=cuda)
    y2 = torch.empty(M, 512, device=cuda)
    cabi.call("omt_layernorm_h", x.to(cuda), 512, y2, 512, yp[0], yp[1], None, xp[0], xp[1], None, 512, g.to(cuda), b.to(cuda),
              M, 512, 1e-5, 0, 0, 0)
    d = (y - y2).abs()
    assert torch.equal(y, y2), f"fp32 output differs between the two entry points: max {d.max().item():.3e}, {int((d > 0).sum())} elements"
    tol = lambda t: 2.0 ** -21 * t.abs().max().item()
    assert (_join(yp[0], yp[1]) - y.cpu()).abs().max().item() <= tol(y.cpu())
    assert (_join(xp[0], xp[1]) - x).abs().max().item() <= tol(x)
    cabi.call("omt_layernorm_h", x.to(cuda), 512, None, 0, yp[0], yp[1], None, None, None, None, 512, g.to(cuda), b.to(cuda),
              M, 512, 1e-5, 0, 0, 0)                             # planes only
    assert (_join(yp[0], yp[1]) - y.cpu()).abs().max().item() <= tol(y.cpu())
    # row-scaled form: hi + lo (unscaled) times the inverse row scale; the scale puts the row maximum in [2^14, 2^15)
    yrs, xrs = torch.zeros(M, device=cuda), torch.zeros(M, device=cuda)
    cabi.call("omt_layernorm_h", x.to(cuda), 512, None, 0, yp[0], yp[1], yrs, xp[0], xp[1], xrs, 512, g.to(cuda), b.to(cuda),
              M, 512, 1e-5, 0, 0, 0)
    for pl, rs, want in ((yp, yrs, y.cpu()), (xp, xrs, x)):
        hi, lo = pl[0].cpu().view(torch.float16).float(), pl[1].cpu().view(torch.float16).float()
        got = (hi + lo) * rs.cpu()[:, None]
        assert ((got - want).abs() <= 2.0 ** -22 * want.abs().amax(dim=1, keepdim=True)).all()
        top = hi.abs().amax(dim=1)
        assert (top >= 2.0 ** 14).all() and (top <= 2.0 ** 15).all()
        h2, l2, inv2 = L.split_rows_rs(want)                      # the host twin agrees bit for bit
        assert torch.equal(inv2, rs.cpu()) and torch.equal(h2.float(), hi) and torch.equal(l2.float(), lo)
    # patch gather
    shape = (2, 3, 5, 64, 64)
    v = _rand(shape, 13, 0.5)
    for is_first, K, rows in ((1, 192, 2 * 64), (0, 768, 2 * 64)):
        lw, lb = _rand((K,), 14) + 1.0, _rand((K,), 15)
        A = torch.empty(rows, K, device=cuda)
        cabi.call("omt_patchify_ln", v.to(cuda), A, None, None, None, lw.to(cuda), lb.to(cuda), 2, 3, 5, 64, 64, 8, 4, is_first, 1e-5)
        Ap = torch.zeros(2, rows, K, dtype=torch.int16, device=cuda)
        cabi.call("omt_patchify_ln", v.to(cuda), None, Ap[0], Ap[1], None, lw.to(cuda), lb.to(cuda), 2, 3, 5, 64, 64, 8, 4,
                  is_first, 1e-5)
        assert (_join(Ap[0], Ap[1]) - A.cpu()).abs().max().item() <= tol(A.cpu())
        ars = torch.zeros(rows, device=cuda)
        cabi.call("omt_patchify_ln", v.to(cuda), None, Ap[0], Ap[1], ars, lw.to(cuda), lb.to(cuda), 2, 3, 5, 64, 64, 8, 4,
                  is_first, 1e-5)
        got = (Ap[0].cpu().view(torch.float16).float() + Ap[1].cpu().view(torch.float16).float()) * ars.cpu()[:, None]
        assert ((got - A.cpu()).abs() <= 2.0 ** -22 * A.cpu().abs().amax(dim=1, keepdim=True)).all()
    # attention cores
    nseq, N = 2, 256
    Ma = nseq * N
    qkv = torch.cat([_rand((Ma, 512), 30, 0.2), _rand((Ma, 512), 31, 0.2), _rand((Ma, 512), 32)], dim=1).contiguous().to(cuda)
    p = qkv.data_ptr()
    o = torch.empty(Ma, 512, device=cuda)
    op = torch.zeros(2, Ma, 512, dtype=torch.int16, device=cuda)
    for kern in (3, 1):
        cabi.set_option("attn_kernel", kern)
        cabi.call("omt_attn_spatial", p, 1536, p + 2048, 1536, p + 4096, 1536, o, None, None, 512, nseq, N, 8, 8.0)
        cabi.call("omt_attn_spatial", p, 1536, p + 2048, 1536, p + 4096, 1536, None, op[0], op[1], 512, nseq, N, 8, 8.0)
        assert (_join(op[0], op[1]) - o.cpu()).abs().max().item() <= tol(o.cpu())
    cabi.set_option("attn_kernel", 3)
    bias = _rand((8, 64, 64), 33).to(cuda)
    cabi.call("omt_attn_window", p, 1536, p + 2048, 1536, p + 4096, 1536, o, None, None, 512, bias, nseq, 16, 16, 8, 8, 0.125)
    cabi.call("omt_attn_window", p, 1536, p + 2048, 1536, p + 4096, 1536, None, op[0], op[1], 512, bias, nseq, 16, 16, 8, 8,
              0.125)
    assert (_join(op[0], op[1]) - o.cpu()).abs().max().item() <= tol(o.cpu())
    cabi.call("omt_attn_temporal", p, 1536, p + 2048, 1536, p + 4096, 1536, o, None, None, 512, 2, 4, 64, 8, 8.0, 1)
    cabi.call("omt_attn_temporal", p, 1536, p + 2048, 1536, p + 4096, 1536, None, op[0], op[1], 512, 2, 4, 64, 8, 8.0, 1)
    assert (_join(op[0], op[1]) - o.cpu()).abs().max().item() <= tol(o.cpu())


@pytest.mark.parametrize("M,N,K", [(64, 512, 512), (320, 192, 512), (1024, 1024, 768), (4160, 2816, 512), (192, 512, 192)])
def test_linear_h_row_scaled(cuda, M, N, K):
    """Single-accumulator form: row-scaled A planes (per-row power-of-two scale, unscaled lo) x per-matrix-scaled W planes,
    rows of very different magnitude in one call (1e-3 .. 1e3)."""
    cabi = _cabi()
    from omnitokenizer_b200 import layout as L
    A, Wt, b, R = _rand((M, K), 1), _rand((N, K), 2, 0.05), _rand((N,), 3), _rand((M, N), 4)
    A = A * torch.logspace(-3, 3, M)[:, None]
    ref = (A.double() @ Wt.double().t() + b.double() + R.double()).float()
    ah, al, ars = [t.to(cuda) for t in L.split_rows_rs(A)]
    wh, wl, wsc = L.split_f16_rs(L.pad_rows(Wt, 256))
    out = torch.full((M, N), float("nan"), device=cuda)
    cabi.linear_h(a_hi=ah, a_lo=al, a_rs=ars, w_scale=wsc, lda=K, w_hi=wh.to(cuda), w_lo=wl.to(cuda), c=out, ldc=N, M=M, N=N, K=K,
                  bias=b.to(cuda), residual=R.to(cuda), ldr=N, epilogue=cabi.EPI_NONE)
    torch.cuda.synchronize()
    scale = A.abs().amax(dim=1, keepdim=True).clamp_min(1.0)              # error bar relative to each row's magnitude
    err = ((out.cpu() - ref).abs() / scale).max().item()
    assert err < 2e-5, f"row-scaled f16x3 M{M} N{N} K{K}: max scaled err {err:.3e}"


def test_linear_h_row_scaled_epilogues(cuda):
    """Row-scaled form through the GEGLU and the dual-A QKV epilogues and the A row map (to_pixels reads X through one)."""
    cabi = _cabi()
    from omnitokenizer_b200 import layout as L
    M, K, inner = 320, 512, 1365
    ku = L.round_up(inner, 64)
    A, W1 = _rand((M, K), 5, 2.0), _rand((2 * inner, K), 6, 0.05)
    y = A.double() @ W1.double().t()
    ref = (oo.gelu_erf(y[:, inner:]) * y[:, :inner]).float()
    ah, al, ars = [t.to(cuda) for t in L.split_rows_rs(A)]
    wh, wl, wsc = L.split_f16_rs(L.pad_rows(L.pack_geglu(W1, inner, ku), 256))
    U = torch.full((2, M, ku), -1, dtype=torch.int16, device=cuda)
    cabi.linear_h(a_hi=ah, a_lo=al, a_rs=ars, w_scale=wsc, lda=K, w_hi=wh.to(cuda), w_lo=wl.to(cuda), u_hi=U[0], u_lo=U[1], ldu=ku,
                  M=M, N=2 * ku, K=K, epilogue=cabi.EPI_GEGLU)
    got = _join(U[0], U[1])
    assert (got[:, :inner] - ref).abs().max().item() < 4e-5 and torch.count_nonzero(U[:, :, inner:]).item() == 0
    # statically scaled U planes (unscaled lo) feeding the second FF GEMM in the single-accumulator form
    us = L.pow2_scale(float(ref.abs().max()) * 4.0)
    cabi.linear_h(a_hi=ah, a_lo=al, a_rs=ars, w_scale=wsc, lda=K, w_hi=wh.to(cuda), w_lo=wl.to(cuda), u_hi=U[0], u_lo=U[1], ldu=ku,
                  M=M, N=2 * ku, K=K, epilogue=cabi.EPI_GEGLU, u_scale=us)
    got = (U[0].cpu().view(torch.float16).float() + U[1].cpu().view(torch.float16).float()) / us
    assert (got[:, :inner] - ref).abs().max().item() < 4e-5
    W2 = _rand((512, inner), 16, 0.05)
    w2h, w2l, w2s = L.split_f16_rs(L.pad_rows(L.pad_cols(W2, ku), 256))
    X = torch.empty(M, 512, device=cuda)
    cabi.linear_h(a_hi=U[0], a_lo=U[1], a_rs_uniform=1.0 / us, w_scale=w2s, lda=ku, w_hi=w2h.to(cuda), w_lo=w2l.to(cuda), c=X, ldc=512,
                  M=M, N=512, K=ku, epilogue=cabi.EPI_NONE)
    assert (X.cpu() - (ref.double() @ W2.double().t()).float()).abs().max().item() < 4e-5
    # dual-A + rope / l2norm / scale
    Mq, N = 640, 128
    A1, A2, Wt = _rand((Mq, K), 70, 0.3), _rand((Mq, K), 71, 40.0), _rand((1536, K), 72, 0.05)
    ref = torch.cat([A1.double() @ Wt[:512].double().t(), A2.double() @ Wt[512:].double().t()], dim=1).float()
    a1 = [t.to(cuda) for t in L.split_rows_rs(A1)]
    a2 = [t.to(cuda) for t in L.split_rows_rs(A2)]
    wh, wl, wsc = L.split_f16_rs(L.pad_rows(Wt, 256))
    qs, ks = _rand((64,), 73, 0.5) + 1.0, _rand((64,), 74, 0.5) + 1.0
    cos, sin = L.rope_tables(N, 64)
    out = torch.full((Mq, 1536), float("nan"), device=cuda)
    cabi.linear_h(a_hi=a1[0], a_lo=a1[1], a_rs=a1[2], a2_hi=a2[0], a2_lo=a2[1], a2_rs=a2[2], w_scale=wsc, n_split=512, lda=K,
                  w_hi=wh.to(cuda), w_lo=wl.to(cuda), c=out, ldc=1536, M=Mq, N=1536, K=K, epilogue=cabi.EPI_QKV, q_scale=qs.to(cuda),
                  k_scale=ks.to(cuda), rope_cos=cos.to(cuda), rope_sin=sin.to(cuda), qk_cols=1024, tokens=N)
    got = out.cpu()
    for sl, sc in ((slice(0, 512), qs), (slice(512, 1024), ks)):
        want = (oo.l2norm(oo.apply_rope(ref[:, sl].reshape(Mq // N, N, 8, 64), cos, sin)) * sc).reshape(Mq, 512)
        assert (got[:, sl] - want).abs().max().item() < 2e-5
    assert ((got[:, 1024:] - ref[:, 1024:]).abs() / 40.0).max().item() < 2e-5
    # A row map: logical rows gather from the canonical buffer, the row scales follow the same map
    B, T, Nt, Kp = 2, 3, 64, 192
    Xc = _rand((B * T * Nt, 512), 7) * torch.logspace(-2, 2, B * T * Nt)[:, None]
    xh, xl, xrs = [t.to(cuda) for t in L.split_rows_rs(Xc)]
    Wp = _rand((Kp, 512), 8, 0.05)
    wh, wl, wsc = L.split_f16_rs(L.pad_rows(Wp, 256))
    rows = B * (T - 1) * Nt
    P = torch.full((rows, Kp), float("nan"), device=cuda)
    cabi.linear_h(a_hi=xh, a_lo=xl, a_rs=xrs, w_scale=wsc, lda=512, a_seg=(T - 1) * Nt, a_seg_stride=T * Nt, a_seg_off=Nt,
                  w_hi=wh.to(cuda), w_lo=wl.to(cuda), c=P, ldc=Kp, M=rows, N=Kp, K=512, epilogue=cabi.EPI_NONE)
    sel = Xc.view(B, T, Nt, 512)[:, 1:].reshape(rows, 512)
    want = (sel.double() @ Wp.double().t()).float()
    assert ((P.cpu() - want).abs() / sel.abs().amax(dim=1, keepdim=True).clamp_min(1.0)).max().item() < 2e-5


def _static_planes(x, ps):
    xs = x.float() * ps
    hi = xs.clamp(-65504, 65504).half()
    return hi, (xs - hi.float()).half()


@pytest.mark.parametrize("ctas", [1, 2])
@pytest.mark.parametrize("ramp", [False, True])
@pytest.mark.parametrize("N", [128, 256, 1024])
def test_attn_spatial_h(cuda, N, ramp, ctas):
    """wgmma f16 attention core on operand planes (V as MN-major B) vs fp64 softmax;
    q, k unit-norm x scale as the QKV epilogue leaves them, v rows of very different magnitude.  ramp: key norms grow
    along the sequence so that the row maxima keep rising from tile to tile -- the in-place rescale of the O accumulator
    (lazy running maximum) fires several times per row."""
    cabi = _cabi()
    cabi.set_option("attn_f16_ctas", ctas)           # both shapes of the kernel (conftest restores the default)
    from omnitokenizer_b200 import layout as L
    nseq, H = 3, 8
    M = nseq * N
    g = torch.Generator().manual_seed(40 + N)
    q = torch.nn.functional.normalize(torch.randn(M, H, 64, generator=g), dim=-1) * (torch.rand(64, generator=g) + 0.5)
    k = torch.nn.functional.normalize(torch.randn(M, H, 64, generator=g), dim=-1) * (torch.rand(64, generator=g) + 0.5)
    if ramp:
        k = k * (0.1 + 2.4 * (torch.arange(M) % N).float() / N)[:, None, None]
    v = torch.randn(M, H, 64, generator=g) * torch.logspace(-2, 2, M)[torch.randperm(M, generator=g)][:, None, None]
    qs, ks = L.pow2_scale(float(q.abs().max())), L.pow2_scale(float(k.abs().max()))
    qh, ql = _static_planes(q.reshape(M, 512), qs)
    kh, kl = _static_planes(k.reshape(M, 512), ks)
    vh, vl, vinv = L.split_rows_rs(v.reshape(M * H, 64))
    vh, vl, vinv = vh.reshape(M, 512), vl.reshape(M, 512), vinv.reshape(M, H).t().contiguous()
    dev = lambda t: t.contiguous().to(cuda)
    qh, ql, kh, kl, vh, vl, vinv = map(dev, (qh, ql, kh, kl, vh, vl, vinv))
    o = torch.full((M, 512), float("nan"), device=cuda)
    cabi.call("omt_attn_spatial_h", qh, ql, 512, kh, kl, 512, vh, vl, 512, vinv, qs * ks, o, None, None, 512, nseq, N, H, 8.0)
    torch.cuda.synchronize()
    qq, kk, vv = (t.view(nseq, N, H, 64).permute(0, 2, 1, 3).double() for t in (q, k, v))
    want = (torch.softmax((qq @ kk.transpose(-1, -2)) * 8.0, dim=-1) @ vv).permute(0, 2, 1, 3).reshape(M, 512).float()
    rel = ((o.cpu() - want).abs() / want.abs().amax(dim=1, keepdim=True).clamp_min(1e-3)).max().item()
    assert rel < 2e-5, f"f16 attention core N={N}: max error relative to the row magnitude {rel:.2e}"
    op = torch.zeros(2, M, 512, dtype=torch.int16, device=cuda)
    cabi.call("omt_attn_spatial_h", qh, ql, 512, kh, kl, 512, vh, vl, 512, vinv, qs * ks, None, op[0], op[1], 512, nseq, N, H, 8.0)
    assert (_join(op[0], op[1]) - o.cpu()).abs().max().item() <= 2.0 ** -21 * o.abs().max().item()


def test_linear_h_qkv_planes(cuda):
    """The QKV GEMM epilogue that feeds the f16 attention core: q / k planes with static power-of-two scales, v planes
    scaled per (row, head) with vinv -- reconstructed values vs the fp32-output epilogue of the same GEMM."""
    cabi = _cabi()
    from omnitokenizer_b200 import layout as L
    M, K, N = 640, 512, 128
    A1, A2, Wt = _rand((M, K), 70, 0.3), _rand((M, K), 71, 5.0), _rand((1536, K), 72, 0.05)
    A2 = A2 * torch.logspace(-2, 1, M)[:, None]
    a1 = [t.to(cuda) for t in L.split_rows_rs(A1)]
    a2 = [t.to(cuda) for t in L.split_rows_rs(A2)]
    wh, wl, wsc = L.split_f16_rs(L.pad_rows(Wt, 256))
    qsc, ksc = _rand((64,), 73, 0.5) + 1.0, _rand((64,), 74, 0.5) + 1.0
    cos, sin = L.rope_tables(N, 64)
    common = dict(a_hi=a1[0], a_lo=a1[1], a_rs=a1[2], a2_hi=a2[0], a2_lo=a2[1], a2_rs=a2[2], w_scale=wsc, n_split=512, lda=K,
                  w_hi=wh.to(cuda), w_lo=wl.to(cuda), M=M, N=1536, K=K, q_scale=qsc.to(cuda), k_scale=ksc.to(cuda),
                  rope_cos=cos.to(cuda), rope_sin=sin.to(cuda), qk_cols=1024, tokens=N)
    ref = torch.full((M, 1536), float("nan"), device=cuda)
    cabi.linear_h(c=ref, ldc=1536, epilogue=cabi.EPI_QKV, **common)
    P = torch.full((2, M, 1536), -1, dtype=torch.int16, device=cuda)
    vinv = torch.zeros(8, M, device=cuda)
    qps, kps = L.pow2_scale(float(qsc.abs().max())), L.pow2_scale(float(ksc.abs().max()))
    cabi.linear_h(u_hi=P[0], u_lo=P[1], ldu=1536, epilogue=cabi.EPI_QKV_PLANES, q_plane_scale=qps, k_plane_scale=kps, vinv=vinv,
                  **common)
    torch.cuda.synchronize()
    val = P[0].cpu().view(torch.float16).float() + P[1].cpu().view(torch.float16).float()
    ref = ref.cpu()
    assert (val[:, :512] / qps - ref[:, :512]).abs().max().item() <= 2.0 ** -21 * float(qsc.abs().max())
    assert (val[:, 512:1024] / kps - ref[:, 512:1024]).abs().max().item() <= 2.0 ** -21 * float(ksc.abs().max())
    vv = val[:, 1024:].view(M, 8, 64) * vinv.cpu().t()[:, :, None]
    rv = ref[:, 1024:].view(M, 8, 64)
    assert ((vv - rv).abs() <= 2.0 ** -21 * rv.abs().amax(dim=-1, keepdim=True)).all()
    top = P[0].cpu().view(torch.float16).float()[:, 1024:].view(M, 8, 64).abs().amax(dim=-1)
    assert (top >= 2.0 ** 14).all() and (top <= 2.0 ** 15).all()
