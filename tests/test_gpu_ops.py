"""GPU op-level parity: every C-ABI kernel vs the oracle's restatement of the same reference op.
Tolerances are fp32 round-off (different summation order), written next to each check."""

import pytest
import torch

from oracle import omni_oracle as oo
from oracle import weights as W

pytestmark = pytest.mark.gpu


def _cabi():
    from omnitokenizer_b200 import _cabi
    _cabi.load()
    return _cabi


def _rand(shape, seed, scale=1.0):
    return (torch.rand(shape, generator=torch.Generator().manual_seed(seed)) - 0.5) * 2 * scale


def _pad128(w):
    from omnitokenizer_b200 import layout as L
    return L.pad_rows(w, 128)


@pytest.mark.parametrize("M,N,K", [(64, 512, 512), (320, 192, 512), (1024, 1024, 768), (200, 512, 192),
                                   (4160, 2752, 512)])
@pytest.mark.parametrize("math", ["fp32", "3xtf32"])
def test_linear_plain_bias_residual(cuda, M, N, K, math):
    cabi = _cabi()
    from omnitokenizer_b200 import layout as L
    # any M: the tensor-core path reads rows past M as zeros (TMA bounds) and stores only rows below M
    A, Wt, b, R = _rand((M, K), 1), _rand((N, K), 2, 0.05), _rand((N,), 3), _rand((M, N), 4)
    ref = (A.double() @ Wt.double().t() + b.double() + R.double()).float()
    Ad, bd, Rd = A.to(cuda), b.to(cuda), R.to(cuda)
    Wp = _pad128(Wt).to(cuda)
    mode = {"fp32": cabi.MATH_FP32, "3xtf32": cabi.MATH_3XTF32}[math]
    Wlo = None
    if math == "3xtf32":
        hi = L.tf32_round(Wp)
        Wlo, Wp = (Wp - hi).contiguous(), hi
    out = torch.full((M, N), float("nan"), device=cuda)
    cabi.call("omt_linear", Ad, K, 0, 0, 0, Wp, Wlo, out, N, 0, 0, 0, M, N, K, bd, Rd, N, cabi.EPI_NONE, mode)
    torch.cuda.synchronize()
    err = (out.cpu() - ref).abs().max().item()
    tol = 2e-5     # |A.W| ~ 1
    assert err < tol, f"{math} M{M} N{N} K{K}: max err {err:.3e}"


@pytest.mark.parametrize("math", ["fp32", "3xtf32"])
def test_linear_geglu_and_rowmaps(cuda, math):
    cabi = _cabi()
    from omnitokenizer_b200 import layout as L
    M, K, inner = 256, 512, 1365
    ku = L.round_up(inner, 32)
    A, W1 = _rand((M, K), 5), _rand((2 * inner, K), 6, 0.05)
    y = A.double() @ W1.double().t()
    ref = (oo.gelu_erf(y[:, inner:]) * y[:, :inner]).float()
    mode = cabi.MATH_FP32 if math == "fp32" else cabi.MATH_3XTF32
    Wp = _pad128(L.pack_geglu(W1, inner, ku)).to(cuda)
    Wlo = None
    if math == "3xtf32":
        hi = L.tf32_round(Wp)
        Wlo, Wp = (Wp - hi).contiguous(), hi
    U = torch.full((M, ku), float("nan"), device=cuda)
    cabi.call("omt_linear", A.to(cuda), K, 0, 0, 0, Wp, Wlo, U, ku, 0, 0, 0, M, 2 * ku, K, None, None, 0,
              cabi.EPI_GEGLU, mode)
    torch.cuda.synchronize()
    assert (U[:, :inner].cpu() - ref).abs().max().item() < 2e-5
    assert torch.count_nonzero(U[:, inner:]).item() == 0          # zero padding columns are exact
    # row maps: logical rows scatter into / gather from the canonical buffer (first-frame / rest-frames)
    B, T, N, Kp = 2, 3, 64, 192
    X = _rand((B * T * N, 512), 7).to(cuda)
    Wt = _rand((Kp, 512), 8, 0.05)
    Wq = _pad128(Wt).to(cuda)
    Wql = None
    if math == "3xtf32":
        hi = L.tf32_round(Wq)
        Wql, Wq = (Wq - hi).contiguous(), hi
    rows = B * (T - 1) * N
    P = torch.empty(rows, Kp, device=cuda)
    cabi.call("omt_linear", X, 512, (T - 1) * N, T * N, N, Wq, Wql, P, Kp, 0, 0, 0, rows, Kp, 512, None, None, 0,
              cabi.EPI_NONE, mode)
    sel = X.view(B, T, N, 512)[:, 1:].reshape(rows, 512).cpu()
    assert (P.cpu() - (sel.double() @ Wt.double().t()).float()).abs().max().item() < 2e-5
    Xo = torch.zeros(B * T * N, 512, device=cuda)
    Wb = _pad128(_rand((512, Kp), 9, 0.05)).to(cuda)
    Wbl = None
    Wb_ref = Wb[:512].cpu()
    if math == "3xtf32":
        hi = L.tf32_round(Wb)
        Wbl, Wb = (Wb - hi).contiguous(), hi
    cabi.call("omt_linear", P, Kp, 0, 0, 0, Wb, Wbl, Xo, 512, (T - 1) * N, T * N, N, rows, 512, Kp, None, None, 0,
              cabi.EPI_NONE, mode)
    want = torch.zeros(B, T, N, 512)
    want[:, 1:] = (P.cpu().double() @ Wb_ref.double().t()).float().view(B, T - 1, N, 512)
    assert (Xo.cpu().view(B, T, N, 512) - want).abs().max().item() < 2e-5


@pytest.mark.parametrize("M,N,K", [(20480, 1024, 1376), (5120, 512, 512), (40960, 512, 512)])
def test_linear_multiwave_deterministic(cuda, M, N, K):
    """gemm_tc2 (CTA-scope remote mbarrier arrives, no MEMBAR.ALL.GPU on the k-block critical path): the same bits
    run after run over several waves of tiles per cluster."""
    cabi = _cabi()
    from omnitokenizer_b200 import layout as L
    A = (torch.rand((M, K), device=cuda, generator=torch.Generator(device=cuda).manual_seed(31)) - 0.5)
    W = (torch.rand((N, K), device=cuda, generator=torch.Generator(device=cuda).manual_seed(32)) - 0.5) * 0.05
    R = (torch.rand((M, N), device=cuda, generator=torch.Generator(device=cuda).manual_seed(33)) - 0.5)
    hi = L.tf32_round(W)
    lo = (W - hi).contiguous()
    outs = []
    for _ in range(4):
        out = torch.full((M, N), float("nan"), device=cuda)
        cabi.call("omt_linear", A, K, 0, 0, 0, hi, lo, out, N, 0, 0, 0, M, N, K, None, R, N, cabi.EPI_NONE,
                  cabi.MATH_3XTF32)
        outs.append(out)
    torch.cuda.synchronize()
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    ref = (A[:256].double() @ W.double().t() + R[:256].double()).float()
    assert (outs[0][:256] - ref).abs().max().item() < 2e-5


def test_layernorm_and_patchify(cuda):
    cabi = _cabi()
    x = _rand((300, 512), 10, 3.0)
    g, b = _rand((512,), 11) + 1.0, _rand((512,), 12)
    y = torch.empty(300, 512, device=cuda)
    cabi.call("omt_layernorm", x.to(cuda), 512, y, 512, g.to(cuda), b.to(cuda), 300, 512, 1e-5, 0, 0, 0)
    assert (y.cpu() - oo.layer_norm(x, g, b)).abs().max().item() < 5e-6
    for shape in [(2, 3, 5, 64, 64), (1, 3, 1, 64, 64)]:
        v = _rand(shape, 13, 0.5)
        first, rest = oo.patchify(v, 8, 4)
        for is_first, ref in ((1, first), (0, rest)):
            if ref is None:
                continue
            K = ref.shape[-1]
            lw, lb = _rand((K,), 14) + 1.0, _rand((K,), 15)
            A = torch.empty(ref.numel() // K, K, device=cuda)
            cabi.call("omt_patchify_ln", v.to(cuda), A, None, None, None, lw.to(cuda), lb.to(cuda), shape[0], 3, shape[2], 64,
                      64, 8, 4, is_first, 1e-5)
            want = oo.layer_norm(ref, lw, lb).reshape(-1, K)
            assert (A.cpu() - want).abs().max().item() < 5e-6
            # un-patchify is the exact inverse permutation
            vid = torch.zeros(shape, device=cuda)
            raw = ref.reshape(-1, K).contiguous().to(cuda)
            cabi.call("omt_unpatchify", raw, vid, shape[0], 3, shape[2], 64, 64, 8, 4, is_first)
            got = vid.cpu()
            want_v = v[:, :, :1] if is_first else v[:, :, 1:]
            got_v = got[:, :, :1] if is_first else got[:, :, 1:]
            assert torch.equal(got_v, want_v)


@pytest.mark.parametrize("pk", [3, 4])
@pytest.mark.parametrize("temporal", [False, True])
@pytest.mark.parametrize("T", [1, 5])
def test_peg(cuda, temporal, T, pk):
    cabi = _cabi()
    cabi.set_option("peg_kernel", pk)
    from omnitokenizer_b200 import layout as L
    B, h, w, C = 2, 8, 8, 512
    X = _rand((B, T, h * w, C), 20)
    wt, bias = _rand((C, 1, 3, 3, 3), 21, 0.3), _rand((C,), 22, 0.1)
    want = oo.peg(X, wt, bias, (h, w), temporal, True) + X
    nbr = L.peg_neighbour_table(T, h, w, temporal, True)
    rows, _ = oo.peg_index_map(T, h, w, temporal, True)
    assert torch.equal(nbr.long(), rows)
    y = torch.empty(B * T * h * w, C, device=cuda)
    cabi.call("omt_peg", X.reshape(-1, C).to(cuda), y, wt.reshape(C, 27).t().contiguous().to(cuda), bias.to(cuda),
              nbr.to(cuda), B, T * h * w, C)
    assert (y.cpu().view_as(want) - want).abs().max().item() < 1e-5
    y2 = torch.empty_like(y)
    cabi.call("omt_peg_volume", X.reshape(-1, C).to(cuda), y2, wt.reshape(C, 27).t().contiguous().to(cuda),
              bias.to(cuda), B, T, h, w, C, int(temporal), 1)
    assert (y2.cpu().view_as(want) - want).abs().max().item() < 1e-5


@pytest.mark.parametrize("T,h,w,temporal,causal", [(9, 16, 16, True, True), (3, 8, 16, False, False),
                                                   (2, 8, 8, True, False), (5, 64, 64, True, True),
                                                   (5, 32, 32, False, True), (5, 32, 32, True, True),
                                                   (3, 6, 9, False, True), (17, 8, 8, True, True), (1, 32, 32, False, True)])
def test_peg_volume_shapes(cuda, T, h, w, temporal, causal):
    """The tiled kernels against the oracle; v4 (cp.async + FFMA2, the default) keeps v3's fma order, so the two are
    bit-identical."""
    cabi = _cabi()
    B, C = 2, 64
    X = _rand((B, T, h * w, C), 23)
    wt, bias = _rand((C, 1, 3, 3, 3), 24, 0.3), _rand((C,), 25, 0.1)
    want = oo.peg(X, wt, bias, (h, w), temporal, causal) + X
    got = {}
    for pk in (3, 4):
        cabi.set_option("peg_kernel", pk)
        y = torch.full((B * T * h * w, C), float("nan"), device=cuda)
        cabi.call("omt_peg_volume", X.reshape(-1, C).to(cuda), y, wt.reshape(C, 27).t().contiguous().to(cuda),
                  bias.to(cuda), B, T, h, w, C, int(temporal), int(causal))
        got[pk] = y.cpu()
        assert (got[pk].view_as(want) - want).abs().max().item() < 1e-5, pk
    assert torch.equal(got[3], got[4])


def _attn_inputs(M, seed):
    q, k, v = _rand((M, 512), seed), _rand((M, 512), seed + 1), _rand((M, 512), seed + 2)
    qkv = torch.cat([q, k, v], dim=1).contiguous()
    return q, k, v, qkv


@pytest.mark.parametrize("kernel,N", [(1, 256), (3, 256), (3, 1024), (1, 64)])
def test_qk_prep_and_spatial_attention(cuda, kernel, N):
    cabi = _cabi()
    cabi.set_option("attn_kernel", kernel)
    from omnitokenizer_b200 import layout as L
    nseq = 3
    M = nseq * N
    q, k, v, qkv = _attn_inputs(M, 30)
    qs, ks = _rand((64,), 33, 0.5) + 1.0, _rand((64,), 34, 0.5) + 1.0
    cos, sin = L.rope_tables(N, 64)
    c2, s2 = oo.rope_table(N, 64)
    assert torch.equal(cos, c2) and torch.equal(sin, s2)
    d = qkv.to(cuda)
    p = d.data_ptr()
    cabi.call("omt_qk_prep", p, 1536, p + 2048, 1536, qs.to(cuda), ks.to(cuda), cos.to(cuda), sin.to(cuda), M, N, 8)
    q4 = oo.l2norm(oo.apply_rope(q.view(nseq, N, 8, 64), cos, sin)) * qs
    k4 = oo.l2norm(oo.apply_rope(k.view(nseq, N, 8, 64), cos, sin)) * ks
    got = d.cpu()
    assert (got[:, :512].reshape(nseq, N, 8, 64) - q4).abs().max().item() < 2e-6
    assert (got[:, 512:1024].reshape(nseq, N, 8, 64) - k4).abs().max().item() < 2e-6
    assert torch.equal(got[:, 1024:], v)
    o = torch.empty(M, 512, device=cuda)
    cabi.call("omt_attn_spatial", p, 1536, p + 2048, 1536, p + 4096, 1536, o, None, None, 512, nseq, N, 8, 8.0)
    qq, kk, vv = q4.permute(0, 2, 1, 3), k4.permute(0, 2, 1, 3), v.view(nseq, N, 8, 64).permute(0, 2, 1, 3)
    want = torch.softmax((qq.double() @ kk.double().transpose(-1, -2)) * 8.0, dim=-1) @ vv.double()
    want = want.permute(0, 2, 1, 3).reshape(M, 512).float()
    err = (o.cpu() - want).abs().max().item()
    cabi.set_option("attn_kernel", 3)
    assert err < (5e-6 if kernel == 1 else 1e-5), f"attention kernel {kernel} N={N}: max err {err:.2e}"


def test_window_attention(cuda):
    cabi = _cabi()
    from omnitokenizer_b200 import layout as L
    cfg = oo.Config()
    frames, h, w = 3, 16, 16
    M = frames * h * w
    q, k, v, qkv = _attn_inputs(M, 40)
    table = _rand((225, 8), 43)
    sd = W.make_state_dict(oo.Config(), 0)
    index = sd["encoder.enc_spatial_transformer.layers.2.1.relative_position_index"]
    bias = L.window_bias(table, index, 8)
    d = qkv.to(cuda)
    p = d.data_ptr()
    o = torch.empty(M, 512, device=cuda)
    cabi.call("omt_attn_window", p, 1536, p + 2048, 1536, p + 4096, 1536, o, None, None, 512, bias.to(cuda), frames, h, w,
              8, 8, 0.125)
    rows = oo.window_rows(h, w, 8)
    def win(t):
        return t.view(frames, h * w, 8, 64)[:, rows].permute(0, 1, 3, 2, 4)       # (f, nW, H, 64, D)
    s = (win(q) * 0.125) @ win(k).transpose(-1, -2) + bias
    ow = (torch.softmax(s, dim=-1) @ win(v)).permute(0, 1, 3, 2, 4).reshape(frames, rows.shape[0], 64, 512)
    want = torch.empty(frames, h * w, 512)
    want[:, rows] = ow
    assert (o.cpu() - want.reshape(M, 512)).abs().max().item() < 5e-6


@pytest.mark.parametrize("T,causal", [(1, 1), (5, 1), (9, 1), (5, 0)])
def test_temporal_attention(cuda, T, causal):
    cabi = _cabi()
    B, N = 2, 64
    M = B * T * N
    q, k, v, qkv = _attn_inputs(M, 50)
    d = qkv.to(cuda)
    p = d.data_ptr()
    o = torch.empty(M, 512, device=cuda)
    cabi.call("omt_attn_temporal", p, 1536, p + 2048, 1536, p + 4096, 1536, o, None, None, 512, B, T, N, 8, 8.0, causal)
    def seq(t):
        return t.view(B, T, N, 8, 64).permute(0, 2, 3, 1, 4)                        # (B,N,H,T,D)
    s = (seq(q) @ seq(k).transpose(-1, -2)) * 8.0
    if causal:
        s = s.masked_fill(torch.ones(T, T, dtype=torch.bool).triu(1), float("-inf"))
    want = (torch.softmax(s.double(), dim=-1) @ seq(v).double()).permute(0, 3, 1, 2, 4).reshape(M, 512).float()
    # un-normalised random q,k give |scale*q.k| ~ 50: exp() carries |s|*2^-24 ~ 3e-6 relative error per term
    assert (o.cpu() - want).abs().max().item() < 2e-5


def test_vq_path(cuda):
    cabi = _cabi()
    M, C = 1000, 512
    x = _rand((M, C), 60)
    Wp, bp = _rand((8, C), 61, 0.05), _rand((8,), 62, 0.1)
    E = torch.rand((8192, 8, 12), generator=torch.Generator().manual_seed(63)).sum(-1) - 6.0
    z = torch.empty(M, 8, device=cuda)
    cabi.call("omt_pre_vq", x.to(cuda), C, Wp.to(cuda), bp.to(cuda), z, M, C, 8, 1)
    zr = x @ Wp.t() + bp
    zr = zr / zr.norm(dim=1, keepdim=True).clamp_min(1e-12)
    assert (z.cpu() - zr).abs().max().item() < 2e-6
    # search on the kernel's own z: must equal the oracle's argmin on the same z bit for bit
    zc = z.cpu()
    out = oo.codebook(E, zc)
    e2 = (E.t() ** 2).sum(dim=0)
    idx = torch.empty(M, dtype=torch.int64, device=cuda)
    counts = torch.zeros(8192, dtype=torch.int32, device=cuda)
    cabi.call("omt_vq_search", z, E.to(cuda), e2.to(cuda), M, 8192, idx, counts)
    assert torch.equal(idx.cpu(), out["idx"])
    assert torch.equal(counts.cpu().long(), torch.bincount(out["idx"], minlength=8192))
    # ties: duplicated codes must resolve to the FIRST index (torch.argmin rule)
    E2 = E.clone(); E2[4096:] = E[:4096]
    e22 = (E2.t() ** 2).sum(dim=0)
    counts.zero_()
    cabi.call("omt_vq_search", z, E2.to(cuda), e22.to(cuda), M, 8192, idx, counts)
    assert torch.equal(idx.cpu(), oo.codebook(E2, zc)["idx"]) and int(idx.max()) < 4096
    # the fused form (projection + normalise + search in one launch) gives the same z bits and the same indices
    for Mf in (M, 512, 513, 37):
        z2 = torch.full((Mf, 8), float("nan"), device=cuda)
        idx2 = torch.full((Mf,), -1, dtype=torch.int64, device=cuda)
        counts.zero_()
        cabi.call("omt_vq_fused", x[:Mf].contiguous().to(cuda), C, Wp.to(cuda), bp.to(cuda), C, 1, z2, E.to(cuda), e2.to(cuda), Mf,
                  8192, idx2, counts)
        dz = (z2 - z[:Mf]).abs()
        assert torch.equal(z2, z[:Mf]), f"fused z differs from omt_pre_vq at M={Mf}: max {dz.max().item():.3e}, {int((dz > 0).sum())} elements, nan {int(torch.isnan(z2).sum())}"
        bad = (idx2.cpu() != out["idx"][:Mf]).nonzero().flatten()
        assert bad.numel() == 0, f"fused idx differs at M={Mf}: {bad.numel()} rows, first {bad[:8].tolist()} got {idx2.cpu()[bad[:8]].tolist()} want {out['idx'][bad[:8]].tolist()}"
        assert torch.equal(counts.cpu().long(), torch.bincount(out["idx"][:Mf], minlength=8192))
    # the 4-rows-per-thread form (taken when the launch fills the GPU): 12 000 rows, with duplicated codes in different slices
    Mb = 12000
    xb = _rand((Mb, C), 66)
    zb = torch.empty(Mb, 8, device=cuda)
    idxb = torch.full((Mb,), -1, dtype=torch.int64, device=cuda)
    counts.zero_()
    cabi.call("omt_vq_fused", xb.to(cuda), C, Wp.to(cuda), bp.to(cuda), C, 1, zb, E2.to(cuda), e22.to(cuda), Mb, 8192, idxb, counts)
    want = oo.codebook(E2, zb.cpu())["idx"]
    assert torch.equal(idxb.cpu(), want) and int(idxb.max()) < 4096
    assert torch.equal(counts.cpu().long(), torch.bincount(want, minlength=8192))
    idxc = torch.full((Mb,), -1, dtype=torch.int64, device=cuda)
    cabi.call("omt_vq_search", zb, E.to(cuda), e2.to(cuda), Mb, 8192, idxc, None)
    assert torch.equal(idxc.cpu(), oo.codebook(E, zb.cpu())["idx"])
    # decode-side gather + post_vq, with and without straight-through rounding
    Wq, bq = _rand((512, 8), 64, 0.3), _rand((512,), 65, 0.1)
    X = torch.empty(M, 512, device=cuda)
    idx_d = out["idx"].to(cuda)
    cabi.call("omt_post_vq", idx_d, E.to(cuda), None, None, None, Wq.to(cuda), bq.to(cuda), X, M, 512, 8)
    assert (X.cpu() - (E[out["idx"]] @ Wq.t() + bq)).abs().max().item() < 2e-6
    zq = torch.empty(M, 8, device=cuda)
    cabi.call("omt_post_vq", idx_d, E.to(cuda), None, z, zq, Wq.to(cuda), bq.to(cuda), X, M, 512, 8)
    st = (E[out["idx"]] - zc) + zc
    assert torch.equal(zq.cpu(), st)
    assert (X.cpu() - (st @ Wq.t() + bq)).abs().max().item() < 2e-6
    cabi.call("omt_post_vq", None, None, z, None, None, Wq.to(cuda), bq.to(cuda), X, M, 512, 8)
    assert (X.cpu() - (zc @ Wq.t() + bq)).abs().max().item() < 2e-6


def test_errors_are_loud(cuda):
    cabi = _cabi()
    x = torch.zeros(4, 512, device=cuda)
    with pytest.raises(RuntimeError, match="omt_layernorm"):
        cabi.call("omt_layernorm", x, 512, x, 512, x, None, 4, 514, 1e-5, 0, 0, 0)
    with pytest.raises(RuntimeError, match="omt_attn_spatial"):
        cabi.call("omt_attn_spatial", x, 512, x, 512, x, 512, x, None, None, 512, 1, 100, 8, 8.0)


@pytest.mark.parametrize("math", ["fp32", "3xtf32"])
def test_linear2_dual_a(cuda, math):
    """q from LN(x), k/v from raw x in one launch (attention.py:407-412)."""
    cabi = _cabi()
    from omnitokenizer_b200 import layout as L
    M, K = 640, 512
    A1, A2, Wt = _rand((M, K), 70), _rand((M, K), 71), _rand((1536, K), 72, 0.05)
    ref = torch.cat([A1.double() @ Wt[:512].double().t(), A2.double() @ Wt[512:].double().t()], dim=1).float()
    Wp = _pad128(Wt).to(cuda)
    Wlo = None
    mode = cabi.MATH_FP32
    if math == "3xtf32":
        hi = L.tf32_round(Wp)
        Wlo, Wp, mode = (Wp - hi).contiguous(), hi, cabi.MATH_3XTF32
    out = torch.full((M, 1536), float("nan"), device=cuda)
    cabi.call("omt_linear2", A1.to(cuda), A2.to(cuda), 512, K, Wp, Wlo, out, 1536, M, 1536, K, mode, None, None, None,
              None, 0, 0)
    assert (out.cpu() - ref).abs().max().item() < 2e-5
    # with the fused q/k preparation (rope + l2norm + scale on the q and k heads, v untouched)
    N = 128
    qs, ks = _rand((64,), 73, 0.5) + 1.0, _rand((64,), 74, 0.5) + 1.0
    cos, sin = L.rope_tables(N, 64)
    for tables in ((cos, sin), (None, None)):
        out.fill_(float("nan"))
        cabi.call("omt_linear2", A1.to(cuda), A2.to(cuda), 512, K, Wp, Wlo, out, 1536, M, 1536, K, mode, qs.to(cuda),
                  ks.to(cuda), None if tables[0] is None else tables[0].to(cuda),
                  None if tables[1] is None else tables[1].to(cuda), 1024, N)
        got = out.cpu()
        for sl, sc in ((slice(0, 512), qs), (slice(512, 1024), ks)):
            t = ref[:, sl].reshape(M // N, N, 8, 64)
            if tables[0] is not None:
                t = oo.apply_rope(t, cos, sin)
            want = (oo.l2norm(t) * sc).reshape(M, 512)
            assert (got[:, sl] - want).abs().max().item() < 2e-5
        assert (got[:, 1024:] - ref[:, 1024:]).abs().max().item() < 2e-5
