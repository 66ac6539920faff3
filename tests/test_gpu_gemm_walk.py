"""The persistent wgmma GEMM (csrc/gemm_wgmma.cuh) across its tile walk, checked bit for bit.

Exact operands.  Every plane value is a small integer times a power of two: hi in {-2 .. 2}, lo worth {-1, 0, 1} * 2^-3.
Each product the kernel forms (hi.hi, lo.hi, hi.lo) is then a multiple of 2^-6, and with K <= 1408 every partial sum
stays below 2^14, i.e. within 20 significant bits.  fp32 holds every partial sum exactly.  So the tensor core's internal
rounding and the accumulation order cannot matter: a correct kernel has exactly one possible pre-epilogue value y, and
fp64 computes it.  The row scales (powers of two) keep y * scale exact.  Any dropped, duplicated or misplaced product
(wrong k-block, stage or phase, wrong 64-row half, wrong A matrix of a dual-A launch, wrong row scale under a row map)
moves y by at least 2^-3 * scale and breaks bit equality, in any tile and on either consumer warpgroup.  The lo.lo
product is not part of the f16x3 / 3xTF32 schemes, so the reference leaves it out too.

The tile-walk sweep picks M and N so that the tile count T is 1, S - 1, S, S + 1, 2S, 2S + 1 or 3S + 1, where S is the
number of SMs (the launcher puts one CTA on each).  The CTAs then walk 1 to 4 tiles, and warpgroup 2 of the ping-pong
schedule gets no tile, a middle tile or the last one.  Every output sits inside a larger NaN-filled buffer whose guard
bands must keep their bits, and three launches must give identical bits.
"""
import math

import pytest
import torch

from omnitokenizer_b200 import layout as L

SENT32 = 0x7FBADBAD          # fp32 NaN pattern that fills every fp32 output buffer before a launch
SENT16 = 0x7E5B              # fp16 NaN pattern for the operand-plane outputs
PRE, POST = 3, 5             # guard rows before and after every output
LO_UNIT = {"rs": 2.0 ** -3, "uniform": 2.0 ** -3, "nacc2": 2.0 ** 8}     # lo plane value for a represented 2^-3
CROSS = {"rs": 1.0, "uniform": 1.0, "nacc2": 2.0 ** -11}                 # weight of the lo plane in the represented value
W_SCALE = 2.0 ** -4


def _cabi():
    from omnitokenizer_b200 import _cabi
    _cabi.load()
    return _cabi


def _gen(seed, dev):
    return torch.Generator(device=dev).manual_seed(seed)


def _ints(shape, lo, hi, g, dev):
    return torch.randint(lo, hi + 1, shape, generator=g, device=dev).float()


def grid_operand(rows, cols, seed, dev, form, amp=2):
    """Operand on the exact grid: hi in {-amp .. amp}, lo worth {-1, 0, 1} * 2^-3.

    form "rs" / "uniform": fp16 planes, lo unscaled (the row-scaled, single-accumulator form);
    "nacc2": fp16 planes, lo scaled by 2^11 (the two-accumulator form);
    "tf32a": one fp32 matrix hi + lo (at most 5 significant bits, so the kernel's tf32 split gives A_hi = A, A_lo = 0);
    "tf32w": fp32 (hi, lo) of a 3xTF32 weight (the kernel takes any hi / lo pair, the split need not be canonical).
    """
    g = _gen(seed, dev)
    hi = _ints((rows, cols), -amp, amp, g, dev)
    lo = _ints((rows, cols), -1, 1, g, dev)
    if form == "tf32a":
        return (hi + lo * 2.0 ** -3,)
    if form == "tf32w":
        return hi, lo * 2.0 ** -3
    return hi.half(), (lo * LO_UNIT[form]).half()


def exact_y(a, w, form):
    """fp64 A . W^T of the products the kernel forms: hi.hi + c (lo.hi + hi.lo), c the lo plane weight.  All terms are
    multiples of 2^-6 below 2^14 in magnitude, so fp64 gets every sum exactly in any order."""
    if form == "tf32":
        (A,), (wh, wl) = a, w
        return A.double() @ (wh.double() + wl.double()).t()
    (ah, al), (wh, wl) = [[t.double() for t in p] for p in (a, w)]
    return ah @ wh.t() + CROSS[form] * (al @ wh.t() + ah @ wl.t())


def pow2_rows(rows, seed, dev, lo, hi):
    """Per-row inverse scales 2^e, e uniform in [lo, hi]."""
    return torch.exp2(_ints((rows,), lo, hi, _gen(seed, dev), dev))


def gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def map_rows(M, seg, stride, off, dev):
    """Physical row of every logical row under a (seg, seg_stride, seg_off) row map (include/omnitok_b200.h)."""
    r = torch.arange(M, device=dev)
    return r if seg <= 0 else (r // seg) * stride + off + r % seg


def _sms():
    return _cabi().device_info()[0]


T_KEYS = {"1": lambda s: 1, "S-1": lambda s: s - 1, "S": lambda s: s, "S+1": lambda s: s + 1, "2S": lambda s: 2 * s,
          "2S+1": lambda s: 2 * s + 1, "3S+1": lambda s: 3 * s + 1}


def _shape(T, n_list, tail):
    """(M, N) with exactly T tiles: the first N of n_list whose 128-column block count divides T; the last m block holds
    `tail` rows (1 .. 128)."""
    for N in n_list:
        nb = (N + 127) // 128
        if T % nb == 0:
            return (T // nb - 1) * 128 + tail, N
    raise AssertionError(f"no N in {n_list} tiles T={T}")


def _f32_buf(rows, cols, dev):
    b = torch.empty(rows, cols, device=dev)
    b.view(torch.int32).fill_(SENT32)
    return b


def _f16_buf(rows, cols, dev):
    return torch.full((2, rows, cols), SENT16, dtype=torch.int16, device=dev)


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _launch3(launch, bufs, reset):
    """Three launches, each into freshly reset buffers.  Every bit of every buffer (guards included) must agree; the
    buffers keep the last launch's output."""
    runs = []
    for _ in range(3):
        reset()
        launch()
        runs.append([_bits(b).clone() for b in bufs])
    torch.cuda.synchronize()
    for r in runs[1:]:
        for x, y in zip(r, runs[0]):
            assert torch.equal(x, y), f"launches differ in {int((x != y).sum())} elements"


def _check_guard(buf, mask, sent, what):
    """Outside the written region (mask False) the sentinel bits survive."""
    out = _bits(buf)[~mask]
    bad = int((out != sent).sum())
    assert bad == 0, f"{what}: {bad} elements outside the written region were overwritten"


def _qkv_layout(N):
    """(qk_cols, n_split) of a QKV GEMM with N columns, shaped like the model's (q | k | v, q from the first A)."""
    qk = max(128, (2 * N // 3) // 128 * 128)
    n_split = max(256, qk // 2 // 256 * 256) if N > 256 else 0
    return qk, n_split


def _qk_ref(z, qk_cols, qs, ks, cos, sin, tokens):
    """fp64 rope + l2norm + per-dim scale of the q / k heads of z [M, N] (attention.py:417-421, 435-437)."""
    M = z.shape[0]
    x = z[:, :qk_cols].reshape(M, qk_cols // 64, 64).clone()
    if cos is not None:
        pos = torch.arange(M, device=z.device) % tokens
        c, s = cos.double()[pos][:, None, :], sin.double()[pos][:, None, :]
        a, b = x[..., 0::2].clone(), x[..., 1::2].clone()
        x[..., 0::2], x[..., 1::2] = a * c - b * s, a * s + b * c
    x = x / x.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    heads = qk_cols // 64
    sc = torch.stack([qs if h < heads // 2 else ks for h in range(heads)]).double()
    return (x * sc).reshape(M, qk_cols), sc.reshape(qk_cols).abs()


# ---- the tile-walk sweep --------------------------------------------------------------------------------------------
# (form, epilogue, T, K, candidate N, rows in the last m block, options).  N lists start with the model's widths (512
# FF2 / to_out, 1536 QKV, 2816 = 2 * 1408 packed GEGLU, 192 / 768 to_pixels) and fall back to narrower ones when their
# block count does not divide T; 544 / 608 / 96 / 64 end in a partial 128-column block.
SWEEP = [
    ("rs", "plain", "1", 64, [64], 1, dict(bias=True, res="sep")),
    ("rs", "plain", "S-1", 128, [96], 127, dict(bias=True, res="sep")),
    ("rs", "plain", "S", 192, [512], 127, dict(bias=True, res="inplace")),
    ("rs", "plain", "S+1", 256, [896, 128], 1, dict(dual=True)),
    ("rs", "plain", "2S", 256, [192, 768, 128], 128, dict(bias=True, res="inplace", amap=True, cmap=True)),
    ("uniform", "plain", "2S+1", 1408, [544, 640, 128], 64, dict(res="sep")),
    ("rs", "plain", "3S+1", 64, [128], 64, dict(bias=True)),
    ("rs", "geglu", "2S", 256, [2816, 128], 64, {}),
    ("rs", "geglu_us", "S+1", 192, [896, 128], 127, {}),
    ("rs", "geglu_us", "3S+1", 64, [128], 1, {}),
    ("rs", "geglu", "S-1", 1408, [128], 128, {}),
    ("rs", "qkv", "2S", 128, [1536, 640, 128], 64, dict(tokens=96)),
    ("rs", "qkv_norope", "S", 256, [1536, 640, 128], 127, dict(tokens=128)),
    ("rs", "qkv", "2S+1", 64, [640, 1536, 128], 1, dict(tokens=96)),
    ("rs", "planes", "S+1", 192, [896, 1536, 640], 64, dict(tokens=96)),
    ("rs", "planes", "2S", 1408, [1536, 896, 640], 128, dict(tokens=128)),
    ("nacc2", "plain", "S+1", 1408, [896, 128], 127, dict(bias=True, res="sep")),
    ("nacc2", "plain", "3S+1", 64, [64], 64, dict(res="inplace")),
    ("nacc2", "geglu", "2S", 128, [2816, 128], 128, {}),
    ("nacc2", "geglu_us", "2S+1", 192, [640, 128], 1, {}),
    ("tf32", "plain", "S", 256, [512, 128], 1, dict(bias=True, res="sep")),
    ("tf32", "plain", "2S+1", 64, [544, 640, 128], 64, dict(res="inplace", cmap=True)),
    ("tf32", "geglu", "S+1", 128, [896, 128], 127, dict(bias=True)),
    ("tf32", "geglu", "3S+1", 1408, [128], 1, dict(bias=True)),
]


def _ops(form, rows, cols, seed, dev, amp=2):
    return grid_operand(rows, cols, seed, dev, "tf32a" if form == "tf32" else form, amp)


def _wops(form, rows, cols, seed, dev, amp=2):
    return grid_operand(rows, cols, seed, dev, "tf32w" if form == "tf32" else form, amp)


def _wpad(w, form):
    """W padded to the launcher's row multiple (256 for the f16 planes, 128 for 3xTF32)."""
    return [L.pad_rows(t, 128 if form == "tf32" else 256) for t in w]


def _f16_args(form, a, ars, a2, a2rs, n_split, K, wp, seg=(0, 0, 0)):
    kw = dict(a_hi=a[0], a_lo=a[1], lda=K, w_hi=wp[0], w_lo=wp[1], a_seg=seg[0], a_seg_stride=seg[1], a_seg_off=seg[2])
    if form == "rs":
        kw.update(a_rs=ars, w_scale=W_SCALE)
    elif form == "uniform":
        kw.update(a_rs_uniform=float(ars), w_scale=W_SCALE)
    if a2 is not None:
        kw.update(a2_hi=a2[0], a2_lo=a2[1], n_split=n_split)
        if form == "rs":
            kw.update(a2_rs=a2rs)
    return kw


def _row_seg(M, mult, extra, off, dev):
    """A row map of up to four segments over M logical rows (segment a multiple of `mult`), `extra` physical rows
    between segments, starting `off` rows in: (seg, stride, off, physical rows, logical -> physical index)."""
    for d in (4, 3, 2, 1):
        if M % (mult * d) == 0:
            seg = M // d
            break
    else:
        raise AssertionError(f"M={M} has no row-map segment that is a multiple of {mult}")
    stride = seg + extra
    return seg, stride, off, d * stride, map_rows(M, seg, stride, off, dev)


def _scales(form, epi, rows, seed, dev):
    """Row scales: per row 2^-20 .. 2^20 for the plain and QKV epilogues.  GEGLU's fp16 planes must hold
    |gelu(gate) * value| <= |y|^2 (scale 2^-4)^2 < 2^15 with |y| <= 4.5 K < 2^13: 2^-12 .. 2^-4 keeps it there (and
    most rows above the planes' subnormal floor)."""
    if form == "rs":
        return pow2_rows(rows, seed, dev, -12, -4) if epi.startswith("geglu") else pow2_rows(rows, seed, dev, -20, 20)
    if form == "uniform":
        return torch.tensor(2.0 ** 3)
    return None


def _case_plain(cabi, dev, form, T, K, n_list, tail, opt):
    M, N = _shape(T, n_list, tail)
    tf32 = form == "tf32"
    if opt.get("amap"):
        aseg, astr, aoff, arows, aidx = _row_seg(M, 64, 192, 128, dev)
    else:
        aseg, astr, aoff, arows, aidx = 0, 0, 0, M, torch.arange(M, device=dev)
    if opt.get("cmap"):
        cseg, cstr, coff, crows, cidx = _row_seg(M, 32, 96, 32, dev)
    else:
        cseg, cstr, coff, crows, cidx = 0, 0, 0, M, torch.arange(M, device=dev)
    a = _ops(form, arows, K, 11, dev)
    w = _wops(form, N, K, 12, dev)
    ars = _scales(form, "plain", arows, 13, dev)
    dual = opt.get("dual", False)
    n_split = 512 if dual else 0
    a2 = _ops(form, arows, K, 14, dev) if dual else None
    a2rs = _scales(form, "plain", arows, 15, dev) if dual else None
    g = _gen(16, dev)
    bias = _ints((N,), -16, 16, g, dev) * 2.0 ** -3 if opt.get("bias") else None
    res_vals = _ints((M, N), -16, 16, g, dev) * 2.0 ** -3 if opt.get("res") else None

    # reference: y exact in fp64, y * scale exact in fp32, then the kernel's two fp32 additions (bias, residual)
    y = exact_y([t[aidx] for t in a], w, "tf32" if tf32 else form)
    if form == "rs":
        y = y * (ars[aidx].double() * W_SCALE)[:, None]
    elif form == "uniform":
        y = y * (float(ars) * W_SCALE)
    if dual:
        y2 = exact_y([t[aidx] for t in a2], w, form)
        if form == "rs":
            y2 = y2 * (a2rs[aidx].double() * W_SCALE)[:, None]
        y[:, n_split:] = y2[:, n_split:]
    want = y.float()
    assert torch.equal(want.double(), y)
    if bias is not None:
        want = want + bias
    if res_vals is not None:
        want = want + res_vals

    ldc = N + 12
    cb = _f32_buf(PRE + crows + POST, ldc, dev)
    C = cb[PRE:]
    res, ldr = None, 0
    if opt.get("res") == "sep":
        res = torch.zeros(crows, N, device=dev)
        res[cidx] = res_vals
        ldr = N
    elif opt.get("res") == "inplace":
        res, ldr = C, ldc

    def reset():
        cb.view(torch.int32).fill_(SENT32)
        if opt.get("res") == "inplace":
            C[cidx, :N] = res_vals

    wp = _wpad(w, form)
    if tf32:
        def launch():
            cabi.call("omt_linear", a[0], K, aseg, astr, aoff, wp[0], wp[1], C, ldc, cseg, cstr, coff, M, N, K, bias,
                      res, ldr, cabi.EPI_NONE, cabi.MATH_3XTF32)
    else:
        kw = _f16_args(form, a, ars, a2, a2rs, n_split, K, wp, (aseg, astr, aoff))

        def launch():
            cabi.linear_h(c=C, ldc=ldc, c_seg=cseg, c_seg_stride=cstr, c_seg_off=coff, M=M, N=N, K=K, bias=bias,
                          residual=res, ldr=ldr, epilogue=cabi.EPI_NONE, **kw)
    _launch3(launch, [cb], reset)
    got = C[cidx, :N]
    assert not torch.isnan(got).any(), "NaN left inside the output"
    bad = got != want
    assert not bad.any(), (f"{int(bad.sum())} of {bad.numel()} outputs differ from the exact result, first at "
                           f"{bad.nonzero()[0].tolist()}, max |diff| {(got - want).abs().max().item():.3e}")
    mask = torch.zeros(cb.shape, dtype=torch.bool, device=dev)
    mask[PRE + cidx, :N] = True
    _check_guard(cb, mask, SENT32, "C")
    return M, N


def _case_geglu(cabi, dev, form, T, K, n_list, tail, opt, static):
    M, N = _shape(T, n_list, tail)
    ku = N // 2
    inner = 1365 if ku == 1408 else ku - 11
    tf32 = form == "tf32"
    # |y| <= K (amp + 1/8)^2 keeps |gelu(gate) * value| < 2^15 for the fp16 planes of the 2^11 form (amp 1, K 128)
    amp = 1 if form == "nacc2" else 2
    a = _ops(form, M, K, 21, dev, amp)
    w = [L.pack_geglu(t, inner, ku) for t in _wops(form, 2 * inner, K, 22, dev, amp)]
    ars = _scales(form, "geglu", M, 23, dev)
    bias = None
    if opt.get("bias"):
        bias = torch.zeros(N, device=dev)
        bias[: 2 * inner] = _ints((2 * inner,), -16, 16, _gen(24, dev), dev) * 2.0 ** -3
    y = exact_y(a, w, "tf32" if tf32 else form)
    if form == "rs":
        y = y * (ars.double() * W_SCALE)[:, None]
    if bias is not None:
        y = y + bias.double()
    assert torch.equal(y.float().double(), y)
    val, gate = y[:, 0::2], y[:, 1::2]
    want = gelu64(gate) * val
    # fp32 gelu_erf(gate) * value: the erff argument (two roundings), erff (<= 2 ulp), 1 + erf and the two products
    # each err by <= 2^-23 of |gate| * |value| / 2, <= 2^-22 |gate| |value| in all; the fp16 planes hold the result to
    # 2^-22 |result| <= 2^-22 |gate| |value| (|gelu(g)| <= |g|).  2^-20 leaves a factor 2 over the sum.
    tol = 2.0 ** -20 * val.abs() * gate.abs()
    us = L.pow2_scale(float(want.abs().max()) * 4.0) if static else 0.0
    wp = _wpad(w, form)
    if tf32:
        ldc = ku + 12
        cb = _f32_buf(PRE + M + POST, ldc, dev)
        C = cb[PRE:]

        def launch():
            cabi.call("omt_linear", a[0], K, 0, 0, 0, wp[0], wp[1], C, ldc, 0, 0, 0, M, N, K, bias, None, 0,
                      cabi.EPI_GEGLU, cabi.MATH_3XTF32)

        _launch3(launch, [cb], lambda: cb.view(torch.int32).fill_(SENT32))
        got = C[:M, :ku].double()
        assert not torch.isnan(got).any()
        mask = torch.zeros(cb.shape, dtype=torch.bool, device=dev)
        mask[PRE: PRE + M, :ku] = True
        _check_guard(cb, mask, SENT32, "C")
    else:
        ldu = ku + 24
        ub = _f16_buf(PRE + M + POST, ldu, dev)
        kw = _f16_args(form, a, ars, None, None, 0, K, wp)

        def launch():
            cabi.linear_h(u_hi=ub[0, PRE:], u_lo=ub[1, PRE:], ldu=ldu, M=M, N=N, K=K, epilogue=cabi.EPI_GEGLU,
                          u_scale=us, **kw)

        _launch3(launch, [ub], lambda: ub.fill_(SENT16))
        hi, lo = (ub[i, PRE: PRE + M, :ku].view(torch.float16).double() for i in (0, 1))
        assert not (hi.isnan().any() or lo.isnan().any()), "NaN left inside the U planes"
        # subnormal floor of the fp16 lo plane: 2^-25 of the scaled value, 2^-35 in the 2^11 form
        if static:
            got, tol = (hi + lo) / us, tol + 2.0 ** -25 / us
        else:
            got, tol = hi + lo / L.F16X3_LO_SCALE, tol + 2.0 ** -35
        mask = torch.zeros(ub.shape, dtype=torch.bool, device=dev)
        mask[:, PRE: PRE + M, :ku] = True
        _check_guard(ub, mask, SENT16, "U planes")
        assert torch.count_nonzero(ub[:, PRE: PRE + M, inner:ku]).item() == 0, "padding columns are not exact zeros"
    err = (got[:, :inner] - want[:, :inner]).abs() - tol[:, :inner]
    assert (err <= 0).all(), (f"GEGLU off by more than its bound at {err.argmax().item()}: "
                              f"{(got - want).abs().max().item():.3e}")
    if tf32:
        assert torch.count_nonzero(got[:, inner:]).item() == 0, "padding columns are not exact zeros"
    return M, N


def _case_qkv(cabi, dev, T, K, n_list, tail, opt, rope, planes):
    M, N = _shape(T, n_list, tail)
    tokens = opt["tokens"]
    qk, n_split = _qkv_layout(N)
    a = _ops("rs", M, K, 31, dev)
    ars = _scales("rs", "qkv", M, 32, dev)
    a2 = _ops("rs", M, K, 33, dev) if n_split else None
    a2rs = _scales("rs", "qkv", M, 34, dev) if n_split else None
    w = _wops("rs", N, K, 35, dev)
    g = _gen(36, dev)
    qs, ks = 0.5 + torch.rand(64, generator=g, device=dev), 0.5 + torch.rand(64, generator=g, device=dev)
    cos, sin = [t.to(dev) for t in L.rope_tables(tokens, 64)] if rope else (None, None)
    z = exact_y(a, w, "rs") * (ars.double() * W_SCALE)[:, None]
    if n_split:
        z[:, n_split:] = (exact_y(a2, w, "rs") * (a2rs.double() * W_SCALE)[:, None])[:, n_split:]
    assert torch.equal(z.float().double(), z)
    qk_want, sc = _qk_ref(z, qk, qs, ks, cos, sin, tokens)
    # rope (<= 2^-22 of the head norm), the sum of 64 squares (18 roundings of positive terms, 2^-19.8), sqrt, the
    # reciprocal and two products: |error| < 2^-19 |scale_d|.  2^-18 leaves a factor 2.
    tol = 2.0 ** -18 * sc
    wp = _wpad(w, "rs")
    kw = _f16_args("rs", a, ars, a2, a2rs, n_split, K, wp)
    kw.update(q_scale=qs, k_scale=ks, rope_cos=cos, rope_sin=sin, qk_cols=qk, tokens=tokens, M=M, N=N, K=K)
    if not planes:
        ldc = N + 12
        cb = _f32_buf(PRE + M + POST, ldc, dev)
        _launch3(lambda: cabi.linear_h(c=cb[PRE:], ldc=ldc, epilogue=cabi.EPI_QKV, **kw), [cb],
                 lambda: cb.view(torch.int32).fill_(SENT32))
        got = cb[PRE: PRE + M, :N]
        assert not torch.isnan(got).any()
        err = (got[:, :qk].double() - qk_want).abs()
        assert (err <= tol).all(), f"q / k off by {(err / tol).max().item():.2f} x the bound"
        assert torch.equal(got[:, qk:], z[:, qk:].float()), "v columns are not exact"
        mask = torch.zeros(cb.shape, dtype=torch.bool, device=dev)
        mask[PRE: PRE + M, :N] = True
        _check_guard(cb, mask, SENT32, "C")
        return M, N
    hv = (N - qk) // 64
    qps, kps = L.pow2_scale(float(qs.max())), L.pow2_scale(float(ks.max()))
    ldu = N + 40
    pb = _f16_buf(PRE + M + POST, ldu, dev)
    vinv = torch.empty(hv * M + 7, device=dev)

    def reset():
        pb.fill_(SENT16)
        vinv.view(torch.int32).fill_(SENT32)

    _launch3(lambda: cabi.linear_h(u_hi=pb[0, PRE:], u_lo=pb[1, PRE:], ldu=ldu, epilogue=cabi.EPI_QKV_PLANES,
                                   q_plane_scale=qps, k_plane_scale=kps, vinv=vinv, **kw), [pb, vinv], reset)
    hi, lo = (pb[i, PRE: PRE + M, :N] for i in (0, 1))
    assert not (hi.view(torch.float16).isnan().any() or lo.view(torch.float16).isnan().any())
    val = hi[:, :qk].view(torch.float16).double() + lo[:, :qk].view(torch.float16).double()
    ps = torch.tensor([qps] * (qk // 2) + [kps] * (qk // 2), device=dev, dtype=torch.float64)
    # the planes hold the scaled value to 2^-22 of itself (|value| <= |scale_d|) above fp16's subnormal floor 2^-25
    err = (val / ps - qk_want).abs()
    assert (err <= 2.0 * tol + 2.0 ** -25 / ps).all(), "q / k planes off by more than their bound"
    vh, vl, vi = L.split_rows_rs(z[:, qk:].float().reshape(M * hv, 64))
    assert torch.equal(hi[:, qk:], vh.view(torch.int16).reshape(M, N - qk)), "v hi plane differs from the host twin"
    assert torch.equal(lo[:, qk:], vl.view(torch.int16).reshape(M, N - qk)), "v lo plane differs from the host twin"
    assert torch.equal(vinv[: hv * M].view(hv, M), vi.view(M, hv).t()), "vinv differs from the host twin"
    mask = torch.zeros(pb.shape, dtype=torch.bool, device=dev)
    mask[:, PRE: PRE + M, :N] = True
    _check_guard(pb, mask, SENT16, "q | k | v planes")
    vmask = torch.zeros(vinv.shape, dtype=torch.bool, device=dev)
    vmask[: hv * M] = True
    _check_guard(vinv, vmask, SENT32, "vinv")
    return M, N


@pytest.mark.gpu
@pytest.mark.parametrize("form,epi,t,K,n_list,tail,opt", SWEEP,
                         ids=[f"{c[0]}-{c[1]}-T{c[2]}-K{c[3]}" + ("-" + "-".join(sorted(c[6])) if c[6] else "")
                              for c in SWEEP])
def test_tile_walk(cuda, form, epi, t, K, n_list, tail, opt):
    cabi = _cabi()
    S = _sms()
    T = T_KEYS[t](S)
    if epi == "plain":
        M, N = _case_plain(cabi, cuda, form, T, K, n_list, tail, opt)
    elif epi in ("geglu", "geglu_us"):
        M, N = _case_geglu(cabi, cuda, form, T, K, n_list, tail, opt, epi == "geglu_us")
    else:
        M, N = _case_qkv(cabi, cuda, T, K, n_list, tail, opt, rope=epi != "qkv_norope", planes=epi == "planes")
    assert ((M + 127) // 128) * ((N + 127) // 128) == T


# ---- placement invariance -------------------------------------------------------------------------------------------
# A row gets the same bits wherever it lands in a launch: sharding a batch of 64-row images moves rows by half a tile.
# Each element gets the same products in the same k order wherever its row and column sit, so every shift below is
# bit-identical, including shifts by 1 and 8 rows.

def _real_operands(form, M, N, K, dev):
    g = _gen(41, dev)
    A = torch.randn(M, K, generator=g, device=dev) * torch.logspace(-3, 3, M, device=dev)[
        torch.randperm(M, generator=g, device=dev)][:, None]
    Wt = torch.randn(N, K, generator=g, device=dev) * 0.05
    bias, R = torch.randn(N, generator=g, device=dev), torch.randn(M, N, generator=g, device=dev)
    extra = 256           # spare zero rows, so a W view shifted by whole n blocks still has its padded rows
    if form == "rs":
        ah, al, ars = L.split_rows_rs(A)
        wh, wl, wsc = L.split_f16_rs(Wt)
        return dict(a=(ah, al), ars=ars, wsc=wsc, w=[L.pad_rows(t, 256) for t in (wh, wl)], extra=extra, bias=bias, R=R)
    if form == "nacc2":
        return dict(a=L.split_f16(A), ars=None, wsc=0.0, w=[L.pad_rows(t, 256) for t in L.split_f16(Wt)], bias=bias,
                    R=R, extra=extra)
    hi = L.tf32_round(Wt)
    return dict(a=(A,), ars=None, wsc=0.0, w=[L.pad_rows(t, 256) for t in (hi, Wt - hi)], bias=bias, R=R, extra=extra)


def _pad_more(w, extra):
    return [torch.cat([t, torch.zeros(extra, t.shape[1], dtype=t.dtype, device=t.device)]) for t in w]


def _plain_launch(cabi, form, op, r, j, M, N, K, out):
    """One launch on rows [r, r + M) of A / residual and on W, bias from n block j."""
    a = [t[r: r + M] for t in op["a"]]
    w = [t[128 * j:] for t in op["w"]]
    bias, R = op["bias"][128 * j: 128 * j + N], op["R"][r: r + M]
    ldr = op["R"].shape[1]
    Rv = R[:, 128 * j:]
    if form == "tf32":
        cabi.call("omt_linear", a[0], K, 0, 0, 0, w[0], w[1], out, out.stride(0), 0, 0, 0, M, N, K, bias, Rv, ldr,
                  cabi.EPI_NONE, cabi.MATH_3XTF32)
        return
    kw = dict(a_hi=a[0], a_lo=a[1], lda=K, w_hi=w[0], w_lo=w[1])
    if form == "rs":
        kw.update(a_rs=op["ars"][r: r + M], w_scale=op["wsc"])
    cabi.linear_h(c=out, ldc=out.stride(0), M=M, N=N, K=K, bias=bias, residual=Rv, ldr=ldr, epilogue=cabi.EPI_NONE, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["rs", "nacc2", "tf32"])
def test_placement_invariance_plain(cuda, form):
    cabi = _cabi()
    S = _sms()
    N, K = 512, 512
    M = -(-(2 * S + 1) // 4) * 128               # T >= 2S + 1: tiles on warpgroup 2 and on later passes of the walk
    op = _real_operands(form, M, N, K, cuda)
    op["w"] = _pad_more(op["w"], op["extra"])
    op["bias"] = torch.cat([op["bias"], torch.zeros(op["extra"], device=cuda)])
    big = torch.full((M, N), float("nan"), device=cuda)
    _plain_launch(cabi, form, op, 0, 0, M, N, K, big)
    Mw = 320                                     # two and a half tiles
    for r, j in ((1, 0), (8, 1), (64, 0), (64, 2), (128, 1), (128 * (M // 256), 0), (M - Mw, 3)):
        Nw = N - 128 * j
        small = torch.full((Mw, Nw), float("nan"), device=cuda)
        _plain_launch(cabi, form, op, r, j, Mw, Nw, K, small)
        want = big[r: r + Mw, 128 * j:]
        d = (small - want).abs().max().item()
        assert torch.equal(small, want), f"rows shifted by {r}, columns by {128 * j}: max |diff| {d:.3e}"


@pytest.mark.gpu
def test_placement_invariance_qkv_planes(cuda):
    """QKV -> planes: offsets are multiples of `tokens` (the rope position of row m is m % tokens); vinv is compared
    per head because its stride is M."""
    cabi = _cabi()
    S = _sms()
    N, K, tokens, qk, n_split = 1536, 512, 32, 1024, 512
    M = -(-(2 * S + 1) // 12) * 128
    g = _gen(51, cuda)
    A1 = torch.randn(M, K, generator=g, device=cuda)
    A2 = torch.randn(M, K, generator=g, device=cuda) * torch.logspace(-2, 2, M, device=cuda)[:, None]
    Wt = torch.randn(N, K, generator=g, device=cuda) * 0.05
    a1, a2 = L.split_rows_rs(A1), L.split_rows_rs(A2)
    wh, wl, wsc = L.split_f16_rs(L.pad_rows(Wt, 256))
    qs, ks = 0.5 + torch.rand(64, generator=g, device=cuda), 0.5 + torch.rand(64, generator=g, device=cuda)
    cos, sin = [t.to(cuda) for t in L.rope_tables(tokens, 64)]
    qps, kps = L.pow2_scale(float(qs.max())), L.pow2_scale(float(ks.max()))
    hv = (N - qk) // 64

    def run(r, m):
        P = torch.full((2, m, N), SENT16, dtype=torch.int16, device=cuda)
        vinv = torch.full((hv, m), float("nan"), device=cuda)
        cabi.linear_h(a_hi=a1[0][r: r + m], a_lo=a1[1][r: r + m], a_rs=a1[2][r: r + m], a2_hi=a2[0][r: r + m],
                      a2_lo=a2[1][r: r + m], a2_rs=a2[2][r: r + m], w_scale=wsc, n_split=n_split, lda=K, w_hi=wh,
                      w_lo=wl, u_hi=P[0], u_lo=P[1], ldu=N, M=m, N=N, K=K, epilogue=cabi.EPI_QKV_PLANES, q_scale=qs,
                      k_scale=ks, rope_cos=cos, rope_sin=sin, qk_cols=qk, tokens=tokens, q_plane_scale=qps,
                      k_plane_scale=kps, vinv=vinv)
        return P, vinv

    Pb, vb = run(0, M)
    Mw = 320
    for r in (32, 64, 128, 128 * (M // 256), M - Mw):
        P, v = run(r, Mw)
        assert torch.equal(P, Pb[:, r: r + Mw]), f"planes differ for rows shifted by {r}"
        for h in range(hv):
            assert torch.equal(v[h], vb[h, r: r + Mw]), f"vinv of v head {h} differs for rows shifted by {r}"


# ---- accumulation precision -----------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("form", ["rs", "nacc2"])
def test_accumulation_bound(cuda, form):
    """Realistic operands at K = 1408 (FF2): all-positive rows, where nothing cancels a biased accumulation, and heavily
    cancelling rows.  |got - ref| <= tau_K (|A_rep| . |W_rep|^T) with tau_K = 2 ceil(3K / 16) 2^-23, i.e. at most two
    ulps per wgmma accumulation step (three k16 wgmmas per 16 columns of K); ref is fp64 of the products the kernel
    forms on the plane-represented values."""
    cabi = _cabi()
    M, N, K = 512, 512, 1408
    g = _gen(61, cuda)
    A = torch.rand(M, K, generator=g, device=cuda) + 2.0 ** -8
    Wt = torch.rand(N, K, generator=g, device=cuda) * 0.05 + 2.0 ** -12
    # rows M/2.. cancel: random signs on A (W stays positive); every other one of them pairs +x with -x against weight
    # pairs that differ by 2^-10, so its sum is about 2^-10 of its magnitude
    A[M // 2:] *= torch.where(torch.rand(M // 2, K, generator=g, device=cuda) < 0.5, -1.0, 1.0)
    A[M // 2::2, 1::2] = -A[M // 2::2, 0::2]
    Wt[:, 1::2] = Wt[:, 0::2] * (1.0 + 2.0 ** -10)
    if form == "rs":
        ah, al, ars = L.split_rows_rs(A)
        wh, wl, wsc = L.split_f16_rs(Wt)
        scale = ars.double()[:, None] * wsc
        c = 1.0
    else:
        ah, al = L.split_f16(A)
        wh, wl = L.split_f16(Wt)
        scale, c = 1.0, 2.0 ** -11
    ahd, ald, whd, wld = (t.double() for t in (ah, al, wh, wl))
    ref = (ahd @ whd.t() + c * (ald @ whd.t() + ahd @ wld.t())) * scale
    mag = ((ahd + c * ald).abs() @ (whd + c * wld).abs().t()) * (scale.abs() if form == "rs" else 1.0)
    out = torch.full((M, N), float("nan"), device=cuda)
    kw = dict(a_rs=ars, w_scale=wsc) if form == "rs" else {}
    wp = [L.pad_rows(t, 256) for t in (wh, wl)]
    cabi.linear_h(a_hi=ah, a_lo=al, lda=K, w_hi=wp[0], w_lo=wp[1], c=out, ldc=N, M=M, N=N, K=K,
                  epilogue=cabi.EPI_NONE, **kw)
    torch.cuda.synchronize()
    tau = 2 * math.ceil(3 * K / 16) * 2.0 ** -23
    ratio = ((out.double() - ref).abs() / (tau * mag))
    pos, canc = ratio[: M // 2].max().item(), ratio[M // 2:].max().item()
    print(f"accumulation {form} K={K}: max |err| / (tau_K |A||W|) = {pos:.4f} (positive rows), {canc:.4f} (cancelling)")
    assert max(pos, canc) <= 1.0


# ---- the exact-grid construction itself (no GPU) --------------------------------------------------------------------

@pytest.mark.parametrize("form", ["rs", "nacc2", "tf32"])
def test_grid_operands_are_exact(form):
    """The plane values are what they claim, the fp64 reference is exact, and fp32 computes every partial sum of it
    exactly in whatever order: the property the GPU tests rely on to ask for bit equality."""
    M, N, K = 48, 40, 1408
    a = grid_operand(M, K, 1, "cpu", "tf32a" if form == "tf32" else form)
    w = grid_operand(N, K, 2, "cpu", "tf32w" if form == "tf32" else form)
    if form == "tf32":
        A = a[0]
        assert torch.equal(L.tf32_round(A), A), "A is not tf32-exact: the kernel's split would leave a lo part"
        assert set(w[0].unique().tolist()) <= {-2.0, -1.0, 0.0, 1.0, 2.0}
        assert set(w[1].unique().tolist()) <= {-0.125, 0.0, 0.125}
        terms = A.double()[:, None, :] * (w[0] + w[1]).double()[None, :, :]
    else:
        hi, lo = a
        assert set(hi.float().unique().tolist()) <= {-2.0, -1.0, 0.0, 1.0, 2.0}
        assert set((lo.float() / LO_UNIT[form]).unique().tolist()) <= {-1.0, 0.0, 1.0}
        ah, al, wh, wl = (t.double() for t in (a[0], a[1], w[0], w[1]))
        terms = (ah[:, None, :] * wh[None] + CROSS[form] * (al[:, None, :] * wh[None] + ah[:, None, :] * wl[None]))
    y = exact_y(a, w, form)
    assert torch.equal(terms.sum(-1), y)
    # every prefix sum (k ascending and descending) is exact in fp32, so no accumulation order can round
    for t in (terms, terms.flip(-1)):
        pre = t.cumsum(-1)
        assert torch.equal(pre.float().double(), pre)
        assert torch.equal(t.float().cumsum(-1).double(), pre)
    assert (terms.abs().sum(-1) < 2.0 ** 14).all()
    # the row scales keep it exact, and the plain reference is the fp32 cast of the fp64 value
    s = pow2_rows(M, 3, "cpu", -20, 20)
    assert set(torch.log2(s).unique().tolist()) <= set(float(e) for e in range(-20, 21))
    z = y * (s.double() * W_SCALE)[:, None]
    assert torch.equal(z.float().double(), z)
    assert torch.equal(z.float(), (y.float() * (s * W_SCALE)[:, None]))
