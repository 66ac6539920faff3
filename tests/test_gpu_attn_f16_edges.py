"""The f16 spatial attention cores (omt_attn_spatial_h / omt_attn_spatial_h1) on the cases of tests/attn_f16_cases.py:
planted one-hot keys at every key position, v rows spread over 2^0 ... 2^30 inside a sequence, and logits up to 2048
with the engine's plane scales at both ends of their binade.

Both entry points write into the sentinel-filled, guarded buffers of test_gpu_attn_walk.py, in fp32 and in plane form.
Planted rows that the host model predicts exactly must equal its bits; every other output must stay within the host
model's bound of fp64 attention (attn_f16_cases.bound_head); three launches must agree bit for bit.  The layer survey
runs the golden configurations and checks that the sweeps cover the vinv spreads and logits the model's layers produce.

The printed ratios read as follows.  The planted rows are sharp: a wrong bit fails them.  Elsewhere the bound is derived
term by term, not fitted, and is worst-case: on the spread and logit cases it sits 100 to 500 times above the x3 error
the kernel shows, so a fault smaller than that margin passes those families and only the planted rows would catch it.
x1 cases whose worst bound/mag exceeds 1 are checked against the hull of the v rows only (attn_f16_cases.LOGIT_SCALES).
"""
import os

import pytest
import torch

import omnitokenizer_b200 as ob
from omnitokenizer_b200 import layout as L
from tests import attn_f16_cases as A
from tests.test_gpu_attn_walk import PRE, SENT16, SENT32, _cabi, _check_guards, _f16_buf, _f32_buf
from tests.util import build_model, flags_namespace, flags_setup, golden_setup, load_golden

pytestmark = pytest.mark.gpu


def _launch(c, mode, dev, planes=False):
    cols = c.H * 64
    ldo = cols + 8
    qh, ql, kh, kl, vh, vl = (t.view(torch.int16).contiguous().to(dev) for t in (c.qh, c.ql, c.kh, c.kl, c.vh, c.vl))
    vinv = c.vinv.contiguous().to(dev)
    if planes:
        buf = _f16_buf(c.M, ldo, dev)
        o, o_hi, o_lo = None, buf[0, PRE:], buf[1, PRE:]
    else:
        buf = _f32_buf(c.M, ldo, dev)
        o, o_hi, o_lo = buf[PRE:], None, None
    if mode == "x3":
        _cabi().call("omt_attn_spatial_h", qh, ql, cols, kh, kl, cols, vh, vl, cols, vinv, c.qs * c.ks, o, o_hi, o_lo,
                     ldo, c.nseq, c.N, c.H, A.SCALE)
    else:
        _cabi().call("omt_attn_spatial_h1", qh, cols, kh, cols, vh, cols, vinv, c.qs * c.ks, o, o_hi, ldo, c.nseq, c.N,
                     c.H, A.SCALE)
    torch.cuda.synchronize()
    _check_guards(buf, c.M, cols, SENT16 if planes else SENT32)
    return buf


def _run(c, mode, dev, target=None):
    cols = c.H * 64
    runs = [_launch(c, mode, dev) for _ in range(3)]
    for b in runs[1:]:
        assert torch.equal(b.view(torch.int32), runs[0].view(torch.int32)), f"{c.name} [{mode}]: launches differ"
    o = runs[0][PRE:PRE + c.M, :cols].cpu()
    ok, r, e, b, bad = A.evaluate(c, mode, out=o, target=target)
    note = " (hull check only, not an accuracy check)" if b >= 1 else ""
    print(f"[attn-f16-edges] {c.name} [{mode}]: worst err/bound {r:.3g}, worst err/mag {e:.2e}, "
          f"worst bound/mag {b:.2e}{note}")
    assert ok, f"{c.name} [{mode}]: {bad} rows differ from the model's exact bits or leave the bound"
    op = _launch(c, mode, dev, planes=True)
    hi, lo = op[0, PRE:PRE + c.M, :cols].cpu(), op[1, PRE:PRE + c.M, :cols].cpu()
    if mode == "x3":
        wh, wl = L.split_f16(o)
        assert torch.equal(hi, wh.view(torch.int16)) and torch.equal(lo, wl.view(torch.int16)), f"{c.name}: O planes"
    else:
        assert torch.equal(hi, o.clamp(-65504, 65504).half().view(torch.int16)), f"{c.name}: O hi plane"
        assert bool((lo == SENT16).all()), f"{c.name}: the x1 core wrote an O lo plane"


@pytest.fixture(scope="module")
def planted():
    return A.planted_cases()


@pytest.mark.parametrize("mode", A.MODES)
@pytest.mark.parametrize("idx", [0, 1, 2])
def test_planted(cuda, planted, idx, mode):
    c, target, _ = planted[idx]
    _run(c, mode, cuda, target)


@pytest.mark.parametrize("mode", A.MODES)
@pytest.mark.parametrize("idx", range(len(A.SPREADS) + 1))
def test_spread(cuda, idx, mode):
    _run(A.spread_cases()[idx], mode, cuda)


@pytest.mark.parametrize("mode", A.MODES)
@pytest.mark.parametrize("idx", range(len(A.LOGIT_SCALES) + 1))
def test_logit_range(cuda, idx, mode):
    _run(A.logit_cases()[idx], mode, cuda)


# ------------------------------------------------------------------------------------------------------ layer survey
class _Dev:
    """A device array view of raw engine memory: [rows, cols] fp16 at `ptr` with row stride `ld` elements."""

    def __init__(self, ptr, rows, cols, ld):
        self.__cuda_array_interface__ = {"shape": (rows, cols), "typestr": "<f2", "data": (ptr, False),
                                         "strides": (ld * 2, 2), "version": 3}


def _survey_calls(monkeypatch, found):
    real = _cabi().call

    def call(name, *a):
        real(name, *a)
        if name not in ("omt_attn_spatial_h", "omt_attn_spatial_h1") or torch.cuda.is_current_stream_capturing():
            return
        if name == "omt_attn_spatial_h":
            qp, ld, kp, vinv, qkps, n_seq, N, H = a[0], a[2], a[3], a[9], a[10], a[15], a[16], a[17]
        else:
            qp, ld, kp, vinv, qkps, n_seq, N, H = a[0], a[1], a[2], a[6], a[7], a[11], a[12], a[13]
        torch.cuda.synchronize()
        M = n_seq * N
        q = torch.as_tensor(_Dev(qp, M, H * 64, ld), device="cuda").float().view(n_seq, N, H, 64).transpose(1, 2)
        k = torch.as_tensor(_Dev(kp, M, H * 64, ld), device="cuda").float().view(n_seq, N, H, 64).transpose(1, 2)
        lg = max(float((q[s] @ k[s].transpose(-1, -2)).abs().max()) for s in range(n_seq)) * A.SCALE / qkps
        vi = vinv[:, :M].reshape(H, n_seq, N)
        sp = float(torch.log2(vi.amax(-1) / vi.amin(-1)).max())
        found.append((lg, sp, name, n_seq, N, H))

    monkeypatch.setattr(_cabi(), "call", call)


def _survey_models(dev, monkeypatch):
    for name in ("img64", "vid5x64", "vid9x128_b2", "img256_cfg1"):
        cfg, sd, x = golden_setup(load_golden(name))
        yield name, build_model(cfg, sd, dev, "f16x3"), [x]
    wg = torch.load(os.path.join(os.path.dirname(__file__), "golden", "widths.pt"), weights_only=False)
    for name in ("w256_h8", "w256_h4", "w512_h4", "w768_h12", "w1024_h16"):
        row = wg[name]
        cfg, sd, xs = flags_setup(row)
        monkeypatch.setenv("OMT_MATH", "f16x3")
        m = ob.OmniTokenizer_VQGAN(flags_namespace(row))
        m.load_state_dict(sd, strict=False)
        m.codebook._need_init = False
        yield name, m.to(dev).eval(), xs


def test_layer_survey(cuda, monkeypatch):
    """Per attention layer of the golden configurations: the largest per-(sequence, head) vinv spread in the engine's
    ws.vinv and the largest |logit|.  The sweeps of attn_f16_cases cover both with 2^6 to spare.  Each layer is read on
    the first (eager) encode and decode of its shape, before any CUDA graph is captured."""
    sweep_sp = max(A.max_logit(c)[1] for c in A.spread_cases())
    sweep_lg = max(A.max_logit(c)[0] for c in A.logit_cases() + [p[0] for p in A.planted_cases()])
    worst_sp, worst_lg, ran = 0.0, 0.0, []
    for name, m, xs in _survey_models(cuda, monkeypatch):
        found = []
        _survey_calls(monkeypatch, found)
        with torch.no_grad():
            for x in xs:
                is_image = x.ndim == 4
                _, idx = m.encode(x.to(cuda), is_image, include_embeddings=True)
                m.decode(idx, is_image)
        monkeypatch.undo()
        if not found:       # token grids of 64 tokens (N % 128 != 0) run the fp32-operand core
            print(f"[attn-f16-survey] {name}: no layer on the f16 core")
            continue
        ran.append(name)
        for i, (lg, sp, entry, n_seq, N, H) in enumerate(found):
            print(f"[attn-f16-survey] {name} call {i} ({entry}, {n_seq} sequences x {N} tokens, {H} heads): "
                  f"|logit| {lg:.2f}, vinv spread 2^{sp:.1f}")
        lg, sp = max(f[0] for f in found), max(f[1] for f in found)
        print(f"[attn-f16-survey] {name}: {len(found)} layer calls, largest |logit| {lg:.2f}, "
              f"largest vinv spread 2^{sp:.1f}")
        worst_sp, worst_lg = max(worst_sp, sp), max(worst_lg, lg)
    print(f"[attn-f16-survey] all: |logit| {worst_lg:.2f} (sweep {sweep_lg:.0f}), spread 2^{worst_sp:.1f} "
          f"(sweep 2^{sweep_sp:.1f})")
    assert {"vid9x128_b2", "img256_cfg1"} <= set(ran)
    assert worst_sp + 6 <= sweep_sp
    assert worst_lg * 64 <= sweep_lg
