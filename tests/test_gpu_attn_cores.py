"""The fp32-operand attention cores across their grids, strides and output forms:

* attn_tc3_kernel (csrc/attention_tc3.cu), the 3xTF32 wgmma spatial core: omt_attn_spatial with N % 128 == 0;
* attn_flash_kernel<false> (csrc/attention_fp32.cu), the CUDA-core spatial core: N % 128 != 0, or attn_kernel = 1;
* attn_flash_kernel<true>, the window core: every window block;
* attn_temporal_kernel<T'> for every T' from 1 to 17: every temporal block.

The operands (tests/attn_cases.py) sit in separate q, k, v buffers with distinct leading dimensions and NaN padding
columns.  Every output lands in a sentinel-filled buffer with guard rows on both sides and a leading dimension wider than
the heads; the guards must survive every launch.  Each shape runs three times into fp32 outputs (the launches must agree
bit for bit) and once into fp16 hi / lo operand planes, which must equal layout.split_f16 of the fp32 output bit for bit:
both forms compute the same value and split it with the rounding split_f16 restates.  Results are compared with fp64
softmax attention relative to each output row's magnitude; planted cases must return v of their target key.  One launch
must equal launches on sub-ranges of its sequences, frames or videos bit for bit, the grids reach 65 535 sequences and
more than 65 535 windows, and bad arguments raise before anything is launched.
"""
import pytest
import torch

from omnitokenizer_b200 import layout as L
from tests import attn_cases as A

pytestmark = pytest.mark.gpu

SENT32 = 0x7FBADBAD          # fp32 NaN pattern of the fp32 output buffers
SENT16 = 0x7E5B              # fp16 NaN pattern of the plane buffers
PRE, POST = 3, 5             # guard rows before and after every output
OUT_EXTRA = 8                # ldo = 64 heads + 8: columns past the heads are guards as well


def _cabi():
    from omnitokenizer_b200 import _cabi
    _cabi.load()
    return _cabi


def _f32_buf(rows, ld, dev):
    b = torch.empty(PRE + rows + POST, ld, device=dev)
    b.view(torch.int32).fill_(SENT32)
    return b


def _f16_buf(rows, ld, dev):
    return torch.full((2, PRE + rows + POST, ld), SENT16, dtype=torch.int16, device=dev)


def _check_guards(buf, rows, cols, sent, what):
    bits = buf.view(torch.int32) if buf.dtype == torch.float32 else buf
    assert bool((bits[..., :PRE, :] == sent).all()), f"{what}: guard rows before the output were written"
    assert bool((bits[..., PRE + rows:, :] == sent).all()), f"{what}: guard rows after the output were written"
    assert bool((bits[..., PRE:PRE + rows, cols:] == sent).all()), f"{what}: columns beyond the heads were written"


def launch(case, out, ldo, planes=False, u0=0, u1=None):
    """Run the case's entry point on units [u0, u1) (sequences, frames or videos) by offsetting every pointer, writing
    rows PRE + ... of `out` (an fp32 buffer, or the [2, rows, ldo] plane pair with planes=True)."""
    t = case.topo
    u1 = t.units if u1 is None else u1
    r0 = u0 * t.unit_rows
    q, k, v = case.qb[r0:], case.kb[r0:], case.vb[r0:]
    o, o_hi, o_lo = (None, out[0, PRE + r0:], out[1, PRE + r0:]) if planes else (out[PRE + r0:], None, None)
    args = (q, case.ldq, k, case.ldk, v, case.ldv, o, o_hi, o_lo, ldo)
    if t.kind == "spatial":
        _cabi().call("omt_attn_spatial", *args, u1 - u0, t.dims["N"], case.H, case.scale)
    elif t.kind == "window":
        _cabi().call("omt_attn_window", *args, case.bias, u1 - u0, t.dims["h"], t.dims["w"], 8, case.H, case.scale)
    else:
        _cabi().call("omt_attn_temporal", *args, u1 - u0, t.dims["T"], t.dims["N"], case.H, case.scale, int(t.causal))


def _check(case, o, bar, what, set_ids=None):
    """Planted: v_t(i) to 1e-6 of the magnitude of each head's 64 columns (the heads of one row return v rows of very
    different magnitude).  Otherwise fp64 attention to `bar` of the row's magnitude, taken as in
    test_gpu_attn_walk._check_accuracy but of softmax(...) |v| rather than of the output itself: the v rows' magnitudes
    spread over four decades and their signs cancel in the weighted sum, so the output of a row can be far smaller than
    the terms it is summed from, and the fp32 rounding of those terms is what any kernel's error scales with."""
    rows = case.rows(set_ids)
    got = o[rows].double()
    assert not bool(torch.isnan(got).any()), f"{what}: NaN in the output (an unwritten row or a read of the padding)"
    if case.family == "planted":
        want = case.answer(set_ids).double().view(got.shape[0], -1, 64)
        got = got.view(want.shape)
        rel = ((got - want).abs() / want.abs().amax(dim=-1, keepdim=True)).max().item()
        bar = 1e-6
    else:
        want, mag = case.reference(set_ids, magnitude=True)
        rel = ((got - want).abs() / mag.amax(dim=1, keepdim=True)).max().item()
    print(f"[attn-cores] {what}: max rel err {rel:.2e} (bar {bar:.0e})")
    assert rel < bar, f"{what}: max error relative to the row magnitude {rel:.2e} >= {bar:.0e}"


def _sweep(case, bar, what):
    """Three fp32 launches (guards, bit-equal), accuracy, and the plane form (guards, = split_f16 bit for bit)."""
    dev, M, C = case.device, case.topo.M, case.H * 64
    ldo = C + OUT_EXTRA
    runs = []
    for _ in range(3):
        buf = _f32_buf(M, ldo, dev)
        launch(case, buf, ldo)
        torch.cuda.synchronize()
        _check_guards(buf, M, C, SENT32, what)
        runs.append(buf)
    for b in runs[1:]:
        assert torch.equal(b.view(torch.int32), runs[0].view(torch.int32)), f"{what}: launches differ"
    o = runs[0][PRE:PRE + M, :C]
    _check(case, o, bar, what)
    op = _f16_buf(M, ldo, dev)
    launch(case, op, ldo, planes=True)
    torch.cuda.synchronize()
    _check_guards(op, M, C, SENT16, what + " planes")
    hi, lo = L.split_f16(o)
    for name, got, want in (("hi", op[0, PRE:PRE + M, :C], hi), ("lo", op[1, PRE:PRE + M, :C], lo)):
        bad = (got != want.view(torch.int16)).sum().item()
        assert bad == 0, f"{what}: {bad} {name} plane elements differ from split_f16 of the fp32 output"


# ---------------------------------------------------------------- tc3 spatial (N % 128 == 0, attn_kernel = 3)

# Error bars, relative to the row magnitude of _check, for up to 1024 keys:
#  * CUDA-core cores, model / ramp operands: 5e-6, test_qk_prep_and_spatial_attention's bar (observed up to 2.1e-6).
#  * tc3, model / ramp: 2e-5.  3xTF32 drops the lo.lo products and the tensor cores read the lo halves as tf32 (their
#    last 13 bits go), so each product carries about 2^-21 where fp32 carries 2^-24; over the 20 M outputs of the cfg-3
#    shape (40 x 1024 tokens, 8 heads) the largest error reaches 1.1e-5, beyond test_qk_prep_and_spatial_attention's
#    1e-5 for 3 sequences.
#  * hot operands, every core: 4e-5.  A logit of ~70 is the fp32 sum of 64 products whose magnitudes add up to ~130, so
#    it carries an absolute rounding error of up to ~130 * 2^-24 * sqrt(64) ~ 6e-5, which exp() hands on as relative
#    error of its weight.  test_temporal_attention's 2e-5 covers up to 9 keys; with 192 .. 1024 keys the row maxima
#    grow and the observed error reaches 3.2e-5.
FP32_BAR, TC3_BAR, HOT_BAR = 5e-6, 2e-5, 4e-5


def _bar(family, base, N=64):
    """The fp32 sums over the keys (P.V and the row sum) gather rounding error at most in proportion to their length,
    so the bars grow with N / 1024 beyond 1024 keys: 4x at N = 4096."""
    return (HOT_BAR if family == "hot" else base) * max(1, N // 1024)


# (N, heads, n_seq, family): every N with every family and every head count; 40 x 1024 x 8 heads is the cfg-3 shape
TC3 = [(128, 1, 37, "model"), (128, 3, 5, "ramp"), (128, 8, 2, "planted"), (128, 8, 3, "hot"),
       (384, 3, 1, "model"), (384, 8, 3, "ramp"), (384, 1, 6, "planted"),
       (1024, 8, 40, "model"), (1024, 1, 2, "ramp"), (1024, 3, 3, "planted"), (1024, 8, 2, "hot"),
       (4096, 1, 2, "model"), (4096, 8, 1, "ramp"), (4096, 3, 1, "planted")]


@pytest.mark.parametrize("N,H,nseq,family", TC3)
def test_tc3_spatial(cuda, N, H, nseq, family):
    case = A.Case(A.Topology.spatial(nseq, N), H, family, 1000 + N + H + nseq, cuda)
    _sweep(case, _bar(family, TC3_BAR, N), f"tc3 N={N} H={H} n_seq={nseq} {family}")


# ---------------------------------------------------------------- CUDA-core spatial (N % 128 != 0, or attn_kernel = 1)

FLASH = [(64, 8, 7, "model"), (64, 1, 3, "planted"), (192, 3, 4, "ramp"), (192, 8, 2, "planted"), (192, 1, 5, "hot"),
         (320, 1, 3, "model"), (320, 8, 1, "planted"), (320, 3, 2, "ramp"),
         (1024, 8, 3, "model"), (1024, 3, 2, "planted"), (1024, 1, 2, "hot"),
         (4096, 1, 2, "ramp"), (4096, 3, 1, "planted"), (4096, 8, 1, "model")]


@pytest.mark.parametrize("N,H,nseq,family", FLASH)
def test_flash_spatial(cuda, N, H, nseq, family):
    if N % 128 == 0:
        _cabi().set_option("attn_kernel", 1)
    case = A.Case(A.Topology.spatial(nseq, N), H, family, 2000 + N + H + nseq, cuda)
    _sweep(case, _bar(family, FP32_BAR, N), f"flash N={N} H={H} n_seq={nseq} {family}")


# ---------------------------------------------------------------- window (8x8 windows, relative position bias)

WINDOW = [(8, 8, 1, 1, "real", "model"), (8, 8, 9, 8, "random", "planted"), (16, 16, 3, 8, "real", "ramp"),
          (16, 16, 2, 1, "real", "planted"), (8, 24, 5, 8, "real", "model"), (8, 24, 2, 1, "random", "hot"),
          (24, 8, 4, 1, "real", "planted"), (24, 8, 7, 8, "real", "ramp"), (16, 16, 1, 8, "random", "model")]


@pytest.mark.parametrize("h,w,frames,H,bias,family", WINDOW)
def test_window(cuda, h, w, frames, H, bias, family):
    b = A.real_window_bias(H, 30 + h + w) if bias == "real" else A.random_window_bias(H, 40 + h + w)
    case = A.Case(A.Topology.window(frames, h, w), H, family, 3000 + h * w + frames + H, cuda, bias=b)
    _sweep(case, _bar(family, FP32_BAR), f"window {h}x{w} frames={frames} H={H} {bias} bias {family}")


# ---------------------------------------------------------------- temporal: every T' the entry point takes

def _temporal_shape(T):
    """(B, N, heads) for T': N over {1, 3, 64, 1024}, heads over {1, 8}; B N heads is not a multiple of 8 (a partial
    last block of 8 warps) at N = 1 and 3 with one head."""
    N = (1, 3, 64, 1024)[T % 4]
    H = 8 if T % 3 == 0 else 1
    B = 3 if N <= 3 else (2 if N == 64 else 1)
    return B, N, H


@pytest.mark.parametrize("causal", [1, 0])
@pytest.mark.parametrize("T", range(1, 18))
def test_temporal(cuda, T, causal):
    B, N, H = _temporal_shape(T)
    topo = A.Topology.temporal(B, T, N, causal)
    for family in ("planted", ("model", "ramp", "hot")[T % 3]):
        case = A.Case(topo, H, family, 4000 + 2 * T + causal, cuda)
        _sweep(case, _bar(family, FP32_BAR), f"temporal T'={T} causal={causal} B={B} N={N} H={H} {family}")


# ---------------------------------------------------------------- placement: one launch = launches on sub-ranges

PLACEMENT = {
    "tc3": (lambda: A.Topology.spatial(7, 256), 3, [(0, 1), (1, 4), (4, 6), (6, 7)]),
    "flash": (lambda: A.Topology.spatial(5, 192), 8, [(0, 2), (2, 3), (3, 5)]),
    "window": (lambda: A.Topology.window(7, 8, 24), 8, [(0, 1), (1, 3), (3, 7)]),
    "temporal": (lambda: A.Topology.temporal(5, 9, 64, 1), 8, [(0, 1), (1, 4), (4, 5)]),
    "temporal-odd": (lambda: A.Topology.temporal(5, 17, 3, 0), 1, [(0, 2), (2, 3), (3, 5)]),
}


@pytest.mark.parametrize("name", list(PLACEMENT))
def test_placement_invariance(cuda, name):
    """Every sequence, window and pixel decodes to the same rows whichever part of the grid runs it, and no launch reads
    rows outside its own range: one launch equals launches on sub-ranges (pointers offset), bit for bit."""
    make, H, parts = PLACEMENT[name]
    topo = make()
    bias = A.real_window_bias(H, 7) if topo.kind == "window" else None
    case = A.Case(topo, H, "ramp", 91, cuda, bias=bias)
    C = H * 64
    ldo = C + OUT_EXTRA
    whole, split = _f32_buf(topo.M, ldo, cuda), _f32_buf(topo.M, ldo, cuda)
    launch(case, whole, ldo)
    for u0, u1 in parts:
        launch(case, split, ldo, u0=u0, u1=u1)
    torch.cuda.synchronize()
    _check_guards(split, topo.M, C, SENT32, name)
    assert torch.equal(whole.view(torch.int32), split.view(torch.int32)), f"{name}: sub-range launches differ"
    _check(case, whole[PRE:PRE + topo.M, :C], TC3_BAR if name == "tc3" else FP32_BAR, f"placement {name}")


# ---------------------------------------------------------------- grid limits

def _sample(n, k, seed):
    """First and last sequence, both sides of the 2^12 and 2^15 boundaries, and k random ones."""
    g = torch.Generator().manual_seed(seed)
    fixed = [s for s in (0, 1, 4095, 4096, 32767, 32768, n - 2, n - 1) if 0 <= s < n]
    return torch.tensor(sorted(set(fixed + torch.randint(0, n, (k,), generator=g).tolist())))


def _grid_limit(case, bar, what):
    """One fp32 launch over the whole grid (about 4 to 10 GB of operands and output); guards, every row written, and
    fp64 attention on a sample of sequences."""
    M = case.topo.M
    ldo = 64 + OUT_EXTRA
    buf = _f32_buf(M, ldo, case.device)
    launch(case, buf, ldo)
    torch.cuda.synchronize()
    _check_guards(buf, M, 64, SENT32, what)
    o = buf[PRE:PRE + M, :64]
    assert bool(torch.isfinite(o).all()), f"{what}: rows left unwritten"
    _check(case, o, bar, what, _sample(case.topo.sets.shape[0], 8, M))


def test_grid_limit_flash_spatial(cuda):
    """n_seq = 65 535 (the gridDim.z limit) at N = 64, one head: the CUDA-core core."""
    _grid_limit(A.Case(A.Topology.spatial(65535, 64), 1, "model", 5, cuda), FP32_BAR, "flash n_seq=65535")


def test_grid_limit_tc3_spatial(cuda):
    """n_seq = 65 535 at N = 128, one head: the tc3 core, whose tensor maps span all 8.4 M rows."""
    _grid_limit(A.Case(A.Topology.spatial(65535, 128), 1, "model", 6, cuda), TC3_BAR, "tc3 n_seq=65535")


def test_grid_limit_window(cuda):
    """65 700 windows, one head (3 windows of an 8x24 grid in each of 21 900 frames): window sequences run on gridDim.x
    so that they can exceed the 65 535 of gridDim.z."""
    topo = A.Topology.window(21900, 8, 24)
    assert topo.sets.shape[0] > 65535
    _grid_limit(A.Case(topo, 1, "model", 7, cuda, bias=A.real_window_bias(1, 8)), FP32_BAR, "window 65700 windows")


# ---------------------------------------------------------------- loud errors

def test_bad_arguments_raise(cuda):
    """Each rejected call raises a RuntimeError whose message names the entry point and the reason, and writes nothing."""
    x = torch.zeros(8 * 1024, 516, device=cuda)
    bias = torch.zeros(8, 64, 64, device=cuda)
    out = _f32_buf(8 * 1024, 516, cuda)

    def io(ldq=512, ldo=512, o=out[PRE:]):
        return (x, ldq, x, 512, x, 512, o, None, None, ldo)

    # entry point, geometry arguments that are valid on their own
    good = {"omt_attn_spatial": (1, 64, 8, 8.0), "omt_attn_window": (bias, 1, 8, 8, 8, 8, 8.0),
            "omt_attn_temporal": (1, 2, 64, 8, 8.0, 1)}
    cases = [("omt_attn_spatial", io() + (1, 96, 8, 8.0), "N=96 must be a multiple of 64"),
             ("omt_attn_spatial", io() + (65536, 64, 1, 8.0), "grid too large"),
             ("omt_attn_window", io() + (bias, 1, 8, 8, 4, 8, 8.0), "window 4x4 unsupported"),
             ("omt_attn_window", io() + (bias, 1, 12, 8, 8, 8, 8.0), "grid 12x8 not divisible"),
             ("omt_attn_temporal", io() + (1, 0, 64, 8, 8.0, 1), r"T'=0 unsupported \(1..17\)"),
             ("omt_attn_temporal", io() + (1, 18, 64, 8, 8.0, 1), r"T'=18 unsupported \(1..17\)")]
    for name, geometry in good.items():
        cases += [(name, io(ldq=514) + geometry, "multiples of 4"),
                  (name, io(ldo=510) + geometry, "multiples of 4"),
                  (name, io(o=None) + geometry, "null pointer")]
    for name, args, reason in cases:
        with pytest.raises(RuntimeError, match=f"{name}: .*{reason}"):
            _cabi().call(name, *args)
    torch.cuda.synchronize()
    assert bool((out.view(torch.int32) == SENT32).all()), "a rejected call wrote its output"


def test_videos_past_the_temporal_limit_raise_before_any_launch(cuda):
    """More than 17 latent frames (69 frames at temporal patch 4) is refused by encode and decode up front, naming the
    temporal core's limit, instead of after the patch embed and the spatial blocks have run; 17 latent frames run."""
    import omnitokenizer_b200 as ob
    from oracle import omni_oracle as oo
    from oracle import weights as W
    from tests.util import namespace_from_cfg
    cfg = oo.Config(resolution=64)
    m = ob.OmniTokenizer_VQGAN(namespace_from_cfg(cfg))
    m.load_state_dict(W.make_state_dict(cfg, 0), strict=False)
    m.codebook._need_init = False
    m = m.to(cuda).eval().prepare()
    cabi = _cabi()
    n0 = cabi.launch_count
    with pytest.raises(NotImplementedError, match="at most 17 latent frames"):
        m.encode(torch.zeros(1, 3, 69, 64, 64, device=cuda), False)
    with pytest.raises(NotImplementedError, match="at most 17 latent frames"):
        m.decode(torch.zeros(1, 18, 8, 8, dtype=torch.int64, device=cuda), False)
    assert cabi.launch_count == n0, "kernels were launched before the frame count was rejected"
    idx = m.encode(torch.zeros(1, 3, 65, 64, 64, device=cuda), False)
    assert tuple(idx.shape) == (1, 17, 8, 8)
    assert tuple(m.decode(idx, False).shape) == (1, 3, 65, 64, 64)
