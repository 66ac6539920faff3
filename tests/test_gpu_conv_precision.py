"""omt_conv3d's 3xTF32 correction products at every conv geometry of the metric networks (conv_cases.py), and the
per-layer error of the four networks that run on it.

* Split-grid operands (non-zero lo parts, every product and partial sum exact in fp32): the output equals the fp64
  A_hi.W_hi + A_lo.W_hi + A_hi.W_lo (+ bias, ReLU) bit for bit, in a sentinel-filled buffer whose guard bands and
  neighbouring columns keep their bits.  A wrong lo descriptor, stage or warpgroup half, or a missing correction wgmma,
  moves an output by a multiple of 2^-12.
* Realistic operands against fp64: max |y - y64| / sqrt(sum (x w)^2 + b^2) <= conv_cases.L2_BOUND.
* Per layer of FIDInception, both I3Ds and the VGG LPIPS, run eagerly: each conv against the fp64 conv of its own GPU
  input (so errors do not compound), next to torch's CPU fp32 conv of the same input; every pool bit for bit.
* omt_i3d_head and omt_lpips_input against direct references, and the grid-stride loops of the pooling and input kernels
  at sizes past their 65 536-block grids."""
import os

import pytest
import torch
import torch.nn.functional as F

from omnitokenizer_b200 import _cabi, fid, fvd, quality
from oracle import fid_oracle as fo
from oracle import fvd_suite_oracle as so
from oracle import i3d_oracle as io
from oracle import quality_oracle as qo
from tests import conv_cases as cc

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
SMS = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else cc.H100_SMS
CASES = cc.all_cases(SMS)
SENTINEL = 0x7FC0BEEF             # a NaN with a payload: any store over it changes the bits
GUARD = 256                       # floats before and after the output rows


def _launch(c: cc.ConvCase, x, w, b, relu):
    """omt_conv3d on the case; returns (output (B, To, Ho, Wo, cout) fp32 on the device, untouched-bits ok)."""
    w_hi, w_lo = cc.pack(w, c)
    xd = cc.to_cl(x, c.Cs).to(DEV)
    n = c.M * c.ldy
    buf = torch.full((GUARD + n + GUARD,), SENTINEL, dtype=torch.int32, device=DEV).view(torch.float32)
    _cabi.call("omt_conv3d", xd, c.Cs, c.B, *c.dims, w_hi.to(DEV), w_lo.to(DEV), c.K, b.to(DEV), c.cout, *c.k, *c.s,
               *c.front, *c.out, buf.data_ptr() + 4 * (GUARD + c.col), c.ldy, int(relu))
    torch.cuda.synchronize()
    bits = buf.view(torch.int32)
    rows = bits[GUARD:GUARD + n].view(c.M, c.ldy)
    kept = torch.cat([bits[:GUARD], bits[GUARD + n:], rows[:, :c.col].reshape(-1), rows[:, c.col + c.cout:].reshape(-1)])
    y = buf[GUARD:GUARD + n].view(c.M, c.ldy)[:, c.col:c.col + c.cout].reshape(c.B, *c.out, c.cout)
    return y, bool((kept == SENTINEL).all())


@pytest.mark.parametrize("relu", [False, True], ids=["linear", "relu"])
@pytest.mark.parametrize("c", CASES, ids=[c.id for c in CASES])
def test_split_grid_bit_exact(c, relu):
    x, w, b = cc.split_grid_operands(c, 11 + relu)
    y, kept = _launch(c, x, w, b, relu)
    ref = cc.split_grid_reference(x.to(DEV), w.to(DEV), b, c, relu)
    assert kept, "a store outside the output columns"
    diff = (y != ref) & ~(torch.isnan(y) & torch.isnan(ref))
    assert not bool(diff.any()), (f"{int(diff.sum())} of {y.numel()} outputs differ, max "
                                  f"{float((y - ref).abs().nan_to_num(float('inf')).max())}")


@pytest.mark.parametrize("c", CASES, ids=[c.id for c in CASES])
def test_realistic_operands_against_fp64(c):
    x, w, b = cc.realistic_operands(c, 21)
    y, kept = _launch(c, x, w, b, False)
    xd, wd, bd = x.to(DEV), w.to(DEV), b.to(DEV)
    err = cc.l2_error(y, cc.conv64(xd, wd, c, bd), cc.l2_scale(xd, wd, bd, c))
    print(f"{c.id}: {err:.2e} of the l2 norm")
    assert kept
    assert err <= cc.L2_BOUND, err


# ---------------------------------------------------------------- per-layer error of the four networks

def _tensors(ws):
    """Every tensor a workspace's launch list refers to (closure cells, default arguments, attributes)."""
    out = [v for v in vars(ws).values() if isinstance(v, torch.Tensor)]
    for op in ws.ops:
        cells = [cl.cell_contents for cl in (op.__closure__ or ())] + list(op.__defaults__ or ())
        out += [v for v in cells if isinstance(v, torch.Tensor) and v.is_cuda]
    return out


def _at(tensors, ptr, rows, ld, n):
    """The (rows, n) fp32 matrix of row stride ld at device address ptr, as a view of the tensor that holds it."""
    for t in tensors:
        if t.dtype == torch.float32 and t.data_ptr() <= ptr < t.data_ptr() + 4 * t.numel():
            return t.as_strided((rows, n), (ld, 1), t.storage_offset() + (ptr - t.data_ptr()) // 4)
    raise AssertionError(f"no workspace tensor holds address {ptr:#x}")


class Recorder:
    """Wraps _cabi.call: after every omt_conv3d it synchronises and measures the layer against the fp64 conv of its
    own GPU input with the unit's w_hi + w_lo and bias, and torch's CPU fp32 conv against the same fp64; every
    omt_maxpool3d / omt_pool2d is checked against torch's CPU pooling bit for bit."""

    def __init__(self, ws):
        self.tensors = _tensors(ws)
        self.layers = []            # (index, geometry, gpu error, cpu fp32 error)
        self.pools = 0
        self.drift = []             # (gpu, cpu fp32) per conv
        self.call = _cabi.call

    def __call__(self, name, *a):
        self.call(name, *a)
        if name == "omt_conv3d":
            torch.cuda.synchronize()
            self.conv(*a)
        elif name in ("omt_maxpool3d", "omt_pool2d"):
            torch.cuda.synchronize()
            getattr(self, name[4:])(*a)
            self.pools += 1

    def conv(self, x, Cs, B, T, H, W, w_hi, w_lo, K, bias, N, kt, kh, kw, st, sh, sw, pt, ph, pw, To, Ho, Wo, y, ldy,
             relu):
        c = cc.ConvCase("", B, Cs, Cs, N, (kt, kh, kw), (st, sh, sw), (pt, ph, pw), (T, H, W), (To, Ho, Wo), 0, ldy)
        x64 = x.reshape(B, T, H, W, Cs).permute(0, 4, 1, 2, 3).double()
        w = (w_hi.double() + w_lo.double())[:N, :c.taps * Cs].reshape(N, kt, kh, kw, Cs).permute(0, 4, 1, 2, 3)
        ref = cc.conv64(x64, w, c, bias)
        got = _at(self.tensors, y if isinstance(y, int) else y.data_ptr(), c.M, ldy, N).reshape(ref.shape)
        scale = cc.l2_scale(x64, w, bias, c)
        fr, bk = c.front, c.back()
        xp = F.pad(x64.float().cpu(), (fr[2], bk[2], fr[1], bk[1], fr[0], bk[0]))
        y32 = F.conv3d(xp, w.float().cpu(), bias.cpu(), stride=c.s).permute(0, 2, 3, 4, 1).to(DEV)
        if relu:
            ref, y32 = ref.clamp_min(0), y32.clamp_min(0)
        e, e32 = ((t.double() - ref) / scale for t in (got, y32))
        self.layers.append((len(self.layers), f"{Cs}->{N} k{kt}{kh}{kw} s{st}{sh}{sw} {T}x{H}x{W}",
                            float(e.abs().max()), float(e32.abs().max())))
        # drift: the mean of error * sign(y64) over the mean |error|: 0 for unbiased rounding, -1 when every output is
        # pulled toward zero
        self.drift.append(tuple(float((t * ref.sign()).mean() / t.abs().mean().clamp_min(1e-300)) for t in (e, e32)))

    def maxpool3d(self, x, Cs, B, T, H, W, kt, kh, kw, st, sh, sw, pt, ph, pw, To, Ho, Wo, y):
        back = [(o - 1) * s + k - n - f for o, s, k, n, f in zip((To, Ho, Wo), (st, sh, sw), (kt, kh, kw), (T, H, W),
                                                                   (pt, ph, pw))]
        xc = x.cpu().permute(0, 4, 1, 2, 3)
        ref = F.max_pool3d(F.pad(xc, (pw, back[2], ph, back[1], pt, back[0])), (kt, kh, kw), (st, sh, sw))
        assert torch.equal(y.cpu(), ref.permute(0, 2, 3, 4, 1)), "omt_maxpool3d differs from torch"

    def pool2d(self, x, Cs, C, B, H, W, kh, kw, sh, sw, ph, pw, Ho, Wo, y, ldy, mode):
        xc = x.reshape(B, H, W, Cs)[..., :C].cpu().permute(0, 3, 1, 2).contiguous()
        if mode == fid.POOL_MAX:
            ref = F.max_pool2d(xc, (kh, kw), (sh, sw), (ph, pw))
        else:
            ref = F.avg_pool2d(xc, (kh, kw), (sh, sw), (ph, pw), count_include_pad=False)
        got = _at(self.tensors, y if isinstance(y, int) else y.data_ptr(), B * Ho * Wo, ldy, C)
        assert torch.equal(got.cpu(), ref.permute(0, 2, 3, 1).reshape(-1, C)), "omt_pool2d differs from torch"


def _fid_ws():
    g = torch.load(os.path.join(GOLDEN, "fid_inception.pt"))
    sd = fo.make_state_dict(g["w_seed"])
    sd.update(g["bn"])
    ws = fid._Workspace(fid.FIDInception(sd, DEV), 1, 64, 80)
    ws.u8.copy_(fo.image_bytes((64, 80), 5)[None])
    return ws


def _i3d_sd(seed_key, bn_key, path):
    g = torch.load(path)
    sd = io.make_state_dict(g[seed_key])
    sd.update(g[bn_key])
    return sd


def _clip(T, seed):
    return torch.randint(0, 256, (1, T, 64, 64, 3), generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


def _videogpt_ws():
    ws = fvd._Workspace(fvd.I3D(_i3d_sd("w_seed", "bn", os.path.join(GOLDEN, "fvd_i3d.pt")), DEV), 1, 9, 64, 64)
    ws.u8.copy_(_clip(9, 6))
    return ws


def _styleganv_ws():
    sd = so.styleganv_keys(_i3d_sd("sgv_seed", "sgv_bn", os.path.join(GOLDEN, "fvd_suite.pt")))
    ws = fvd._Workspace(fvd.load_i3d_styleganv(DEV, sd), 1, 10, 64, 64)
    ws.u8.copy_(_clip(10, 7))
    return ws


def _lpips_ws():
    g = torch.load(os.path.join(GOLDEN, "quality.pt"))
    ws = quality._Workspace(DEV, quality.FORM_U8, 1, 48, 64, None, quality.LPIPS(qo.make_state_dict(g["w_seed"]), DEV))
    for t, seed in ((ws.a, 8), (ws.b, 9)):
        t.copy_(torch.randint(0, 256, tuple(t.shape), generator=torch.Generator().manual_seed(seed), dtype=torch.uint8))
    return ws


NETS = {"fid": (_fid_ws, 94, 14), "i3d_videogpt": (_videogpt_ws, 57, 13), "i3d_styleganv": (_styleganv_ws, 57, 13),
        "lpips": (_lpips_ws, 13, 4)}


@pytest.mark.parametrize("net", list(NETS))
def test_network_layers_against_fp64(net, monkeypatch):
    make, n_conv, n_pool = NETS[net]
    ws = make()
    rec = Recorder(ws)
    monkeypatch.setattr(_cabi, "call", rec)
    with torch.no_grad():
        ws.run()
    monkeypatch.undo()
    assert len(rec.layers) == n_conv and rec.pools == n_pool
    gpu = torch.tensor([e for *_, e, _ in rec.layers])
    cpu = torch.tensor([e for *_, e in rec.layers])
    print(f"\n{net}: {n_conv} convs, error / l2 norm: 3xTF32 max {float(gpu.max()):.2e} median "
          f"{float(gpu.median()):.2e}; CPU fp32 max {float(cpu.max()):.2e} median {float(cpu.median()):.2e}; "
          f"ratio of medians {float(gpu.median() / cpu.median()):.2f}")
    for i, geom, e, e32 in sorted(rec.layers, key=lambda r: -r[2])[:5]:
        print(f"  layer {i:2d} {geom}: 3xTF32 {e:.2e}, CPU fp32 {e32:.2e}, drift {rec.drift[i][0]:+.2f} / "
              f"{rec.drift[i][1]:+.2f}")
    d = torch.tensor(rec.drift)
    print(f"  drift (mean signed error / mean |error|), median over the convs: 3xTF32 {float(d[:, 0].median()):+.2f}, "
          f"CPU fp32 {float(d[:, 1].median()):+.2f}")
    assert float(gpu.max()) <= cc.L2_BOUND, float(gpu.max())


# ---------------------------------------------------------------- omt_i3d_head, omt_lpips_input, grid-stride loops

@pytest.mark.parametrize("B, T, Cs, N", [(2, 2, 1056, 400), (3, 9, 1024, 401), (2, 5, 1088, 7), (1, 3, 1024, 400)])
def test_i3d_head_against_fp64(B, T, Cs, N):
    g = torch.Generator().manual_seed(B * 100 + T)
    x = torch.randn(B, T, 7, 7, Cs, generator=g).clamp_min(0)
    x[..., 1024:] = 1e30                                    # columns past C must not be read
    w = torch.randn(N, 1024, generator=g) / 32
    b = torch.randn(N, generator=g)
    out = torch.full((B, N), float("nan"), device=DEV)
    _cabi.call("omt_i3d_head", x.to(DEV), Cs, 1024, B, T, w.to(DEV), b.to(DEV), N, out)
    torch.cuda.synchronize()
    x64 = x[..., :1024].double()
    pooled = (x64[:, :-1] + x64[:, 1:]).sum(dim=(2, 3)) / 98               # (B, T - 1, C)
    ref = (pooled @ w.double().t() + b.double()).mean(dim=1)
    scale = (pooled @ w.double().abs().t() + b.double().abs()).mean(dim=1)
    err = float(((out.cpu().double() - ref).abs() / scale).max())
    print(f"B={B} T={T} Cs={Cs} N={N}: {err:.2e}")
    assert err <= 2e-5, err


def test_lpips_input_f32_bit_exact():
    P, H, W = 2, 13, 17
    x = torch.rand(P, H, W, 3, generator=torch.Generator().manual_seed(3))
    shift, scale = torch.tensor(quality.SHIFT), torch.tensor(quality.SCALE)
    out = torch.full((P, H, W, 4), float("nan"), device=DEV)
    _cabi.call("omt_lpips_input", x.to(DEV), None, None, torch.cat([shift, scale]).to(DEV), quality.FORM_F32, P, H, W,
               out)
    torch.cuda.synchronize()
    ref = ((x * 2 - 1) - shift) / scale
    assert torch.equal(out.cpu()[..., :3], ref)
    assert bool((out.cpu()[..., 3] == 0).all())


def _lpips_u8(P, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    u8 = torch.randint(0, 256, (P, H, W, 3), generator=g, dtype=torch.uint8)
    lut = torch.randn(2, 3, 256, generator=g)
    sel = torch.arange(P, dtype=torch.int32) % 2
    out = torch.full((P, H, W, 4), float("nan"), device=DEV)
    _cabi.call("omt_lpips_input", u8.to(DEV), lut.to(DEV), sel.to(DEV), None, quality.FORM_U8, P, H, W, out)
    torch.cuda.synchronize()
    ref = lut[sel.long().view(P, 1, 1, 1), torch.arange(3).view(1, 1, 1, 3), u8.long()]
    out = out.cpu()
    assert torch.equal(out[..., :3], ref)
    assert bool((out[..., 3] == 0).all())


def test_lpips_input_u8_table_per_frame():
    _lpips_u8(3, 11, 9, 4)


GRID_THREADS = 65536 * 256                                  # the pooling / input kernels' largest grid


def test_grid_stride_lpips_input():
    assert 2 * 2048 * 4100 > GRID_THREADS
    _lpips_u8(2, 2048, 4100, 5)


def test_grid_stride_maxpool3d():
    dims, k, s = (2, 1032, 1024), (1, 3, 3), (1, 1, 1)
    front, o = fvd.same_geometry(k, s, dims)
    assert dims[0] * dims[1] * dims[2] * 8 > GRID_THREADS
    x = torch.randn(1, 32, *dims, generator=torch.Generator().manual_seed(6))
    y = torch.full((1, *o, 32), float("nan"), device=DEV)
    _cabi.call("omt_maxpool3d", x.permute(0, 2, 3, 4, 1).contiguous().to(DEV), 32, 1, *dims, *k, *s, *front, *o, y)
    torch.cuda.synchronize()
    ref = F.max_pool3d(F.pad(x, io.same_pad(k, s, dims)), k, s)
    assert torch.equal(y.cpu(), ref.permute(0, 2, 3, 4, 1))


def test_grid_stride_pool2d():
    B, C, H, W = 2, 32, 1032, 1024
    assert B * H * W * C // 4 > GRID_THREADS
    x = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(7))
    y = torch.full((B, H, W, C), float("nan"), device=DEV)
    _cabi.call("omt_pool2d", x.permute(0, 2, 3, 1).contiguous().to(DEV), C, C, B, H, W, 3, 3, 1, 1, 1, 1, H, W, y, C,
               fid.POOL_AVG)
    torch.cuda.synchronize()
    ref = F.avg_pool2d(x, 3, 1, 1, count_include_pad=False)
    assert torch.equal(y.cpu(), ref.permute(0, 2, 3, 1))
