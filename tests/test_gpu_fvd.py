"""The FVD feature network on the GPU: omt_conv3d on exact-grid operands at every I3D geometry, omt_maxpool3d and the
preprocess against torch's CPU bits, I3D logits against the reference fixture, and determinism."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from omnitokenizer_b200 import _cabi
from omnitokenizer_b200 import fvd
from oracle import i3d_oracle as io

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "fvd_i3d.pt")


def to_cl(x, cs):
    """(B, C, T, H, W) -> channels-last (B, T, H, W, cs), pad channels zero."""
    y = torch.zeros(x.shape[0], *x.shape[2:], cs, dtype=x.dtype)
    y[..., :x.shape[1]] = x.permute(0, 2, 3, 4, 1)
    return y


def conv_ref(x, w, b, k, s, relu):
    """float64 F.pad (SAME) + conv3d, cast to fp32, channels-last (B, T, H, W, cout)."""
    y = F.conv3d(F.pad(x.double(), io.same_pad((k,) * 3, (s,) * 3, x.shape[2:])), w.double(), b.double(), stride=s)
    if relu:
        y = F.relu(y)
    return y.float().permute(0, 2, 3, 4, 1)


def run_conv(x, w, b, k, s, relu, col=0, ldy=None, fill=float("nan")):
    B, cin, T, H, W = x.shape
    cout = w.shape[0]
    cs = fvd.cpad(cin)
    wp, K = fvd.pack_weight(w)
    hi = fvd.L.tf32_round(wp)
    front, o = fvd.same_geometry((k,) * 3, (s,) * 3, (T, H, W))
    ldy = ldy or cout
    xd = to_cl(x, cs).to(DEV)
    y = torch.full((B, *o, ldy), fill, device=DEV)
    _cabi.call("omt_conv3d", xd, cs, B, T, H, W, hi.to(DEV), (wp - hi).to(DEV), K, b.to(DEV), cout, k, k, k, s, s, s,
               *front, *o, y.data_ptr() + 4 * col, ldy, int(relu))
    torch.cuda.synchronize()
    return y.cpu()


# (B, cin, cout, T, H, W, k, s): every I3D geometry, odd sizes (asymmetric SAME), and tile counts that give each
# persistent CTA of a 132-SM H100 1 to 4 tiles (254, 270 and 450 tiles of 128 rows)
CASES = [
    (1, 3, 64, 9, 21, 19, 7, 2),        # Conv3d_1a: the 4-channel input, 8 taps per k-block
    (2, 64, 64, 5, 11, 9, 1, 1),        # Conv3d_2b (64-wide tile)
    (1, 64, 192, 5, 9, 7, 3, 1),        # Conv3d_2c
    (1, 16, 32, 3, 7, 5, 3, 1),         # b2b of Mixed_3b: 16 channels padded to 32
    (1, 96, 208, 3, 6, 5, 3, 1),        # b1b of Mixed_4b
    (1, 528, 256, 3, 5, 5, 1, 1),       # b0 of Mixed_4f
    (1, 832, 384, 2, 7, 7, 1, 1),       # b0 of Mixed_5c
    (1, 24, 64, 2, 3, 3, 3, 1),
    (1, 192, 16, 5, 9, 7, 1, 1),        # b2a of Mixed_3b: N = 16 on the 64-wide tile
    (1, 512, 24, 3, 7, 9, 1, 1),        # b2a of Mixed_4c: N = 24
    (1, 832, 400, 1, 1, 1, 1, 1),       # a logits-sized GEMM: 4 column tiles, the last one partial
    (1, 32, 64, 9, 60, 60, 1, 1),       # 254 tiles: 1 to 2 per CTA
    (1, 32, 128, 9, 64, 60, 1, 1),      # 270 tiles: 2 to 3 per CTA
    (1, 32, 128, 9, 80, 80, 1, 1),      # 450 tiles: 3 to 4 per CTA
    (1, 32, 192, 4, 31, 33, 3, 2),      # stride 2 on a 3x3x3 kernel, odd sizes
]


@pytest.mark.parametrize("case", CASES, ids=[f"{c[1]}to{c[2]}_k{c[6]}s{c[7]}_{c[3]}x{c[4]}x{c[5]}" for c in CASES])
@pytest.mark.parametrize("relu", [True, False])
def test_conv3d_exact_grid(case, relu):
    B, cin, cout, T, H, W, k, s = case
    g = torch.Generator().manual_seed(hash(case) % 1000 + relu)
    x = torch.randint(-3, 4, (B, cin, T, H, W), generator=g).float()
    w = torch.randint(-3, 4, (cout, cin, k, k, k), generator=g).float()
    b = torch.randint(-8, 9, (cout,), generator=g).float()
    y = run_conv(x, w, b, k, s, relu)
    ref = conv_ref(x, w, b, k, s, relu)
    assert torch.equal(y, ref), f"max diff {float((y - ref).abs().max())}"


@pytest.mark.parametrize("cin, cout, k, col, ldy", [(96, 208, 3, 192, 544), (192, 16, 1, 0, 32), (480, 16, 1, 400, 512),
                                                    (512, 24, 1, 64, 96), (32, 48, 3, 128, 544)])
def test_conv3d_column_slice(cin, cout, k, col, ldy):
    """A branch writes exactly its N columns at its offset of the concat buffer: the neighbours keep their bits."""
    g = torch.Generator().manual_seed(7 + cout)
    x = torch.randint(-3, 4, (1, cin, 3, 6, 5), generator=g).float()
    w = torch.randint(-3, 4, (cout, cin, k, k, k), generator=g).float()
    b = torch.randint(-8, 9, (cout,), generator=g).float()
    y = run_conv(x, w, b, k, 1, True, col=col, ldy=ldy, fill=-7.0)
    assert torch.equal(y[..., col:col + cout], conv_ref(x, w, b, k, 1, True))
    assert bool((y[..., :col] == -7).all()) and bool((y[..., col + cout:] == -7).all())


def test_conv3d_random_operands():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 192, 5, 9, 11, generator=g)
    w = torch.randn(96, 192, 3, 3, 3, generator=g) / 50
    b = torch.randn(96, generator=g)
    y = run_conv(x, w, b, 3, 1, False)
    ref = F.conv3d(F.pad(x.double(), io.same_pad((3,) * 3, (1,) * 3, x.shape[2:])), w.double(), b.double())
    scale = F.conv3d(F.pad(x.double().abs(), io.same_pad((3,) * 3, (1,) * 3, x.shape[2:])), w.double().abs(),
                     b.double().abs())
    err = ((y.double() - ref.permute(0, 2, 3, 4, 1)).abs() / scale.permute(0, 2, 3, 4, 1).clamp_min(1e-30)).max()
    print(f"relative error {float(err):.2e}")
    assert float(err) < 1e-6, float(err)


@pytest.mark.parametrize("win", [((1, 3, 3), (1, 2, 2)), ((3, 3, 3), (1, 1, 1)), ((3, 3, 3), (2, 2, 2)),
                                 ((2, 2, 2), (2, 2, 2))])
@pytest.mark.parametrize("dims", [(9, 23, 17), (4, 7, 7), (5, 14, 15)])
def test_maxpool3d_exact(win, dims):
    k, s = win
    g = torch.Generator().manual_seed(sum(dims))
    x = torch.randn(2, 40, *dims, generator=g)          # negative values: the zero padding wins at the border
    ref = F.max_pool3d(F.pad(x, io.same_pad(k, s, dims)), k, s)
    front, o = fvd.same_geometry(k, s, dims)
    assert tuple(ref.shape[2:]) == o
    xd = to_cl(x, 64).to(DEV)
    y = torch.full((2, *o, 64), float("nan"), device=DEV)
    _cabi.call("omt_maxpool3d", xd, 64, 2, *dims, *k, *s, *front, *o, y)
    torch.cuda.synchronize()
    assert torch.equal(y.cpu()[..., :40], ref.permute(0, 2, 3, 4, 1))
    assert bool((y.cpu()[..., 40:] == 0).all())


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN)


@pytest.fixture(scope="module")
def net(golden):
    sd = io.make_state_dict(golden["w_seed"])
    sd.update(golden["bn"])
    assert io.conv_fingerprint(sd) == golden["fingerprint"]
    return fvd.I3D(sd, DEV)


def clip(shape, seed):
    if seed is None:
        return torch.full(tuple(shape) + (3,), 200, dtype=torch.uint8)
    return torch.randint(0, 256, tuple(shape) + (3,), generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


@pytest.mark.parametrize("shape", [(17, 256, 256), (9, 64, 64), (3, 240, 320), (2, 97, 131)])
def test_preprocess_bit_exact(shape, net):
    u8 = clip(shape, 5)[None].repeat(2, 1, 1, 1, 1)
    u8[1] = 255 - u8[1]
    B, T, H, W = 2, *shape
    x = torch.full((B, T, 224, 224, 4), float("nan"), device=DEV)
    tv = fvd.L.clip_axis_table(H, 224, float(np.float32(H) / np.float32(224))).reshape(-1)
    th = fvd.L.clip_axis_table(W, 224, float(np.float32(W) / np.float32(224))).reshape(-1)
    tab = torch.from_numpy(np.concatenate([tv, th]).astype(np.int32))
    desc = torch.zeros(B, fvd.CLIP_DESC_WORDS, dtype=torch.int32)
    desc[:, :2] = (torch.arange(B, dtype=torch.int64) * (T * H * W * 3)).view(torch.int32).view(B, 2)
    desc[:, 2:] = torch.tensor([H, W, 0, 0, H, W, 224, 224, 0, 0, 0, 0, tv.size, 0], dtype=torch.int32)
    src = u8.to(DEV)
    _cabi.call("omt_fvd_preprocess", src, src.numel(), desc.to(DEV), desc, tab.to(DEV), tab, tab.numel(),
               net.byte_lut, None, B, T, 224, 224, x)
    torch.cuda.synchronize()
    ref = io.preprocess(u8.numpy())                      # (B, 3, T, 224, 224)
    got = x.cpu()
    assert torch.equal(got[..., :3], ref.permute(0, 2, 3, 4, 1))
    assert bool((got[..., 3] == 0).all())


def test_logits_match_fixture(golden, net):
    """Against the reference's fp32 CPU logits (and, printed, an fp64 run of the oracle)."""
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in io.make_state_dict(golden["w_seed"]).items()}
    sd64.update({k: v.double() for k, v in golden["bn"].items()})
    for name, e in golden["clips"].items():
        u8 = clip(e["shape"], e["seed"])[None]
        got = net.logits(u8.to(DEV)).cpu()[0]
        ref = e["logits"]
        with torch.no_grad():
            r64 = io.forward(sd64, io.preprocess(u8.numpy()).double())[0]
        rel = float((got - ref).abs().max() / ref.abs().max())
        rel64 = float((got.double() - r64).abs().max() / r64.abs().max())
        ref64 = float((ref.double() - r64).abs().max() / r64.abs().max())
        print(f"{name}: max|logit| {float(ref.abs().max()):.3f}  vs reference {rel:.2e}  vs fp64 {rel64:.2e}  "
              f"(reference vs fp64 {ref64:.2e})")
        assert rel <= 1e-4, name


def test_fvd_matches_oracle(net):
    """FVD between two sets of 8 clips from the device logits and from the oracle's CPU logits (the reference's bits:
    tests/test_oracle_fvd.py).  The distance runs in float64 on both sides: with 8 samples in 400 dimensions the
    covariances are singular, and fp32's square roots of its rounding noise would swamp the comparison."""
    real = torch.stack([clip((9, 64, 80), 300 + i) for i in range(8)])
    fake = real.clone()
    fake[..., 1:, :] = fake[..., :-1, :]                  # a shifted copy: close to the real set, not equal
    fake = (fake.int() * 7 // 8 + 16).to(torch.uint8)
    dev_r, dev_f = (net.logits(v.to(DEV)).clone().cpu().double() for v in (real, fake))
    sd = io.make_state_dict(torch.load(GOLDEN)["w_seed"])
    sd.update(torch.load(GOLDEN)["bn"])
    with torch.no_grad():
        cpu_r, cpu_f = (io.forward(sd, io.preprocess(v.numpy())).double() for v in (real, fake))
    got, ref = float(fvd.frechet_distance(dev_r, dev_f)), float(fvd.frechet_distance(cpu_r, cpu_f))
    print(f"FVD device {got:.6f}  oracle {ref:.6f}  relative {abs(got / ref - 1):.2e}")
    assert abs(got / ref - 1) <= 1e-4


def test_graph_replay_equals_eager(net):
    u8 = clip((9, 64, 64), 3)[None].repeat(3, 1, 1, 1, 1).to(DEV)
    u8[1:] = 255 - u8[1:]
    net._ws.pop((3, 9, 64, 64, None), None)
    outs = [net.logits(u8).clone() for _ in range(3)]      # eager, capture + replay, replay
    assert isinstance(net._ws[(3, 9, 64, 64, None)].graphs["i3d"], tuple)
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


def test_clip_alone_equals_batch_of_16(net):
    batch = torch.stack([clip((9, 72, 88), 40 + i) for i in range(16)]).to(DEV)
    together = net.logits(batch).clone()
    for i in (0, 7, 15):
        assert torch.equal(net.logits(batch[i:i + 1]).clone()[0], together[i]), i


def test_get_fvd_logits_numpy_equals_device(net):
    u8 = torch.stack([clip((10, 100, 120), 50 + i) for i in range(2)])
    a = fvd.get_fvd_logits(u8.numpy(), net, DEV)
    b = fvd.get_fvd_logits(u8.to(DEV), net, DEV)
    assert a.device == DEV and torch.equal(a, b)


def test_refusals_launch_nothing(net):
    n0 = _cabi.launch_count
    for bad in (torch.zeros(1, 9, 32, 32, 3, device=DEV),                      # fp32
                torch.zeros(1, 9, 32, 32, 4, dtype=torch.uint8, device=DEV),   # 4 channels
                torch.zeros(9, 32, 32, 3, dtype=torch.uint8, device=DEV),      # rank 4
                torch.zeros(1, 8, 32, 32, 3, dtype=torch.uint8, device=DEV),   # T = 8
                torch.zeros(1, 9, 32, 32, 3, dtype=torch.uint8)):              # host tensor to logits
        with pytest.raises((TypeError, ValueError)):
            net.logits(bad)
    assert _cabi.launch_count == n0


def test_script_device_and_numpy_input(tmp_path, golden):
    """vqgan_eval.py:59 passes torch.device('cuda') (no index) to load_fvd_model, then numpy bytes to get_fvd_logits."""
    sd = io.make_state_dict(golden["w_seed"])
    sd.update(golden["bn"])
    path = tmp_path / "i3d.pt"
    torch.save({k: v for k, v in sd.items() if not k.endswith("num_batches_tracked")}, path)
    i3d = fvd.load_fvd_model(torch.device("cuda"), str(path))
    assert i3d.device == torch.device("cuda", torch.cuda.current_device())
    u8 = torch.stack([clip((9, 64, 64), 70 + i) for i in range(2)])
    a = fvd.get_fvd_logits(u8.numpy(), i3d=i3d, device=torch.device("cuda"))
    b = fvd.get_fvd_logits(u8.to(DEV), i3d=i3d, device=torch.device("cuda"))
    assert torch.equal(a, b)


def test_eval_step_fvd_equals_script_bytes(net):
    """eval_step_fvd == get_fvd_logits on the byte tensors vqgan_eval.py builds (:144-148), bit for bit, with one clip
    in VideoNorm's max <= 1 branch."""
    import omnitokenizer_b200 as ob
    from omnitokenizer_b200 import consumers as C
    from oracle import omni_oracle as oo
    from oracle import weights as W
    args = ob.canonical_args()
    m = ob.OmniTokenizer_VQGAN(args)
    m.load_state_dict(W.make_state_dict(oo.Config.from_args(args), 0), strict=False)
    m.codebook._need_init = False
    m = m.to(DEV).eval()
    u8 = torch.stack([clip((9, 128, 128), 80), clip((9, 128, 128), 81) % 2])    # clip 1: bytes 0 / 1 only
    frames = u8.to(DEV)
    usage = torch.zeros(8192, device=DEV)
    real_l, fake_l, vq_output = C.eval_step_fvd(m, frames, net, usage)
    # the script: the loader's VideoNorm'd clip, real_videos = video + 0.5, shift_dim(real_videos * 255, 1, -1).byte()
    video = fvd.L.u8_normalize(u8, C.VIDEO_NORM)
    real_bytes = ((video + 0.5) * 255).movedim(1, -1).byte()
    fake_bytes, vq2 = C.eval_step_u8(m, frames)
    assert torch.equal(real_l, fvd.get_fvd_logits(real_bytes.numpy(), net, DEV))
    assert torch.equal(fake_l, fvd.get_fvd_logits(fake_bytes, net, DEV))
    assert torch.equal(vq_output["batch_usage"], vq2["batch_usage"]) and bool(usage.sum() > 0)
