"""The FID feature network on the GPU: omt_pool2d and omt_conv3d at every 2-D geometry InceptionV3 uses against torch's
CPU bits, the preprocess against torch's CPU bits (and, reported, torch's CUDA F.interpolate), the pool3 features
against the reference fixture, determinism, eval_step_fid, and the FID end to end against the oracle in float64."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from omnitokenizer_b200 import _cabi
from omnitokenizer_b200 import fid
from omnitokenizer_b200 import fvd
from oracle import fid_oracle as fo

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "fid_inception.pt")


def to_cl(x, cs):
    """(B, C, H, W) -> channels-last (B, H, W, cs), pad channels zero."""
    y = torch.zeros(x.shape[0], *x.shape[2:], cs, dtype=x.dtype)
    y[..., :x.shape[1]] = x.permute(0, 2, 3, 1)
    return y


# (C, H, W, mode, k, s, p, col, ldy): every pool of the network, at its size, column offset and row width
POOLS = [(64, 147, 147, fid.POOL_MAX, 3, 2, 0, 0, 64),        # block 0's MaxPool2d(3, 2)
         (192, 71, 71, fid.POOL_MAX, 3, 2, 0, 0, 192),        # block 1's
         (288, 35, 35, fid.POOL_MAX, 3, 2, 0, 480, 768),      # Mixed_6a's pool branch in its concat slice
         (768, 17, 17, fid.POOL_MAX, 3, 2, 0, 512, 1280),     # Mixed_7a's
         (2048, 8, 8, fid.POOL_MAX, 3, 1, 1, 0, 2048),        # FIDInceptionE_2's max_pool2d(3, 1, 1)
         (192, 35, 35, fid.POOL_AVG, 3, 1, 1, 0, 192),        # FIDInceptionA (Mixed_5b)
         (288, 35, 35, fid.POOL_AVG, 3, 1, 1, 0, 288),        # Mixed_5d
         (768, 17, 17, fid.POOL_AVG, 3, 1, 1, 0, 768),        # FIDInceptionC
         (1280, 8, 8, fid.POOL_AVG, 3, 1, 1, 0, 1280),        # FIDInceptionE_1
         (2048, 8, 8, fid.POOL_AVG, 8, 1, 0, 0, 2048),        # AdaptiveAvgPool2d(1) -> the features
         (64, 13, 10, fid.POOL_AVG, 3, 2, 1, 32, 128)]        # odd sizes, stride 2 with padding, a column offset


@pytest.mark.parametrize("case", POOLS, ids=[f"{'max' if c[3] == 0 else 'avg'}{c[4]}s{c[5]}p{c[6]}_{c[0]}x{c[1]}x{c[2]}"
                                             f"_col{c[7]}" for c in POOLS])
def test_pool2d_exact(case):
    C, H, W, mode, k, s, p, col, ldy = case
    g = torch.Generator().manual_seed(C + H + mode)
    x = torch.randn(2, C, H, W, generator=g)                 # negative values: a zero padding would win at the border
    if mode == fid.POOL_MAX:
        ref = F.max_pool2d(x, k, s, p)
    else:
        ref = F.avg_pool2d(x, k, s, p, count_include_pad=False)
    Ho, Wo = (fid.out_size(n, k, s, p) for n in (H, W))
    assert tuple(ref.shape[2:]) == (Ho, Wo)
    y = torch.full((2, Ho, Wo, ldy), -7.0, device=DEV)
    xd = to_cl(x, C).to(DEV)
    _cabi.call("omt_pool2d", xd, C, C, 2, H, W, k, k, s, s, p, p, Ho, Wo, y.data_ptr() + 4 * col, ldy, mode)
    torch.cuda.synchronize()
    y = y.cpu()
    assert torch.equal(y[..., col:col + C], ref.permute(0, 2, 3, 1))
    assert bool((y[..., :col] == -7).all()) and bool((y[..., col + C:] == -7).all())


def conv_ref(x, w, b, s, p):
    """float64 conv2d + ReLU, cast to fp32, channels-last (B, H, W, cout)."""
    return F.relu(F.conv2d(x.double(), w.double(), b.double(), stride=s, padding=p)).float().permute(0, 2, 3, 1)


def run_conv(x, w, b, s, p, col=0, ldy=None, fill=float("nan")):
    B, cin, H, W = x.shape
    cout, _, kh, kw = w.shape
    cs = fvd.cpad(cin)
    wp, K = fvd.pack_weight(w.unsqueeze(2))
    hi = fvd.L.tf32_round(wp)
    Ho, Wo = fid.out_size(H, kh, s, p[0]), fid.out_size(W, kw, s, p[1])
    ldy = ldy or fvd.cpad(cout)
    y = torch.full((B, Ho, Wo, ldy), fill, device=DEV)
    _cabi.call("omt_conv3d", to_cl(x, cs).to(DEV), cs, B, 1, H, W, hi.to(DEV), (wp - hi).to(DEV), K, b.to(DEV), cout,
               1, kh, kw, 1, s, s, 0, p[0], p[1], 1, Ho, Wo, y.data_ptr() + 4 * col, ldy, 1)
    torch.cuda.synchronize()
    return y.cpu()


# (B, cin, cout, H, W, (kh, kw), s, (ph, pw), col, ldy): the network's 2-D geometries (sizes shrunk where the shape
# does not matter), the padded channel strides 4 / 64 / 96 in and 96 out, and concat slices at their offsets
CONVS = [(2, 3, 32, 41, 37, (3, 3), 2, (0, 0), 0, None),        # Conv2d_1a: 4-channel input, stride 2, pad 0
         (1, 32, 32, 29, 31, (3, 3), 1, (0, 0), 0, None),       # Conv2d_2a
         (1, 32, 64, 29, 31, (3, 3), 1, (1, 1), 0, None),       # Conv2d_2b
         (1, 64, 80, 23, 21, (1, 1), 1, (0, 0), 0, None),       # Conv2d_3b: 80 columns of a 96-wide row
         (1, 80, 192, 19, 17, (3, 3), 1, (0, 0), 0, None),      # Conv2d_4a: Cs = 96 input
         (2, 48, 64, 35, 35, (5, 5), 1, (2, 2), 64, 256),       # Mixed_5b.branch5x5_2: Cs = 64 input, concat slice
         (1, 288, 384, 35, 35, (3, 3), 2, (0, 0), 0, 768),      # Mixed_6a.branch3x3: strided, pad 0
         (1, 96, 96, 35, 35, (3, 3), 2, (0, 0), 384, 768),      # Mixed_6a.branch3x3dbl_3
         (1, 128, 128, 17, 17, (1, 7), 1, (0, 3), 0, None),     # Mixed_6b.branch7x7_2
         (1, 160, 192, 17, 17, (7, 1), 1, (3, 0), 192, 768),    # Mixed_6c.branch7x7_3
         (1, 192, 192, 17, 17, (3, 3), 2, (0, 0), 320, 1280),   # Mixed_7a.branch7x7x3_4
         (2, 384, 384, 8, 8, (1, 3), 1, (0, 1), 1088, 2048),    # Mixed_7c.branch3x3dbl_3a
         (2, 384, 384, 8, 8, (3, 1), 1, (1, 0), 1472, 2048),    # Mixed_7c.branch3x3dbl_3b
         (2, 448, 384, 8, 8, (3, 3), 1, (1, 1), 0, None),       # Mixed_7b.branch3x3dbl_2
         (2, 2048, 192, 8, 8, (1, 1), 1, (0, 0), 1856, 2048)]   # Mixed_7c.branch_pool


@pytest.mark.parametrize("case", CONVS, ids=[f"{c[1]}to{c[2]}_k{c[5][0]}x{c[5][1]}s{c[6]}_{c[3]}x{c[4]}_col{c[8]}"
                                             for c in CONVS])
def test_conv2d_exact_grid(case):
    B, cin, cout, H, W, k, s, p, col, ldy = case
    g = torch.Generator().manual_seed(cin * 7 + cout + k[0])
    x = torch.randint(-3, 4, (B, cin, H, W), generator=g).float()
    w = torch.randint(-3, 4, (cout, cin) + k, generator=g).float()
    b = torch.randint(-8, 9, (cout,), generator=g).float()
    y = run_conv(x, w, b, s, p, col=col, ldy=ldy, fill=-7.0)
    ref = conv_ref(x, w, b, s, p)
    assert torch.equal(y[..., col:col + cout], ref), f"max diff {float((y[..., col:col + cout] - ref).abs().max())}"
    assert bool((y[..., :col] == -7).all()) and bool((y[..., col + cout:] == -7).all())


def preprocess_device(u8, lut):
    B, H, W, _ = u8.shape
    oh, ow = fid.TARGET_RESOLUTION
    tv = fvd.L.clip_axis_table(H, oh, float(np.float32(H) / np.float32(oh))).reshape(-1)
    th = fvd.L.clip_axis_table(W, ow, float(np.float32(W) / np.float32(ow))).reshape(-1)
    tab = torch.from_numpy(np.concatenate([tv, th]).astype(np.int32))
    desc = torch.zeros(B, fvd.CLIP_DESC_WORDS, dtype=torch.int32)
    desc[:, :2] = (torch.arange(B, dtype=torch.int64) * (H * W * 3)).view(torch.int32).view(B, 2)
    desc[:, 2:] = torch.tensor([H, W, 0, 0, H, W, oh, ow, 0, 0, 0, 0, tv.size, 0], dtype=torch.int32)
    x = torch.full((B, oh, ow, 4), float("nan"), device=DEV)
    src = u8.to(DEV)
    _cabi.call("omt_fid_preprocess", src, src.numel(), desc.to(DEV), desc, tab.to(DEV), tab, tab.numel(),
               lut.to(DEV), None, B, oh, ow, x)
    torch.cuda.synchronize()
    return x.cpu()


@pytest.mark.parametrize("shape", [(256, 256), (128, 128), (299, 299), (320, 480), (97, 131)])
def test_preprocess_bit_exact(shape):
    from omnitokenizer_b200.consumers import IMAGE_NORM
    u8 = torch.stack([fo.image_bytes(shape, 5), 255 - fo.image_bytes(shape, 5)])
    for lut in (fid.byte_lut()[0], fid.byte_lut(IMAGE_NORM)[0]):
        got = preprocess_device(u8, lut)
        ref = fo.preprocess(u8, lut=lut)                          # torch's CPU F.interpolate
        assert torch.equal(got[..., :3], ref.permute(0, 2, 3, 1))
        assert bool((got[..., 3] == 0).all())
    # pytorch-fid itself resizes on the device: torch's CUDA bilinear kernel (reported, not a bit-exactness claim)
    x01 = u8.permute(0, 3, 1, 2).contiguous().float().div(255).to(DEV)
    cuda = (2 * F.interpolate(x01, size=(299, 299), mode="bilinear", align_corners=False) - 1).cpu()
    got = preprocess_device(u8, fid.byte_lut()[0])
    print(f"{shape}: max |kernel - torch CUDA F.interpolate| = {float((got[..., :3] - cuda.permute(0, 2, 3, 1)).abs().max()):.2e}")


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN)


@pytest.fixture(scope="module")
def sd(golden):
    sd = fo.make_state_dict(golden["w_seed"])
    sd.update(golden["bn"])
    assert fo.conv_fingerprint(sd) == golden["fingerprint"]
    return sd


@pytest.fixture(scope="module")
def net(sd):
    return fid.FIDInception(sd, DEV)


def test_features_match_fixture(golden, net, sd):
    """Against the reference's fp32 CPU features (and, printed, an fp64 run of the oracle).  The bound is 3e-4 of
    max |feature|: on the noise image up_256 the seeded network carries the 3xTF32 convs' rounding to 2e-4 of it (the
    fp32 reference's own distance from fp64 is 2.7e-5 there); the FID itself agrees far closer (the end-to-end test)."""
    worst = 0.0
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    for name, e in golden["images"].items():
        u8 = fo.image_bytes(e["shape"], e["seed"])[None]
        got = net.features(u8.to(DEV)).cpu()[0]
        ref = e["features"]
        with torch.no_grad():
            r64 = fo.forward(sd64, fo.preprocess(u8).double())[0]
        rel = float((got - ref).abs().max() / ref.abs().max())
        rel64 = float((got.double() - r64).abs().max() / r64.abs().max())
        ref64 = float((ref.double() - r64).abs().max() / r64.abs().max())
        print(f"{name}: max|feature| {float(ref.abs().max()):.3f}  vs reference {rel:.2e}  vs fp64 {rel64:.2e}  "
              f"(reference vs fp64 {ref64:.2e})")
        worst = max(worst, rel)
    assert worst <= 3e-4, worst


def test_graph_replay_equals_eager(net):
    u8 = torch.stack([fo.image_bytes((64, 80), 3 + i) for i in range(3)]).to(DEV)
    key = (3, 64, 80, None)
    net._ws.pop(key, None)
    outs = [net.features(u8).clone() for _ in range(3)]       # eager, capture + replay, replay
    assert isinstance(net._ws[key].graphs["fid"], tuple)
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


def test_image_alone_equals_batch(net):
    batch = torch.stack([fo.image_bytes((48, 40), 40 + i) for i in range(12)]).to(DEV)
    together = net.features(batch).clone()
    for i in (0, 5, 11):
        assert torch.equal(net.features(batch[i:i + 1]).clone()[0], together[i]), i


def test_refusals_launch_nothing(net):
    n0 = _cabi.launch_count
    for bad in (torch.zeros(1, 32, 32, 3, device=DEV),                       # fp32
                torch.zeros(1, 32, 32, 4, dtype=torch.uint8, device=DEV),    # 4 channels
                torch.zeros(32, 32, 3, dtype=torch.uint8, device=DEV),       # rank 3
                torch.zeros(0, 32, 32, 3, dtype=torch.uint8, device=DEV),    # empty
                torch.zeros(1, 32, 32, 3, dtype=torch.uint8)):               # host tensor
        with pytest.raises((TypeError, ValueError)):
            net.features(bad)
    assert _cabi.launch_count == n0


def test_paths_and_script_device(tmp_path, sd):
    """load_fid_model with torch.device('cuda') (no index); path_features over a PNG directory laid out as
    vqgan_eval.py writes it (<root>/<class>/<file>.png), in batches of 3, equal to the features of the same bytes;
    fid_given_paths over two .npz statistics files."""
    from PIL import Image
    path = tmp_path / "inception.pth"
    torch.save(sd, path)
    model = fid.load_fid_model(torch.device("cuda"), str(path))
    assert model.device == torch.device("cuda", torch.cuda.current_device())
    ims = [fo.image_bytes((40, 48), i) for i in range(7)]
    for i, im in enumerate(ims):
        (tmp_path / "input" / f"c{i % 2}").mkdir(parents=True, exist_ok=True)
        Image.fromarray(im.numpy()).save(tmp_path / "input" / f"c{i % 2}" / f"{i}.png")
    order = sorted(range(7), key=lambda i: (f"c{i % 2}", f"{i}.png"))
    want = model.features(torch.stack([ims[i] for i in order]).to(DEV)).clone()
    got = fid.path_features(fid.image_files(tmp_path / "input"), model, batch_size=3)
    assert torch.equal(got, want)
    fd = torch.load(GOLDEN)["fd"]
    for name, x in (("a.npz", fd["x1"]), ("b.npz", fd["x2"])):
        mu, sigma = fid.activation_statistics(x)
        np.savez(tmp_path / name, mu=mu, sigma=sigma)
    v = fid.fid_given_paths([str(tmp_path / "a.npz"), str(tmp_path / "b.npz")], model)
    assert abs(v / fd["value"] - 1) < 1e-12


def test_eval_step_fid_equals_separate_bytes(net):
    """eval_step_fid's real side == features of the host transform (layout.resize_u8) with the script's real byte map;
    its fake side == features of forward_u8's output on those bytes."""
    import omnitokenizer_b200 as ob
    from omnitokenizer_b200 import consumers as C
    from omnitokenizer_b200 import layout as L
    from oracle import omni_oracle as oo
    from oracle import weights as W
    args = ob.canonical_args()
    m = ob.OmniTokenizer_VQGAN(args)
    m.load_state_dict(W.make_state_dict(oo.Config.from_args(args), 0), strict=False)
    m.codebook._need_init = False
    m = m.to(DEV).eval()
    images = [fo.image_bytes(s, 90 + i) for i, s in enumerate([(150, 200), (128, 128), (97, 131)])]
    resize = L.resizecrop_resize(128)
    params = [(3, 50, False), (10, 0, False), (0, 64, False)]
    usage = torch.zeros(8192, device=DEV)
    # the accessor: the encode_u8 slot holds the transformed input bytes of the last call
    fake, vq_output = m.forward_images_u8(images, resize, C.IMAGE_NORM, C.EVAL_U8, params=params)
    real_dev = m.engine().encode_u8_frames(tuple(fake.shape)).clone()
    host = torch.stack([L.resize_u8(im, resize, p_) for im, p_ in zip(images, params)])
    assert torch.equal(real_dev[:, 0].cpu(), host)
    torch.manual_seed(5)
    real_f, fake_f, vq_output = C.eval_step_fid(m, images, resize, net, usage)
    torch.manual_seed(5)
    drawn = L.resize_params(len(images), resize)
    host = torch.stack([L.resize_u8(im, resize, p_) for im, p_ in zip(images, drawn)])
    x = L.u8_normalize(host.unsqueeze(1), C.IMAGE_NORM)[:, :, 0]                         # (B, 3, h, w)
    script = ((x.permute(0, 2, 3, 1) + 0.5).numpy() * 255).astype(np.uint8)             # vqgan_eval.py:204-205
    want_real = net.features(torch.from_numpy(script).to(DEV)).clone()
    fake_bytes, vq2 = C.eval_step_u8(m, host.to(DEV), None, C.IMAGE_NORM)
    want_fake = net.features(fake_bytes[:, 0].contiguous()).clone()
    assert torch.equal(real_f, want_real)
    assert torch.equal(fake_f, want_fake)
    assert torch.equal(vq_output["batch_usage"], vq2["batch_usage"]) and bool(usage.sum() > 0)


def test_fid_end_to_end_matches_oracle_fp64(net, sd):
    """FID between two sets of 2 560 seeded images (more than 2048, so both covariances are full rank): from the
    device features and from the oracle run in float64 on the device, through the same calculate_frechet_distance."""
    n, bs = 2560, 64
    g = torch.Generator().manual_seed(77)
    real = torch.randint(0, 256, (n, 24, 24, 3), generator=g, dtype=torch.uint8)   # upscaled: smooth, varied images
    fake = (real.int() * 3 // 4 + torch.randint(0, 64, real.shape, generator=g, dtype=torch.int32)).to(torch.uint8)
    sd64 = {k: (v.double().to(DEV) if v.is_floating_point() else v) for k, v in sd.items()}
    stats_dev, stats_64 = [], []
    for imgs in (real, fake):
        dev, o64 = [], []
        for i in range(0, n, bs):
            b = imgs[i:i + bs]
            dev.append(net.features(b.to(DEV)).clone().cpu())
            with torch.no_grad():
                o64.append(fo.forward(sd64, fo.preprocess(b).double().to(DEV)).cpu())
        dev, o64 = torch.cat(dev), torch.cat(o64)
        print(f"features: max rel diff vs fp64 oracle {float((dev.double() - o64).abs().max() / o64.abs().max()):.2e}")
        stats_dev.append(fid.activation_statistics(dev))
        stats_64.append(fid.activation_statistics(o64))
    got = fid.calculate_frechet_distance(*stats_dev[0], *stats_dev[1])
    ref = fid.calculate_frechet_distance(*stats_64[0], *stats_64[1])
    print(f"FID device {got:.6f}  fp64 oracle {ref:.6f}  relative {abs(got / ref - 1):.2e}")
    assert abs(got / ref - 1) <= 1e-3
