"""Host logic of omnitokenizer_b200.fid without a GPU: the network's geometry and concat layout, BatchNorm folding and
weight packing, the real side's byte map, the statistics and the Frechet distance, and refusals before any launch."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from omnitokenizer_b200 import _cabi
from omnitokenizer_b200 import fid
from omnitokenizer_b200 import fvd
from omnitokenizer_b200 import layout as L
from oracle import fid_oracle as fo

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "fid_inception.pt")


def test_conv_list_matches_oracle():
    got = [(c.name, c.cin, c.cout, c.k, c.s, c.p) for c in fid.conv_list()]
    assert len(got) == 94
    assert got == fo.convs()
    assert set(fid.expected_keys()) == {f"{c[0]}.{s}" for c in fo.convs()
                                        for s in ("conv.weight", "bn.weight", "bn.bias", "bn.running_mean",
                                                  "bn.running_var")}


def test_geometry_of_every_conv_and_pool():
    """The spatial path of a 299^2 input (149 -> 147 -> 73 -> 71 -> 35 -> 17 -> 8), every conv's output size against
    F.conv2d's, and every block's branches landing on the block's output size and its concat columns."""
    path, hw = [], (299, 299)
    for layer in fid.STEM:
        if isinstance(layer, fid.Conv):
            o = tuple(fid.out_size(n, k, layer.s, p) for n, k, p in zip(hw, layer.k, layer.p))
            ref = F.conv2d(torch.empty(1, layer.cin, *hw, device="meta"), torch.empty(layer.cout, layer.cin, *layer.k,
                           device="meta"), stride=layer.s, padding=layer.p).shape[2:]
        else:
            o = tuple(fid.out_size(n, layer.k, layer.s, layer.p) for n in hw)
            ref = F.max_pool2d(torch.empty(1, 1, *hw, device="meta"), layer.k, layer.s, layer.p).shape[2:]
        assert o == tuple(ref)
        if o != hw:
            path.append(o[0])
        hw = o
    for name, convs, pool, cout in fid.BLOCKS:
        shapes = {"x": hw, "p": hw}
        o_blk = hw if pool.col is None else tuple(fid.out_size(n, pool.k, pool.s, pool.p) for n in hw)
        cols = [] if pool.col is None else [(pool.col, pool.col + convs[0].cin)]
        for c in convs:
            src = shapes[c.src]
            o = tuple(fid.out_size(n, k, c.s, p) for n, k, p in zip(src, c.k, c.p))
            ref = F.conv2d(torch.empty(1, c.cin, *src, device="meta"), torch.empty(c.cout, c.cin, *c.k, device="meta"),
                           stride=c.s, padding=c.p).shape[2:]
            assert o == tuple(ref), f"{name}.{c.name}"
            shapes[c.name] = o
            if c.col is not None:
                assert o == o_blk, f"{name}.{c.name}"
                cols.append((c.col, c.col + c.cout))
        cols.sort()
        assert cols[0][0] == 0 and cols[-1][1] == cout and all(a[1] == b[0] for a, b in zip(cols, cols[1:])), name
        assert all(a % 32 == 0 for a, _ in cols), name
        if o_blk != hw:
            path.append(o_blk[0])
        hw = o_blk
    assert path == [149, 147, 73, 71, 35, 17, 8]
    assert hw == (8, 8) and fid.BLOCKS[-1][3] == 2048


@pytest.mark.parametrize("prefix", ["Conv2d_1a_3x3", "Conv2d_4a_3x3", "Mixed_5b.branch5x5_2", "Mixed_6b.branch7x7_2",
                                    "Mixed_6b.branch7x7_3", "Mixed_7a.branch7x7x3_2", "Mixed_7b.branch3x3_2a",
                                    "Mixed_7c.branch3x3dbl_3b"])
def test_bn_folding_and_packing(prefix):
    """BatchNorm eps 1e-3, and the packed layout of 1x7 / 7x1 / 1x3 / 3x1 kernels and of the padded channel strides
    (3 -> 4, 48 -> 64, 80 -> 96): row n, column (dh kw + dw) cs + c holds W[n, c, dh, dw], everything else zero."""
    sd = fo.make_state_dict(2)
    g = torch.Generator().manual_seed(4)
    cout = sd[prefix + ".bn.weight"].numel()
    sd[prefix + ".bn.running_mean"] = torch.rand(cout, generator=g) - 0.5
    sd[prefix + ".bn.running_var"] = torch.rand(cout, generator=g) * 0.01 + 1e-4     # eps 1e-3 vs 1e-5 matters
    args = [sd[f"{prefix}.bn.{f}"] for f in ("weight", "bias", "running_mean", "running_var")]
    w, b = fid.fold_bn(sd[prefix + ".conv.weight"], *args)
    wo, bo = fo.fold_bn(sd, prefix)
    assert torch.equal(w, wo) and torch.equal(b, bo)
    assert not torch.equal(w, fo.fold_bn(sd, prefix, eps=1e-5)[0])
    conv = next(c for c in fid.conv_list() if c.name == prefix)
    u = fid._Unit(conv, w, b, "cpu")
    packed = u.w_hi + u.w_lo
    cout, cin, kh, kw = w.shape
    cs = fvd.cpad(cin)
    assert cs == {3: 4, 48: 64, 80: 96}.get(cin, cin)
    assert u.K == L.round_up(kh * kw * cs, 32) and packed.shape == (L.round_up(cout, 128), u.K)
    assert torch.equal(u.w_hi, L.tf32_round(u.w_hi))
    unpacked = packed[:cout, :kh * kw * cs].reshape(cout, kh, kw, cs)
    assert torch.equal(unpacked[..., :cin].permute(0, 3, 1, 2), wo)
    assert float(unpacked[..., cin:].abs().sum()) == 0 and float(packed[cout:].abs().sum()) == 0
    assert float(packed[:, kh * kw * cs:].abs().sum()) == 0


def test_folded_conv_equals_conv_then_bn():
    sd = fo.make_state_dict(3)
    p = "Mixed_6c.branch7x7dbl_3"
    sd[p + ".bn.running_mean"] = torch.linspace(-0.3, 0.3, 160)
    sd[p + ".bn.running_var"] = torch.linspace(0.2, 2.0, 160)
    x = torch.randn(1, 160, 9, 11, generator=torch.Generator().manual_seed(1))
    ref = fo.basic_conv(x, sd, p)
    w, b = fid.fold_bn(sd[p + ".conv.weight"], *(sd[f"{p}.bn.{f}"] for f in ("weight", "bias", "running_mean",
                                                                              "running_var")))
    got = F.relu(F.conv2d(x, w, b, padding=(0, 3)))
    assert float((got - ref).abs().max()) < 1e-5


def test_byte_lut_is_to_tensor():
    assert torch.equal(fid.byte_lut()[0], torch.arange(256, dtype=torch.uint8).float().div(255))


def test_real_byte_lut_matches_script():
    """The real side's lut for IMAGE_NORM over all 256 bytes: the loader's ToTensor + Normalize((.5,) * 3, (1,) * 3),
    vqgan_eval.py:204-205's ((x + 0.5).numpy() * 255).astype(np.uint8) written as a PNG, and pytorch-fid's ToTensor
    of the decoded byte."""
    from omnitokenizer_b200.consumers import IMAGE_NORM
    img = torch.arange(256, dtype=torch.uint8).view(1, 256, 1).expand(1, 256, 3).contiguous()
    t = img.permute(2, 0, 1).contiguous().float().div(255)                       # ToTensor
    t = (t - torch.tensor([0.5, 0.5, 0.5]).view(3, 1, 1)) / torch.tensor([1.0, 1.0, 1.0]).view(3, 1, 1)   # Normalize
    saved = ((t.permute(1, 2, 0) + 0.5).numpy() * 255).astype(np.uint8)          # (1, 256, 3)
    read = torch.from_numpy(saved).float().div(255)
    lut = fid.byte_lut(IMAGE_NORM)
    assert lut.shape == (1, 256)
    for c in range(3):
        assert torch.equal(lut[0], read[0, :, c])
    assert not torch.equal(lut[0], fid.byte_lut()[0])           # bytes 0 .. 255 do not all survive the round trip


def test_preprocess_arithmetic_matches_fixture():
    """The kernel's arithmetic (layout.clip_axis_table, torch's separable bilinear form, byte / 255 first, 2 y - 1)
    on the host equals the reference preprocess the fixture stored."""
    golden = torch.load(GOLDEN)
    for name, e in golden["images"].items():
        H, W = e["shape"]
        u8 = fo.image_bytes((H, W), e["seed"])
        v = u8.numpy().astype(np.float32) / np.float32(255)
        th = L.clip_axis_table(H, 299, float(np.float32(H) / np.float32(299)))
        tw = L.clip_axis_table(W, 299, float(np.float32(W) / np.float32(299)))
        l0h, l1h = (th[:, k].view(np.float32)[:, None, None] for k in (2, 3))
        l0w, l1w = (tw[:, k].view(np.float32)[None, :, None] for k in (2, 3))
        r0, r1 = v[th[:, 0]], v[th[:, 1]]
        x00, x01, x10, x11 = r0[:, tw[:, 0]], r0[:, tw[:, 1]], r1[:, tw[:, 0]], r1[:, tw[:, 1]]
        y = L.fma32(L.fma32(x00, l0w, x01 * l1w), l0h, L.fma32(x10, l0w, x11 * l1w) * l1h)
        y = np.float32(2) * y - np.float32(1)
        ref = torch.from_numpy(np.ascontiguousarray(y.transpose(2, 0, 1)))      # (3, 299, 299)
        assert torch.equal(ref.flatten()[e["pre_idx"]], e["pre_val"]), name


def test_activation_statistics_match_numpy():
    g = np.random.default_rng(3)
    act = g.standard_normal((300, 16)).astype(np.float32)
    mu, sigma = fid.activation_statistics(torch.from_numpy(act))
    assert mu.dtype == np.float64 and sigma.shape == (16, 16)
    assert np.array_equal(mu, np.mean(act.astype(np.float64), axis=0))
    assert np.array_equal(sigma, np.cov(act.astype(np.float64), rowvar=False))


def test_frechet_distance_matches_fixture():
    fd = torch.load(GOLDEN)["fd"]
    m1, s1 = fid.activation_statistics(fd["x1"])
    m2, s2 = fid.activation_statistics(fd["x2"])
    got = fid.calculate_frechet_distance(m1, s1, m2, s2)
    assert abs(got / fd["value"] - 1) < 1e-12, (got, fd["value"])
    assert abs(fid.calculate_frechet_distance(m1, s1, m1, s1)) < 1e-9


def test_frechet_distance_singular_product_retries():
    """Rank-deficient covariances: the eps retry still gives a finite, real distance."""
    g = np.random.default_rng(5)
    a, b = g.standard_normal((4, 12)), g.standard_normal((4, 12))
    m1, s1 = fid.activation_statistics(a)
    m2, s2 = fid.activation_statistics(b)
    v = fid.calculate_frechet_distance(m1, s1, m2, s2)
    assert np.isfinite(v) and np.isrealobj(v)


def test_state_dict_checks_name_keys_and_ignore_fc():
    sd = fo.make_state_dict(0)
    assert "fc.weight" in sd
    fid.FIDInception(sd, "cpu")                                   # with fc.* and num_batches_tracked
    sd2 = {k: v for k, v in sd.items() if not k.endswith("num_batches_tracked") and not k.startswith("fc.")}
    sd2["AuxLogits.fc.weight"] = torch.zeros(1000, 768)
    fid.FIDInception(sd2, "cpu")
    bad = dict(sd)
    del bad["Mixed_6e.branch7x7dbl_4.bn.running_var"]
    bad["Mixed_8a.branch1x1.conv.weight"] = torch.zeros(1)
    with pytest.raises(KeyError, match=r"Mixed_6e\.branch7x7dbl_4\.bn\.running_var.*Mixed_8a\.branch1x1\.conv\.weight"):
        fid.FIDInception(bad, "cpu")
    bad = dict(sd)
    bad["Mixed_6b.branch7x7_2.conv.weight"] = torch.zeros(128, 128, 7, 1)
    with pytest.raises(ValueError, match=r"Mixed_6b\.branch7x7_2\.conv\.weight"):
        fid.FIDInception(bad, "cpu")


def test_refusals_before_any_launch(tmp_path):
    from omnitokenizer_b200.layout import U8Norm
    net = fid.FIDInception(fo.make_state_dict(0), "cpu")
    n0 = _cabi.launch_count
    cases = [(torch.zeros(1, 32, 32, 3), TypeError),                           # fp32 images
             (np.zeros((1, 32, 32, 3), np.uint8), TypeError),                   # numpy
             (torch.zeros(1, 32, 32, 4, dtype=torch.uint8), ValueError),       # 4 channels
             (torch.zeros(32, 32, 3, dtype=torch.uint8), ValueError),          # rank 3
             (torch.zeros(1, 1, 32, 32, 3, dtype=torch.uint8), ValueError),    # rank 5
             (torch.zeros(0, 32, 32, 3, dtype=torch.uint8), ValueError)]       # empty batch
    for images, err in cases:
        with pytest.raises(err):
            net.features(images)
    with pytest.raises(ValueError, match="per channel"):
        net.features(torch.zeros(1, 32, 32, 3, dtype=torch.uint8), real_norm=U8Norm("x", (0.4, 0.5, 0.6), (1.0,) * 3))
    with pytest.raises(ValueError, match="2048"):
        fid.load_fid_model("cpu", str(tmp_path / "none.pth"), dims=768)
    with pytest.raises(ValueError, match="2048"):
        fid.fid_given_paths([str(tmp_path), str(tmp_path)], net, dims=192)
    assert _cabi.launch_count == n0


def test_image_files_order(tmp_path):
    """fid_score.py's listing: the sorted */*.ext files when there are any, else the sorted *.ext files."""
    (tmp_path / "b").mkdir()
    (tmp_path / "a").mkdir()
    for p in ("b/2.png", "a/9.jpg", "a/1.png", "top.png"):
        (tmp_path / p).write_bytes(b"")
    assert [f.relative_to(tmp_path).as_posix() for f in fid.image_files(tmp_path)] == ["a/1.png", "a/9.jpg", "b/2.png"]
    flat = tmp_path / "flat"
    flat.mkdir()
    for p in ("z.webp", "c.png", "x.txt"):
        (flat / p).write_bytes(b"")
    assert [f.name for f in fid.image_files(flat)] == ["c.png", "z.webp"]


def test_eval_step_fid_refuses_per_channel_norm():
    from omnitokenizer_b200 import consumers as C
    from omnitokenizer_b200.layout import U8Norm
    n0 = _cabi.launch_count
    with pytest.raises(ValueError, match="per channel"):
        C.eval_step_fid(object(), [torch.zeros(8, 8, 3, dtype=torch.uint8)], L.image_resize(64), None,
                        norm=U8Norm("x", (0.4, 0.5, 0.6), (1.0,) * 3))
    with pytest.raises(ValueError, match="at least one image"):
        C.eval_step_fid(object(), [], L.image_resize(64), None)
    assert _cabi.launch_count == n0
