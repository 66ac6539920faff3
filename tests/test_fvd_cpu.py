"""Host logic of omnitokenizer_b200.fvd without a GPU: SAME geometry, BatchNorm folding and packing, state_dict checks,
the preprocess arithmetic the kernel runs, and refusals before any launch."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from omnitokenizer_b200 import _cabi
from omnitokenizer_b200 import fvd
from omnitokenizer_b200 import layout as L
from oracle import i3d_oracle as io

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "fvd_i3d.pt")


def layers():
    """(kernel, stride) of every conv and pool in order, with the spatial path of a 224^2 input."""
    out = []
    for name, kind, spec in fvd.ARCH:
        if kind == "unit":
            out.append(((spec[2],) * 3, (spec[3],) * 3))
        elif kind == "pool":
            out.append(spec)
        else:
            out += [((1, 1, 1), (1, 1, 1)), ((3, 3, 3), (1, 1, 1))]
    return out


@pytest.mark.parametrize("T", [9, 17, 33])
def test_same_padding_matches_compute_pad(T):
    dims = (T, 224, 224)
    for k, s in layers():
        front, o = fvd.same_geometry(k, s, dims)
        pads = io.same_pad(k, s, dims)                 # (w_f, w_b, h_f, h_b, t_f, t_b)
        assert front == (pads[4], pads[2], pads[0])
        x = torch.empty(1, 1, *dims, device="meta")
        ref = F.max_pool3d(F.pad(x, pads), k, s).shape[2:]
        assert o == tuple(ref)
        if s == (1, 1, 1):
            continue
        dims = o


def test_arch_matches_oracle():
    assert [(n, 3 if k == "unit" else 1) for n, k, _ in fvd.ARCH] == [(n, 3 if k == "unit" else 1) for n, k, _ in io.ARCH]
    assert [(p, ci, co, (k,) * 3, (s,) * 3) for p, ci, co, k, s in fvd.unit_names()] == io.units()


def test_bn_folding_and_packing_match_oracle():
    sd = io.make_state_dict(2)
    g = torch.Generator().manual_seed(4)
    for prefix, cin, cout, k, _ in fvd.unit_names():
        sd[prefix + ".bn.running_mean"] = torch.rand(cout, generator=g) - 0.5
        sd[prefix + ".bn.running_var"] = torch.rand(cout, generator=g) + 0.1
    for prefix in ("Conv3d_1a_7x7", "Mixed_3b.b2a", "Mixed_4e.b1b", "Mixed_5c.b3b"):
        w, b = fvd.fold_bn(sd[prefix + ".conv3d.weight"],
                           *(sd[f"{prefix}.bn.{f}"] for f in ("weight", "bias", "running_mean", "running_var")))
        wo, bo = io.fold_bn(sd, prefix)
        assert torch.equal(w, wo) and torch.equal(b, bo)
        packed, K = fvd.pack_weight(w)
        cout, cin, kt, kh, kw = w.shape
        cs = fvd.cpad(cin)
        assert K == L.round_up(kt * kh * kw * cs, 32) and packed.shape == (L.round_up(cout, 128), K)
        # row n, column ((dt kh + dh) kw + dw) cs + c holds W[n, c, dt, dh, dw]; everything else is zero
        unpacked = packed[:cout, :kt * kh * kw * cs].reshape(cout, kt, kh, kw, cs)
        assert torch.equal(unpacked[..., :cin].permute(0, 4, 1, 2, 3), wo)
        assert float(unpacked[..., cin:].abs().sum()) == 0 and float(packed[cout:].abs().sum()) == 0
        assert float(packed[:, kt * kh * kw * cs:].abs().sum()) == 0


def test_folded_unit_equals_conv_then_bn():
    sd = io.make_state_dict(3)
    sd["Mixed_3b.b1b.bn.running_mean"] = torch.linspace(-0.3, 0.3, 128)
    sd["Mixed_3b.b1b.bn.running_var"] = torch.linspace(0.2, 2.0, 128)
    x = torch.randn(1, 96, 3, 5, 6, generator=torch.Generator().manual_seed(1))
    ref = io.unit3d(x, sd, "Mixed_3b.b1b", (3, 3, 3), (1, 1, 1))
    w, b = fvd.fold_bn(sd["Mixed_3b.b1b.conv3d.weight"],
                       *(sd[f"Mixed_3b.b1b.bn.{f}"] for f in ("weight", "bias", "running_mean", "running_var")))
    got = F.relu(F.conv3d(F.pad(x, io.same_pad((3, 3, 3), (1, 1, 1), x.shape[2:])), w, b))
    assert float((got - ref).abs().max()) < 1e-5


def test_preprocess_arithmetic_matches_fixture():
    """The kernel's arithmetic (layout.clip_axis_table, torch's separable bilinear form, 2 y / 255 - 1) on the host
    equals the reference preprocess the fixture stored, whatever this host's thread count."""
    golden = torch.load(GOLDEN)
    for name, e in golden["clips"].items():
        T, H, W = e["shape"]
        u8 = (torch.full((T, H, W, 3), 200, dtype=torch.uint8) if e["seed"] is None else
              torch.randint(0, 256, (T, H, W, 3), generator=torch.Generator().manual_seed(e["seed"]), dtype=torch.uint8))
        v = u8.numpy().astype(np.float32)
        th = L.clip_axis_table(H, 224, float(np.float32(H) / np.float32(224)))
        tw = L.clip_axis_table(W, 224, float(np.float32(W) / np.float32(224)))
        l0h, l1h = (th[:, k].view(np.float32)[None, :, None, None] for k in (2, 3))
        l0w, l1w = (tw[:, k].view(np.float32)[None, None, :, None] for k in (2, 3))
        r0, r1 = v[:, th[:, 0]], v[:, th[:, 1]]
        x00, x01, x10, x11 = r0[:, :, tw[:, 0]], r0[:, :, tw[:, 1]], r1[:, :, tw[:, 0]], r1[:, :, tw[:, 1]]
        y = L.fma32(L.fma32(x00, l0w, x01 * l1w), l0h, L.fma32(x10, l0w, x11 * l1w) * l1h)
        y = np.float32(2) * y / np.float32(255) - np.float32(1)
        ref = torch.from_numpy(np.ascontiguousarray(y.transpose(3, 0, 1, 2)))     # (3, T, 224, 224)
        assert torch.equal(ref.flatten()[e["pre_idx"]], e["pre_val"]), name


def test_state_dict_checks_name_keys():
    sd = io.make_state_dict(0)
    fvd.I3D(sd, "cpu")                                   # with num_batches_tracked
    fvd.I3D({k: v for k, v in sd.items() if not k.endswith("num_batches_tracked")}, "cpu")
    bad = dict(sd)
    del bad["Mixed_4e.b1b.bn.running_var"]
    bad["Mixed_9z.b0.conv3d.weight"] = torch.zeros(1)
    with pytest.raises(KeyError, match=r"Mixed_4e\.b1b\.bn\.running_var.*Mixed_9z\.b0\.conv3d\.weight"):
        fvd.I3D(bad, "cpu")
    bad = dict(sd)
    bad["Mixed_3b.b0.conv3d.weight"] = torch.zeros(64, 192, 3, 3, 3)
    with pytest.raises(ValueError, match="Mixed_3b.b0.conv3d.weight"):
        fvd.I3D(bad, "cpu")
    sd101 = io.make_state_dict(0, num_classes=101)
    assert fvd.I3D(sd101, "cpu").num_classes == 101


def test_refusals_before_any_launch():
    net = fvd.I3D(io.make_state_dict(0), "cpu")
    n0 = _cabi.launch_count
    cases = [(torch.zeros(1, 9, 32, 32, 3), TypeError),                       # fp32 frames
             (np.zeros((1, 9, 32, 32, 3), np.uint8), TypeError),              # numpy to logits
             (torch.zeros(1, 9, 32, 32, 4, dtype=torch.uint8), ValueError),   # 4 channels
             (torch.zeros(9, 32, 32, 3, dtype=torch.uint8), ValueError),      # rank 4
             (torch.zeros(1, 8, 32, 32, 3, dtype=torch.uint8), ValueError),   # T = 8: the reference's AvgPool3d raises
             (torch.zeros(0, 9, 32, 32, 3, dtype=torch.uint8), ValueError)]   # empty batch
    for frames, err in cases:
        with pytest.raises(err):
            net.logits(frames)
    with pytest.raises(ValueError, match="T >= 9"):
        fvd.get_fvd_logits(np.zeros((2, 8, 16, 16, 3), np.uint8), net, "cpu")
    assert _cabi.launch_count == n0


def test_frechet_distance_matches_fixture():
    fd = torch.load(GOLDEN)["fd"]
    assert abs(float(fvd.frechet_distance(fd["x1"], fd["x2"])) / float(fd["value"]) - 1) < 1e-6


@pytest.mark.parametrize("branch", [0, 1])
def test_real_byte_map_matches_script(branch):
    """real_byte_table against vqgan_eval.py's real_videos = batch['video'] + 0.5; shift_dim(real_videos * 255, 1,
    -1).byte() of VideoNorm (video_utils.py:46-58) applied to a clip holding every byte value (branch 0: max > 1, / 255)
    or, for branch 1, the undivided expression (VideoNorm's max <= 1 branch, used only for clips of 0 / 1 bytes)."""
    from omnitokenizer_b200.consumers import VIDEO_NORM
    img = torch.arange(256, dtype=torch.uint8).float().view(1, 1, 1, 256).expand(1, 3, 1, 256).clone()
    mean, std = torch.tensor([0.5, 0.5, 0.5]).view(1, 3, 1, 1), torch.tensor([1.0, 1.0, 1.0]).view(1, 3, 1, 1)
    if branch == 0:
        img.div_(255.0)
    video = img.sub_(mean).div_(std)
    script = ((video + 0.5) * 255).byte()                 # (1, 3, 1, 256)
    tab = fvd.real_byte_table(VIDEO_NORM)
    assert tab.shape == (2, 256)
    for c in range(3):
        assert torch.equal(tab[branch], script[0, c, 0])


def test_real_byte_map_refuses_per_channel_norms():
    from omnitokenizer_b200.layout import U8Norm
    with pytest.raises(ValueError, match="per channel"):
        fvd.real_byte_table(U8Norm("x", (0.4, 0.5, 0.6), (1.0, 1.0, 1.0)))


def test_eval_step_fvd_refuses_before_any_launch():
    from omnitokenizer_b200 import consumers as C
    net = fvd.I3D(io.make_state_dict(0), "cpu")
    n0 = _cabi.launch_count
    with pytest.raises(ValueError, match="T >= 9"):
        C.eval_step_fvd(object(), torch.zeros(1, 5, 64, 64, 3, dtype=torch.uint8), net)
    with pytest.raises(TypeError):
        C.eval_step_fvd(object(), torch.zeros(1, 9, 64, 64, 3), net)
    assert _cabi.launch_count == n0
