"""The Inception Score on the GPU: omt_pool2d's count_include_pad average and omt_is_preprocess against torch's CPU
bits, omt_softmax_rows and omt_inception_score against float64 / scipy, the network's logits and scores against the
reference fixture, determinism, independence from chunk-mates, and the uint8 form."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from omnitokenizer_b200 import _cabi
from omnitokenizer_b200 import fid
from omnitokenizer_b200 import iscore
from omnitokenizer_b200 import layout as L
from omnitokenizer_b200.engine import CLIP_DESC_WORDS
from oracle import fid_oracle as fo
from oracle import is_oracle as io

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "is_inception.pt")


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN, weights_only=False)


@pytest.fixture(scope="module")
def model(golden):
    sd = io.fixture_state_dict(golden)
    assert fo.conv_fingerprint(sd) == golden["fingerprint"]
    return iscore.ISInception(sd, DEV)


def to_cl(x, cs):
    y = torch.zeros(x.shape[0], *x.shape[2:], cs, dtype=x.dtype)
    y[..., :x.shape[1]] = x.permute(0, 2, 3, 1)
    return y


# (C, H, W, k, s, p, col, ldy): torchvision's avg_pool2d(3, 1, 1) branch pools at their sizes, then a column offset,
# odd sizes with stride 2, and windows whose padded edge cuts the count (k 4, p 2; k 5 s 3 p 2)
POOLS = [(192, 35, 35, 3, 1, 1, 0, 192), (256, 35, 35, 3, 1, 1, 0, 256), (288, 35, 35, 3, 1, 1, 0, 288),
         (768, 17, 17, 3, 1, 1, 0, 768), (1280, 8, 8, 3, 1, 1, 0, 1280), (2048, 8, 8, 3, 1, 1, 0, 2048),
         (64, 9, 9, 3, 1, 1, 32, 128), (64, 13, 10, 3, 2, 1, 0, 64), (32, 11, 7, 4, 2, 2, 0, 32),
         (32, 13, 12, 5, 3, 2, 32, 96)]


@pytest.mark.parametrize("case", POOLS, ids=[f"k{c[3]}s{c[4]}p{c[5]}_{c[0]}x{c[1]}x{c[2]}_col{c[6]}" for c in POOLS])
def test_pool2d_avg_pad_exact(case):
    C, H, W, k, s, p, col, ldy = case
    g = torch.Generator().manual_seed(C + H + k)
    x = torch.randn(2, C, H, W, generator=g)
    ref = F.avg_pool2d(x, k, s, p, count_include_pad=True)
    Ho, Wo = (fid.out_size(n, k, s, p) for n in (H, W))
    assert tuple(ref.shape[2:]) == (Ho, Wo)
    y = torch.full((2, Ho, Wo, ldy), -7.0, device=DEV)
    _cabi.call("omt_pool2d", to_cl(x, C).to(DEV), C, C, 2, H, W, k, k, s, s, p, p, Ho, Wo, y.data_ptr() + 4 * col, ldy,
               fid.POOL_AVG_PAD)
    torch.cuda.synchronize()
    y = y.cpu()
    assert torch.equal(y[..., col:col + C], ref.permute(0, 2, 3, 1))
    assert bool((y[..., :col] == -7).all()) and bool((y[..., col + C:] == -7).all())


def run_preprocess(src, form, H, W, resize):
    N = src.shape[0]
    oh, ow = iscore.TARGET_RESOLUTION if resize else (H, W)
    tab_host = torch.from_numpy(np.concatenate([iscore.axis_table(H, oh if resize else None).reshape(-1),
                                                iscore.axis_table(W, ow if resize else None).reshape(-1)]))
    desc = torch.zeros(N, CLIP_DESC_WORDS, dtype=torch.int32)
    desc[:, :2] = (torch.arange(N, dtype=torch.int64) * (3 * H * W)).view(torch.int32).view(N, 2)
    desc[:, 2:] = torch.tensor([H, W, 0, 0, H, W, oh, ow, 0, 0, 0, 0, 4 * oh, L.INTERP_SEPARABLE], dtype=torch.int32)
    out = torch.full((N, oh, ow, 4), float("nan"), device=DEV)
    srcd = src.contiguous().to(DEV)
    _cabi.call("omt_is_preprocess", srcd, srcd.numel(), form, desc.to(DEV), desc, tab_host.to(DEV), tab_host,
               tab_host.numel(), N, 1, oh, ow, out)
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("form", ["f32", "u8"])
@pytest.mark.parametrize("hw,resize", [((64, 64), True), ((336, 400), True), ((32, 32), True), ((48, 80), True),
                                       ((299, 299), True), ((96, 128), False), ((75, 81), False)])
def test_preprocess_exact(form, hw, resize):
    H, W = hw
    g = torch.Generator().manual_seed(H * 1000 + W)
    u8 = torch.randint(0, 256, (3, H, W, 3), generator=g, dtype=torch.uint8)
    x = u8.permute(0, 3, 1, 2).float() / 255 if form == "u8" else torch.randn(3, 3, H, W, generator=g)
    ref = io.preprocess(x, resize)
    got = run_preprocess(u8 if form == "u8" else x, iscore.FORM_U8 if form == "u8" else iscore.FORM_F32, H, W, resize)
    assert torch.equal(got[..., :3], ref.permute(0, 2, 3, 1))
    assert bool((got[..., 3] == 0).all())
    if resize:
        cuda = F.interpolate(x.to(DEV), size=(299, 299), mode="bilinear", align_corners=False).cpu()
        print(f"{form} {H}x{W}: max|torch CUDA interpolate - CPU| {float((cuda - ref).abs().max()):.2e}")


def test_softmax_rows_against_float64(golden):
    for name, g in golden["cases"].items():
        lg = g["logits"]
        y = torch.full_like(lg, float("nan"), device=DEV)
        _cabi.call("omt_softmax_rows", lg.to(DEV), lg.shape[1], lg.shape[0], lg.shape[1], y, lg.shape[1])
        ref = torch.softmax(lg.double(), 1)
        err = (y.cpu().double() - ref).abs()
        assert bool((err <= 1e-6 * ref + 1e-44).all()), (name, float((err / ref.clamp_min(1e-30)).max()))


def test_score_reduction_against_scipy(golden):
    from scipy.stats import entropy
    for name, g in golden["cases"].items():
        splits = g["spec"]["splits"]
        preds = g["probs"].double().numpy()
        N, n = preds.shape[0], preds.shape[0] // splits
        scores = []
        for k in range(splits):
            part = preds[k * n:(k + 1) * n]
            py = np.mean(part, axis=0)
            scores.append(np.exp(np.mean([entropy(part[i], py) for i in range(part.shape[0])])))
        mean, std = iscore.score(g["probs"].to(DEV), splits)
        assert abs(mean - np.mean(scores)) <= 1e-12 * np.mean(scores), name
        assert abs(std - np.std(scores)) <= 1e-12 * np.mean(scores), name
        assert mean == g["mean"] or abs(mean - g["mean"]) <= 1e-12 * g["mean"]
        again = iscore.score(g["probs"].to(DEV), splits)
        assert again == (mean, std)


def _case_frames(spec):
    x, u8 = io.case_input(spec)
    if spec["fn"] == "calculate_is":
        return x.reshape(-1, *x.shape[2:]), u8
    return x, None


@pytest.mark.parametrize("name", list(io.CASES))
def test_network_against_fixture(golden, model, name):
    g = golden["cases"][name]
    spec = g["spec"]
    frames, _ = _case_frames(spec)
    resize = spec.get("resize", True)
    probs = model.probabilities(frames.to(DEV), resize=resize).clone()
    oh, ow = iscore.TARGET_RESOLUTION if resize else tuple(frames.shape[2:])
    logits = model._ws[(frames.shape[0], oh, ow)].logits.cpu()
    scale = float(g["logits"].abs().max())
    err = float((logits - g["logits"]).abs().max()) / scale
    if spec["fn"] == "calculate_is":
        mean, std = iscore.calculate_is(io.case_input(spec)[0], DEV, spec["splits"], model=model)
    else:
        mean, std = iscore.inception_score(frames, batch_size=spec["batch_size"], resize=resize, splits=spec["splits"],
                                           model=model)
    print(f"{name}: logits max|diff| / max|logit| {err:.2e}; IS {mean:.6f} vs {g['mean']:.6f} "
          f"(rel {abs(mean - g['mean']) / g['mean']:.2e}), std {std:.6f} vs {g['std']:.6f}")
    assert err <= 3e-4
    assert abs(mean - g["mean"]) <= 1e-4 * g["mean"]
    assert abs(std - g["std"]) <= 1e-4 * g["mean"]
    assert torch.equal(model.probabilities(frames.to(DEV), resize=resize).cpu(), probs.cpu())   # the graph replay


def test_uint8_equals_float_of_bytes(model):
    spec = io.CASES["calc_u8_48x64"]
    x, u8 = io.case_input(spec)
    a = model.probabilities(u8.reshape(-1, *u8.shape[2:]).to(DEV)).cpu()
    b = model.probabilities(x.reshape(-1, *x.shape[2:]).to(DEV)).cpu()
    assert torch.equal(a, b)
    assert iscore.calculate_is(u8, DEV, 2, model=model) == iscore.calculate_is(x, DEV, 2, model=model)
    assert iscore.calculate_is(u8.to(DEV), DEV, 2, model=model) == iscore.calculate_is(u8, DEV, 2, model=model)


def test_frame_rows_do_not_depend_on_chunk_mates(model):
    N = 2 * iscore.CHUNK_FRAMES + 5
    frames = io.frames((N, 40, 48), 909).to(DEV)
    batch = model.probabilities(frames).cpu()
    for i in range(N):
        alone = model.probabilities(frames[i:i + 1]).cpu()
        assert torch.equal(alone[0], batch[i]), i
