"""Per-frame PSNR / SSIM / VGG LPIPS on the GPU: omt_psnr_ssim against the fp64 oracle and the reference fixture,
omt_lpips_head against fp64, LPIPS end to end against the fixture, determinism and graph replay, the real-side
selector, eval_step_quality, and the drop-ins on the suite's float input.  Measured worst cases are printed."""
import os

import numpy as np
import pytest
import torch

from omnitokenizer_b200 import _cabi, quality
from omnitokenizer_b200.fvd import real_byte_table
from oracle import quality_oracle as qo

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "quality.pt")
# LPIPS per frame, relative: measured worst 3.4e-6 against the fp32 reference (the constant pair, whose value is a
# hundred times smaller than a noisy pair's); the bound leaves room for the 3xTF32 convs' larger error on other weights
LPIPS_REL = 1e-4


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN)


@pytest.fixture(scope="module")
def model(golden):
    sd = qo.make_state_dict(golden["w_seed"])
    assert qo.fingerprint(sd) == golden["fingerprint"]
    return quality.LPIPS(sd, DEV), sd


def _oracle_frame(a_u8, b_u8, taps):
    a, b = qo.to01(a_u8).double().numpy(), qo.to01(b_u8).double().numpy()
    sse = float(((a - b) ** 2).sum())
    return sse, qo.ssim(a, b, taps)


def _noisy_batch(P, H, W, seed):
    pairs = [qo.frame_pair((H, W, "noise", seed + i)) for i in range(P)]
    return torch.stack([p[0] for p in pairs]), torch.stack([p[1] for p in pairs])


def _raw_psnr_ssim(a, b, taps):
    P, H, W = a.shape[:3]
    lut = (torch.arange(256, dtype=torch.float32) / 255).to(DEV)
    sse = torch.empty(P, dtype=torch.float64, device=DEV)
    ssim = torch.empty(P, dtype=torch.float64, device=DEV)
    _cabi.call("omt_psnr_ssim", a.to(DEV), lut, None, b.to(DEV), lut, None, quality.FORM_U8, P, H, W, taps.to(DEV),
               sse, ssim)
    torch.cuda.synchronize()
    return sse.cpu(), ssim.cpu()


@pytest.mark.parametrize("P,H,W", [(136, 64, 64), (3, 256, 256), (5, 67, 93), (4, 11, 11), (2, 45, 12)])
def test_psnr_ssim_against_fp64_oracle(golden, P, H, W):
    a, b = _noisy_batch(P, H, W, 100 + H)
    sse, ssim = _raw_psnr_ssim(a, b, golden["taps"])
    taps = golden["taps"].numpy()
    worst_sse = worst_ssim = 0.0
    for p in range(P):
        s, m = _oracle_frame(a[p], b[p], taps)
        worst_sse = max(worst_sse, abs(float(sse[p]) - s) / s)
        worst_ssim = max(worst_ssim, abs(float(ssim[p]) - m))
    print(f"P={P} {H}x{W}: sse rel {worst_sse:.1e}, ssim abs {worst_ssim:.1e}")
    assert worst_sse <= 1e-12 and worst_ssim <= 1e-12


def test_psnr_ssim_against_reference_fixture(golden, model):
    net, _ = model
    worst_p = worst_s = worst_l = 0.0
    for name, e in golden["cases"].items():
        a, b = qo.frame_pair(e["spec"])
        lp = net if e["lpips"] is not None else None
        psnr, ssim, lpv = quality.frame_metrics(a[None, None].to(DEV), b[None, None].to(DEV), lp)
        psnr, ssim = float(psnr[0, 0]), float(ssim[0, 0])
        dp = abs(psnr - e["psnr"])
        worst_p, worst_s = max(worst_p, dp), max(worst_s, abs(ssim - e["ssim"]))
        assert dp <= 1e-9 and abs(ssim - e["ssim"]) <= 1e-9, name
        if e["psnr"] == 100:
            assert psnr == 100.0, name
        if lp is not None:
            got, ref = float(lpv[0, 0]), e["lpips"]
            if ref == 0.0:
                assert got == 0.0, name
                continue
            rel = abs(got - ref) / abs(ref)
            worst_l = max(worst_l, rel)
            print(f"{name}: lpips {got:.9g} vs {ref:.9g}, rel {rel:.1e}")
            assert rel <= LPIPS_REL, name
    print(f"fixture: psnr abs {worst_p:.1e}, ssim abs {worst_s:.1e}, lpips rel {worst_l:.1e}")


def test_fixture_cases_batched_on_the_136_grid(golden):
    """Every psnr / ssim fixture case of one size inside a P = 136 (8 x 17) batch, at rotating positions."""
    for name, e in golden["cases"].items():
        a, b = qo.frame_pair(e["spec"])
        H, W = a.shape[:2]
        fa, fb = _noisy_batch(136, H, W, 7)
        pos = (len(name) * 13) % 136
        fa[pos], fb[pos] = a, b
        psnr, ssim, _ = quality.frame_metrics(fa.view(8, 17, H, W, 3).to(DEV), fb.view(8, 17, H, W, 3).to(DEV))
        assert abs(float(psnr.flatten()[pos]) - e["psnr"]) <= 1e-9, name
        assert abs(float(ssim.flatten()[pos]) - e["ssim"]) <= 1e-9, name


@pytest.mark.parametrize("C,h,w,P", [(64, 37, 29, 3), (128, 16, 16, 2), (512, 1, 1, 4), (256, 8, 13, 5)])
def test_lpips_head_against_fp64(C, h, w, P):
    g = torch.Generator().manual_seed(C + h)
    x = torch.relu(torch.randn(2 * P, h, w, C, generator=g))
    x[0, 0, 0] = 0                                   # an all-zero feature vector: normalises to zero via the 1e-10
    x[2 * P - 1, -1, -1] = 0                        # in another pair, so no pair's reference value is 0
    lin = torch.rand(C, generator=g)
    taps = torch.full((5, P), -1.0, device=DEV)
    total = torch.full((P,), -1.0, device=DEV)
    # fill taps 0..2 first so tap 3's total adds them in order
    prev = torch.rand(3, P, generator=g)
    taps[:3] = prev.to(DEV)
    _cabi.call("omt_lpips_head", x.to(DEV), C, C, P, h, w, lin.to(DEV), 3, taps, total)
    torch.cuda.synchronize()
    xc = x.permute(0, 3, 1, 2)
    ref = qo.lpips_head64(xc[:P], xc[P:], lin)
    got = taps[3].cpu().double()
    rel = float(((got - ref).abs() / ref.abs()).max())
    print(f"head C={C} {h}x{w}: rel {rel:.1e}")
    assert rel <= 2e-6
    want = prev[0] + prev[1] + prev[2] + taps[3].cpu()
    assert torch.equal(total.cpu(), ((prev[0] + prev[1]) + prev[2]) + taps[3].cpu()) and torch.allclose(total.cpu(), want)


def test_determinism_and_graph_replay(model):
    net, _ = model
    a, b = _noisy_batch(6, 64, 80, 300)
    a, b = a.view(2, 3, 64, 80, 3).to(DEV), b.view(2, 3, 64, 80, 3).to(DEV)
    outs = [tuple(t.clone() for t in quality.frame_metrics(a, b, net)) for _ in range(3)]   # eager, capture, replay
    for o in outs[1:]:
        assert all(torch.equal(x, y) for x, y in zip(o, outs[0]))
    ws = net._ws[(DEV, quality.FORM_U8, 6, 64, 80, None)]
    assert isinstance(ws.graphs.get("quality"), tuple)


def test_real_side_selector(model):
    """real_norm=VIDEO_NORM: clip 1 has bytes 0 / 1 only (VideoNorm's undivided branch); the metrics equal those of the
    bytes the script makes of the normalised clips, mapped on the host."""
    from omnitokenizer_b200.consumers import VIDEO_NORM
    net, _ = model
    a, b = _noisy_batch(6, 32, 48, 400)
    a = a.view(2, 3, 32, 48, 3).clone()
    a[1] %= 2
    b = b.view(2, 3, 32, 48, 3)
    got = quality.frame_metrics(a.to(DEV), b.to(DEV), net, real_norm=VIDEO_NORM)
    tab = real_byte_table(VIDEO_NORM)
    sel = (a.reshape(2, -1).amax(1) <= 1).long()
    mapped = torch.stack([tab[sel[i]][a[i].long()] for i in range(2)])
    want = quality.frame_metrics(mapped.to(DEV), b.to(DEV), net)
    assert int(sel[1]) == 1 and int(sel[0]) == 0
    assert all(torch.equal(x, y) for x, y in zip(got, want))


def test_eval_step_quality(model):
    import omnitokenizer_b200 as ob
    from omnitokenizer_b200 import consumers as C
    from oracle import omni_oracle as oo
    from oracle import weights as W
    net, sd = model
    args = ob.canonical_args()
    m = ob.OmniTokenizer_VQGAN(args)
    m.load_state_dict(W.make_state_dict(oo.Config.from_args(args), 0), strict=False)
    m.codebook._need_init = False
    m = m.to(DEV).eval()
    g = torch.Generator().manual_seed(5)
    u8 = torch.randint(0, 256, (2, 5, 64, 64, 3), generator=g, dtype=torch.uint8)
    frames = u8.to(DEV)
    psnr, ssim, lp, fake, vq = C.eval_step_quality(m, frames, net)
    fake2, _ = C.eval_step_u8(m, frames)
    assert torch.equal(fake, fake2)
    video = C.u8_normalize(u8, C.VIDEO_NORM)                          # the script's real_videos bytes
    real_bytes = ((video + 0.5) * 255).movedim(1, -1).byte()
    fk = fake.cpu()
    taps = quality.gaussian_taps().numpy()
    for i in range(2):
        for t in range(5):
            a, b = qo.to01(real_bytes[i, t]).double().numpy(), qo.to01(fk[i, t]).double().numpy()
            assert abs(float(psnr[i, t]) - qo.psnr(a, b)) <= 1e-9
            assert abs(float(ssim[i, t]) - qo.ssim(a, b, taps)) <= 1e-11
    with torch.no_grad():
        ref = qo.lpips(sd, qo.to01(real_bytes.flatten(0, 1)), qo.to01(fk.flatten(0, 1)))
    rel = float(((lp.cpu().flatten() - ref).abs() / ref.abs()).max())
    print(f"eval_step_quality lpips rel {rel:.1e}")
    assert rel <= LPIPS_REL


def test_dropins_on_float_videos(model):
    net, sd = model
    g = torch.Generator().manual_seed(9)
    v1 = torch.rand(3, 2, 3, 40, 52, generator=g)
    v2 = (v1 + 0.05 * torch.randn(3, 2, 3, 40, 52, generator=g)).clamp(0, 1)
    rp, rs = quality.calculate_psnr(v1, v2), quality.calculate_ssim(v1.to(DEV), v2.to(DEV))
    rl = quality.calculate_lpips_vgg(v1, v2, net)
    taps = quality.gaussian_taps().numpy()
    per_p = [[qo.psnr(v1[i, t].double().numpy(), v2[i, t].double().numpy()) for t in range(2)] for i in range(3)]
    per_s = [[qo.ssim(v1[i, t].double().numpy(), v2[i, t].double().numpy(), taps) for t in range(2)] for i in range(3)]
    with torch.no_grad():
        per_l = qo.lpips(sd, v1.flatten(0, 1), v2.flatten(0, 1)).view(3, 2).double().numpy()
    for r, per, tol in ((rp, per_p, 1e-9), (rs, per_s, 1e-11)):
        assert r["video_setting"] == v1[0].shape and r["video_setting_name"] == "time, channel, heigth, width"
        for t in range(2):
            assert abs(r["value"][t] - np.mean(np.array(per)[:, t])) <= tol
            assert abs(r["value_std"][t] - np.std(np.array(per)[:, t])) <= 10 * tol
    for t in range(2):
        assert abs(rl["value"][t] - np.mean(per_l[:, t])) <= LPIPS_REL * abs(np.mean(per_l[:, t]))
