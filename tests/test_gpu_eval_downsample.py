"""vqgan_eval.py's --infer_downsample and --replacewithgt on the device: omt_eval_downsample and the LANCZOS
omt_resample_u8 against tests/golden/eval_downsample.pt and against torch / Pillow run live, eval_step_fvd and
eval_step_fid with the flags against the networks on the script's bytes, a CUDA-graph replay, and refusals before
any launch."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from omnitokenizer_b200 import _cabi, consumers as C, downsample, fid, fvd
from omnitokenizer_b200 import layout as L
from tests.util import load_golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def fx():
    return load_golden("eval_downsample")


@pytest.fixture(scope="module")
def model():
    import omnitokenizer_b200 as ob
    from oracle import omni_oracle as oo
    from oracle import weights as W
    args = ob.canonical_args()
    m = ob.OmniTokenizer_VQGAN(args)
    m.load_state_dict(W.make_state_dict(oo.Config.from_args(args), 0), strict=False)
    m.codebook._need_init = False
    return m.to(DEV).eval()


@pytest.fixture(scope="module")
def i3d():
    from oracle import i3d_oracle as io
    g = load_golden("fvd_i3d")
    sd = io.make_state_dict(g["w_seed"])
    sd.update(g["bn"])
    return fvd.I3D(sd, DEV)


@pytest.fixture(scope="module")
def inception():
    from oracle import fid_oracle as fo
    g = load_golden("fid_inception")
    sd = fo.make_state_dict(g["w_seed"])
    sd.update(g["bn"])
    return fid.FIDInception(sd, DEV)


def _clips(seed, B=2, T=9, S=128):
    g = torch.Generator().manual_seed(seed)
    u8 = torch.randint(0, 256, (B, T, S, S, 3), generator=g, dtype=torch.uint8)
    u8[-1] %= 2                                               # VideoNorm's max <= 1 branch
    return u8


def _script_video(u8, x_recons, d, k=None):
    """vqgan_eval.py:121-148 on the host: the bytes get_fvd_logits receives for each side."""
    real_videos = L.u8_normalize(u8, C.VIDEO_NORM) + 0.5
    fake_videos = torch.clamp(x_recons.cpu() + 0.5, 0, 1)
    if d is not None:
        B = u8.shape[0]
        real_videos, fake_videos = (
            F.interpolate(v.permute(0, 2, 1, 3, 4).flatten(0, 1), scale_factor=1 / d, mode="bilinear",
                          align_corners=False).unflatten(0, (B, -1)).permute(0, 2, 1, 3, 4)
            for v in (real_videos, fake_videos))
    if k is not None:
        fake_videos = torch.cat((real_videos[:, :, :k], fake_videos[:, :, k:]), dim=2)
    return tuple((v * 255).movedim(1, -1).byte().contiguous() for v in (real_videos, fake_videos))


def test_kernel_equals_fixture(fx):
    for case in fx["video"] + fx["replace"]:
        c = fx["clips"][case["clip"]]
        d, one = case["d"], case["one_thread"]
        real = downsample.clips_u8(c["u8"].to(DEV), d, real_norm=C.VIDEO_NORM, one_thread=one)
        fake = downsample.clips_u8(c["recons"].to(DEV), d, one_thread=one)
        k = case.get("k", 0)
        fake[:, :k] = real[:, :k]
        assert torch.equal(real.cpu(), case["real"]), (c["shape"], d, one)
        assert torch.equal(fake.cpu(), case["fake"]), (c["shape"], d, one, k)


def test_lanczos_kernel_equals_fixture(fx):
    im = fx["images"]
    real = downsample.clips_u8(im["u8"].unsqueeze(1).to(DEV), 1, real_norm=C.IMAGE_NORM)[:, 0]
    fake = downsample.clips_u8(im["recons"].unsqueeze(2).to(DEV), 1)[:, 0]
    for d, (want_real, want_fake) in im["out"].items():
        assert torch.equal(downsample.images_u8(real, d).cpu(), want_real), d
        assert torch.equal(downsample.images_u8(fake, d).cpu(), want_fake), d


@pytest.mark.parametrize("d", [2, 3, 4])
def test_kernel_equals_torch_on_the_models_reconstruction(model, d):
    frames = _clips(11).to(DEV)
    x_recons, _ = model.forward_u8(frames, C.VIDEO_NORM, None)
    assert x_recons.dtype == torch.float32 and tuple(x_recons.shape) == (2, 3, 9, 128, 128)
    host = x_recons.cpu()
    old = torch.get_num_threads()
    try:
        for threads in (1, max(2, old)):
            torch.set_num_threads(threads)
            want = torch.clamp(host + 0.5, 0, 1).permute(0, 2, 1, 3, 4).flatten(0, 1)
            want = F.interpolate(want, scale_factor=1 / d, mode="bilinear", align_corners=False)
            want = (want * 255).byte().unflatten(0, (2, 9)).permute(0, 1, 3, 4, 2)
            got = downsample.clips_u8(x_recons, d, one_thread=threads == 1)
            assert torch.equal(got.cpu(), want), (d, threads)
    finally:
        torch.set_num_threads(old)


@pytest.mark.parametrize("d, k", [(2, None), (2, 2), (3, 0), (None, 2), (4, 9)])
def test_eval_step_fvd_equals_script(model, i3d, d, k):
    u8 = _clips(20)
    frames = u8.to(DEV)
    usage = torch.zeros(8192, device=DEV)
    real_l, fake_l, vq_output = C.eval_step_fvd(model, frames, i3d, usage, infer_downsample=d, replacewithgt=k,
                                                sequence_length=9)
    x_recons, vq2 = model.forward_u8(frames, C.VIDEO_NORM, None)
    real_b, fake_b = _script_video(u8, x_recons, d, k)
    if k:
        assert torch.equal(fake_b[:, :k], real_b[:, :k])
    assert torch.equal(real_l, i3d.logits(real_b.to(DEV)))
    assert torch.equal(fake_l, i3d.logits(fake_b.to(DEV)))
    assert torch.equal(vq_output["batch_usage"], vq2["batch_usage"]) and bool(usage.sum() > 0)


def test_replacewithgt_swaps_exactly_k_frames(model, i3d):
    frames = _clips(30).to(DEV)
    x_recons, _ = model.forward_u8(frames, C.VIDEO_NORM, None)
    real = downsample.clips_u8(frames, 2, real_norm=C.VIDEO_NORM)
    fake = downsample.clips_u8(x_recons, 2)
    assert all(not torch.equal(real[:, t], fake[:, t]) for t in range(9))
    for k in (0, 2, 9):
        _, fake_l, _ = C.eval_step_fvd(model, frames, i3d, infer_downsample=2, replacewithgt=k)
        assert torch.equal(fake_l, i3d.logits(torch.cat([real[:, :k], fake[:, k:]], dim=1)))


@pytest.mark.parametrize("d", [2, 3])
def test_eval_step_fid_equals_script(model, inception, d):
    from PIL import Image
    from oracle import fid_oracle as fo
    images = [fo.image_bytes(s, 60 + i) for i, s in enumerate([(150, 200), (128, 128), (97, 131)])]
    resize = L.image_resize(128)
    usage = torch.zeros(8192, device=DEV)
    real_f, fake_f, vq_output = C.eval_step_fid(model, images, resize, inception, usage, infer_downsample=d)
    host = torch.stack([L.resize_u8(im, resize) for im in images])
    x = L.u8_normalize(host.unsqueeze(1), C.IMAGE_NORM)[:, :, 0]
    antialias = getattr(Image, "ANTIALIAS", Image.LANCZOS)
    side = 128 // d
    real_saved = ((x.permute(0, 2, 3, 1) + 0.5).numpy() * 255).astype(np.uint8)          # vqgan_eval.py:204-208
    fake_bytes, vq2 = C.eval_step_u8(model, host.to(DEV), None, C.IMAGE_NORM)
    fake_saved = fake_bytes[:, 0].cpu().numpy()                                          # :214-219
    real_small = np.stack([np.asarray(Image.fromarray(a).resize((side, side), antialias)) for a in real_saved])
    fake_small = np.stack([np.asarray(Image.fromarray(a).resize((side, side), antialias)) for a in fake_saved])
    assert torch.equal(real_f, inception.features(torch.from_numpy(real_small).to(DEV)).clone())
    assert torch.equal(fake_f, inception.features(torch.from_numpy(fake_small).to(DEV)).clone())
    assert torch.equal(vq_output["batch_usage"], vq2["batch_usage"]) and bool(usage.sum() > 0)


def test_graph_replay_equals_eager(fx):
    c = fx["clips"][1]
    u8, recons = c["u8"].to(DEV), c["recons"].to(DEV)
    for one in (True, False):
        eager = (downsample.clips_u8(u8, 3, real_norm=C.VIDEO_NORM, one_thread=one),
                 downsample.clips_u8(recons, 3, one_thread=one))
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            downsample.clips_u8(u8, 3, real_norm=C.VIDEO_NORM, one_thread=one)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            outs = (downsample.clips_u8(u8, 3, real_norm=C.VIDEO_NORM, one_thread=one),
                    downsample.clips_u8(recons, 3, one_thread=one))
        for o in outs:
            o.zero_()
        graph.replay()
        torch.cuda.synchronize()
        for a, b in zip(eager, outs):
            assert torch.equal(a, b), one


@pytest.mark.parametrize("kw", [dict(infer_downsample=0), dict(infer_downsample=2.5), dict(infer_downsample=129),
                                dict(replacewithgt=10), dict(replacewithgt=-1),
                                dict(infer_downsample=2, replacewithgt=3, sequence_length=16)])
def test_fvd_refusals_launch_nothing(model, i3d, kw):
    frames = _clips(40).to(DEV)
    n0 = _cabi.launch_count
    with pytest.raises((ValueError, TypeError)):
        C.eval_step_fvd(model, frames, i3d, **kw)
    assert _cabi.launch_count == n0


@pytest.mark.parametrize("d", [0, 129, 2.0])
def test_fid_refusals_launch_nothing(model, inception, d):
    from oracle import fid_oracle as fo
    n0 = _cabi.launch_count
    with pytest.raises((ValueError, TypeError)):
        C.eval_step_fid(model, [fo.image_bytes((128, 128), 1)], L.image_resize(128), inception, infer_downsample=d)
    assert _cabi.launch_count == n0


def test_defaults_launch_what_they_launched(model, i3d):
    """Without the flags eval_step_fvd runs its earlier path: forward_u8's bytes and the real-byte map in the I3D."""
    u8 = _clips(50)
    frames = u8.to(DEV)
    real_l, fake_l, _ = C.eval_step_fvd(model, frames, i3d)
    assert torch.equal(real_l, i3d.logits(frames, real_norm=C.VIDEO_NORM))
    fake_bytes, _ = C.eval_step_u8(model, frames)
    assert torch.equal(fake_l, i3d.logits(fake_bytes))
