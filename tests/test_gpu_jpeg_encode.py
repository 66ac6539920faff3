"""JPEG files through the model on the device: encode_jpeg_u8 / forward_jpeg_u8 equal encode_images_u8 /
forward_images_u8 of Pillow's decoded images bit for bit (codes, embeddings, VAE latents, usage statistics, CPU RNG
state afterwards), for VQ and VAE and for batches mixing JPEG files and decoded host tensors; eval_step_fid from JPEG
sources equals eval_step_fid from the decoded images for saved_as "png" and "jpeg" and with infer_downsample=2; a
refused file raises before any launch and a corrupt one before the resize."""
import os
import tempfile

import numpy as np
import pytest
import torch

from oracle import jpeg_decode_oracle as D
from oracle import omni_oracle as oo
from oracle import weights as W
from omnitokenizer_b200 import _cabi, consumers as C, fid
from omnitokenizer_b200 import layout as L
from tests.util import build_model, load_golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")

CASES = [(375, 500, "4:2:0", 90, "smooth", {}), (31, 17, "4:4:4", 75, "noise", {"optimize": True}),
         (64, 64, "4:2:2", 50, "blocky", {"restart_marker_rows": 1}), (96, 120, "L", 95, "smooth", {}),
         (1, 3, "4:2:0", 10, "noise", {}), (300, 200, "4:2:0", 75, "checker", {"restart_marker_blocks": 2})]


def _files():
    return [D.fixture(H, W_, sub, q, kind, 900 + i, **o) for i, (H, W_, sub, q, kind, o) in enumerate(CASES)]


def _pillow(files):
    return [torch.from_numpy(D.pillow_rgb(f).copy()) for f in files]


def _usage(m):
    return m.codebook.codebook_usage.clone(), m.codebook.call_cnt


def _set_usage(m, st):
    m.codebook.codebook_usage.data = st[0].clone()
    m.codebook.call_cnt = st[1]


def _eq(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_eq(a[k], b[k]) for k in a)
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(_eq(x, y) for x, y in zip(a, b))
    if a is None or b is None:
        return a is b
    return torch.equal(a, b)


def _same_run(m, seed, want_fn, got_fn):
    st0 = _usage(m)
    torch.manual_seed(seed)
    want = want_fn()
    st_want, rng_want = _usage(m), torch.get_rng_state()
    _set_usage(m, st0)
    torch.manual_seed(seed)
    got = got_fn()
    assert _eq(got, want)
    assert _eq(_usage(m)[0], st_want[0]) and _usage(m)[1] == st_want[1]
    assert torch.equal(torch.get_rng_state(), rng_want)


@pytest.mark.parametrize("vae", [False, True])
def test_encode_and_forward_jpeg_u8_equal_images_u8(cuda, vae):
    cfg = oo.Config(resolution=64, use_vae=vae)
    m = build_model(cfg, W.make_state_dict(cfg, 4), cuda, "f16x3")
    files = _files()
    decoded = _pillow(files)
    mixed = [files[i] if i % 2 == 0 else decoded[i] for i in range(len(files))]
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for i, f in enumerate(files):
            paths.append(os.path.join(tmp, f"im{i}.jpg"))
            with open(paths[-1], "wb") as fh:
                fh.write(f)
        for rz in (L.image_resize(64), L.resizecrop_resize(64), L.dit_resize(64)):
            for sources in (files, mixed, paths):
                for emb in ((False, True) if not vae else (False,)):
                    for rep in range(2):          # the encode_u8 slot's eager run, then its graph capture
                        _same_run(m, 11 + rep, lambda: m.encode_images_u8(decoded, rz, include_embeddings=emb),
                                  lambda: m.encode_jpeg_u8(sources, rz, include_embeddings=emb))
                _same_run(m, 12, lambda: m.forward_images_u8(decoded, rz), lambda: m.forward_jpeg_u8(sources, rz))


def test_refused_and_corrupt_files(cuda):
    import io
    from PIL import Image
    cfg = oo.Config(resolution=64)
    m = build_model(cfg, W.make_state_dict(cfg, 4), cuda, "f16x3")
    files = _files()
    f = io.BytesIO()
    Image.fromarray(np.zeros((16, 16, 3), np.uint8)).save(f, "JPEG", progressive=True)
    n0 = _cabi.launch_count
    rng = torch.get_rng_state()
    with pytest.raises(NotImplementedError, match="source 2.*progressive"):
        m.encode_jpeg_u8(files[:2] + [f.getvalue()], L.image_resize(64))
    assert _cabi.launch_count == n0 and torch.equal(torch.get_rng_state(), rng)
    bad = files[0][:len(files[0]) // 2]
    with pytest.raises(ValueError, match="source 1: corrupt JPEG scan"):
        m.encode_jpeg_u8([files[1], bad], L.image_resize(64))
    # the model is still usable afterwards
    torch.manual_seed(3)
    want = m.encode_images_u8(_pillow(files), L.image_resize(64))
    torch.manual_seed(3)
    assert _eq(m.encode_jpeg_u8(files, L.image_resize(64)), want)


@pytest.fixture(scope="module")
def eval_model():
    import omnitokenizer_b200 as ob
    args = ob.canonical_args()
    m = ob.OmniTokenizer_VQGAN(args)
    m.load_state_dict(W.make_state_dict(oo.Config.from_args(args), 0), strict=False)
    m.codebook._need_init = False
    return m.to(DEV).eval()


@pytest.fixture(scope="module")
def inception():
    from oracle import fid_oracle as fo
    g = load_golden("fid_inception")
    sd = fo.make_state_dict(g["w_seed"])
    sd.update(g["bn"])
    return fid.FIDInception(sd, DEV)


@pytest.mark.parametrize("saved_as,d", [("png", None), ("jpeg", None), ("png", 2), ("jpeg", 2)])
def test_eval_step_fid_from_jpeg_sources(eval_model, inception, saved_as, d):
    files = _files()[:4]
    decoded = _pillow(files)
    resize = L.image_resize(128)
    outs = []
    for images in (decoded, files, [files[0], decoded[1], files[2], decoded[3]]):
        usage = torch.zeros(8192, device=DEV)
        torch.manual_seed(21)
        real_f, fake_f, vq = C.eval_step_fid(eval_model, images, resize, inception, usage, infer_downsample=d,
                                             saved_as=saved_as)
        outs.append((real_f.clone(), fake_f.clone(), usage.clone(), vq["batch_usage"].clone()))
    for o in outs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(o, outs[0]))
