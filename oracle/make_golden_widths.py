"""Records the reference's encode / decode at model widths other than 512 and at attention widths apart from the model's, so
that the engine is checked wherever it keeps the model width C (--embedding_dim) and the attention width A
(--heads x --dim_head) apart.

    OMT_REFERENCE_ROOT=<reference checkout> python -m oracle.make_golden_widths     (writes tests/golden/widths.pt)

Rows in the layout of make_golden_flags (argv, drop, cfg, weight seed, W.fingerprint, inputs), plus the reference's own
state_dict key -> shape list (its discriminators and perceptual model left out).  VQ inputs store the reference's
encode(..., include_embeddings=True) indices and embeddings and decode(indices); the VAE row stores the noise draw, the
latent and decode(latent), as make_golden does.  Every input and weight is regenerated from the seeds by the tests.
"""
import dataclasses
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import omni_oracle as oo  # noqa: E402
from oracle import ref_loader as rl  # noqa: E402
from oracle import weights as W  # noqa: E402
from oracle.make_golden import _sub  # noqa: E402
from oracle.make_golden_flags import edit_argv  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "widths.pt")
REC_CAP = 16_000          # pixels kept per reconstruction (strided sample + checksums): the file stays near 1 MB
NOT_MODEL = ("image_discriminator", "video_discriminator", "perceptual_model")

C = rl.CANON
TTTT = dict(enc_block="tttt", dec_block="tttt")
# name, argv, weight seed, [(input shape, input seed)]
ROWS = [
    # A = 512 > C = 256: to_q / to_kv widen the stream, to_out narrows it back
    ("w256_h8", edit_argv(C, embedding_dim=256, heads=8, **TTTT), 30, [((1, 3, 9, 64, 64), 3001), ((1, 3, 64, 64), 3002)]),
    # C = A = 256: window heads of 64 at C = 256; at 128^2 the f16 spatial core and 256-wide GEMMs
    ("w256_h4", edit_argv(C, embedding_dim=256, heads=4), 31, [((1, 3, 5, 128, 128), 3101)]),
    # A = 256 < C = 512
    ("w512_h4", edit_argv(C, heads=4, **TTTT), 32, [((1, 3, 5, 64, 64), 3201)]),
    # C = A = 768: LayerNorm of 6 chunks per lane; the QKV input switch at column 768 (not a multiple of 256)
    ("w768_h12", edit_argv(C, embedding_dim=768, heads=12), 33, [((1, 3, 5, 128, 128), 3301), ((1, 3, 128, 128), 3302)]),
    # C = A = 1024: LayerNorm of 8 chunks per lane, post_vq past 512 channels
    ("w1024_h16", edit_argv(C, embedding_dim=1024, heads=16), 34, [((1, 3, 5, 64, 64), 3401)]),
    # VAE moments at C = 768
    ("w768_vae", edit_argv(C, embedding_dim=768, heads=12) + ["--use_vae"], 35, [((1, 3, 5, 64, 64), 3501)]),
    # window blocks with heads of C / heads = 32: the engine refuses it; the oracle is pinned to the reference here
    ("w256_h8_win", edit_argv(C, embedding_dim=256, heads=8), 36, [((1, 3, 5, 64, 64), 3601)]),
]


def main():
    assert rl.available(), "the reference tree is needed (OMT_REFERENCE_ROOT)"
    torch.set_num_threads(os.cpu_count())
    ot, _ = rl.load()
    g = {}
    for name, argv, wseed, inputs in ROWS:
        args = rl.make_args(argv)
        cfg = oo.Config.from_args(args)
        torch.manual_seed(0)
        m = ot.VQGAN(args).eval()
        m.codebook._need_init = False
        sd = W.make_state_dict(cfg, wseed)
        res = m.load_state_dict(sd, strict=False)
        assert not res.unexpected_keys and not [k for k in res.missing_keys if not k.startswith(NOT_MODEL)], res
        shapes = [(k, tuple(v.shape)) for k, v in m.state_dict().items() if not k.startswith(NOT_MODEL)]
        row = {"argv": list(argv), "drop": [], "cfg": dataclasses.asdict(cfg), "wseed": wseed,
               "fingerprint": W.fingerprint(sd), "state_shapes": shapes, "inputs": []}
        for shape, xseed in inputs:
            x = W.synthetic_input(shape, xseed)
            is_image = x.ndim == 4
            r = {"shape": shape, "xseed": xseed, "x_sum64": float(x.double().sum())}
            with torch.no_grad():
                if cfg.use_vae:
                    h = m.pre_vq_conv(m.encoder(x, is_image))
                    noise = torch.rand(h.shape[0], h.shape[1] // 2, *h.shape[2:],
                                       generator=torch.Generator().manual_seed(xseed + 1)) * 2 - 1
                    _orig = torch.randn
                    try:        # the reference's sampler (vae.py:15-17) with the recorded draw in place of the global RNG
                        torch.randn = lambda *a, **k: noise.clone()
                        z = m.encode(x, is_image)
                    finally:
                        torch.randn = _orig
                    rec = m.decode(z if is_image else z.permute(0, 2, 3, 4, 1), is_image)
                    r.update(noise=noise, z=_sub(z, cap=REC_CAP), rec=_sub(rec, cap=REC_CAP))
                else:
                    emb, idx = m.encode(x, is_image, include_embeddings=True)
                    rec = m.decode(idx, is_image)
                    r.update(idx=idx.to(torch.int16), emb=_sub(emb, cap=REC_CAP), rec=_sub(rec, cap=REC_CAP))
            row["inputs"].append(r)
            print(name, shape, "state_dict entries", len(shapes))
        g[name] = row
    g["torch"] = torch.__version__
    torch.save(g, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
