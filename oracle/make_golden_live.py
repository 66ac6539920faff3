"""Records what the live-reference tests compare against, so that they run without the reference tree.

    OMT_REFERENCE_ROOT=<reference checkout> python -m oracle.make_golden_live     (writes tests/golden/live_reference.pt)

Stored: the reference's state-dict layout (key -> shape, dtype) and parser defaults (test_boundary), its encode / decode
outputs on the synthetic inputs of test_oracle_matches_live_reference, Net2NetTransformer.encode_to_z outputs and the
uint8 conversion of test_consumer_restatements_match_live_reference (on the weights of oracle/weights.py, seed 3), and per-tensor
sha256 digests of the inflate_gen results of test_inflate_gen_matches_live_reference.  Every input is regenerated from the same seeds by the tests.
"""
import argparse
import hashlib
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import omni_oracle as oo  # noqa: E402
from oracle import ref_loader as rl  # noqa: E402
from oracle import weights as W  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "live_reference.pt")
ORACLE_SHAPES = [(1, 3, 64, 64), (1, 3, 5, 64, 64)]
U8_SHAPE, U8_SEED = (2, 3, 5, 8, 8), 11


def u8_input():
    return torch.rand(U8_SHAPE, generator=torch.Generator().manual_seed(U8_SEED)) - 0.5


def tensor_digests(sd):
    """key -> (shape, dtype, sha256 of the raw bytes): a bit-for-bit fingerprint of a state dict"""
    return {k: (tuple(v.shape), str(v.dtype), hashlib.sha256(v.detach().contiguous().view(torch.uint8).numpy().tobytes()).hexdigest())
            for k, v in sd.items()}


def main():
    assert rl.available(), "the reference tree is needed (OMT_REFERENCE_ROOT)"
    g = {}
    # ---- state dict layout and parser defaults
    ref, args = rl.make_model(perturb=False)
    g["state_dict_layout"] = {k: (tuple(v.shape), str(v.dtype)) for k, v in ref.state_dict().items()
                              if not k.startswith(("image_discriminator", "video_discriminator", "perceptual_model"))}
    ot, base = rl.load()
    rp = ot.VQGAN.add_model_specific_args(base.VQGAN.add_model_specific_args(argparse.ArgumentParser()))
    g["parser_defaults"] = vars(rp.parse_args([]))
    g["latent_shape"] = tuple(ref.latent_shape)
    g["model_args"] = vars(args)
    # ---- encode / decode on synthetic inputs
    cfg = oo.Config.from_args(args)
    sd = W.make_state_dict(cfg, 3)
    ref.load_state_dict(sd, strict=False)
    for shape in ORACLE_SHAPES:
        x = W.synthetic_input(shape, 99)
        is_image = x.ndim == 4
        with torch.no_grad():
            emb, idx = ref.encode(x, is_image, include_embeddings=True)
            rec = ref.decode(idx, is_image)
        g["encode_decode", shape] = {"emb": emb.clone(), "idx": idx.clone(), "rec": rec.clone()}
    # ---- consumers: Net2NetTransformer.encode_to_z, shift_dim + uint8
    ref, _ = rl.make_model(seed=3)
    ref.load_state_dict(W.make_state_dict(oo.Config(), 3), strict=False)
    import OmniTokenizer.lm_transformer as lt
    from OmniTokenizer.utils import shift_dim
    x = W.synthetic_input((1, 3, 9, 64, 64), 55)
    for n in (0, 2):
        stub = types.SimpleNamespace(vtokens=False, first_stage_model=ref, sample_every_n_latent_frames=n)
        with torch.no_grad():
            emb, tgt = lt.Net2NetTransformer.encode_to_z(stub, x, False)
        g["encode_to_z", n] = {"emb": emb.clone(), "tgt": tgt.clone()}
    v = u8_input()
    g["u8"] = shift_dim(torch.clamp(v + 0.5, 0, 1) * 255, 1, -1).byte()
    # ---- checkpoint inflation
    from OmniTokenizer.utils import inflate_gen
    sd = W.make_state_dict(oo.Config(), 4)
    for strategy in ("average", "first"):
        g["inflate_gen", strategy] = tensor_digests(inflate_gen(sd, 4, 8, strategy=strategy))
    torch.save(g, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e6:.1f} MB)")


if __name__ == "__main__":
    main()
