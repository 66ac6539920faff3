"""Records the reference's encode / decode on architecture flags other than the canonical ones, so that the engine is checked
on every flag it reads and sends to a kernel.

    OMT_REFERENCE_ROOT=<reference checkout> python -m oracle.make_golden_flags     (writes tests/golden/flags.pt)

One entry per row of ROWS: the command line (argv) and the Namespace keys deleted from it afterwards (drop, an old
checkpoint's Namespace that the model back-fills), the oracle Config the back-filled Namespace gives, the weight seed and
W.fingerprint, and per input (seed, shape, float64 sum) the reference's encode(..., include_embeddings=True) indices (full)
and embeddings, and decode(indices) (sampled like make_golden._sub).  Every input and weight is regenerated from the seeds
by the tests.
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

OUT = os.path.join(ROOT, "tests", "golden", "flags.pt")
REC_CAP = 25_000          # pixels kept per reconstruction (strided sample + checksums): the file stays near 1 MB
# keys an old checkpoint's Namespace lacks (the reference back-fills them, omnitokenizer.py:70-125)
OLD_NAMESPACE_DROP = ("enc_block", "dec_block", "twod_window_size", "spatial_pos", "use_vae", "kl_weight", "gen_upscale",
                      "resolution_scale")


def edit_argv(argv, remove=(), **values):
    """argv without the store_true flags in `remove` and without the valued flags set to None in `values`; other
    `values` replace (or append) '--flag value'."""
    out, i = [], 0
    argv = list(argv)
    while i < len(argv):
        a = argv[i]
        name = a[2:]
        if name in remove:
            i += 1
        elif name in values:
            i += 2
        else:
            out.append(a)
            i += 1
    for k, v in values.items():
        if v is not None:
            out += ["--" + k, str(v)]
    return out


C = rl.CANON
# name, argv, drop, weight seed, [(input shape, input seed)]
ROWS = [
    # an old checkpoint as load_from_checkpoint builds it: enc / dec tttt, rel, non-causal, no l2 -- and at 128^2 the f16
    # spatial core with the no-rope q | k | v planes epilogue
    ("backfill", edit_argv(C, remove=("causal_in_temporal_transformer", "causal_in_peg", "l2_code")), OLD_NAMESPACE_DROP,
     20, [((1, 3, 9, 128, 128), 2001), ((1, 3, 128, 128), 2002)]),
    # the stage-1 training recipe (scripts/recons/train.sh): temporal patch 2 (patch K 384, to_pixels N 384), rel
    ("stage1", edit_argv(C, temporal_patch_size=2, spatial_pos=None), (), 21, [((1, 3, 5, 128, 128), 2101)]),
    # the two causal flags on their own: an engine that hands one kernel the other's flag fails one of these rows
    ("attn_causal_only", edit_argv(C, remove=("causal_in_peg",)), (), 22, [((1, 3, 9, 64, 64), 2201)]),
    ("peg_causal_only", edit_argv(C, remove=("causal_in_temporal_transformer",)), (), 23, [((1, 3, 9, 64, 64), 2301)]),
    # window layers in the decoder (each with its own bias table), other layer orders, two temporal layers
    ("blocks", edit_argv(C, enc_block="wtwt", dec_block="twwt", temporal_depth=2), (), 24, [((1, 3, 5, 128, 128), 2401)]),
    # GEGLU widths: inner 682 (K of FF2 padded to whole k-blocks) and 1024
    ("ff2", edit_argv(C, ff_mult=2), (), 25, [((1, 3, 5, 64, 64), 2501)]),
    ("ff3", edit_argv(C, ff_mult=3), (), 26, [((1, 3, 5, 64, 64), 2601)]),
    # z not l2-normalised before the codebook search
    ("nol2", edit_argv(C, remove=("l2_code",)), (), 27, [((1, 3, 5, 128, 128), 2701)]),
]


def main():
    assert rl.available(), "the reference tree is needed (OMT_REFERENCE_ROOT)"
    torch.set_num_threads(os.cpu_count())
    ot, _ = rl.load()
    g = {}
    for name, argv, drop, wseed, inputs in ROWS:
        args = rl.make_args(argv)
        for k in drop:
            delattr(args, k)
        cfg = oo.Config.from_args(args)                   # before the reference back-fills the Namespace in place
        torch.manual_seed(0)
        m = ot.VQGAN(args).eval()
        m.codebook._need_init = False
        assert oo.Config.from_args(args) == cfg, "the oracle's back-fills differ from the reference's"
        sd = W.make_state_dict(cfg, wseed)
        res = m.load_state_dict(sd, strict=False)
        assert not res.unexpected_keys and not [k for k in res.missing_keys if not k.startswith(
            ("image_discriminator", "video_discriminator", "perceptual_model"))], res
        row = {"argv": list(argv), "drop": list(drop), "cfg": dataclasses.asdict(cfg), "wseed": wseed,
               "fingerprint": W.fingerprint(sd), "inputs": []}
        for shape, xseed in inputs:
            x = W.synthetic_input(shape, xseed)
            is_image = x.ndim == 4
            with torch.no_grad():
                emb, idx = m.encode(x, is_image, include_embeddings=True)
                rec = m.decode(idx, is_image)
            row["inputs"].append({"shape": shape, "xseed": xseed, "x_sum64": float(x.double().sum()),
                                  "idx": idx.to(torch.int16), "emb": emb.clone(), "rec": _sub(rec, cap=REC_CAP)})
            print(name, shape, "codes", tuple(idx.shape))
        g[name] = row
    g["torch"] = torch.__version__
    torch.save(g, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
