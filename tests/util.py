"""Shared helpers for the parity tests (oracle = oracle/omni_oracle.py, test infrastructure)."""
import dataclasses
import os

import torch

from oracle import omni_oracle as oo
from oracle import weights as W

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLDEN_CASES = ["img64", "vid5x64", "vid9x128_b2", "img256_cfg1", "vae_vid5x64", "vae_img64", "cnn_vid5x64"]


def load_golden(name):
    return torch.load(os.path.join(GOLDEN, name + ".pt"), weights_only=False)


def golden_setup(fx):
    """Rebuild (cfg, state_dict, input) of a fixture and prove the recipe reproduced the same bits."""
    cfg = oo.Config(use_vae=bool(fx["use_vae"]), patch_embed=fx.get("patch_embed", "linear"),
                    resolution=fx.get("resolution", 256))
    sd = W.make_state_dict(cfg, fx["wseed"])
    assert W.fingerprint(sd) == fx["fingerprint"], "synthetic checkpoint differs from the one the golden run used"
    x = W.synthetic_input(fx["shape"], fx["xseed"])
    assert float(x.double().sum()) == fx["x_sum64"]
    return cfg, sd, x


def check_sub(sub, t, atol, what=""):
    """Compare tensor ``t`` with a fixture entry written by oracle/make_golden._sub."""
    t = t.detach().float().cpu().contiguous()
    if "full" in sub:
        ref = sub["full"]
        assert tuple(ref.shape) == tuple(t.shape), f"{what}: shape {tuple(t.shape)} vs {tuple(ref.shape)}"
        err = (ref - t).abs().max().item()
    else:
        assert tuple(sub["shape"]) == tuple(t.shape), f"{what}: shape {tuple(t.shape)} vs {sub['shape']}"
        err = (sub["sample"] - t.reshape(-1)[:: sub["stride"]]).abs().max().item()
        s = float(t.double().sum())
        assert abs(s - sub["sum64"]) <= atol * t.numel(), f"{what}: checksum {s} vs {sub['sum64']}"
    assert err <= atol, f"{what}: max abs err {err:.3e} > {atol:.1e}"
    return err


def namespace_from_cfg(cfg: oo.Config, **over):
    """argparse Namespace as vqgan_eval.py would build it (canonical flags + overrides)."""
    import omnitokenizer_b200 as ob
    extra = []
    if cfg.use_vae:
        extra.append("--use_vae")
    if cfg.patch_embed != "linear":
        extra += ["--patch_embed", cfg.patch_embed]
    if cfg.resolution != 256:
        extra += ["--resolution", str(cfg.resolution)]
    a = ob.canonical_args(extra)
    for k, v in over.items():
        setattr(a, k, v)
    return a


def flags_namespace(row):
    """A fresh argparse Namespace of a tests/golden/flags.pt row: its command line, minus the keys an old checkpoint's
    Namespace lacks (the model back-fills them in place, so every model gets its own)."""
    from omnitokenizer_b200.vqgan import parse_args
    a = parse_args(row["argv"])
    for k in row["drop"]:
        delattr(a, k)
    return a


def flags_setup(row):
    """(cfg, state_dict, [input, ...]) of a tests/golden/flags.pt row, proven to be the ones the reference run used."""
    cfg = oo.Config.from_args(flags_namespace(row))
    assert dataclasses.asdict(cfg) == row["cfg"], "the Namespace reads as a different model than the reference built"
    sd = W.make_state_dict(cfg, row["wseed"])
    assert W.fingerprint(sd) == row["fingerprint"], "synthetic checkpoint differs from the one the golden run used"
    xs = []
    for inp in row["inputs"]:
        x = W.synthetic_input(inp["shape"], inp["xseed"])
        assert float(x.double().sum()) == inp["x_sum64"]
        xs.append(x)
    return cfg, sd, xs


def build_model(cfg, sd, device, math=None):
    import omnitokenizer_b200 as ob
    if math is not None:
        os.environ["OMT_MATH"] = math
    m = ob.OmniTokenizer_VQGAN(namespace_from_cfg(cfg))
    res = m.load_state_dict(sd, strict=False)
    assert not res.missing_keys and not res.unexpected_keys, (res.missing_keys[:3], res.unexpected_keys[:3])
    m.codebook._need_init = False
    return m.to(device).eval()
