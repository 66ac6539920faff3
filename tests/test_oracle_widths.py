"""CPU tests: the oracle at model widths other than 512 and attention widths apart from the model's, against the reference's
outputs recorded by oracle/make_golden_widths.py (tests/golden/widths.pt); the module's parameter containers against the
reference's state_dict keys and shapes; and, per row, that an engine which confuses the two widths would land far from the
fixture."""
import dataclasses
import os

import pytest
import torch
import torch.nn.functional as F

import omnitokenizer_b200 as ob
from oracle import omni_oracle as oo
from tests.util import GOLDEN, check_sub, flags_namespace, flags_setup

ROWS = ["w256_h8", "w256_h4", "w512_h4", "w768_h12", "w1024_h16", "w768_vae", "w256_h8_win"]
PIX_TOL = 2e-6
VAE_PIX_TOL = 5e-6      # pixels of an unnormalised latent: 2.5 x PIX_TOL, as test_oracle.py allows its VAE goldens


def widths_golden():
    return torch.load(os.path.join(GOLDEN, "widths.pt"), weights_only=False)


def _a_as_c(sd, cfg):
    """The attention width taken as the model width: C / 64 heads, the q | k | v columns of the stacked [to_q; to_kv]
    projection split at C and 2C, and to_out read as C x C (rows past the stack and columns past A are zero padding)."""
    C, A = cfg.embedding_dim, cfg.heads * cfg.dim_head
    sd = dict(sd)
    for pre in {k[: -len(".to_q.weight")] for k in sd if k.endswith(".to_q.weight")}:
        qkv = torch.cat([sd[pre + ".to_q.weight"], sd[pre + ".to_kv.weight"]])
        qkv = torch.cat([qkv, qkv.new_zeros(max(0, 3 * C - 3 * A), C)])
        sd[pre + ".to_q.weight"], sd[pre + ".to_kv.weight"] = qkv[:C], qkv[C: 3 * C]
        wo = sd[pre + ".to_out.weight"]
        sd[pre + ".to_out.weight"] = F.pad(wo, (0, C - A)) if A < C else wo[:, :C]
    return sd, dataclasses.replace(cfg, heads=C // cfg.dim_head)


def _to_out_k_as_c(sd, cfg):
    """to_out given K = C: the [C, A] weight read as a dense [C, C] matrix and the attention output read C columns wide
    (zero past A).  Returns a MATMUL_MODEL that applies it to the to_out products only."""
    C = cfg.embedding_dim
    ptrs = {v.data_ptr() for k, v in sd.items() if k.endswith(".to_out.weight")}

    def mm(a, b):
        if b.data_ptr() not in ptrs:
            return a @ b
        w = b.t().reshape(-1)
        w = torch.cat([w, w.new_zeros(max(0, C * C - w.numel()))])[: C * C].view(C, C)
        A = a.shape[-1]
        return (F.pad(a, (0, C - A)) if A < C else a[..., :C]) @ w.t()
    return mm


def _window_head_dim_from_dim_head(orig):
    """Window attention with heads of --dim_head channels (C / dim_head heads, the first columns of the bias table)
    instead of the reference's C / heads."""
    def f(sd, pre, cfg, X, hw):
        H = X.shape[-1] // cfg.dim_head
        sd = dict(sd)
        sd[pre + ".relative_position_bias_table"] = sd[pre + ".relative_position_bias_table"][:, :H]
        return orig(sd, pre, dataclasses.replace(cfg, heads=H), X, hw)
    return f


# row -> the broken wirings the fixture must tell apart from it (rows where the two widths differ)
SENSITIVITY = {"w256_h8": ("a_as_c", "to_out_k_as_c"), "w512_h4": ("a_as_c", "to_out_k_as_c"),
               "w256_h8_win": ("to_out_k_as_c", "window_head_dim")}


def _run(sd, cfg, x, r):
    is_image = x.ndim == 4
    with torch.no_grad():
        if cfg.use_vae:
            z = oo.encode(sd, cfg, x, noise=r["noise"])
            zr = r["z"]["full"]          # decode the reference's latent, as the VQ rows decode its codes
            return None, None, z, oo.decode(sd, cfg, zr if is_image else zr.permute(0, 2, 3, 4, 1), is_image)
        emb, idx = oo.encode(sd, cfg, x, include_embeddings=True)
        return idx, emb, None, oo.decode(sd, cfg, r["idx"].long(), is_image)


def test_fixture_covers_every_row():
    g = widths_golden()
    assert sorted(k for k in g if k != "torch") == sorted(ROWS)


def test_rows_differ_from_canonical_as_described():
    g = widths_golden()
    canon = dataclasses.asdict(oo.Config())
    tttt = dict(enc_block="tttt")            # the canonical decoder is tttt already
    want = {"w256_h8": dict(embedding_dim=256, **tttt), "w256_h4": dict(embedding_dim=256, heads=4),
            "w512_h4": dict(heads=4, **tttt), "w768_h12": dict(embedding_dim=768, heads=12),
            "w1024_h16": dict(embedding_dim=1024, heads=16), "w768_vae": dict(embedding_dim=768, heads=12, use_vae=True),
            "w256_h8_win": dict(embedding_dim=256)}
    for name in ROWS:
        cfg, _, _ = flags_setup(g[name])
        diff = {k: v for k, v in dataclasses.asdict(cfg).items() if v != canon[k]}
        assert diff == want[name], (name, diff)


@pytest.mark.parametrize("name", ROWS)
def test_oracle_matches_widths_golden(name):
    row = widths_golden()[name]
    cfg, sd, xs = flags_setup(row)
    for x, r in zip(xs, row["inputs"]):
        idx, emb, z, rec = _run(sd, cfg, x, r)
        if cfg.use_vae:
            check_sub(r["z"], z, PIX_TOL, f"{name} latent")
        else:
            mism = int((idx != r["idx"].long()).sum())
            assert mism == 0, f"{name} {tuple(x.shape)}: {mism}/{idx.numel()} code indices differ from the reference"
            check_sub(r["emb"], emb, 1e-6, f"{name} embeddings")
        err = check_sub(r["rec"], rec, VAE_PIX_TOL if cfg.use_vae else PIX_TOL, f"{name} {tuple(x.shape)} reconstruction")
        print(f"{name} {tuple(x.shape)}: max |dpixel| {err:.2e}")


@pytest.mark.parametrize("name", ROWS)
def test_module_state_dict_matches_reference(name):
    """The module's parameter containers give the reference's state_dict keys and shapes (checkpoints load strictly)."""
    row = widths_golden()[name]
    m = ob.OmniTokenizer_VQGAN(flags_namespace(row))
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    want = dict(row["state_shapes"])
    assert sorted(set(got) ^ set(want)) == []
    assert {k: v for k, v in got.items() if want[k] != v} == {}


@pytest.mark.parametrize("name", sorted(SENSITIVITY))
def test_widths_golden_is_sensitive_to_width_wiring(name, monkeypatch):
    row = widths_golden()[name]
    cfg, sd, xs = flags_setup(row)
    x, r = xs[0], row["inputs"][0]
    for label in SENSITIVITY[name]:
        with monkeypatch.context() as mp:
            sd2, cfg2 = sd, cfg
            if label == "a_as_c":
                sd2, cfg2 = _a_as_c(sd, cfg)
            elif label == "to_out_k_as_c":
                mp.setattr(oo, "MATMUL_MODEL", _to_out_k_as_c(sd, cfg))
            else:
                mp.setattr(oo, "window_attention", _window_head_dim_from_dim_head(oo.window_attention))
            idx, _, _, rec = _run(sd2, cfg2, x, r)
        mism = int((idx != r["idx"].long()).sum())
        err = check_sub(r["rec"], rec, float("inf"), label)
        print(f"{name} / {label}: {mism}/{idx.numel()} codes differ, max |dpixel| {err:.2e}")
        # the window row decodes through tttt: its window wiring shows in the codes alone
        assert mism > 0 or err > 1e-2, f"{name}: the fixture does not tell the row from '{label}'"
