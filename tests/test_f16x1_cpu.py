"""CPU checks of the f16x1 numerics model (tests/f16x1_model.py) that DESIGN.md section 4 quotes, and of the near-tie
test the GPU golden checks apply to flipped codes."""
import pytest
import torch

from oracle import omni_oracle as oo
from tests.f16x1_model import mm_f16x1, provable_near_tie
from tests.util import check_sub, golden_setup, load_golden

VQ_CASES = ["img64", "vid5x64", "vid9x128_b2", "img256_cfg1", "cnn_vid5x64"]


def test_model_rounds_one_product():
    """Single fp16 product on power-of-two-scaled operands: exact on fp16-representable grids, 2^-11-relative otherwise."""
    g = torch.Generator().manual_seed(1)
    a = torch.randint(-2048, 2048, (16, 64), generator=g).float() * 2.0 ** -30
    b = torch.randint(-2048, 2048, (64, 8), generator=g).float() * 2.0 ** 7
    assert torch.equal(mm_f16x1(a, b), a @ b)          # 11-bit integers times powers of two: every step exact
    a, b = torch.randn(32, 256, generator=g), torch.randn(256, 48, generator=g)
    ref = a.double() @ b.double()
    mag = a.double().abs() @ b.double().abs()
    err = (mm_f16x1(a, b).double() - ref).abs()
    assert (err <= 2.0 ** -10 * mag + 1e-6).all()
    assert err.max() > 2.0 ** -14 * mag.max()          # and it is not fp32-grade
    # batched right operand: one scale per matrix
    bb = torch.randn(3, 256, 48, generator=g)
    assert torch.equal(mm_f16x1(a, bb)[1], mm_f16x1(a, bb[1]))


@pytest.mark.parametrize("name", VQ_CASES)
def test_model_on_goldens(name, monkeypatch):
    """At most one flipped code per golden case and a decode-only pixel error <= 2e-3 (DESIGN.md section 4)."""
    fx = load_golden(name)
    cfg, sd, x = golden_setup(fx)
    monkeypatch.setattr(oo, "MATMUL_MODEL", mm_f16x1)
    with torch.no_grad():
        idx = oo.encode(sd, cfg, x)
        rec = oo.decode(sd, cfg, fx["idx"].long(), x.ndim == 4)
    flips = int((idx != fx["idx"].long()).sum())
    err = check_sub(fx["rec"], rec, 1.0, "rec")
    print(f"{name}: f16x1 model flips {flips}/{idx.numel()}, decode-only max |dpx| {err:.2e}")
    assert flips <= 1
    assert err <= 2e-3


def _unit(v):
    return v / v.norm(dim=-1, keepdim=True)


def test_near_tie_constructed():
    """z exactly between two codes flips under any perturbation; a clear winner survives a small one, and a flip there is
    rejected; the bound scales with |z' - z| and with |E_a - E_b|."""
    g = torch.Generator().manual_seed(3)
    E = _unit(torch.randn(16, 8, generator=g))
    a, b = torch.tensor([2]), torch.tensor([9])
    mid = _unit((E[2] + E[9]) / 2)[None]             # equidistant from codes 2 and 9: gap 0
    eps = 1e-4 * _unit(torch.randn(1, 8, generator=g))
    assert provable_near_tie(mid, mid + eps, E, a, b, slack=0.0).all()
    # z = E_a: gap = |E_a - E_b|^2, far beyond 2 |dz| |E_a - E_b| for a small move
    za = E[2][None]
    assert not provable_near_tie(za, za + eps, E, a, b).any()
    # exactly at the bound: z' - z parallel to E_a - E_b with 2 |dz| |E_a - E_b| = gap
    d = (E[2] - E[9])
    gap = float(((za - E[9]) ** 2).sum() - ((za - E[2]) ** 2).sum())
    step = gap / (2 * float(d.norm()))
    move = -(d / d.norm())[None]
    assert provable_near_tie(za, za + move * step * 1.001, E, a, b, slack=0.0).all()
    assert not provable_near_tie(za, za + move * step * 0.99, E, a, b, slack=0.0).any()
    # several rows at once
    zs = torch.cat([mid, za])
    got = provable_near_tie(zs, zs + eps, E, torch.tensor([2, 2]), torch.tensor([9, 9]))
    assert got.tolist() == [True, False]
