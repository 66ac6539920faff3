"""The operand construction of tests/attn_cases.py, checked without a GPU: the planted answers are exact, the targets sit
where the plan puts them, and the poisoned padding columns never overlap the operands."""
import pytest
import torch

from oracle import omni_oracle as oo
from tests import attn_cases as A

TOPOLOGIES = {
    "spatial-256": lambda: (A.Topology.spatial(2, 256), None),
    "spatial-4096": lambda: (A.Topology.spatial(1, 4096), None),
    "window-16x24": lambda: (A.Topology.window(2, 16, 24), A.real_window_bias(2, 5)),
    "window-24x8-random-bias": lambda: (A.Topology.window(1, 24, 8), A.random_window_bias(2, 6)),
    **{f"temporal-T{T}-{'causal' if c else 'full'}": (lambda T=T, c=c: (A.Topology.temporal(2, T, 3, c), None))
       for T in range(1, 18) for c in (0, 1)},
}


def _planted(name, H=2):
    topo, bias = TOPOLOGIES[name]()
    return A.Case(topo, H, "planted", 11, bias=bias)


@pytest.mark.parametrize("name", list(TOPOLOGIES))
def test_planted_gap(name):
    """At least 100 between the target's logit and every other one of its row: exactly on the stored fp32 operands,
    and with the scores formed in fp32."""
    case = _planted(name, H=1 if name == "spatial-4096" else 2)
    if case.topo.L == 1:
        return
    g64, g32 = case.gap(torch.float64), case.gap(torch.float32)
    assert g64 >= A.PLANT_GAP and g32 >= A.PLANT_GAP, (g64, g32)


@pytest.mark.parametrize("name", [n for n in TOPOLOGIES if n != "spatial-4096"])
def test_planted_answer_is_exact(name):
    """fp64 softmax(...) @ v returns v_t(i) to 1e-30 of its magnitude: every other weight is below e^-100."""
    case = _planted(name)
    want = case.answer().view(-1, case.H, 64)
    got = case.reference().view(-1, case.H, 64)
    rel = ((got - want.double()).abs().amax(-1) / want.double().abs().amax(-1)).max().item()
    assert rel < 1e-30, rel


def test_spatial_targets():
    for N in (64, 128, 256, 384, 4096):
        topo = A.Topology.spatial(3, N)
        t = A.target_plan(topo, 3)
        hit = set(t.unique().tolist())
        assert {k for k in (0, 63, 64, 127, 128, N - 1) if k < N} <= hit
        assert {k // 64 for k in hit} == set(range(N // 64)), "a key tile without a target"
        assert bool(((t >= 0) & (t < N)).all())


def test_window_targets_and_sets():
    topo = A.Topology.window(2, 8, 24)
    t = A.target_plan(topo, 2)
    assert set(t.unique().tolist()) >= {0, 7, 56, 63}
    # every window gets every corner as some query's target
    for w in range(topo.sets.shape[0]):
        assert set(t[w].unique().tolist()) >= {0, 7, 56, 63}
    # the sets tile each frame with 8x8 blocks: every row once, slot (sy, sx) at (8 wy + sy, 8 wx + sx)
    assert torch.equal(topo.sets.reshape(-1).sort().values, torch.arange(topo.M))
    rows = oo.window_rows(8, 24, 8)
    for win in range(rows.shape[0]):
        y, x = rows[win] // 24, rows[win] % 24
        assert int(y.max() - y.min()) == 7 and int(x.max() - x.min()) == 7
        assert torch.equal(y - y.min(), torch.arange(64) // 8) and torch.equal(x - x.min(), torch.arange(64) % 8)


@pytest.mark.parametrize("causal", [0, 1])
def test_temporal_targets(causal):
    for T in range(1, 18):
        topo = A.Topology.temporal(2, T, 3, causal)
        t = A.target_plan(topo, 2)
        i = torch.arange(T)[None, :, None]
        if causal:
            assert bool((t <= i).all()), "a target after its query under the causal mask"
            assert bool((t == i).any()) and bool((t == 0).any())
            assert bool((t[:, 0] == 0).all()), "frame 0 of a causal row can only attend to itself"
        else:
            assert bool((t == T - 1).any()) and bool((t == 0).any())
        assert t.shape == (2 * 3, T, 2)
        # row (b T + t) N + n of the set of pixel n of video b
        assert torch.equal(topo.sets[4], (1 * T + torch.arange(T)) * 3 + 1)


@pytest.mark.parametrize("family", A.FAMILIES)
def test_poisoned_padding(family):
    """Columns past 64 H are NaN and disjoint from the operand columns; the operands are finite; the leading
    dimensions differ and keep rows 16-byte aligned."""
    case = A.Case(A.Topology.window(3, 16, 8), 2, family, 3, bias=A.real_window_bias(2, 4))
    C = case.H * 64
    lds = (case.ldq, case.ldk, case.ldv)
    assert len(set(lds)) == 3 and all(ld % 4 == 0 and ld > C for ld in lds)
    for buf, view, ld in ((case.qb, case.q, case.ldq), (case.kb, case.k, case.ldk), (case.vb, case.v, case.ldv)):
        assert buf.shape == (case.topo.M, ld) and buf.is_contiguous()
        assert view.data_ptr() == buf.data_ptr() and view.stride() == (ld, 1) and view.shape[1] == C
        assert bool(torch.isnan(buf[:, C:]).all()) and bool(torch.isfinite(buf[:, :C]).all())
    assert len({case.qb.data_ptr(), case.kb.data_ptr(), case.vb.data_ptr()}) == 3


def test_families():
    """model: unit rows times a per-dimension scale in [0.5, 1.5]; ramp: key norms rising along each sequence; hot:
    scores up to about 60; v rows spread over 1e-2 .. 1e2."""
    topo = A.Topology.spatial(2, 512)
    m = A.Case(topo, 2, "model", 1)
    n = m.q.reshape(-1, 2, 64).norm(dim=-1)
    assert 0.5 <= float(n.min()) and float(n.max()) <= 1.5
    r = A.Case(topo, 2, "ramp", 1)
    kn = r.k.reshape(2, 512, 2, 64).norm(dim=-1).mean(dim=(0, 2))
    assert float(kn[:64].mean()) * 5 < float(kn[-64:].mean())
    h = A.Case(topo, 2, "hot", 1)
    s = (h.q.reshape(-1, 2, 64)[:512, 0] @ h.k.reshape(-1, 2, 64)[:512, 0].t()) * A.SCALE
    assert 40 < float(s.abs().max()) < 120
    vm = m.v.abs().amax(dim=1)
    assert float(vm.min()) < 0.05 and float(vm.max()) > 20
