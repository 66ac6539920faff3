"""The f16 spatial attention cores' cases, host model and error bound (tests/attn_f16_cases.py), on the CPU: the planted
cases cover every key position, the unmutated model stays inside its bound on every case, and every mutant of the model
fails the GPU test's check on every planted case."""
import pytest
import torch

from omnitokenizer_b200 import layout as L
from tests import attn_f16_cases as A


@pytest.fixture(scope="module")
def planted():
    return A.planted_cases()


def test_planted_targets_cover_every_key(planted):
    """Every key position of every (sequence, head) is some row's target: every ring stage, every jj, qd, both h, both
    P'' tiles of a pair; the target beats every other key by more than 128 in ex2's argument."""
    for c, target, partner in planted:
        for s in range(c.nseq):
            for h in range(c.H):
                r0 = s * c.N
                t = target[r0:r0 + c.N, h]
                assert torch.equal(t.sort().values, torch.arange(c.N)), c.name
                lg = (c.q[r0:r0 + c.N, h] @ c.k[r0:r0 + c.N, h].t()) * A.SCALE * 1.4426950408889634
                one = partner[r0:r0 + c.N, h] < 0
                best = lg[torch.arange(c.N), t]
                rest = lg.clone()
                rest[torch.arange(c.N), t] = -1e30
                assert bool((best[one] - rest[one].max(1).values >= 128).all()), c.name
                pr = ~one
                assert bool(pr.any()) and bool((best[pr] > lg[torch.arange(c.N), partner[r0:r0 + c.N, h].clamp_min(0)][pr]).all())


@pytest.mark.parametrize("mode", A.MODES)
def test_model_within_bound_planted(planted, mode):
    for c, target, _ in planted:
        ok, r, e, b, bad = A.evaluate(c, mode, target=target)
        print(f"{c.name} [{mode}]: model err/bound {r:.3f}, err/mag {e:.2e}, bound/mag {b:.2e}")
        assert ok, f"{c.name} [{mode}]: {bad} rows outside the bound"
        exact = sum(int(A.exact_rows(c, s, h, mode, target).sum()) for s in range(c.nseq) for h in range(c.H))
        assert exact >= c.M * c.H // 3, f"{c.name}: only {exact} exact rows"


@pytest.mark.parametrize("mode", A.MODES)
def test_mutants_fail_every_planted_case(planted, mode):
    for c, target, _ in planted:
        for m in A.mutants(mode):
            ok, r, _, _, bad = A.evaluate(c, mode, mutant=m, target=target)
            print(f"{c.name} [{mode}] mutant {m}: {bad} rows fail, worst err/bound {r:.3g}")
            assert not ok, f"{c.name} [{mode}]: mutant {m} passes the check"


@pytest.mark.parametrize("mode", A.MODES)
@pytest.mark.parametrize("family", ["spread", "logit"])
def test_model_within_bound(family, mode):
    cases = A.spread_cases() if family == "spread" else A.logit_cases()
    for c in cases:
        ok, r, e, b, bad = A.evaluate(c, mode)
        lg, sp = A.max_logit(c)
        print(f"{c.name} [{mode}]: max logit {lg:.1f}, vinv spread 2^{sp:.1f}: model err/bound {r:.3f}, "
              f"err/mag {e:.2e}, bound/mag {b:.2e}")
        assert ok, f"{c.name} [{mode}]: {bad} rows outside the bound"


def test_sweep_ranges():
    """The spread sweep reaches a vinv spread of 2^30; each logit case takes the engine's plane scales, pow2_scale of
    its q / k scale maxima, and reaches its bound 8 qmax kmax (up to 2048); the ramp case puts every row's maximum in
    its last key tile."""
    sp = max(A.max_logit(c)[1] for c in A.spread_cases())
    assert sp >= 30
    cases = A.logit_cases()
    for c, (qm, km) in zip(cases, A.LOGIT_SCALES):
        assert (c.qs, c.ks) == (L.pow2_scale(qm), L.pow2_scale(km)), c.name
        assert A.max_logit(c)[0] == 8 * qm * km, c.name
        # the hi planes hold fp16(qmax qs) / fp16(kmax ks) as their largest element
        for x, ps, hi in ((qm, c.qs, c.qh), (km, c.ks, c.kh)):
            assert 2.0 ** 14 <= x * ps < 2.0 ** 15
            assert float(hi.float().abs().max()) == float(torch.tensor(x * ps).half()), c.name
    ends = [x * ps for c, (qm, km) in zip(cases, A.LOGIT_SCALES) for x, ps in ((qm, c.qs), (km, c.ks))]
    assert 2.0 ** 14 in ends and any(2.0 ** 15 - e <= 16 for e in ends)     # both ends of the binade
    assert max(A.max_logit(c)[0] for c in cases) == 2048
    c = cases[-1]
    lg = c.q[:, 0] @ c.k[:, 0].t()
    assert bool((lg.argmax(1) >= c.N - A.KT).all())
