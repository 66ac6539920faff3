"""The operand grids of the codebook-lookup GPU tests (tests/vq_cases.py), checked on the CPU.

For every (row, code): each intermediate of the kernel's distance (sum z^2 in sequence, __fmul_rn then seven fmaf for
2 z.E, (zz - dot) + ek) equals its fp64 value, so fp32 rounding never acts; the oracle's fp32 distances equal the fp64
ones too.  The planted winners are the first fp64 minima, the planted runners-up sit exactly 0 or 1 ulp away, and
oracle.omni_oracle.codebook returns the planted winners (its first-minimum rule)."""
import pytest
import torch

from oracle import omni_oracle as oo
from tests import vq_cases as V


def _exact(t):
    """fp64 values that fp32 holds exactly."""
    return bool(torch.equal(t.float().double(), t))


def _kernel_order_exact(z, E, e2):
    """Every intermediate of the kernel's sequence, evaluated in fp64, is an fp32 value; returns the fp64 distances."""
    zd, Ed, e2d = z.double(), E.double(), e2.double()
    zz = zd[:, 0] * zd[:, 0]
    assert _exact(zz)
    for c in range(1, 8):
        zz = zz + zd[:, c] * zd[:, c]
        assert _exact(zz), f"sum z^2 after channel {c}"
    z2 = 2.0 * zd
    dot = z2[:, None, 0] * Ed[None, :, 0]                       # __fmul_rn
    assert _exact(dot)
    for c in range(1, 8):                                       # fmaf: one rounding of the exact sum
        dot = dot + z2[:, None, c] * Ed[None, :, c]
        assert _exact(dot), f"2 z.E after channel {c}"
    diff = zz[:, None] - dot
    assert _exact(diff)
    d = diff + e2d[None, :]
    assert _exact(d)
    assert _exact(e2d) and torch.equal(e2d, (Ed * Ed).sum(1))
    assert torch.equal(d, ((zd[:, None, :] - Ed[None]) ** 2).sum(-1)), "the expansion is not the distance"
    return d


def _oracle_distances(z, E):
    """The oracle's fp32 expression (oracle/omni_oracle.codebook), whatever order torch sums in."""
    return (z ** 2).sum(dim=1, keepdim=True) - (2 * z) @ E.t() + (E.t() ** 2).sum(dim=0, keepdim=True)


@pytest.mark.parametrize("n_codes", [64, 128, 1024])
def test_tie_grid_exact(n_codes):
    z, E = V.tie_grid(700, n_codes, 11)
    d = _kernel_order_exact(z, E, V.e2_of(E))
    assert torch.equal(_oracle_distances(z, E).double(), d)
    want = torch.argmin(d, dim=1)
    assert torch.equal(V.ref_argmin(z, E), want)
    assert torch.equal(oo.codebook(E, z)["idx"], want)
    # the grid is coarse enough that the first-minimum rule decides many rows
    ties = (d == d.min(dim=1, keepdim=True).values).sum(1)
    assert int((ties > 1).sum()) > 20


@pytest.mark.parametrize("kind", V.KINDS)
@pytest.mark.parametrize("n_codes,rows_per_block", [(64, 256), (128, 512), (1024, 512), (2048, 256)])
def test_ulp_grid_planted(n_codes, rows_per_block, kind):
    E, plants = V.ulp_table(n_codes, kind, 5)
    M = 3 * rows_per_block + 17
    z, rows, want = V.ulp_rows(M, rows_per_block, plants, 6)
    d = _kernel_order_exact(z, E, V.e2_of(E))
    assert float(d.min()) >= 2.0 ** 23 and float(d.max()) < 2.0 ** 24, "distances outside [2^23, 2^24)"
    assert torch.equal(_oracle_distances(z, E).double(), d)
    first = torch.argmin(d, dim=1)
    assert torch.equal(V.ref_argmin(z, E), first)
    # every tuple is planted at every offset that exists in a block, and each planted winner is the first fp64 minimum
    lr = [x for x in V.LROWS if x < rows_per_block]
    assert rows.numel() == 3 * len(lr) + sum(x < 17 for x in lr)
    assert torch.equal(first[rows], want)
    assert set(want.tolist()) == {p[1] for p in plants}
    D = float(V.A_PLANT) ** 2
    for r, w in zip(rows.tolist(), want.tolist()):
        codes = next(p[0] for p in plants if p[1] == w)
        dr = d[r].float()
        assert float(dr[w]) == D
        for k in codes:                     # runners-up: exactly 0 ulp (tie) or 1 ulp away
            if k != w:
                up = torch.nextafter(dr[w], torch.tensor(float("inf")))
                assert (kind == "tie" and dr[k] == dr[w]) or (kind != "tie" and dr[k] == up), (r, k, w)
        others = torch.ones(n_codes, dtype=torch.bool)
        others[list(codes)] = False
        assert float(dr[others].min()) >= D + 4
    assert torch.equal(oo.codebook(E, z)["idx"], first)


def test_grid_projection_exact():
    E, plants = V.ulp_table(128, "tie", 1)
    for z in (V.ulp_rows(300, 256, plants, 2)[0], V.tie_grid(300, 64, 3)[0]):
        x, Wt, b = V.grid_projection(z, 512, 4)
        # any order: every partial sum is bounded by the sum of |terms| and lies on the grid of z (2^-3)
        bound = (x.double().abs() @ Wt.double().abs().t() + b.double().abs()).max()
        assert float(bound) < 2.0 ** 12
        assert torch.equal(x.double() @ Wt.double().t() + b.double(), z.double())
        assert torch.equal((x * 8).round(), x * 8)
