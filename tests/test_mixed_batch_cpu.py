"""CPU tests of the packed-batch host logic: BatchLayout (sorting, groups, offsets, per-sample rows and slots) and the
C ABI of the layout-table entry points."""
import os
import re

from omnitokenizer_b200 import _cabi
from omnitokenizer_b200.engine import BatchLayout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_layout_sorts_stably_and_groups_equal_lengths():
    tps = [5, 1, 3, 5, 1, 17, 3, 5]
    lay = BatchLayout(tps, 8, 8)
    assert lay.order == [1, 4, 2, 6, 0, 3, 7, 5]            # stable: equal lengths keep the caller's order
    assert [(g.tp, g.s0, g.n, g.f0) for g in lay.groups] == [(1, 0, 2, 0), (3, 2, 2, 2), (5, 4, 3, 8), (17, 7, 1, 23)]
    assert lay.t_off == [0, 1, 2, 5, 8, 13, 18, 23, 40]
    assert lay.frames == 40 and lay.M == 40 * 64 and not lay.uniform
    # every sample owns its own rows, they tile [0, M) and the slot points at the same place
    seen = []
    for i, tp in enumerate(tps):
        r = lay.rows(i)
        assert r.stop - r.start == tp * 64
        gi, k = lay.slot[i]
        g = lay.groups[gi]
        assert g.tp == tp and lay.order[g.s0 + k] == i
        assert r.start == (g.f0 + k * g.tp) * 64
        seen.append((r.start, r.stop))
    seen.sort()
    assert seen[0][0] == 0 and seen[-1][1] == lay.M and all(a[1] == b[0] for a, b in zip(seen, seen[1:]))


def test_uniform_layout_is_the_one_group_case():
    lay = BatchLayout([5, 5, 5], 16, 16)
    assert lay.uniform and lay.order == [0, 1, 2] and len(lay.groups) == 1
    assert lay.groups[0] == (5, 0, 3, 0) and [lay.rows(i).start for i in range(3)] == [0, 5 * 256, 10 * 256]


def test_layouts_with_equal_rows_have_different_keys():
    a, b, c = BatchLayout([2, 1, 3], 8, 8), BatchLayout([3, 3], 8, 8), BatchLayout([3, 1, 2], 8, 8)
    assert a.M == b.M == c.M
    assert a.key != b.key
    assert a.key == c.key and a.order != c.order        # same packing, other caller order: same kernels, other slots


def test_varlen_entry_points_are_declared_and_bound():
    hdr = open(os.path.join(ROOT, "include", "omnitok_b200.h")).read()
    for name in ("omt_peg_volume_varlen", "omt_attn_temporal_varlen"):
        assert re.search(r"\bint %s\(" % name, hdr), name
        assert name in _cabi.SIGNATURES
    assert len(_cabi.SIGNATURES["omt_peg_volume_varlen"][1]) == 14
    assert len(_cabi.SIGNATURES["omt_attn_temporal_varlen"][1]) == 19
