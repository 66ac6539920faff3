"""CPU tests of the workspace's static-buffer policy (Workspace.static / graphs_of): one buffer set per slot, replacing a
slot's set drops exactly the graphs captured over that slot, and layout tables live only as long as a set holds their
layout.  No kernel runs: the graphs and layout tables are sentinels."""
import pytest
import torch

from omnitokenizer_b200.engine import BatchLayout, Workspace

SLOTS = ("encode", "encode_batch", "encode_u8", "decode", "decode_u8", "decode_batch", "decode_batch_u8")


def _ws():
    return Workspace("cpu", 64, C=16, A=16, ku=32, kmax=48, cd=16, planes=False)


def _make(groups=1):
    return lambda: [torch.zeros(4) for _ in range(groups)]


def _refuse():
    raise AssertionError("a set of the held layout was rebuilt")


def test_same_layout_returns_the_same_tensors():
    ws = _ws()
    key = BatchLayout((2, 1, 3), 8, 8).key
    bufs = ws.static("encode_batch", key, _make(2))
    ws.graphs[("encode_batch", key, "vq", None)] = sentinel = object()
    again = ws.static("encode_batch", key, _refuse)
    assert again is bufs and all(a is b for a, b in zip(again, bufs))
    assert ws.graphs_of("encode_batch") == {("encode_batch", key, "vq", None): sentinel}
    # the same layout key in another slot is another set
    other = ws.static("encode", key, _make(1))
    assert other is not bufs and ws.static("encode_batch", key, _refuse) is bufs


@pytest.mark.parametrize("slot", SLOTS)
def test_replacing_a_set_drops_exactly_that_slots_graphs(slot):
    ws = _ws()
    k_old, k_new = BatchLayout((1, 2), 8, 8).key, BatchLayout((3,), 8, 8).key
    sets = {s: ws.static(s, k_old, _make()) for s in SLOTS}
    seeded = {s: {(s, k_old, mode, extra): object()
                  for mode, extra in (("vq", None), ("raw", None), ("idx", (1.0, 0.0, 0.0, 255.0, 1.0)))} for s in SLOTS}
    for g in seeded.values():
        ws.graphs.update(g)
    new = ws.static(slot, k_new, _make(2))
    assert new is not sets[slot] and ws.static(slot, k_new, _refuse) is new
    assert ws.graphs_of(slot) == {}
    kept = {}
    for s in SLOTS:
        if s != slot:
            assert ws.static(s, k_old, _refuse) is sets[s]
            assert ws.graphs_of(s) == seeded[s]
            assert all(ws.graphs[k] is v for k, v in seeded[s].items())
            kept.update(seeded[s])
    assert ws.graphs == kept


def test_layout_tables_keep_only_held_layouts():
    ws = _ws()
    a, b, c, d = (BatchLayout(t, 8, 8).key for t in ((1, 2), (2, 3), (1, 1, 4), (5,)))
    ws.static("encode_batch", a, _make())
    ws.static("decode_batch", a, _make())
    ws.static("decode_batch_u8", b, _make())
    ws.layout_tables.update({a: "table a", b: "table b", d: "table d"})
    # encode_batch leaves a: decode_batch still holds it
    ws.static("encode_batch", c, _make())
    assert set(ws.layout_tables) == {a, b}
    ws.layout_tables[c] = "table c"
    ws.static("decode_batch", c, _make())
    assert set(ws.layout_tables) == {b, c}
    ws.static("decode_batch_u8", c, _make())
    assert set(ws.layout_tables) == {c} and ws.layout_tables[c] == "table c"
