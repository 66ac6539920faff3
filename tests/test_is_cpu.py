"""The Inception Score's host side without a GPU: the accepted state_dict against torchvision's Inception3, the
refusals (all raised before any launch), split bookkeeping, the pool wiring and the preprocess tables."""
import numpy as np
import pytest
import torch

from omnitokenizer_b200 import fid
from omnitokenizer_b200 import iscore
from omnitokenizer_b200 import layout as L


def _torchvision_keys():
    torchvision = pytest.importorskip("torchvision")
    sd = torchvision.models.Inception3(aux_logits=True, init_weights=False).state_dict()
    return {k: tuple(v.shape) for k, v in sd.items()
            if not (k.startswith("AuxLogits.") or k.endswith(".num_batches_tracked"))}


def test_keys_equal_torchvision_inception3():
    assert iscore.expected_keys() == _torchvision_keys()


def _fake_state_dict():
    return {k: torch.zeros(s) for k, s in iscore.expected_keys().items()}


def test_state_dict_refusals_name_the_key():
    sd = _fake_state_dict()
    del sd["fc.bias"]
    with pytest.raises(KeyError, match="fc.bias"):
        iscore.ISInception(sd, "cuda:0")
    sd = _fake_state_dict()
    sd["fc.weight"] = torch.zeros(1008, 2048)
    with pytest.raises(ValueError, match="fc.weight"):
        iscore.ISInception(sd, "cuda:0")
    sd = _fake_state_dict()
    sd["Mixed_7c.extra.weight"] = torch.zeros(1)
    with pytest.raises(KeyError, match="Mixed_7c.extra.weight"):
        iscore.ISInception(sd, "cuda:0")


def test_aux_logits_and_counters_are_ignored_and_the_device_must_be_cuda():
    sd = _fake_state_dict()
    sd["AuxLogits.fc.weight"] = torch.zeros(1000, 768)
    sd["Conv2d_1a_3x3.bn.num_batches_tracked"] = torch.tensor(0)
    with pytest.raises(ValueError, match="CUDA"):
        iscore.ISInception(sd, "cpu")


def _model():
    m = object.__new__(iscore.ISInception)          # refusals come before any use of the network
    m.device = torch.device("cuda", 0)
    return m


@pytest.mark.parametrize("frames,err", [
    (torch.zeros(2, 4, 4, 80, 80), ValueError),                  # C = 4
    (torch.zeros(2, 4, 80, 80, 4, dtype=torch.uint8), ValueError),
    (torch.zeros(2, 4, 3, 80, 80, dtype=torch.float64), TypeError),
    (torch.zeros(2, 4, 3, 80, 80, dtype=torch.int32), TypeError),
    (torch.zeros(0, 4, 3, 80, 80), ValueError),                  # empty
    (torch.zeros(2, 4, 3, 0, 80), ValueError),
    (torch.zeros(2, 3, 80, 80), ValueError),                     # not (B, T, ...)
], ids=["c4_f32", "c4_u8", "f64", "i32", "empty_batch", "empty_frame", "4d"])
def test_calculate_is_refuses_bad_videos(frames, err):
    with pytest.raises(err):
        iscore.calculate_is(frames, "cuda:0", 1, model=_model())


def test_calculate_is_refusals():
    v = torch.zeros(1, 7, 3, 32, 32)
    with pytest.raises(TypeError):
        iscore.calculate_is(v, "cuda:0", 1)                     # model= is required
    for splits in (0, 8, -1, 1.5):
        with pytest.raises(ValueError):
            iscore.calculate_is(v, "cuda:0", splits, model=_model())
    with pytest.raises(ValueError, match="CUDA"):
        iscore.calculate_is(v, "cpu", 1, model=_model())
    with pytest.raises(ValueError):
        iscore.calculate_is(v, "cuda:1", 1, model=_model())


def test_inception_score_refusals():
    m = _model()
    with pytest.raises(ValueError):
        iscore.inception_score(torch.zeros(4, 3, 74, 299), resize=False, model=m)        # under 75 x 75
    with pytest.raises(ValueError):
        iscore.inception_score(torch.zeros(4, 3, 80, 80), cuda=False, model=m)
    with pytest.raises(ValueError):
        iscore.inception_score(torch.zeros(4, 3, 80, 80), batch_size=0, model=m)
    with pytest.raises(ValueError):
        iscore.inception_score([], model=m)
    with pytest.raises(TypeError):
        iscore.inception_score([np.zeros((3, 80, 80), dtype=np.uint8)], model=m)
    with pytest.raises(ValueError):
        iscore.inception_score(torch.zeros(4, 3, 80, 80), splits=5, model=m)
    iscore.check_frames(torch.zeros(1, 3, 75, 75), resize=False)                    # the least accepted size
    iscore.check_frames(torch.zeros(1, 3, 8, 8), resize=True)


def test_split_bookkeeping():
    assert iscore.split_rows(7, 3) == 2 and iscore.split_rows(5, 2) == 2 and iscore.split_rows(6, 1) == 6
    assert iscore.split_rows(7, 7) == 1
    for N, s in ((7, 0), (7, 8), (0, 1)):
        with pytest.raises(ValueError):
            iscore.split_rows(N, s)


def test_pool_wiring():
    tv = {name: pool.mode for name, _, pool, _ in iscore.BLOCKS if pool.col is None}
    assert tv and all(m == fid.POOL_AVG_PAD for m in tv.values()) and "Mixed_7c" in tv
    modes = {name: pool.mode for name, _, pool, _ in fid.BLOCKS if pool.col is None}
    assert modes.pop("Mixed_7c") == fid.POOL_MAX and set(modes.values()) == {fid.POOL_AVG}
    assert [(n, c) for n, c, _, _ in iscore.BLOCKS] == [(n, c) for n, c, _, _ in fid.BLOCKS]


@pytest.mark.parametrize("hw,out", [((299, 299), (8, 8)), ((75, 75), (1, 1)), ((96, 128), (1, 2)),
                                    ((320, 480), (8, 13))])
def test_trunk_size(hw, out):
    assert iscore.trunk_size(*hw) == out


def test_trunk_size_below_75():
    assert min(iscore.trunk_size(74, 299)) < 1 and min(iscore.trunk_size(299, 74)) < 1


def test_axis_tables():
    ident = iscore.axis_table(97, None)
    assert ident.shape == (97, 4)
    assert (ident[:, 0] == np.arange(97)).all() and (ident[:, 1] == ident[:, 0]).all()
    assert (ident[:, 2].view(np.float32) == 1).all() and (ident[:, 3].view(np.float32) == 0).all()
    up = iscore.axis_table(64, 299)
    assert np.array_equal(up, L.clip_axis_table(64, 299, float(np.float32(64) / np.float32(299))))
    assert up.shape == (299, 4) and up[:, 1].max() == 63
