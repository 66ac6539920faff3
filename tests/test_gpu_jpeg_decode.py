"""omt_jpeg_decode_u8 on the device (jpeg.decode_u8): Image.open(f).convert("RGB") byte for byte against Pillow run
live and tests/golden/jpeg_decode.pt over oracle/jpeg_decode_oracle.py's matrix of sizes, subsamplings, qualities,
custom tables, optimised tables, restart intervals, metadata segments and content kinds; mixed batches of 8, 64 and
256 files; no write outside the output, sources untouched, identical bytes on a second launch; refusals before any
launch; corrupt scans raising ValueError with the file's name."""
import numpy as np
import pytest
import torch

from oracle import jpeg_decode_oracle as D
from omnitokenizer_b200 import _cabi, jpeg
from tests.util import load_golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _check(files):
    got = jpeg.decode_u8(files, DEV)
    torch.cuda.synchronize()
    bad = [i for i, (g, f) in enumerate(zip(got, files)) if not np.array_equal(g.cpu().numpy(), D.pillow_rgb(f))]
    return bad


def test_golden_files():
    import hashlib
    g = load_golden("jpeg_decode")
    got = jpeg.decode_u8(g["files"], DEV)
    bad = [c for c, t, s in zip(g["cases"], got, g["sha256"]) if hashlib.sha256(t.cpu().numpy().tobytes()).hexdigest() != s]
    assert not bad, bad


@pytest.mark.parametrize("size", D.SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_matrix_one_file_at_a_time(size):
    cases = [c for c in D.matrix() if (c[0], c[1]) == size]
    bad = []
    for H, W, sub, q, kind, seed, opts in cases:
        f = D.fixture(H, W, sub, q, kind, seed, **opts)
        if _check([f]):
            bad.append((H, W, sub, q, kind, sorted(opts)))
    assert not bad, bad


@pytest.mark.parametrize("B", [8, 64, 256])
def test_mixed_batches(B):
    rng = np.random.default_rng(B)
    cases = D.matrix([(int(h), int(w)) for h, w in rng.integers(1, 300, (B // 4 + 1, 2))], seed=100 + B)[:B]
    files = [D.fixture(H, W, sub, q, kind, seed, **opts) for H, W, sub, q, kind, seed, opts in cases]
    assert not _check(files)


def test_every_quality_and_subsampling_at_500x375():
    files = [D.fixture(375, 500, sub, q, "smooth", 11 + i, **opts)
             for i, (sub, q, opts) in enumerate((s, q, o) for s in D.SUBSAMPLINGS for q in D.QUALITIES
                                                for o in ({}, {"optimize": True, "restart_marker_rows": 2}))]
    assert not _check(files)


def test_no_write_outside_out_and_repeatable():
    files = [D.fixture(H, W, sub, q, kind, seed, **opts) for H, W, sub, q, kind, seed, opts in D.matrix()[:24]]
    copies = [bytes(f) for f in files]
    hdrs, desc, blob, out_bytes, scratch_bytes = jpeg.stage(files)
    guard = 4096
    outs = []
    for _ in range(2):
        big = torch.full((out_bytes + 2 * guard,), 0xA5, dtype=torch.uint8, device=DEV)
        out = big[guard:guard + out_bytes]
        scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=DEV)
        status = torch.empty(len(files), dtype=torch.int32, device=DEV)
        dev, host, o_blob = jpeg._upload(DEV, desc, blob)
        _cabi.call("omt_jpeg_decode_u8", dev.data_ptr() + o_blob, blob.nbytes, dev, host.data_ptr(), len(files),
                   scratch, scratch_bytes, out, out_bytes, status)
        assert int(status.abs().sum()) == 0
        assert bool((big[:guard] == 0xA5).all()) and bool((big[guard + out_bytes:] == 0xA5).all())
        outs.append(out.cpu())
    assert torch.equal(outs[0], outs[1])
    assert files == copies
    for e, h, f in zip(desc, hdrs, files):
        got = outs[0][int(e["out"]):int(e["out"]) + 3 * h.H * h.W].numpy().reshape(h.H, h.W, 3)
        assert np.array_equal(got, D.pillow_rgb(f))


def test_refused_file_raises_before_any_launch():
    import io
    from PIL import Image
    good = D.fixture(16, 16, "4:2:0", 75, "noise", 1)
    f = io.BytesIO()
    Image.fromarray(np.zeros((16, 16, 3), np.uint8)).save(f, "JPEG", progressive=True)
    n0 = _cabi.launch_count
    with pytest.raises(NotImplementedError, match="source 1.*progressive"):
        jpeg.decode_u8([good, f.getvalue()], DEV)
    assert _cabi.launch_count == n0


def _corrupt(data: bytes, how: str) -> bytes:
    hdr = jpeg.parse(data)
    b = bytearray(data)
    if how == "truncated":
        return bytes(b[:hdr.scan + (len(b) - hdr.scan) // 2])
    if how == "no_eoi":
        return bytes(b[:-2])
    if how == "ff_run":                          # fill bytes, then a marker that is not EOI
        mid = hdr.scan + (len(b) - hdr.scan) // 3
        b[mid:mid + 64] = b"\xff" * 64
        return bytes(b)
    raise ValueError(how)


@pytest.mark.parametrize("how", ["truncated", "no_eoi", "ff_run"])
def test_corrupt_scan_raises_naming_the_file(how):
    good = D.fixture(64, 80, "4:2:0", 90, "noise", 3)
    bad = _corrupt(good, how)
    with pytest.raises(ValueError) as e:
        D.decode(bad)
    guard = 4096
    hdrs, desc, blob, out_bytes, scratch_bytes = jpeg.stage([good, bad])
    big = torch.full((out_bytes + 2 * guard,), 0xA5, dtype=torch.uint8, device=DEV)
    with pytest.raises(ValueError, match="source 1: corrupt JPEG scan"):
        jpeg.decode_u8([good, bad], DEV)
    scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=DEV)
    status = torch.empty(2, dtype=torch.int32, device=DEV)
    dev, host, o_blob = jpeg._upload(DEV, desc, blob)
    _cabi.call("omt_jpeg_decode_u8", dev.data_ptr() + o_blob, blob.nbytes, dev, host.data_ptr(), 2, scratch,
               scratch_bytes, big[guard:guard + out_bytes], out_bytes, status)
    st = status.cpu().tolist()
    assert st[0] == 0 and st[1] == e.value.code, (st, str(e.value))
    assert bool((big[:guard] == 0xA5).all()) and bool((big[guard + out_bytes:] == 0xA5).all())
