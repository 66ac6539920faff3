"""The host side of the JPEG decoder (omnitokenizer_b200/jpeg.py parse / probe) and its oracle
(oracle/jpeg_decode_oracle.py), no GPU: headers against Pillow over the fixture matrix, every refusal with its reason,
malformed headers, the serial oracle decode against Pillow byte for byte, the self-synchronising restatement against the
serial decode at subsequence sizes from 32 bits, and tests/golden/jpeg_decode.pt."""
import hashlib
import io

import numpy as np
import pytest
from PIL import Image, JpegImagePlugin

from oracle import jpeg_decode_oracle as D
from omnitokenizer_b200 import jpeg
from tests.util import load_golden

SMALL = [s for s in D.SIZES if s[0] * s[1] <= 127 * 255]


def _files(sizes):
    return [(c, D.fixture(*c[:6], **c[6])) for c in D.matrix(sizes)]


@pytest.fixture(scope="module")
def small_files():
    return _files(SMALL)


def test_header_matches_pillow():
    for (H, W, sub, q, kind, seed, opts), f in _files(D.SIZES):
        h = jpeg.parse(f)
        im = Image.open(io.BytesIO(f))
        assert (h.W, h.H) == im.size
        assert im.mode == ("L" if sub == "L" else "RGB")
        if sub != "L":
            assert JpegImagePlugin.get_sampling(im) == {"4:4:4": 0, "4:2:2": 1, "4:2:0": 2}[sub]
            assert D.SAMPLINGS_OF[sub] == (h.comps[0][1], h.comps[0][2])
        assert {k: list(v) for k, v in h.qt.items()} == {k: list(v) for k, v in im.quantization.items()}
        want = opts.get("restart_marker_blocks", 0) or opts.get("restart_marker_rows", 0) * h.mcus[0]
        assert h.restart == want
        assert jpeg.probe(f) is None


def _pillow(**kw):
    f = io.BytesIO()
    mode = kw.pop("mode", "RGB")
    Image.fromarray(np.full((24, 40, 3), 100, np.uint8)).convert(mode).save(f, "JPEG", **kw)
    return f.getvalue()


def _sof(data: bytes) -> int:
    return data.index(b"\xff\xc0")


def _patch(data: bytes, at: int, value: int) -> bytes:
    b = bytearray(data)
    b[at] = value
    return bytes(b)


def _second_sos(data: bytes) -> bytes:
    """The first scan covers Y alone and a second SOS follows: a sequential multi-scan file."""
    h = jpeg.parse(data)
    sos = data.rindex(b"\xff\xda", 0, h.scan)
    one = b"\xff\xda\x00\x08\x01" + data[sos + 5:sos + 7] + b"\x00\x3f\x00"
    return data[:sos] + one + data[h.scan:-2] + data[sos:]


REFUSALS = {
    "progressive": (lambda: _pillow(progressive=True), "progressive"),
    "cmyk": (lambda: _pillow(mode="CMYK"), "4-component"),
    "keep_rgb": (lambda: _pillow(keep_rgb=True), "RGB"),
    "4:1:1": (lambda: _patch(_pillow(subsampling="4:4:4"), _sof(_pillow(subsampling="4:4:4")) + 11, 0x41), "sampling"),
    "4:4:0": (lambda: _patch(_pillow(subsampling="4:4:4"), _sof(_pillow(subsampling="4:4:4")) + 11, 0x12), "sampling"),
    "arithmetic": (lambda: _patch(_pillow(), _sof(_pillow()) + 1, 0xC9), "arithmetic"),
    "12-bit": (lambda: _patch(_pillow(), _sof(_pillow()) + 4, 12), "12-bit"),
    "second_sos": (lambda: _second_sos(_pillow()), "multi-scan"),
    "dnl": (lambda: _patch(_patch(_pillow(), _sof(_pillow()) + 5, 0), _sof(_pillow()) + 6, 0), "DNL"),
}


@pytest.mark.parametrize("what", sorted(REFUSALS))
def test_refusals_name_the_file_and_reason(what):
    make, reason = REFUSALS[what]
    data = make()
    with pytest.raises(NotImplementedError, match=f"f.jpg: .*{reason}"):
        jpeg.parse(data, "f.jpg")
    assert reason in jpeg.probe(data)


def _oversubscribed(data: bytes) -> bytes:
    i = data.index(b"\xff\xc4")
    return _patch(data, i + 5, 3)              # three 1-bit codes in the first DC table


MALFORMED = {
    "not_jpeg": lambda d: b"\x89PNG" + d[4:],
    "segment_length": lambda d: _patch(d, d.index(b"\xff\xdb") + 3, 0xFF),
    "missing_huffman_table": lambda d: d.replace(b"\xff\xc4", b"\xff\xe5"),
    "missing_quant_table": lambda d: d.replace(b"\xff\xdb", b"\xff\xe5"),
    "oversubscribed": _oversubscribed,
    "short_file": lambda d: d[:_sof(d) + 6],
    "sos_before_sof": lambda d: _patch(d, _sof(d) + 1, 0xE6),
}


@pytest.mark.parametrize("what", sorted(MALFORMED))
def test_malformed_headers_raise_value_error(what):
    data = MALFORMED[what](_pillow())
    with pytest.raises(ValueError, match="bad.jpg"):
        jpeg.parse(data, "bad.jpg")


def test_oracle_decode_equals_pillow(small_files):
    bad = [c for c, f in small_files if not np.array_equal(D.decode(f), D.pillow_rgb(f))]
    assert not bad, bad


@pytest.mark.parametrize("S", [32, 33, 45, 64, 100, 257, 1024])
def test_sync_restatement_equals_serial_decode(small_files, S):
    for c, f in small_files[::3]:
        h = jpeg.parse(f)
        serial = D.decode_serial(h, f)
        for group in (1, 2, 4):
            got = D.decode_sync(h, f, S, group)
            assert all(np.array_equal(a, b) for a, b in zip(got, serial)), (c, S, group)


def test_golden_sha_matches():
    g = load_golden("jpeg_decode")
    for f, sha, c in zip(g["files"], g["sha256"], g["cases"]):
        assert hashlib.sha256(D.decode(f).tobytes()).hexdigest() == sha, c
        assert hashlib.sha256(D.pillow_rgb(f).tobytes()).hexdigest() == sha, c


def test_work_layout_bounds_the_subsequences():
    for (H, W, sub, q, kind, seed, opts), f in _files(SMALL):
        h = jpeg.parse(f)
        n = len(f) - h.scan
        assert jpeg.subsequences(h, n) % jpeg.GROUP == 0
        assert jpeg.subsequences(h, n) >= -(-8 * n // jpeg.SUB_BITS) + h.segments
