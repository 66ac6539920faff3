"""JPEG on the device, byte for byte as Pillow (libjpeg-turbo's integer chain: ISLOW IDCT, fancy upsampling).

roundtrip_u8: the pixels of a JPEG save and reload, what Pillow's img.save(f, "JPEG", quality=q) followed by
Image.open(f).convert("RGB") gives (baseline 4:2:0; oracle/jpeg_oracle.py is the step-by-step host restatement).
vqgan_eval.py saves every input and reconstruction of a dataset whose paths end in .jpg / .JPEG this way, and
pytorch-fid reads them back (consumers.eval_step_fid(saved_as="jpeg")).  No file and no bitstream is made: entropy
coding is lossless, so the pixels depend only on the integer transform chain, which omt_jpeg_roundtrip_u8 runs in two
launches.  Every check runs before the launch.

decode_u8: Image.open(f).convert("RGB") of JPEG files, decoded on the device (omt_jpeg_decode_u8,
oracle/jpeg_decode_oracle.py).  The forms Pillow writes are accepted -- sequential Huffman, 8-bit, one interleaved scan,
grayscale or YCbCr at 4:4:4, 4:2:2 and 4:2:0, any tables, restart intervals, APPn / COM segments -- and everything
else is refused by probe() / parse() before any launch.  A corrupt scan raises ValueError after the decode; libjpeg-turbo
decodes such files anyway, with a warning or (a coefficient index past 63) silently.
"""
from __future__ import annotations

import ctypes
import functools
import os
from dataclasses import dataclass
from typing import List, Optional, Tuple

import numpy as np
import torch

from . import _cabi
from .metricnet import bounded

DEFAULT_QUALITY = 75            # Pillow's JPEG quality when save() is given none
MAX_SCRATCH = 4                 # scratch buffers kept per process; the oldest goes first
_scratch = {}
_tables = {}

# ITU-T T.81 Annex K, tables K.1 (luminance) and K.2 (chrominance), natural order
_BASE = np.array([
    [16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55,
     14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
     18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
     49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99],
    [17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99,
     24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99] + [99] * 32], dtype=np.int64)


def check_quality(quality, what: str = "jpeg") -> int:
    if isinstance(quality, bool) or not isinstance(quality, (int, np.integer)) or not 1 <= int(quality) <= 100:
        raise ValueError(f"{what}: JPEG quality {quality!r} is not an integer in 1..100")
    return int(quality)


def quant_tables(quality: int = DEFAULT_QUALITY) -> np.ndarray:
    """uint16 [2, 64] (luminance, chrominance) in natural order, the tables Pillow writes at this quality
    (Image.open(f).quantization): libjpeg's scaling of Annex K, s = 5000 / q below 50 and 200 - 2 q from 50,
    (base s + 50) / 100 clamped to 1..255 (baseline)."""
    q = check_quality(quality, "quant_tables")
    s = 5000 // q if q < 50 else 200 - 2 * q
    return np.clip((_BASE * s + 50) // 100, 1, 255).astype(np.uint16)


def scratch_bytes(B: int, H: int, W: int) -> int:
    """omt_jpeg_roundtrip_u8's scratch: B images' decoded Y plane and two half-size chroma planes, sides rounded to 16."""
    hp, wp = -(-H // 16) * 16, -(-W // 16) * 16
    return B * hp * wp * 3 // 2


def roundtrip_u8(images: torch.Tensor, quality: int = DEFAULT_QUALITY) -> torch.Tensor:
    """(B, H, W, 3) uint8 RGB on a CUDA device -> a new (B, H, W, 3) uint8 tensor: each image saved as a JPEG of this
    quality by Pillow and read back as RGB.  The scratch is kept per device and size (at most MAX_SCRATCH of them), so a
    later call of the same shape can be captured in a CUDA graph."""
    q = check_quality(quality, "roundtrip_u8")
    if not isinstance(images, torch.Tensor) or images.dtype != torch.uint8:
        raise TypeError(f"roundtrip_u8: expected uint8 images, got {getattr(images, 'dtype', type(images))}")
    if images.dim() != 4 or images.shape[-1] != 3:
        raise ValueError(f"roundtrip_u8: expected (B, H, W, 3) RGB images, got shape {tuple(images.shape)}")
    if images.device.type != "cuda":
        raise ValueError(f"roundtrip_u8: images on {images.device}, not a CUDA device")
    B, H, W, _ = (int(v) for v in images.shape)
    if H < 1 or W < 1:
        raise ValueError(f"roundtrip_u8: empty {H}x{W} images")
    out = torch.empty_like(images, memory_format=torch.contiguous_format)
    if B == 0:
        return out
    src = images.contiguous()
    tables = bounded(_tables, 100, q, lambda: np.ascontiguousarray(quant_tables(q)))
    n = scratch_bytes(B, H, W)
    scratch = bounded(_scratch, MAX_SCRATCH, (src.device, n),
                      lambda: torch.empty(n, dtype=torch.uint8, device=src.device))
    _cabi.call("omt_jpeg_roundtrip_u8", src, out, B, H, W, tables.ctypes.data, scratch)
    return out


# ------------------------------------------------------------------------------------------------ decoding: the header
# zigzag position -> natural (row-major) position (jpeg_natural_order)
NATURAL = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
    28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
    54, 47, 55, 62, 63], dtype=np.int64)
SAMPLINGS = {(1, 1): "4:4:4", (2, 1): "4:2:2", (2, 2): "4:2:0"}   # luma (h, v) with chroma 1 x 1
_REFUSED_SOF = {0xC2: "progressive", 0xC3: "lossless", 0xC5: "hierarchical", 0xC6: "hierarchical",
                0xC7: "hierarchical", 0xC9: "arithmetic-coded", 0xCA: "arithmetic-coded (progressive)",
                0xCB: "arithmetic-coded (lossless)", 0xCD: "arithmetic-coded (hierarchical)",
                0xCE: "arithmetic-coded (hierarchical)", 0xCF: "arithmetic-coded (hierarchical)"}


@dataclass
class HuffTable:
    """A DHT table and libjpeg's derived form (jpeg_make_d_derived_tbl): lookup[256] = len << 8 | value for codes of at
    most 8 bits (9 << 8: longer), maxcode[18] / valoffset[18] by code length (maxcode -1: no code of that length,
    maxcode[17] the sentinel), values[256]."""
    counts: np.ndarray
    values: np.ndarray
    lookup: np.ndarray
    maxcode: np.ndarray
    valoffset: np.ndarray


@dataclass
class Header:
    """What omt_jpeg_decode_u8 needs of one accepted file.  comps: (id, h, v, quant table id, DC table id, AC table id)
    in frame order; for one component h = v = 1 (its scan's MCU is one block).  qt: id -> uint16 [64] natural order.
    scan: byte offset of the entropy-coded data, which runs to the end of the file."""
    name: str
    H: int
    W: int
    comps: List[Tuple[int, int, int, int, int, int]]
    qt: dict
    dc: dict
    ac: dict
    restart: int
    scan: int

    @property
    def hmax(self):
        return max(c[1] for c in self.comps)

    @property
    def vmax(self):
        return max(c[2] for c in self.comps)

    @property
    def mcus(self):
        """(MCU columns, MCU rows): ceil(W / 8 Hmax) x ceil(H / 8 Vmax)."""
        return -(-self.W // (8 * self.hmax)), -(-self.H // (8 * self.vmax))

    @property
    def blocks_per_mcu(self):
        return sum(c[1] * c[2] for c in self.comps)

    @property
    def segments(self):
        """Restart intervals in the scan (1 without DRI)."""
        n = self.mcus[0] * self.mcus[1]
        return -(-n // self.restart) if self.restart else 1


def derive_huffman(counts, values, is_dc: bool, name: str) -> HuffTable:
    """libjpeg's jpeg_make_d_derived_tbl, with its checks: at most 256 symbols, no over-subscribed code length (the
    all-ones code of a length is refused too), DC symbols at most 15.  Files mostly share a few tables, so the derived
    forms are cached by the table's bytes."""
    try:
        return _derive(bytes(np.asarray(counts, dtype=np.uint8)), bytes(np.asarray(values, dtype=np.uint8)), is_dc)
    except ValueError as e:
        raise ValueError(f"{name}: {e}") from None


@functools.lru_cache(maxsize=256)
def _derive(counts: bytes, values: bytes, is_dc: bool) -> HuffTable:
    counts = np.frombuffer(counts, dtype=np.uint8).astype(np.int64)
    values = np.frombuffer(values, dtype=np.uint8).astype(np.int64)
    n = int(counts.sum())
    if n > 256 or n != values.size:
        raise ValueError(f"Huffman table with {n} symbols")
    sizes = np.repeat(np.arange(1, 17), counts)
    codes = np.zeros(n, dtype=np.int64)
    code, p = 0, 0
    for length in range(1, 17):
        for _ in range(int(counts[length - 1])):
            codes[p] = code
            code += 1
            p += 1
        if code >= 1 << length:
            raise ValueError(f"over-subscribed Huffman table at code length {length}")
        code <<= 1
    maxcode = np.full(18, -1, dtype=np.int64)
    valoffset = np.zeros(18, dtype=np.int64)
    p = 0
    for length in range(1, 17):
        if counts[length - 1]:
            valoffset[length] = p - codes[p]
            p += int(counts[length - 1])
            maxcode[length] = codes[p - 1]
    maxcode[17] = 0xFFFFF
    lookup = np.full(256, 9 << 8, dtype=np.int64)
    for i in range(n):
        if sizes[i] <= 8:
            shift = 8 - int(sizes[i])
            lookup[int(codes[i]) << shift:(int(codes[i]) + 1) << shift] = int(sizes[i]) << 8 | int(values[i])
    if is_dc and n and values.max() > 15:
        raise ValueError(f"DC Huffman symbol {int(values.max())} above 15")
    return HuffTable(counts, values, lookup, maxcode, valoffset)


def _name(data, name):
    return name if name is not None else (str(data) if isinstance(data, (str, os.PathLike)) else "<jpeg bytes>")


def parse(data, name: Optional[str] = None) -> Header:
    """The header of a JPEG file (bytes-like or a path) that omt_jpeg_decode_u8 decodes.  Raises NotImplementedError
    naming the file and the reason for a form it does not decode, ValueError for a malformed header.  Reads the
    segments before the scan only, never the scan's bytes."""
    name = _name(data, name)
    if isinstance(data, (str, os.PathLike)):
        with open(data, "rb") as f:
            data = f.read()
    d = memoryview(data).cast("B")
    n = len(d)

    def bad(msg):
        return ValueError(f"{name}: {msg}")

    def refuse(msg):
        return NotImplementedError(f"{name}: {msg} JPEG files are not decoded on the device")

    if n < 4 or d[0] != 0xFF or d[1] != 0xD8:
        raise bad("not a JPEG file (no SOI marker)")
    pos = 2
    qt, dc, ac = {}, {}, {}
    frame, restart, jfif, adobe = None, 0, False, None
    while True:
        if pos + 2 > n or d[pos] != 0xFF:
            raise bad(f"expected a marker at byte {pos}")
        while pos + 1 < n and d[pos + 1] == 0xFF:          # fill bytes
            pos += 1
        if pos + 4 > n:
            raise bad("file ends inside a marker segment")
        m = d[pos + 1]
        if m in (0xD8, 0xD9) or 0xD0 <= m <= 0xD7 or m == 0x01 or m == 0:
            raise bad(f"unexpected marker FF{m:02X} before the scan")
        length = d[pos + 2] << 8 | d[pos + 3]
        if length < 2 or pos + 2 + length > n:
            raise bad(f"segment FF{m:02X} at byte {pos} has length {length}")
        seg = d[pos + 4:pos + 2 + length]
        pos += 2 + length
        if m in _REFUSED_SOF:
            raise refuse(_REFUSED_SOF[m])
        if m == 0xCC:
            raise refuse("arithmetic-coded")
        if m in (0xDE, 0xDF):
            raise refuse("hierarchical")
        if m == 0xDC:
            raise refuse("DNL")
        if m in (0xC0, 0xC1):
            if frame is not None:
                raise bad("two SOF segments")
            if len(seg) < 6:
                raise bad("short SOF segment")
            P, H, W, nf = seg[0], seg[1] << 8 | seg[2], seg[3] << 8 | seg[4], seg[5]
            if len(seg) != 6 + 3 * nf:
                raise bad(f"SOF segment of {len(seg)} bytes for {nf} components")
            if P != 8:
                raise refuse(f"{P}-bit")
            if H == 0:
                raise refuse("DNL (height 0 in the frame header)")
            if W == 0 or nf == 0:
                raise bad(f"{H}x{W} frame of {nf} components")
            comps = []
            for i in range(nf):
                cid, hv, tq = seg[6 + 3 * i], seg[7 + 3 * i], seg[8 + 3 * i]
                h, v = hv >> 4, hv & 15
                if not (1 <= h <= 4 and 1 <= v <= 4) or tq > 3:
                    raise bad(f"component {cid}: sampling {h}x{v}, quantisation table {tq}")
                comps.append([cid, h, v, tq])
            frame = (H, W, comps)
        elif m == 0xDB:
            i = 0
            while i < len(seg):
                pq, tq = seg[i] >> 4, seg[i] & 15
                size = 64 * (pq + 1)
                if pq > 1 or tq > 3 or i + 1 + size > len(seg):
                    raise bad(f"DQT table {tq} of precision {pq} in a {len(seg)}-byte segment")
                raw = np.frombuffer(bytes(seg[i + 1:i + 1 + size]), dtype=">u2" if pq else np.uint8).astype(np.int64)
                if raw.min() == 0:
                    raise bad(f"DQT table {tq} has a zero entry")
                t = np.zeros(64, dtype=np.int64)
                t[NATURAL] = raw
                qt[tq] = t.astype(np.uint16)
                i += 1 + size
        elif m == 0xC4:
            i = 0
            while i < len(seg):
                tc, th = seg[i] >> 4, seg[i] & 15
                if tc > 1 or th > 3 or i + 17 > len(seg):
                    raise bad(f"DHT table class {tc} id {th} in a {len(seg)}-byte segment")
                counts = np.frombuffer(bytes(seg[i + 1:i + 17]), dtype=np.uint8).astype(np.int64)
                k = int(counts.sum())
                if i + 17 + k > len(seg):
                    raise bad(f"DHT table of {k} symbols overruns its segment")
                values = np.frombuffer(bytes(seg[i + 17:i + 17 + k]), dtype=np.uint8).astype(np.int64)
                (ac if tc else dc)[th] = derive_huffman(counts, values, not tc, f"{name}: {'AC' if tc else 'DC'} table {th}")
                i += 17 + k
        elif m == 0xDD:
            if len(seg) != 2:
                raise bad(f"DRI segment of {len(seg)} bytes")
            restart = seg[0] << 8 | seg[1]
        elif m == 0xE0:
            jfif = jfif or (len(seg) >= 14 and bytes(seg[:5]) == b"JFIF\0")
        elif m == 0xEE:
            if len(seg) >= 12 and bytes(seg[:5]) == b"Adobe":
                adobe = seg[11]
        elif m == 0xDA:
            if frame is None:
                raise bad("SOS before SOF")
            H, W, comps = frame
            ns = seg[0] if len(seg) else 0
            if len(seg) != 4 + 2 * ns or ns == 0:
                raise bad(f"SOS segment of {len(seg)} bytes for {ns} components")
            if ns != len(comps):
                raise refuse(f"multi-scan (the first scan has {ns} of {len(comps)} components)")
            ss, se, ahal = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]
            if ss != 0 or se != 63 or ahal != 0:
                raise bad(f"sequential scan with Ss={ss} Se={se} Ah/Al={ahal:#x}")
            by_id = {c[0]: c for c in comps}
            if len(by_id) != len(comps):
                raise bad("two components with one id")
            for i in range(ns):
                cid, t = seg[1 + 2 * i], seg[2 + 2 * i]
                if cid not in by_id or len(by_id[cid]) > 4:
                    raise bad(f"scan component {cid} is not in the frame or repeated")
                by_id[cid].extend((t >> 4, t & 15))
            if [seg[1 + 2 * i] for i in range(ns)] != [c[0] for c in comps]:
                raise refuse("a scan whose component order differs from the frame's")
            for c in comps:
                if c[3] not in qt:
                    raise bad(f"component {c[0]} uses quantisation table {c[3]}, which is not defined")
                if c[4] not in dc or c[5] not in ac:
                    raise bad(f"component {c[0]} uses Huffman tables DC {c[4]} / AC {c[5]}, not both defined")
            if len(comps) == 3:
                ids = tuple(c[0] for c in comps)
                if not jfif and (adobe == 0 if adobe is not None else ids == (82, 71, 66)):
                    raise refuse("RGB (untransformed, e.g. keep_rgb=True)")
                if (comps[0][1], comps[0][2]) not in SAMPLINGS or any(c[1:3] != [1, 1] for c in comps[1:]):
                    raise refuse("sampling " + ", ".join(f"{c[1]}x{c[2]}" for c in comps))
            elif len(comps) == 1:
                comps[0][1:3] = [1, 1]      # a one-component scan's MCU is one block whatever the factors say
            else:
                raise refuse(f"{len(comps)}-component" + (" (CMYK / YCCK)" if len(comps) == 4 else ""))
            if pos >= n:
                raise bad("no scan data after SOS")
            return Header(name, H, W, [tuple(int(v) for v in c) for c in comps],
                          {c[3]: qt[c[3]] for c in comps}, {c[4]: dc[c[4]] for c in comps},
                          {c[5]: ac[c[5]] for c in comps}, restart, pos)
        elif m in (0xC8,) or 0xF0 <= m <= 0xFD:
            raise refuse(f"extension marker FF{m:02X}")
        elif not (0xE0 <= m <= 0xEF or m == 0xFE):
            raise bad(f"unexpected marker FF{m:02X}")


def probe(data) -> Optional[str]:
    """None if omt_jpeg_decode_u8 decodes this file (bytes-like or a path), else the reason it does not: the message
    parse() would raise."""
    try:
        parse(data)
    except (NotImplementedError, ValueError) as e:
        return str(e)
    return None


# ------------------------------------------------------------------------------------------------ decoding: the device
GROUP, SUB_BITS = 128, 1024              # csrc/jpeg_decode.cu: subsequences per CTA, bits per subsequence
DESC = np.dtype([("scan", "<i8"), ("scan_bytes", "<i8"), ("tables", "<i8"), ("out", "<i8"), ("work", "<i8"),
                 ("H", "<i4"), ("W", "<i4"), ("ncomp", "<i4"), ("h", "<i4", 3), ("v", "<i4", 3), ("restart", "<i4"),
                 ("nsub", "<i4"), ("reserved", "<i4")])                                     # omt_jpeg_desc
TABLES = np.dtype([("q", "<i4", (3, 64)), ("lookup", "<u2", (6, 256)), ("maxcode", "<i4", (6, 18)),
                   ("valoffset", "<i4", (6, 18)), ("values", "u1", (6, 256))])             # omt_jpeg_tables
STATUS = {1: "the scan has no end marker", 2: "restart marker out of order", 3: "wrong number of restart intervals",
          4: "invalid Huffman code", 5: "coefficient index past 63", 6: "scan data ends inside an MCU",
          7: "the scan is not followed by EOI", 8: "extraneous data before a marker"}
_staging = {}


def _up(x: int, a: int) -> int:
    return -(-x // a) * a


def subsequences(hdr: Header, scan_bytes: int) -> int:
    """Subsequence slots of a file: every restart interval's bits cut into SUB_BITS pieces fit, whatever the stuffing."""
    return _up(-(-8 * scan_bytes // SUB_BITS) + hdr.segments, GROUP)


def work_bytes(hdr: Header, scan_bytes: int) -> int:
    """Size of a file's work area in omt_jpeg_decode_u8's scratch (csrc/jpeg_decode.cu work_of)."""
    mx, my = hdr.mcus
    nseg, nsub = hdr.segments, subsequences(hdr, scan_bytes)
    o = 256
    o = _up(o + 4 * (nseg + 1), 256)
    o = _up(o + 4 * (nseg + 1), 256)
    o = _up(o + scan_bytes + 16, 256)
    o += 48 * nsub
    o = _up(o + 128 * mx * my * hdr.blocks_per_mcu, 256)
    for c in hdr.comps:
        o = _up(o + mx * c[1] * 8 * my * c[2] * 8, 256)
    return o


def _table_struct(hdr: Header) -> np.ndarray:
    t = np.zeros(1, dtype=TABLES)[0]
    for i, (_, _, _, tq, td, ta) in enumerate(hdr.comps):
        t["q"][i] = hdr.qt[tq]
        for j, h in ((2 * i, hdr.dc[td]), (2 * i + 1, hdr.ac[ta])):
            t["lookup"][j] = h.lookup
            t["maxcode"][j] = h.maxcode
            t["valoffset"][j] = h.valoffset
            t["values"][j, :h.values.size] = h.values
    return t


def _read(src, i: int):
    if isinstance(src, (str, os.PathLike)):
        with open(src, "rb") as f:
            return f.read(), str(src)
    if isinstance(src, (bytes, bytearray, memoryview, np.ndarray)):
        return bytes(memoryview(src).cast("B")) if not isinstance(src, bytes) else src, f"source {i}"
    raise TypeError(f"source {i}: expected JPEG bytes or a path, got {type(src).__name__}")


def stage(sources, names=None):
    """Parse every file (refusals and malformed headers raise here) and lay out one batch: (headers, desc [B] DESC,
    blob bytes, out bytes, scratch bytes).  The blob holds each file's omt_jpeg_tables, then its scan."""
    datas = [_read(s, i) for i, s in enumerate(sources)]
    if names is not None:
        datas = [(d, n) for (d, _), n in zip(datas, names)]
    hdrs = [parse(d, n) for d, n in datas]
    desc = np.zeros(len(hdrs), dtype=DESC)
    parts, o_blob, o_out, o_work = [], 0, 0, 256
    for i, ((d, _), h) in enumerate(zip(datas, hdrs)):
        e = desc[i]
        scan = memoryview(d)[h.scan:]
        e["tables"], o_blob = o_blob, o_blob + TABLES.itemsize
        e["scan"], e["scan_bytes"] = o_blob, len(scan)
        parts += [(int(e["tables"]), _table_struct(h).tobytes()), (o_blob, scan)]
        o_blob = _up(o_blob + len(scan), 16)
        e["out"], o_out = o_out, o_out + 3 * h.H * h.W
        e["work"], o_work = o_work, o_work + work_bytes(h, len(scan))
        e["H"], e["W"], e["ncomp"], e["restart"] = h.H, h.W, len(h.comps), h.restart
        e["h"][:len(h.comps)] = [c[1] for c in h.comps]
        e["v"][:len(h.comps)] = [c[2] for c in h.comps]
        e["nsub"] = subsequences(h, len(scan))
    blob = np.zeros(o_blob, dtype=np.uint8)
    for off, b in parts:
        blob[off:off + len(b)] = np.frombuffer(b, dtype=np.uint8)
    return hdrs, desc, blob, o_out, o_work


def _upload(device, desc: np.ndarray, blob: np.ndarray):
    """desc and blob through one grow-only pinned buffer per device in one asynchronous H2D copy on the current stream.
    Returns (device buffer, host buffer, blob offset)."""
    o_blob = _up(desc.nbytes, 256)
    total = o_blob + blob.nbytes
    st = _staging.get(device)
    if st is not None:
        st[2].synchronize()                 # the previous batch's copy has read the pinned buffer
    if st is None or st[0].numel() < total:
        cap = max(total, 3 * (0 if st is None else st[0].numel()) // 2)
        st = (torch.empty(cap, dtype=torch.uint8, pin_memory=True), torch.empty(cap, dtype=torch.uint8, device=device),
              torch.cuda.Event())
        _staging[device] = st
    host, dev, done = st
    h = host.numpy()
    h[:desc.nbytes] = desc.view(np.uint8)
    h[o_blob:total] = blob
    dev[:total].copy_(host[:total], non_blocking=True)
    done.record()
    return dev, host, o_blob


def _names(sources):
    return [str(s) if isinstance(s, (str, os.PathLike)) else f"source {i}" for i, s in enumerate(sources)]


def decode_into(staged, names, out: torch.Tensor, offsets, timings: Optional[dict] = None):
    """Decode a batch stage() laid out into the uint8 device tensor `out` (any contiguous buffer), file i's (H, W, 3)
    bytes at byte offset offsets[i], on out's device and torch's current stream.  A corrupt scan raises ValueError naming
    the first bad file (names[i]) after one 4 B-byte read back, before any later launch can use out.  timings: if a
    dict is given, it receives the per-stage device times in ms and the synchronisation's launch count."""
    hdrs, desc, blob, _, scratch_bytes = staged
    if not hdrs:
        return
    desc["out"] = np.asarray(offsets, dtype=np.int64)
    device = out.device
    with torch.cuda.device(device):
        scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=device)
        status = torch.empty(len(hdrs), dtype=torch.int32, device=device)
        dev, host, o_blob = _upload(device, desc, blob)
        args = (dev.data_ptr() + o_blob, blob.nbytes, dev, host.data_ptr(), len(hdrs), scratch, scratch_bytes, out,
                out.numel(), status)
        ms, launches = (ctypes.c_float * 5)(), ctypes.c_int()
        _cabi.call("omt_jpeg_decode_u8_timed", *args, None if timings is None else ctypes.addressof(ms),
                   ctypes.addressof(launches))
        _cabi.launch_count += 4 + launches.value        # 5 kernels and the synchronisation's; call() counted one
        if timings is not None:
            timings.update(zip(("destuff", "sync", "decode", "idct", "pixels"), list(ms)))
            timings["sync_launches"] = launches.value
        bad = status.cpu().numpy()
    for i in np.flatnonzero(bad):
        raise ValueError(f"{names[i]}: corrupt JPEG scan: {STATUS.get(int(bad[i]), f'status {int(bad[i])}')}")


def decode_u8(sources, device, timings: Optional[dict] = None) -> List[torch.Tensor]:
    """Image.open(f).convert("RGB") of each source -- JPEG bytes (bytes-like) or a path -- decoded on `device`: a list of
    (H_i, W_i, 3) uint8 tensors (views of one buffer), equal to Pillow's bytes.  Every file is parsed first; a refused
    form raises NotImplementedError and a malformed header ValueError, naming the file, before any launch.  A corrupt
    scan raises ValueError naming the first bad file (decode_into).  timings: see decode_into."""
    sources = list(sources)
    device = torch.device(device)
    if device.type != "cuda":
        raise ValueError(f"decode_u8: {device} is not a CUDA device")
    device = torch.device("cuda", device.index if device.index is not None else torch.cuda.current_device())
    names = _names(sources)
    staged = stage(sources, names)
    hdrs, desc, _, out_bytes, _ = staged
    out = torch.empty(max(out_bytes, 1), dtype=torch.uint8, device=device)
    offsets = [int(e["out"]) for e in desc]
    decode_into(staged, names, out, offsets, timings)
    return [out[o:o + 3 * h.H * h.W].view(h.H, h.W, 3) for o, h in zip(offsets, hdrs)]


class Pending:
    """A JPEG file of a mixed sources list (split_sources), standing in for its decoded (H, W, 3) image until the device
    decodes it in place: .shape, and .index into the batch's staged files."""

    def __init__(self, H: int, W: int, index: int):
        self.shape = (H, W, 3)
        self.index = index


def split_sources(sources):
    """A sources list of JPEG files (bytes-like or paths) and decoded (H, W, C) uint8 host tensors -> (images, jpegs):
    images keeps the tensors and puts a Pending of the file's size in each JPEG's place; jpegs is None without JPEG
    files, else (staged batch, names) for decode_into.  Every file is parsed here: a refused or malformed one raises
    before any launch."""
    sources = list(sources)
    at = [i for i, s in enumerate(sources) if not isinstance(s, torch.Tensor)]
    if not at:
        return sources, None
    names = [str(sources[i]) if isinstance(sources[i], (str, os.PathLike)) else f"source {i}" for i in at]
    staged = stage([sources[i] for i in at], names)
    images = list(sources)
    for k, (i, h) in enumerate(zip(at, staged[0])):
        images[i] = Pending(h.H, h.W, k)
    return images, (staged, names)
