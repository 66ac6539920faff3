"""Image.open(f).convert("RGB") of the JPEG files omt_jpeg_decode_u8 accepts (omnitokenizer_b200.jpeg.parse), restated on
the host in plain Python and NumPy int64:

    destuff(scan)                 the entropy-coded bytes -> restart segments of plain bytes, and the end marker
    decode_serial(hdr, data)      the serial Huffman decode -> per component quantised coefficients
    decode_sync(hdr, data, S)     the same coefficients through the self-synchronising subsequence scheme
    pixels(hdr, coefs)            dequantise, ISLOW IDCT, fancy upsampling (h2v1, h2v2) and colour -> (H, W, 3) uint8
    decode(data)                  decode_serial then pixels

Errors the device reports in its status word raise ValueError here with the same wording (STATUS).
"""
from __future__ import annotations

import numpy as np

from omnitokenizer_b200 import jpeg as J
from oracle import jpeg_oracle as JO

# status words of omt_jpeg_decode_u8 (include/omnitok_b200.h)
STATUS = {1: "the scan has no end marker", 2: "restart marker out of order", 3: "wrong number of restart intervals",
          4: "invalid Huffman code", 5: "coefficient index past 63", 6: "scan data ends inside an MCU",
          7: "the scan is not followed by EOI", 8: "extraneous data before a marker"}


class DecodeError(ValueError):
    def __init__(self, code: int):
        super().__init__(STATUS[code])
        self.code = code


# ------------------------------------------------------------------------------------------------------------ destuff
def destuff(scan: bytes):
    """Scan bytes -> (segments, end marker code): FF00 -> FF, fill FFs dropped, RSTn split segments (checked in order),
    the first other marker ends the scan."""
    segs, cur, i, n, nrst = [], bytearray(), 0, len(scan), 0
    while True:
        if i >= n:
            raise DecodeError(1)
        b = scan[i]
        if b != 0xFF:
            cur.append(b)
            i += 1
            continue
        if i + 1 >= n:
            raise DecodeError(1)
        nx = scan[i + 1]
        if nx == 0x00:
            cur.append(0xFF)
            i += 2
        elif nx == 0xFF:
            i += 1
        elif 0xD0 <= nx <= 0xD7:
            if nx != 0xD0 + (nrst & 7):
                raise DecodeError(2)
            nrst += 1
            segs.append(bytes(cur))
            cur = bytearray()
            i += 2
        else:
            segs.append(bytes(cur))
            return segs, nx


# ------------------------------------------------------------------------------------------------------------ symbols
def _extend(r, s):
    return r - (1 << s) + 1 if r < 1 << (s - 1) else r


class Stream:
    """One segment's bits, MSB first; reads past the end give zeros."""

    def __init__(self, data: bytes):
        self.v = int.from_bytes(data + b"\0" * 8, "big")
        self.nbits = 8 * len(data)
        self.total = 8 * (len(data) + 8)

    def peek32(self, pos: int) -> int:
        if pos + 32 > self.total:
            return (self.v << (pos + 32 - self.total)) & 0xFFFFFFFF if pos < self.total else 0
        return (self.v >> (self.total - pos - 32)) & 0xFFFFFFFF


def huff(t: J.HuffTable, w: int):
    """(length, symbol) of the code at the top of the 32-bit window w; (0, -1) if none matches."""
    e = int(t.lookup[w >> 24])
    if e >> 8 <= 8:
        return e >> 8, e & 255
    for length in range(9, 17):
        code = w >> (32 - length)
        if code <= t.maxcode[length]:
            return length, int(t.values[(code + int(t.valoffset[length])) & 255])
    return 0, -1


def step(hdr: J.Header, slots, st: Stream, pos: int, slot: int, z: int):
    """Decode one symbol from state (pos, slot, z); z = 0: the next symbol is a DC one.  Returns the new state and the
    event: ("dc", diff), ("ac", k, value), ("zeros",) or ("err", status).  An error ends the block, so speculative
    decoding stays deterministic."""
    c = slots[slot]
    w = st.peek32(pos)
    if z == 0:
        length, s = huff(hdr.dc[hdr.comps[c][4]], w)
        if length == 0:
            return pos + 16, (slot + 1) % len(slots), 0, ("err", 4)
        diff = _extend((w << length & 0xFFFFFFFF) >> (32 - s), s) if s else 0
        return pos + length + s, slot, 1, ("dc", diff)
    length, rs = huff(hdr.ac[hdr.comps[c][5]], w)
    nxt = lambda zz: (slot, zz) if zz < 64 else ((slot + 1) % len(slots), 0)
    if length == 0:
        return pos + 16, (slot + 1) % len(slots), 0, ("err", 4)
    r, s = rs >> 4, rs & 15
    if s:
        k = z + r
        if k > 63:
            return pos + length + s, (slot + 1) % len(slots), 0, ("err", 5)
        val = _extend((w << length & 0xFFFFFFFF) >> (32 - s), s)
        sl, zz = nxt(k + 1)
        return pos + length + s, sl, zz, ("ac", k, val)
    if r == 15:
        if z + 16 > 64:
            return pos + length, (slot + 1) % len(slots), 0, ("err", 5)
        sl, zz = nxt(z + 16)
        return pos + length, sl, zz, ("zeros",)
    return pos + length, (slot + 1) % len(slots), 0, ("zeros",)


def mcu_slots(hdr: J.Header):
    """Component of each block slot of an MCU, in scan order."""
    return [c for c, comp in enumerate(hdr.comps) for _ in range(comp[1] * comp[2])]


def _store(hdr, slots, coefs, block: int, k: int, val: int):
    """Coefficient k (zigzag) of serial block `block` into its component's plane of blocks."""
    bpm = len(slots)
    mx_n = hdr.mcus[0]
    mcu, slot = divmod(block, bpm)
    c = slots[slot]
    h, v = hdr.comps[c][1], hdr.comps[c][2]
    first = slots.index(c)
    by, bx = divmod(slot - first, h)
    my, mx = divmod(mcu, mx_n)
    coefs[c][my * v + by, mx * h + bx, J.NATURAL[k]] = val


def _planes(hdr):
    mx, my = hdr.mcus
    return [np.zeros((my * c[2], mx * c[1], 64), dtype=np.int64) for c in hdr.comps]


def _segment_blocks(hdr, k: int) -> int:
    n = hdr.mcus[0] * hdr.mcus[1]
    per = hdr.restart or n
    return min(per, n - k * per) * hdr.blocks_per_mcu


def _check_segments(hdr, segs, end):
    if len(segs) != hdr.segments:
        raise DecodeError(3)
    if end != 0xD9:
        raise DecodeError(7)


def _finish_segment(st: Stream, pos: int):
    if pos > st.nbits:
        raise DecodeError(6)
    if st.nbits - pos >= 8:
        raise DecodeError(8)


def _int16(v: int) -> int:
    return (v + 32768) % 65536 - 32768


def decode_serial(hdr: J.Header, data: bytes):
    """The scan -> per component int64 (rows, cols, 64) natural-order coefficients over the whole MCU grid (the dummy
    blocks of edge MCUs included), DC values summed per component and reset at each restart, stored as int16."""
    segs, end = destuff(bytes(data[hdr.scan:]))
    _check_segments(hdr, segs, end)
    slots, coefs = mcu_slots(hdr), _planes(hdr)
    block = 0
    for k, seg in enumerate(segs):
        st, pos, slot, z, last = Stream(seg), 0, 0, 0, [0] * len(hdr.comps)
        todo = _segment_blocks(hdr, k)
        while todo:
            c = slots[slot]
            pos, nslot, z, ev = step(hdr, slots, st, pos, slot, z)
            if pos > st.nbits:
                raise DecodeError(6)
            if ev[0] == "err":
                raise DecodeError(ev[1])
            if ev[0] == "dc":
                last[c] += ev[1]
                _store(hdr, slots, coefs, block, 0, _int16(last[c]))
            elif ev[0] == "ac":
                _store(hdr, slots, coefs, block, ev[1], ev[2])
            if z == 0:
                block += 1
                todo -= 1
            slot = nslot
        _finish_segment(st, pos)
    return coefs


# ------------------------------------------------------------------------------------------------------------ sync
def decode_sync(hdr: J.Header, data: bytes, S: int, group: int = 4):
    """decode_serial through Weissenberger & Schmidt's self-synchronising scheme, as omt_jpeg_decode_u8 runs it: each
    segment is cut into S-bit subsequences, each decoded from its first bit with a guessed state (slot 0, z 0); within a
    group of `group` subsequences each takes its predecessor's exit state as its entry until no entry changes, then the
    groups do the same across their boundaries ("launches") until nothing changes.  Then every subsequence decodes
    again from its entry, placing its blocks by a prefix sum of per-subsequence block counts and its DC values by a
    per-component prefix sum of the differences."""
    segs, end = destuff(bytes(data[hdr.scan:]))
    _check_segments(hdr, segs, end)
    slots, coefs = mcu_slots(hdr), _planes(hdr)
    ncomp = len(hdr.comps)
    subs = []                                       # (segment, start, end) in order
    for k, seg in enumerate(segs):
        nbits = 8 * len(seg)
        subs += [(k, a, min(a + S, nbits)) for a in range(0, nbits, S)]
    streams = [Stream(s) for s in segs]

    def run(i, entry):
        k, a, b = subs[i]
        pos, slot, z = entry
        nblk, dc = 0, [0] * ncomp
        while pos < b:
            c = slots[slot]
            pos, slot, z, ev = step(hdr, slots, streams[k], pos, slot, z)
            if ev[0] == "dc":
                nblk += 1
                dc[c] += ev[1]
        return (pos, slot, z), nblk, dc

    n = len(subs)
    head = [i == 0 or subs[i][0] != subs[i - 1][0] for i in range(n)]
    entry = [(subs[i][1], 0, 0) for i in range(n)]
    res = [run(i, entry[i]) for i in range(n)]
    launches = 0
    while True:
        changed = False
        for g0 in range(0, n, group):
            while True:                              # inside the group: until no entry changes
                moved = False
                for i in range(g0, min(g0 + group, n)):
                    if head[i] or (i == g0 and launches == 0):
                        continue
                    if entry[i] != res[i - 1][0]:
                        entry[i] = res[i - 1][0]
                        res[i] = run(i, entry[i])
                        moved = True
                        changed = changed or i == g0
                if not moved:
                    break
        launches += 1
        if launches > 1 and not changed:
            break
    # the decode: block and DC prefix sums within each segment
    for k, seg in enumerate(segs):
        idx = [i for i in range(n) if subs[i][0] == k]
        base = sum(_segment_blocks(hdr, j) for j in range(k))
        todo = _segment_blocks(hdr, k)
        done = False
        nb, dcs = 0, [0] * ncomp
        for i in idx:
            pos, slot, z = entry[i]
            block = base + nb - 1                  # the block in progress; a DC symbol starts the next
            last = list(dcs)
            started = nb
            b_end = subs[i][2]
            if started > todo or (started == todo and z == 0):
                break
            while pos < b_end:
                c = slots[slot]
                pos, nslot, z, ev = step(hdr, slots, streams[k], pos, slot, z)
                if pos > streams[k].nbits:
                    raise DecodeError(6)
                if ev[0] == "err":
                    raise DecodeError(ev[1])
                if ev[0] == "dc":
                    block, started = block + 1, started + 1
                    last[c] += ev[1]
                    _store(hdr, slots, coefs, block, 0, _int16(last[c]))
                elif ev[0] == "ac":
                    _store(hdr, slots, coefs, block, ev[1], ev[2])
                slot = nslot
                if z == 0 and started == todo:
                    _finish_segment(streams[k], pos)
                    done = True
                    break
            nb += res[i][1]
            dcs = [a + b for a, b in zip(dcs, res[i][2])]
            if done:
                break
        if not done:
            raise DecodeError(6)
    return coefs


# ------------------------------------------------------------------------------------------------------------ pixels
def idct_plane(coefs: np.ndarray, qt: np.ndarray) -> np.ndarray:
    """(rows, cols, 64) coefficients -> the component's samples, (8 rows, 8 cols)."""
    rows, cols = coefs.shape[:2]
    q = coefs.reshape(rows, cols, 8, 8).astype(np.int64)
    return JO.from_blocks(JO.idct_islow(q, qt.astype(np.int64)))


def upsample_h2v1(c: np.ndarray, W: int) -> np.ndarray:
    """h2v1_fancy_upsample of the (rows, cw) real samples -> (rows, W): (3 this + left + 1) >> 2 and (3 this + right +
    2) >> 2, the outer two outputs copied; a plane at most 2 samples wide is replicated."""
    cw = c.shape[1]
    if cw <= 2:
        return np.repeat(c, 2, axis=1)[:, :W]
    left = np.concatenate([c[:, :1], c[:, :-1]], axis=1)
    right = np.concatenate([c[:, 1:], c[:, -1:]], axis=1)
    out = np.empty((c.shape[0], 2 * cw), dtype=np.int64)
    out[:, 0::2] = (3 * c + left + 1) >> 2
    out[:, 1::2] = (3 * c + right + 2) >> 2
    out[:, 0], out[:, -1] = c[:, 0], c[:, -1]
    return out[:, :W]


def pixels(hdr: J.Header, coefs) -> np.ndarray:
    H, W = hdr.H, hdr.W
    planes = [idct_plane(p, hdr.qt[c[3]]) for p, c in zip(coefs, hdr.comps)]
    y = planes[0][:H, :W]
    if len(planes) == 1:
        return np.repeat(y[..., None], 3, axis=2).astype(np.uint8)
    h = hdr.comps[0][1:3]
    ch, cw = -(-H // h[1]), -(-W // h[0])
    if tuple(h) == (1, 1):
        cb, cr = (p[:H, :W] for p in planes[1:])
    elif tuple(h) == (2, 1):
        cb, cr = (upsample_h2v1(p[:ch, :cw], W) for p in planes[1:])
    else:
        cb, cr = (JO.upsample_chroma(p, H, W) for p in planes[1:])
    return JO.ycc_to_rgb(y, cb, cr)


def decode(data: bytes, S: int = 0) -> np.ndarray:
    """Image.open(f).convert("RGB") of an accepted file: the serial decode, or with S the synchronised one."""
    hdr = J.parse(data)
    coefs = decode_sync(hdr, data, S) if S else decode_serial(hdr, data)
    return pixels(hdr, coefs)


# ------------------------------------------------------------------------------------------------------------ fixtures
SUBSAMPLINGS = ("4:4:4", "4:2:2", "4:2:0", "L")
SAMPLINGS_OF = {"4:4:4": (1, 1), "4:2:2": (2, 1), "4:2:0": (2, 2)}      # luma (h, v) Pillow writes
QUALITIES = (1, 10, 50, 75, 95, 100)
SIZES = ((1, 1), (1, 17), (7, 13), (8, 8), (15, 16), (16, 17), (31, 33), (127, 255), (375, 500), (500, 375), (8, 2048),
         (2048, 8), (1024, 1024))
OPTIONS = ({}, {"optimize": True}, {"restart_marker_blocks": 3}, {"restart_marker_rows": 1},
           {"exif": b"Exif\0\0" + bytes(range(40)), "comment": "a comment"}, {"icc_profile": bytes(200) + b"icc"},
           {"qtables": [list(range(1, 65)), [17] * 64]}, {"optimize": True, "restart_marker_blocks": 1})


def fixture(H: int, W: int, sub: str, quality: int, kind: str, seed: int, **opts) -> bytes:
    """A seeded JPEG file as Pillow writes it: jpeg_oracle.content(kind) saved with this subsampling ("L": grayscale),
    quality and keyword options (qtables replace the quality)."""
    from io import BytesIO
    from PIL import Image
    im = Image.fromarray(JO.content(kind, H, W, seed))
    kw = dict(opts)
    if "qtables" not in kw:
        kw["quality"] = quality
    if sub == "L":
        im = im.convert("L")
    else:
        kw["subsampling"] = sub
    f = BytesIO()
    im.save(f, "JPEG", **kw)
    return f.getvalue()


def matrix(sizes=SIZES, seed: int = 7):
    """(H, W, subsampling, quality, kind, seed, options) cases: every size, with subsampling, quality, content kind and
    options cycling so that every value of each appears at several sizes."""
    cases = []
    i = 0
    for H, W in sizes:
        for j in range(4):
            cases.append((H, W, SUBSAMPLINGS[(i + j) % 4], QUALITIES[i % len(QUALITIES)], JO.KINDS[i % len(JO.KINDS)],
                          seed + i, OPTIONS[i % len(OPTIONS)]))
            i += 1
    return cases


def pillow_rgb(data: bytes) -> np.ndarray:
    from io import BytesIO
    from PIL import Image
    return np.asarray(Image.open(BytesIO(data)).convert("RGB"))
