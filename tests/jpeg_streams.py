"""Test-only baseline JPEG writer: builds a stream from chosen quantised coefficient blocks, DQT / DHT tables, table slots,
restart interval and sampling, with control over the bytes of the entropy-coded segment (fill bytes before a restart
marker shift every later byte, so a stuffed FF 00 or an RSTn can be put on a chosen offset of the scan).  Pillow decodes
every stream built here, so Pillow is the reference for each; a stream Pillow refuses expects "Pillow raises".

A stream is described by `Spec` (width, height, components, tables, coefficients in zig-zag order) and written by
`encode`.  The sync-limit streams of `sync_stream` are derived in its docstring."""
import struct
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np

# zig-zag index -> natural index (F3R_JPEG_NATURAL)
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7,
                   14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39,
                   46, 53, 60, 61, 54, 47, 55, 62, 63])

DC_SYMBOLS = list(range(12))
AC_SYMBOLS = [0x00, 0xF0] + [(r << 4) | s for s in range(1, 11) for r in range(16)]


@dataclass
class Huff:
    """A DHT table: counts[l] codes of length l + 1, symbols in code order."""
    counts: List[int]
    symbols: List[int]

    def codes(self) -> Dict[int, Tuple[int, int]]:
        out, code, k = {}, 0, 0
        for ln in range(1, 17):
            for _ in range(self.counts[ln - 1]):
                out.setdefault(self.symbols[k], (code, ln))
                code += 1
                k += 1
            code <<= 1
        return out


def huff(symbols, min_len=1, max_len=16, fixed=None) -> Huff:
    """Canonical table for `symbols` (shortest codes first), lengths >= min_len, never the all-ones code: each symbol takes
    the shortest length that leaves room for the rest at max_len.  fixed=L gives every symbol an L-bit code."""
    counts = [0] * 16
    if fixed:
        assert len(symbols) < (1 << fixed)
        counts[fixed - 1] = len(symbols)
        return Huff(counts, list(symbols))
    room, ln, n = 1 << 16, min_len, len(symbols)  # code space in units of 2^-16
    for i in range(n):
        while room - (1 << (16 - ln)) < (n - i - 1) * (1 << (16 - max_len)) + 1:
            ln += 1
        assert ln <= max_len, "symbols do not fit"
        counts[ln - 1] += 1
        room -= 1 << (16 - ln)
    return Huff(counts, list(symbols))


@dataclass
class Comp:
    h: int = 1
    v: int = 1
    tq: int = 0
    td: int = 0
    ta: int = 0
    cid: int = 0


@dataclass
class Spec:
    width: int
    height: int
    comps: List[Comp]
    qt: Dict[int, np.ndarray]              # slot -> 64 values, natural order
    dc: Dict[int, Huff]
    ac: Dict[int, Huff]
    coef: List[np.ndarray]                 # per component [bh][bw][64] zig-zag order
    dri: int = 0
    qt16: bool = False
    fill: Dict[int, int] = field(default_factory=dict)  # restart marker index -> fill bytes before it
    pad_ones: bool = True                  # pad each segment with one bits (libjpeg's encoder does)
    extra_dht: bytes = b""                 # raw DHT payloads written before the used tables
    orientation: int = 0                   # EXIF orientation (0: no EXIF segment)


def blocks_shape(spec: Spec, c: int) -> Tuple[int, int]:
    hmax = max(k.h for k in spec.comps)
    vmax = max(k.v for k in spec.comps)
    if len(spec.comps) == 1:
        return (spec.height + 7) // 8, (spec.width + 7) // 8
    mcux, mcuy = -(-spec.width // (8 * hmax)), -(-spec.height // (8 * vmax))
    return mcuy * spec.comps[c].v, mcux * spec.comps[c].h


def mcu_count(spec: Spec) -> Tuple[int, int]:
    if len(spec.comps) == 1:
        return (spec.width + 7) // 8, (spec.height + 7) // 8
    hmax = max(k.h for k in spec.comps)
    vmax = max(k.v for k in spec.comps)
    return -(-spec.width // (8 * hmax)), -(-spec.height // (8 * vmax))


class _Bits:
    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def put(self, v, n):
        for i in range(n - 1, -1, -1):
            self.acc = (self.acc << 1) | ((v >> i) & 1)
            self.n += 1
            if self.n == 8:
                self.out.append(self.acc)
                if self.acc == 0xFF:
                    self.out.append(0)
                self.acc, self.n = 0, 0

    def flush(self, ones=True):
        if self.n:
            self.put((1 << (8 - self.n)) - 1 if ones else 0, 8 - self.n)


def _category(v):
    return 0 if v == 0 else int(abs(int(v))).bit_length()


def _bits(v, s):
    return v if v >= 0 else v + (1 << s) - 1


def scan_bytes(spec: Spec) -> bytes:
    """The entropy-coded segment (stuffed, with RSTn markers and the requested fill bytes), without EOI."""
    mcux, mcuy = mcu_count(spec)
    mcus = mcux * mcuy
    ri = spec.dri or mcus
    dct = {k: v.codes() for k, v in spec.dc.items()}
    act = {k: v.codes() for k, v in spec.ac.items()}
    out, bw, rst = bytearray(), _Bits(), 0
    pred = [0, 0, 0]
    gray = len(spec.comps) == 1
    for m in range(mcus):
        if m and m % ri == 0:
            bw.flush(spec.pad_ones)
            out += bw.out
            out += b"\xFF" * spec.fill.get(rst, 0) + bytes([0xFF, 0xD0 + (rst & 7)])
            bw, rst, pred = _Bits(), rst + 1, [0, 0, 0]
        mx, my = m % mcux, m // mcux
        for c, k in enumerate(spec.comps):
            hh, vv = (1, 1) if gray else (k.h, k.v)
            for dy in range(vv):
                for dx in range(hh):
                    blk = spec.coef[c][my * vv + dy, mx * hh + dx]
                    diff = int(blk[0]) - pred[c]
                    pred[c] = int(blk[0])
                    s = _category(diff)
                    code, ln = dct[k.td][s]
                    bw.put(code, ln)
                    bw.put(_bits(diff, s), s)
                    run = 0
                    last = max([z for z in range(1, 64) if blk[z]] + [0])
                    for z in range(1, last + 1):
                        if blk[z] == 0:
                            run += 1
                            continue
                        while run > 15:
                            bw.put(*act[k.ta][0xF0])
                            run -= 16
                        s = _category(blk[z])
                        bw.put(*act[k.ta][(run << 4) | s])
                        bw.put(_bits(int(blk[z]), s), s)
                        run = 0
                    if last < 63:
                        bw.put(*act[k.ta][0x00])
    bw.flush(spec.pad_ones)
    out += bw.out
    return bytes(out)


def _seg(marker, payload):
    return struct.pack(">BBH", 0xFF, marker, len(payload) + 2) + payload


def dht_payload(tc, th, t: Huff) -> bytes:
    return bytes([(tc << 4) | th] + list(t.counts) + list(t.symbols))


def encode(spec: Spec, scan: Optional[bytes] = None) -> bytes:
    """JFIF stream of `spec` (or of `spec`'s headers around a given entropy-coded segment)."""
    out = bytearray(b"\xFF\xD8")
    out += _seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    if spec.orientation:  # little-endian TIFF, IFD0 with the one entry 0x0112 (SHORT)
        tiff = b"II*\x00" + struct.pack("<I", 8) + struct.pack("<H", 1) + struct.pack("<HHIHH", 0x0112, 3, 1,
                                                                                    spec.orientation, 0)
        out += _seg(0xE1, b"Exif\x00\x00" + tiff + struct.pack("<I", 0))
    for slot in sorted(spec.qt):
        q = np.asarray(spec.qt[slot]).reshape(64)[ZIGZAG]
        if spec.qt16:
            out += _seg(0xDB, bytes([0x10 | slot]) + b"".join(struct.pack(">H", int(v)) for v in q))
        else:
            out += _seg(0xDB, bytes([slot] + [int(v) for v in q]))
    ncomp = len(spec.comps)
    sof = struct.pack(">BHHB", 8, spec.height, spec.width, ncomp)
    for i, k in enumerate(spec.comps):
        sof += bytes([k.cid or i + 1, (k.h << 4) | k.v, k.tq])
    out += _seg(0xC0, sof)
    if spec.extra_dht:
        out += _seg(0xC4, spec.extra_dht)
    for th in sorted(spec.dc):
        out += _seg(0xC4, dht_payload(0, th, spec.dc[th]))
    for th in sorted(spec.ac):
        out += _seg(0xC4, dht_payload(1, th, spec.ac[th]))
    if spec.dri:
        out += _seg(0xDD, struct.pack(">H", spec.dri))
    sos = bytes([ncomp])
    for i, k in enumerate(spec.comps):
        sos += bytes([k.cid or i + 1, (k.td << 4) | k.ta])
    out += _seg(0xDA, sos + b"\x00\x3F\x00")
    out += scan if scan is not None else scan_bytes(spec)
    out += b"\xFF\xD9"
    return bytes(out)


def scan_offset(data: bytes) -> int:
    """First byte of the entropy-coded segment (after the SOS header)."""
    p = data.index(b"\xFF\xDA")
    return p + 2 + (data[p + 2] << 8 | data[p + 3])


# ---------------------------------------------------------------------------------------------------- coefficient content
def random_coef(spec_shape, rng, extreme=False, density=0.3):
    """[bh][bw][64] zig-zag blocks of small random values at `density`.  extreme=True (with unit quantisers): DC values
    alternating near +-600, so the differences are of category 11, one AC value of category 10 at a random z, a zero run
    longer than 16 (ZRL) before it, and +-1 at z = 63 (no EOB).  Dequantised values stay inside the range of 8-bit
    samples: libjpeg-turbo's SIMD IDCT is exact only there."""
    bh, bw = spec_shape
    c = np.zeros((bh, bw, 64), np.int32)
    if extreme:
        sign = np.where((np.arange(bh)[:, None] + np.arange(bw)[None, :]) % 2 == 0, 1, -1)
        c[..., 0] = sign * rng.integers(540, 700, (bh, bw))
        z = rng.integers(20, 62, (bh, bw))
        np.put_along_axis(c, z[..., None], (rng.choice([-1, 1], (bh, bw)) * rng.integers(512, 700, (bh, bw)))[..., None], 2)
        c[..., 63] = rng.choice([-1, 1], (bh, bw))
        return c
    c[..., 0] = rng.integers(-60, 61, (bh, bw))
    mask = rng.random((bh, bw, 63)) < density
    mag = rng.integers(1, 16, (bh, bw, 63))
    c[..., 1:] = np.where(mask, mag * rng.choice([-1, 1], (bh, bw, 63)), 0)
    return c


def qtable(rng, lo=1, hi=16):
    return rng.integers(lo, hi + 1, 64)


def make_spec(width, height, sampling="420", rng=None, dri=0, tables="long", slots="pillow", qt16=False, extreme=False,
              density=0.3, **kw) -> Spec:
    """A stream of random coefficients.  sampling: gray / 444 / 422 / 420.  tables: "long" (all 162 AC symbols, codes up to
    16 bits, most of them longer than the 9-bit LUT) or "short" (every code <= 9 bits).  slots: "pillow" (luma DC/AC 0,
    chroma 1, quant 0 / 1), "zero" (chroma on DC/AC table 0), "swap" (luma on tables 1, chroma on 0) or "q23" (quant
    slots 2 and 3).  qt16: 16-bit DQT entries.  extreme: see random_coef."""
    rng = rng if rng is not None else np.random.default_rng(0)
    hv = dict(gray=(1, 1), s444=(1, 1), s422=(2, 1), s420=(2, 2))["s" + sampling if sampling != "gray" else "gray"]
    n = 1 if sampling == "gray" else 3
    t0, t1 = (0, 1) if slots in ("pillow", "q23") else (0, 0) if slots == "zero" else (1, 0)
    q0, q1 = (2, 3) if slots == "q23" else (0, 1)
    comps = [Comp(hv[0], hv[1], q0, t0, t0)] + [Comp(1, 1, q1, t1, t1) for _ in range(n - 1)]
    mk = (lambda s: huff(s, max_len=9)) if tables == "short" else (lambda s: huff(s, min_len=2))
    dc = {0: mk(DC_SYMBOLS), 1: mk(DC_SYMBOLS[::-1])}
    ac = {0: mk(AC_SYMBOLS), 1: mk(AC_SYMBOLS[:2] + AC_SYMBOLS[2:][::-1])}
    qt = {q0: qtable(rng, 1, 40), q1: qtable(rng, 1, 60)}
    if extreme:
        qt = {q0: np.ones(64, np.int64), q1: np.ones(64, np.int64)}
    spec = Spec(width, height, comps, qt, dc, ac, [], dri=dri, qt16=qt16, **kw)
    for c in range(n):
        spec.coef.append(random_coef(blocks_shape(spec, c), rng, extreme, density))
    if n == 1:
        spec.dc, spec.ac = {t0: dc[t0]}, {t0: ac[t0]}
    return spec


# ----------------------------------------------------------------------------------------------------- sync-limit streams
SUB_BITS, SYNC_THREADS, MAX_ROUNDS = 1024, 128, 12  # jpeg.cu:36-38
SYNC_BLOCK_BITS = 8 + 63 * 9                        # one block of sync_stream: 575 bits


def sync_stream(ctas: int) -> bytes:
    """A 4:4:4 stream whose decode needs exactly `ctas` grid-wide sync rounds, because no guessed start is ever right.

    Every block is the 8-bit DC code 0x00 (difference 0) followed by 63 AC coefficients of +1, each the 8-bit code 0x80 and
    one value bit 1, so no EOB (z = 63 ends the block): 575 bits.  The bit pattern after the DC code is (100000001)*, which
    never holds eight zeros in a row, so the DC table decodes only at a true block start and a guessed start anywhere else
    ends in ST_ERR (jpeg.cu:170).  At a true block start a guess (block 0 of the MCU, z = 0) is right only at an MCU start:
    MCUs are 3 x 575 = 1725 bits, and 1024 i is a multiple of 1725 only for i a multiple of 1725, so with fewer than 1725
    subsequences thread 0 is the only right guess.  A wrong block index never corrects itself (every block decodes the
    same way), and a wrong start ending in ST_ERR restarts the next thread at its own wrong guess.

    So (jpeg.cu:333-373): round 0 decodes CTA 0 exactly (thread 0 starts at the true state and the block-local iterations
    carry it to thread 127); round r makes CTA r exact, its thread 0 reading the end state CTA r - 1 wrote in round r - 1;
    each of these rounds changes an end state of CTA r, so changed[r] = 1 for r < ctas, and round `ctas` changes nothing.
    The finish rule (jpeg.cu:467) reports F3R_JPEG_ERR_SYNC when changed[MAX_ROUNDS - 1] is set: a stream of
    ctas <= MAX_ROUNDS - 1 = 11 CTAs decodes with status 0; at exactly MAX_ROUNDS CTAs the last round completes the decode
    but changed an end state, so the status reports SYNC (the rule cannot tell a last change from a missing one); above it
    the decode has not converged and the status must report SYNC.  The stream is sized to put its last subsequence in the
    middle of CTA ctas - 1, and stays below 1725 subsequences (ctas <= 13)."""
    assert 1 <= ctas <= 13
    nsub_target = SYNC_THREADS * (ctas - 1) + SYNC_THREADS // 2
    mcus = max(1, nsub_target * SUB_BITS // (3 * SYNC_BLOCK_BITS))
    mcux = 32
    mcuy = -(-mcus // mcux)
    # DC: one 8-bit code 0x00 -> 0.  AC: the 1-bit code 0 -> EOB (never coded) and the 8-bit code 0x80 -> 0x01.
    spec = Spec(8 * mcux, 8 * mcuy, [Comp(1, 1, 0, 0, 0), Comp(1, 1, 0, 0, 0), Comp(1, 1, 0, 0, 0)],
                {0: np.full(64, 2)}, {0: Huff([0] * 7 + [1] + [0] * 8, [0])},
                {0: Huff([1] + [0] * 6 + [1] + [0] * 8, [0x00, 0x01])}, [])
    for c in range(3):
        blk = np.zeros((mcuy, mcux, 64), np.int32)
        blk[..., 1:] = 1
        spec.coef.append(blk)
    return encode(spec)
