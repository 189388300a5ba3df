"""Launch keys of image ingest, for the tests: which code runs for a call of the baseline-JPEG decode (f3r_jpeg_decode,
fast3r_b200/csrc/jpeg.cu) and of the resize / crop / normalise (f3r_ingest_rgb8, fast3r_b200/csrc/ingest.cu), and the
table of GPU cases that tests/test_ingest_plans_gpu.py runs and tests/test_ingest_plans_cpu.py checks the callers
(load_images, decode_jpeg, ingest_rgb8) against.

A decode call is described by its stream bytes and (orientation, rotate, crop); an ingest call by the arguments
ingest_rgb8 passes to the library.  Each key function cites the lines it restates."""
import struct

import numpy as np

# jpeg.cu:36-39
SUB_BITS, SYNC_THREADS, MAX_ROUNDS = 1024, 128, 12
UNSTUFF_BYTES, UNSTUFF_CHUNK = 16, 4096
LUT_BITS = 9  # jpeg_parse.h:18
# ingest.cu:18-19, 29, 92
ING_COLS, ING_ROWS, ING_ROWS_PER_BLOCK, ING_SMEM_CAP = 64, 8, 32, 200 * 1024


def _flags(*pairs):
    return "".join(" " + f for f, on in pairs if on)


# ------------------------------------------------------------------------------------------------------------- decode
def parse_headers(data: bytes) -> dict:
    """The header facts the decode's branches read: SOF geometry and sampling, DQT precisions, the longest code of each
    DHT slot, DRI, the SOS table slots and the scan's byte range (the layout jpeg_parse.h reads)."""
    p, out = 2, dict(qt16=False, maxlen={}, dri=0, orientation_exif=False)
    while True:
        while data[p] != 0xFF:
            p += 1
        while data[p] == 0xFF:
            p += 1
        m = data[p]
        p += 1
        if m in (0xD8, 0x01) or 0xD0 <= m <= 0xD7:
            continue
        ln = data[p] << 8 | data[p + 1]
        s = data[p + 2:p + ln]
        if m in (0xC0, 0xC1):
            out["height"], out["width"], n = struct.unpack(">HHB", s[1:6])
            out["comps"] = [(s[7 + 3 * c] >> 4, s[7 + 3 * c] & 15, s[8 + 3 * c]) for c in range(n)]
        elif m == 0xDB:
            q = 0
            while q < len(s):
                out["qt16"] |= bool(s[q] >> 4)
                q += 1 + 64 * ((s[q] >> 4) + 1)
        elif m == 0xC4:
            q = 0
            while q < len(s):
                counts = list(s[q + 1:q + 17])
                out["maxlen"][(s[q] >> 4, s[q] & 15)] = max([i + 1 for i in range(16) if counts[i]] + [0])
                q += 17 + sum(counts)
        elif m == 0xDD:
            out["dri"] = s[0] << 8 | s[1]
        elif m == 0xE1 and s[:6] == b"Exif\x00\x00":
            out["orientation_exif"] = True
        elif m == 0xDA:
            out["slots"] = [(s[2 + 2 * i] >> 4, s[2 + 2 * i] & 15) for i in range(s[0])]
            start = p + ln
            end = data.rindex(b"\xFF\xD9")
            out["scan"] = data[start:end]
            return out
        p += ln


def scan_markers(scan: bytes):
    """(stuffed FF positions, RST FF positions, fill bytes, unstuffed segment starts) of an entropy-coded segment."""
    stuffed, rst, fill, seg, kept = [], [], 0, [], 0
    i = 0
    while i < len(scan):
        if scan[i] != 0xFF:
            kept += 1
            i += 1
            continue
        r = i + 1
        while scan[r] == 0xFF:
            r += 1
        fill += r - i - 1
        if scan[r] == 0:
            stuffed.append(r - 1)
            kept += 1
        else:
            rst.append(r - 1)
            seg.append(kept)
        i = r + 1
    return stuffed, rst, fill, seg, kept


def decode_key(data: bytes, orientation: int, rotate: bool, left: int, top: int, out_w: int, out_h: int) -> str:
    """jpeg.cu:546-622 for a call of f3r_jpeg_decode and the kernels it launches:
      sampling   gray / 444 / 422 / 420 (jpeg_parse.h:183-201: the MCU layout run() walks, jpeg.cu:177-181)
      edge_r/b   a partial MCU at the right / bottom edge (padding blocks decoded, not stored)
      cw2        chroma width <= 2 (jpeg_math.h upsample: the box branch)
      ri_*       restart interval none / divides the MCU count / does not / 1 (jpeg.cu:146-163, 148)
      chunks     more than one 4096-byte unstuff chunk (jpeg.cu:234-323); ff_span / ff_chunk: a stuffed FF or an RST's
                 FF on the last byte of a 16-byte thread span / 4096-byte chunk, so prev / next cross it (:225-231)
      fill       fill bytes before a marker (:229-230)
      cta1/2/n   subsequences in 1, 2 or more sync CTAs (:603); seg_sub: a restart segment starts on a 1024-bit
                 subsequence boundary (:146, :161 reset on the boundary)
      lutmiss    a slot the scan uses has codes longer than the 9-bit LUT (:101-107)
      slots      chroma on DC/AC table 0, luma on table 1, or quant slots 2 / 3 (:169, :187, :434, :568)
      dqt16      16-bit DQT entries (jpeg_parse.h:125)
      o<k>/rot/crop  the orientation map class (jpeg_math.h:123-145; crop: the box is smaller than the oriented image,
                 jpeg.cu:558-562), wrap: out_w > 256 and not a multiple of 256
                 (jpeg.cu:617: a partial last 256-pixel block)"""
    h = parse_headers(data)
    w, ht, comps = h["width"], h["height"], h["comps"]
    if len(comps) == 1:
        samp, hm, vm = "gray", 1, 1
    else:
        hm, vm = comps[0][0], comps[0][1]
        samp = {(1, 1): "444", (2, 1): "422", (2, 2): "420"}[(hm, vm)]
    mcux, mcuy = -(-w // (8 * hm)), -(-ht // (8 * vm))
    mcus = mcux * mcuy
    w2, h2 = (ht, w) if orientation >= 5 else (w, ht)
    w2, h2 = (h2, w2) if rotate else (w2, h2)
    crop = (left, top, out_w, out_h) != (0, 0, w2, h2)
    ri = h["dri"]
    rik = "ri_none" if ri == 0 else "ri_1" if ri == 1 else "ri_div" if mcus % ri == 0 else "ri_nodiv"
    stuffed, rst, fill, seg, kept = scan_markers(h["scan"])
    marks = stuffed + rst
    nsub = -(-len(h["scan"]) * 8 // SUB_BITS)
    ctas = -(-nsub // SYNC_THREADS)
    used = {(0, td) for td, _ in h["slots"]} | {(1, ta) for _, ta in h["slots"]}
    tq = [c[2] for c in comps]
    pillow_slots = [(0, 0)] + [(1, 1)] * (len(comps) - 1)
    nondefault = h["slots"] != pillow_slots or any(t > 1 for t in tq) or (len(comps) == 3 and tq != [0, 1, 1])
    return (f"decode {samp}" + _flags(
        ("edge_r", w % (8 * hm) != 0), ("edge_b", ht % (8 * vm) != 0),
        ("cw2", len(comps) == 3 and -(-w // hm) <= 2), ("chunks", len(h["scan"]) > UNSTUFF_CHUNK),
        ("ff_span", any(m % UNSTUFF_BYTES == UNSTUFF_BYTES - 1 for m in marks)),
        ("ff_chunk", any(m % UNSTUFF_CHUNK == UNSTUFF_CHUNK - 1 for m in marks)), ("fill", fill > 0),
        ("cta1", ctas == 1), ("cta2", ctas == 2), ("ctan", ctas > 2),
        ("seg_sub", any(s * 8 % SUB_BITS == 0 for s in seg)),
        ("lutmiss", any(h["maxlen"].get(k, 0) > LUT_BITS for k in used)), ("slots", nondefault),
        ("dqt16", h["qt16"]), ("rot", rotate), ("crop", crop), ("wrap", out_w > 256 and out_w % 256 != 0))
        + f" {rik} o{orientation}")


def decode_axes(key: str):
    return set(key.split()[1:])


# ------------------------------------------------------------------------------------------------------------- ingest
def h_smem(hks, span):
    """ingest.cu:147-149 (resize_h_kernel's dynamic shared memory)."""
    return hks * ING_COLS * 4 + ING_ROWS * (((span * 3 + 3) & ~3) + 4)


def ingest_key(d) -> str:
    """ingest.cu:152-170 for a call of f3r_ingest_rgb8 (d: h, w, oh, ow, filt, hks, span, left, top, cw, ch, size,
    square_ok):
      lanczos / bicubic / copy   the filter of the taps; copy: no tap tables (the image already has the size)
      h / v               horizontal pass (hk given, :155) / vertical taps (vk given, :124)
      smem48 / optin / direct   resize_h_kernel with <= 48 KB, with opt-in shared memory, or resize_h_direct_kernel
                          above ING_SMEM_CAP (:156-163)
      cb1 / cbpart        one column block / a partial last column block (:38)
      rowstep / rowblk    a partial 8-row step / a partial 32-row block (:49-53)
      lastword            the image's last word is assembled from bytes ((h w 3) mod 4 != 0, :63-67)
      ph<k>               the source phases b0 & 3 the horizontal pass meets (w mod 4 fixes the cycle of 3 w y mod 4)
      crop_l / crop_t     crop offsets (:122)
      cw256               cw a multiple of 256 (no partial block in the vertical pass)
      s224 / sq           size 224 / square_ok"""
    h, w, oh, ow = d["h"], d["w"], d["oh"], d["ow"]
    hp, vp = ow != w, oh != h
    k = "ingest " + ("lanczos" if d["filt"] == 1 else "bicubic" if hp or vp else "copy")
    if hp:
        sm = h_smem(d["hks"], d["span"])
        k += " h " + ("direct" if sm > ING_SMEM_CAP else "optin" if sm > 48 * 1024 else "smem48")
        if sm <= ING_SMEM_CAP:
            k += _flags(("cb1", ow <= ING_COLS), ("cbpart", ow % ING_COLS != 0), ("rowstep", h % ING_ROWS != 0),
                        ("rowblk", h % ING_ROWS_PER_BLOCK != 0))
        k += _flags(("lastword", (h * w * 3) % 4 != 0)) + f" ph{w % 4}"
    k += _flags(("v", vp), ("crop_l", d["left"] > 0), ("crop_t", d["top"] > 0), ("cw256", d["cw"] % 256 == 0),
                ("s224", d["size"] == 224), ("sq", d["square_ok"]))
    return k


# ---------------------------------------------------------------------------------------------------- the case table
# Decode cases: a stream recipe (built by tests/jpeg_streams.py or Pillow's encoder, see test_ingest_plans_gpu.build)
# and (orientation, rotate, crop).  recipe = (kind, args); kind "pil": Pillow-encoded photo (w, h, quality, subsampling,
# restart rows); "spec": jpeg_streams.make_spec(w, h, sampling, seed, **kw); "sync": jpeg_streams.sync_stream(ctas).
def _dec(name, recipe, orientation=1, rot=False, crop=False, status=0):
    return dict(name=name, op="decode", recipe=recipe, orientation=orientation, rot=rot, crop=crop, status=status)


def _ing(name, h, w, size=512, square_ok=False, offset=0):
    return dict(name=name, op="ingest", h=h, w=w, size=size, square_ok=square_ok, offset=offset)


DECODE = [
    # ---- the callers' geometries: phone photos stored 4032 x 3024 or 3024 x 4032, EXIF 1 / 6 / 8
    _dec("photo_4032x3024_q90_420_o1", ("pil", (4032, 3024, 90, 2, 0))),
    _dec("photo_4032x3024_q90_420_o6", ("pil", (4032, 3024, 90, 2, 0)), orientation=6),
    _dec("photo_4032x3024_q90_422_o8", ("pil", (4032, 3024, 90, 1, 0)), orientation=8),
    _dec("photo_3024x4032_q90_420_o6_rot_crop", ("pil", (3024, 4032, 90, 2, 0)), orientation=6, rot=True, crop=True),
    _dec("photo_4000x3000_q90_420_rst", ("pil", (4000, 3000, 90, 2, 4))),
    _dec("photo_1920x1080_q90_422_crop", ("pil", (1920, 1080, 90, 1, 0)), crop=True),
    _dec("photo_1080x1920_q90_420_o3_rot", ("pil", (1080, 1920, 90, 2, 0)), orientation=3, rot=True),
]
# ---- the contract: every sampling x table shape x slots, restart intervals, extreme categories, 16-bit DQT, tiny images,
# the orientation classes, byte placement and the sync limit
_SEED = 0
for _samp in ("gray", "444", "422", "420"):
    for _tab, _slots in (("long", "pillow"), ("short", "zero"), ("long", "swap"), ("short", "q23")):
        _SEED += 1
        DECODE.append(_dec(f"spec_{_samp}_{_tab}_{_slots}_77x45", ("spec", (77, 45, _samp, _SEED, dict(tables=_tab,
                                                                                                      slots=_slots)))))
    for _ri in (1, 3, 5):
        _SEED += 1
        DECODE.append(_dec(f"spec_{_samp}_ri{_ri}_61x37", ("spec", (61, 37, _samp, _SEED, dict(dri=_ri)))))
    _SEED += 1
    DECODE.append(_dec(f"spec_{_samp}_extreme_dqt16_40x24", ("spec", (40, 24, _samp, _SEED, dict(extreme=True, qt16=True)))))
    for _w, _h in ((1, 1), (2, 2), (3, 5), (8, 8), (2, 9), (17, 3)):
        _SEED += 1
        DECODE.append(_dec(f"spec_{_samp}_{_w}x{_h}", ("spec", (_w, _h, _samp, _SEED, {}))))
for _o in range(1, 9):
    for _rot, _crop in ((False, False), (True, True), (True, False), (False, True)):
        DECODE.append(_dec(f"orient_o{_o}_rot{int(_rot)}_crop{int(_crop)}_600x331",
                           ("spec", (600, 331, "420", 100 + _o, dict(density=0.05))), _o, _rot, _crop))
DECODE += [
    _dec("place_ff00_span_gray", ("place", ("ff00", UNSTUFF_BYTES, "gray", 201))),
    _dec("place_rst_span_420", ("place", ("rst", UNSTUFF_BYTES, "420", 202))),
    _dec("place_ff00_chunk_444", ("place", ("ff00", UNSTUFF_CHUNK, "444", 203))),
    _dec("place_rst_chunk_420", ("place", ("rst", UNSTUFF_CHUNK, "420", 204))),
    _dec("segsub_420_ri1", ("segsub", ("420", 205))),
    _dec("sync_ctas1", ("sync", 1)),
    _dec("sync_ctas2", ("sync", 2)),
    _dec("sync_ctas11_below_limit", ("sync", MAX_ROUNDS - 1)),
    _dec("sync_ctas12_at_limit", ("sync", MAX_ROUNDS), status=1),
    _dec("sync_ctas13_above_limit", ("sync", MAX_ROUNDS + 1), status=1),
]

INGEST = [_ing("call_3024x3024_512_sq", 3024, 3024, 512, True)]
# ---- the callers' geometries: load_images at 512 and 224 on photos both ways (bench.py ingests 4032 x 3024 at 512),
# 16:9 both ways and the 4:3 crops of a 16:9 frame and of a rotated portrait photo
for _w, _h in ((4032, 3024), (3024, 4032), (4000, 3000), (1920, 1080), (1080, 1920), (1440, 1080), (3024, 2268)):
    for _size in (512, 224):
        INGEST.append(_ing(f"call_{_w}x{_h}_{_size}", _h, _w, _size))
for _w, _h in ((1, 1), (2, 1), (1, 2), (3, 3), (5, 7), (8, 8), (7, 4), (6, 2)):
    for _size in (512, 224):
        INGEST.append(_ing(f"tiny_{_w}x{_h}_{_size}", _h, _w, _size))
for _w, _h in ((513, 200), (200, 513), (513, 384), (512, 513), (1027, 33), (1026, 61), (1025, 47), (1024, 1029),
               (640, 481), (700, 29), (64, 600), (5000, 170), (200, 4097), (2000, 350), (1000, 1000)):
    for _size, _sq in ((512, False), (224, False), (512, True)):
        INGEST.append(_ing(f"mat_{_w}x{_h}_{_size}" + ("_sq" if _sq else ""), _h, _w, _size, _sq))
INGEST += [
    # panoramas on both sides of ING_SMEM_CAP at size 512 (cap at a landscape width of 32 770 px)
    _ing("pano_32000x1000", 1000, 32000), _ing("pano_33000x1000", 1000, 33000), _ing("pano_40000x2000", 2000, 40000),
    _ing("pano_40000x2000_224", 2000, 40000, 224), _ing("pano_2000x40000", 40000, 2000),
    # images that already have the size: no tap tables, the crop / normalise only
    _ing("copy_512x384_512", 384, 512), _ing("copy_512x512_512_sq", 512, 512, 512, True),
    # row slices of an image whose width is not a multiple of 4: base off by 1..3 bytes (copied to an aligned base)
    _ing("offset1_501x301", 301, 501, offset=1), _ing("offset2_501x301", 301, 501, offset=2),
    _ing("offset3_333x201", 201, 333, offset=3),
]

CASES = DECODE + INGEST

# ---- the key each case is built to reach.  tests/test_ingest_plans_cpu.py runs every case through its real caller and
# fails when the key its call reaches differs from the one declared here.
DECLARED = {
    'photo_4032x3024_q90_420_o1': 'decode 420 chunks ff_span ff_chunk ctan lutmiss wrap ri_none o1',
    'photo_4032x3024_q90_420_o6': 'decode 420 chunks ff_span ff_chunk ctan lutmiss wrap ri_none o6',
    'photo_4032x3024_q90_422_o8': 'decode 422 chunks ff_span ff_chunk ctan lutmiss wrap ri_none o8',
    'photo_3024x4032_q90_420_o6_rot_crop': 'decode 420 chunks ff_span ff_chunk ctan lutmiss rot crop wrap ri_none o6',
    'photo_4000x3000_q90_420_rst': 'decode 420 edge_b chunks ff_span ff_chunk ctan lutmiss wrap ri_div o1',
    'photo_1920x1080_q90_422_crop': 'decode 422 chunks ff_span ff_chunk ctan lutmiss crop wrap ri_none o1',
    'photo_1080x1920_q90_420_o3_rot': 'decode 420 edge_r chunks ff_span ff_chunk ctan lutmiss rot wrap ri_none o3',
    'spec_gray_long_pillow_77x45': 'decode gray edge_r edge_b ff_span cta1 lutmiss ri_none o1',
    'spec_gray_short_zero_77x45': 'decode gray edge_r edge_b ff_span cta1 ri_none o1',
    'spec_gray_long_swap_77x45': 'decode gray edge_r edge_b ff_span cta1 lutmiss slots ri_none o1',
    'spec_gray_short_q23_77x45': 'decode gray edge_r edge_b ff_span cta1 slots ri_none o1',
    'spec_gray_ri1_61x37': 'decode gray edge_r edge_b ff_span cta1 lutmiss ri_1 o1',
    'spec_gray_ri3_61x37': 'decode gray edge_r edge_b ff_span cta1 lutmiss ri_nodiv o1',
    'spec_gray_ri5_61x37': 'decode gray edge_r edge_b ff_span cta1 lutmiss ri_div o1',
    'spec_gray_extreme_dqt16_40x24': 'decode gray cta1 lutmiss dqt16 ri_none o1',
    'spec_gray_1x1': 'decode gray edge_r edge_b cta1 lutmiss ri_none o1',
    'spec_gray_2x2': 'decode gray edge_r edge_b ff_span cta1 lutmiss ri_none o1',
    'spec_gray_3x5': 'decode gray edge_r edge_b cta1 lutmiss ri_none o1',
    'spec_gray_8x8': 'decode gray cta1 lutmiss ri_none o1',
    'spec_gray_2x9': 'decode gray edge_r edge_b cta1 lutmiss ri_none o1',
    'spec_gray_17x3': 'decode gray edge_r edge_b ff_span cta1 lutmiss ri_none o1',
    'spec_444_long_pillow_77x45': 'decode 444 edge_r edge_b chunks ff_span ff_chunk cta1 lutmiss ri_none o1',
    'spec_444_short_zero_77x45': 'decode 444 edge_r edge_b chunks ff_span cta1 slots ri_none o1',
    'spec_444_long_swap_77x45': 'decode 444 edge_r edge_b chunks ff_span ff_chunk cta1 lutmiss slots ri_none o1',
    'spec_444_short_q23_77x45': 'decode 444 edge_r edge_b chunks ff_span cta1 slots ri_none o1',
    'spec_444_ri1_61x37': 'decode 444 edge_r edge_b chunks ff_span cta1 seg_sub lutmiss ri_1 o1',
    'spec_444_ri3_61x37': 'decode 444 edge_r edge_b chunks ff_span cta1 lutmiss ri_nodiv o1',
    'spec_444_ri5_61x37': 'decode 444 edge_r edge_b chunks ff_span cta1 lutmiss ri_div o1',
    'spec_444_extreme_dqt16_40x24': 'decode 444 ff_span cta1 lutmiss dqt16 ri_none o1',
    'spec_444_1x1': 'decode 444 edge_r edge_b cw2 ff_span cta1 lutmiss ri_none o1',
    'spec_444_2x2': 'decode 444 edge_r edge_b cw2 ff_span cta1 lutmiss ri_none o1',
    'spec_444_3x5': 'decode 444 edge_r edge_b ff_span cta1 lutmiss ri_none o1',
    'spec_444_8x8': 'decode 444 ff_span cta1 lutmiss ri_none o1',
    'spec_444_2x9': 'decode 444 edge_r edge_b cw2 ff_span cta1 lutmiss ri_none o1',
    'spec_444_17x3': 'decode 444 edge_r edge_b ff_span cta1 lutmiss ri_none o1',
    'spec_422_long_pillow_77x45': 'decode 422 edge_r edge_b chunks ff_span cta1 lutmiss ri_none o1',
    'spec_422_short_zero_77x45': 'decode 422 edge_r edge_b cta1 slots ri_none o1',
    'spec_422_long_swap_77x45': 'decode 422 edge_r edge_b chunks ff_span cta1 lutmiss slots ri_none o1',
    'spec_422_short_q23_77x45': 'decode 422 edge_r edge_b ff_span cta1 slots ri_none o1',
    'spec_422_ri1_61x37': 'decode 422 edge_r edge_b chunks ff_span cta1 lutmiss ri_1 o1',
    'spec_422_ri3_61x37': 'decode 422 edge_r edge_b chunks ff_span cta1 lutmiss ri_nodiv o1',
    'spec_422_ri5_61x37': 'decode 422 edge_r edge_b chunks ff_span cta1 lutmiss ri_div o1',
    'spec_422_extreme_dqt16_40x24': 'decode 422 edge_r ff_span cta1 lutmiss dqt16 ri_none o1',
    'spec_422_1x1': 'decode 422 edge_r edge_b cw2 ff_span cta1 lutmiss ri_none o1',
    'spec_422_2x2': 'decode 422 edge_r edge_b cw2 ff_span cta1 lutmiss ri_none o1',
    'spec_422_3x5': 'decode 422 edge_r edge_b cw2 ff_span cta1 lutmiss ri_none o1',
    'spec_422_8x8': 'decode 422 edge_r ff_span cta1 lutmiss ri_none o1',
    'spec_422_2x9': 'decode 422 edge_r edge_b cw2 ff_span cta1 lutmiss ri_none o1',
    'spec_422_17x3': 'decode 422 edge_r edge_b ff_span cta1 lutmiss ri_none o1',
    'spec_420_long_pillow_77x45': 'decode 420 edge_r edge_b chunks ff_span cta1 lutmiss ri_none o1',
    'spec_420_short_zero_77x45': 'decode 420 edge_r edge_b ff_span cta1 slots ri_none o1',
    'spec_420_long_swap_77x45': 'decode 420 edge_r edge_b chunks ff_span cta1 lutmiss slots ri_none o1',
    'spec_420_short_q23_77x45': 'decode 420 edge_r edge_b ff_span cta1 slots ri_none o1',
    'spec_420_ri1_61x37': 'decode 420 edge_r edge_b ff_span cta1 lutmiss ri_1 o1',
    'spec_420_ri3_61x37': 'decode 420 edge_r edge_b ff_span cta1 lutmiss ri_div o1',
    'spec_420_ri5_61x37': 'decode 420 edge_r edge_b ff_span cta1 lutmiss ri_nodiv o1',
    'spec_420_extreme_dqt16_40x24': 'decode 420 edge_r edge_b ff_span cta1 lutmiss dqt16 ri_none o1',
    'spec_420_1x1': 'decode 420 edge_r edge_b cw2 ff_span cta1 lutmiss ri_none o1',
    'spec_420_2x2': 'decode 420 edge_r edge_b cw2 ff_span cta1 lutmiss ri_none o1',
    'spec_420_3x5': 'decode 420 edge_r edge_b cw2 ff_span cta1 lutmiss ri_none o1',
    'spec_420_8x8': 'decode 420 edge_r edge_b ff_span cta1 lutmiss ri_none o1',
    'spec_420_2x9': 'decode 420 edge_r edge_b cw2 ff_span cta1 lutmiss ri_none o1',
    'spec_420_17x3': 'decode 420 edge_r edge_b ff_span cta1 lutmiss ri_none o1',
    'orient_o1_rot0_crop0_600x331': 'decode 420 edge_r edge_b chunks ff_span ctan lutmiss wrap ri_none o1',
    'orient_o1_rot1_crop1_600x331': 'decode 420 edge_r edge_b chunks ff_span ctan lutmiss rot crop wrap ri_none o1',
    'orient_o1_rot1_crop0_600x331': 'decode 420 edge_r edge_b chunks ff_span ctan lutmiss rot wrap ri_none o1',
    'orient_o1_rot0_crop1_600x331': 'decode 420 edge_r edge_b chunks ff_span ctan lutmiss crop wrap ri_none o1',
    'orient_o2_rot0_crop0_600x331': 'decode 420 edge_r edge_b chunks ff_span ctan lutmiss wrap ri_none o2',
    'orient_o2_rot1_crop1_600x331': 'decode 420 edge_r edge_b chunks ff_span ctan lutmiss rot crop wrap ri_none o2',
    'orient_o2_rot1_crop0_600x331': 'decode 420 edge_r edge_b chunks ff_span ctan lutmiss rot wrap ri_none o2',
    'orient_o2_rot0_crop1_600x331': 'decode 420 edge_r edge_b chunks ff_span ctan lutmiss crop wrap ri_none o2',
    'orient_o3_rot0_crop0_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss wrap ri_none o3',
    'orient_o3_rot1_crop1_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss rot crop wrap ri_none o3',
    'orient_o3_rot1_crop0_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss rot wrap ri_none o3',
    'orient_o3_rot0_crop1_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss crop wrap ri_none o3',
    'orient_o4_rot0_crop0_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss wrap ri_none o4',
    'orient_o4_rot1_crop1_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss rot crop wrap ri_none o4',
    'orient_o4_rot1_crop0_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss rot wrap ri_none o4',
    'orient_o4_rot0_crop1_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss crop wrap ri_none o4',
    'orient_o5_rot0_crop0_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss wrap ri_none o5',
    'orient_o5_rot1_crop1_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss rot crop wrap ri_none o5',
    'orient_o5_rot1_crop0_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss rot wrap ri_none o5',
    'orient_o5_rot0_crop1_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss crop wrap ri_none o5',
    'orient_o6_rot0_crop0_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss wrap ri_none o6',
    'orient_o6_rot1_crop1_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss rot crop wrap ri_none o6',
    'orient_o6_rot1_crop0_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss rot wrap ri_none o6',
    'orient_o6_rot0_crop1_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss crop wrap ri_none o6',
    'orient_o7_rot0_crop0_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss wrap ri_none o7',
    'orient_o7_rot1_crop1_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss rot crop wrap ri_none o7',
    'orient_o7_rot1_crop0_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss rot wrap ri_none o7',
    'orient_o7_rot0_crop1_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss crop wrap ri_none o7',
    'orient_o8_rot0_crop0_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss wrap ri_none o8',
    'orient_o8_rot1_crop1_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss rot crop wrap ri_none o8',
    'orient_o8_rot1_crop0_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss rot wrap ri_none o8',
    'orient_o8_rot0_crop1_600x331': 'decode 420 edge_r edge_b chunks ff_span ff_chunk ctan lutmiss crop wrap ri_none o8',
    'place_ff00_span_gray': 'decode gray chunks ff_span fill cta2 seg_sub ri_1 o1',
    'place_rst_span_420': 'decode 420 edge_r edge_b chunks ff_span ff_chunk fill ctan seg_sub ri_1 o1',
    'place_ff00_chunk_444': 'decode 444 chunks ff_span ff_chunk fill ctan seg_sub wrap ri_1 o1',
    'place_rst_chunk_420': 'decode 420 edge_b chunks ff_span ff_chunk fill ctan seg_sub wrap ri_1 o1',
    'segsub_420_ri1': 'decode 420 chunks ff_span ctan seg_sub ri_1 o1',
    'sync_ctas1': 'decode 444 chunks cta1 slots ri_none o1',
    'sync_ctas2': 'decode 444 chunks cta2 slots ri_none o1',
    'sync_ctas11_below_limit': 'decode 444 chunks ctan slots ri_none o1',
    'sync_ctas12_at_limit': 'decode 444 chunks ctan slots ri_none o1',
    'sync_ctas13_above_limit': 'decode 444 chunks ctan slots ri_none o1',
    'call_3024x3024_512_sq': 'ingest lanczos h smem48 rowblk ph0 v cw256 sq',
    'call_4032x3024_512': 'ingest lanczos h smem48 rowblk ph0 v cw256',
    'call_4032x3024_224': 'ingest lanczos h smem48 cbpart rowblk ph0 v crop_l s224',
    'call_3024x4032_512': 'ingest lanczos h smem48 ph0 v',
    'call_3024x4032_224': 'ingest lanczos h smem48 cbpart ph0 v crop_t s224',
    'call_4000x3000_512': 'ingest lanczos h smem48 rowblk ph0 v cw256',
    'call_4000x3000_224': 'ingest lanczos h smem48 cbpart rowblk ph0 v crop_l s224',
    'call_1920x1080_512': 'ingest lanczos h smem48 rowblk ph0 v cw256',
    'call_1920x1080_224': 'ingest lanczos h smem48 cbpart rowblk ph0 v crop_l s224',
    'call_1080x1920_512': 'ingest lanczos h smem48 cbpart ph0 v',
    'call_1080x1920_224': 'ingest lanczos h smem48 cbpart ph0 v crop_t s224',
    'call_1440x1080_512': 'ingest lanczos h smem48 rowblk ph0 v cw256',
    'call_1440x1080_224': 'ingest lanczos h smem48 cbpart rowblk ph0 v crop_l s224',
    'call_3024x2268_512': 'ingest lanczos h smem48 rowstep rowblk ph0 v cw256',
    'call_3024x2268_224': 'ingest lanczos h smem48 cbpart rowstep rowblk ph0 v crop_l s224',
    'tiny_1x1_512': 'ingest bicubic h smem48 rowstep rowblk lastword ph1 v crop_t cw256',
    'tiny_1x1_224': 'ingest bicubic h smem48 cbpart rowstep rowblk lastword ph1 v s224',
    'tiny_2x1_512': 'ingest bicubic h smem48 rowstep rowblk lastword ph2 v cw256',
    'tiny_2x1_224': 'ingest bicubic h smem48 rowstep rowblk lastword ph2 v crop_l s224',
    'tiny_1x2_512': 'ingest bicubic h smem48 rowstep rowblk lastword ph1 v cw256',
    'tiny_1x2_224': 'ingest bicubic h smem48 cbpart rowstep rowblk lastword ph1 v crop_t s224',
    'tiny_3x3_512': 'ingest bicubic h smem48 rowstep rowblk lastword ph3 v crop_t cw256',
    'tiny_3x3_224': 'ingest bicubic h smem48 cbpart rowstep rowblk lastword ph3 v s224',
    'tiny_5x7_512': 'ingest bicubic h smem48 cbpart rowstep rowblk lastword ph1 v crop_l',
    'tiny_5x7_224': 'ingest bicubic h smem48 cbpart rowstep rowblk lastword ph1 v crop_t s224',
    'tiny_8x8_512': 'ingest bicubic h smem48 rowblk ph0 v crop_t cw256',
    'tiny_8x8_224': 'ingest bicubic h smem48 cbpart rowblk ph0 v s224',
    'tiny_7x4_512': 'ingest bicubic h smem48 rowstep rowblk ph3 v crop_t cw256',
    'tiny_7x4_224': 'ingest bicubic h smem48 cbpart rowstep rowblk ph3 v crop_l s224',
    'tiny_6x2_512': 'ingest bicubic h smem48 rowstep rowblk ph2 v crop_t cw256',
    'tiny_6x2_224': 'ingest bicubic h smem48 cbpart rowstep rowblk ph2 v crop_l s224',
    'mat_513x200_512': 'ingest lanczos h smem48 rowblk ph1 crop_t cw256',
    'mat_513x200_224': 'ingest bicubic h smem48 cbpart rowblk ph1 v crop_l s224',
    'mat_513x200_512_sq': 'ingest lanczos h smem48 rowblk ph1 crop_t cw256 sq',
    'mat_200x513_512': 'ingest lanczos v crop_l',
    'mat_200x513_224': 'ingest bicubic h smem48 cbpart rowstep rowblk ph0 v crop_t s224',
    'mat_200x513_512_sq': 'ingest lanczos v crop_l sq',
    'mat_513x384_512': 'ingest lanczos h smem48 ph1 v crop_t cw256',
    'mat_513x384_224': 'ingest lanczos h smem48 cbpart ph1 v crop_l s224',
    'mat_513x384_512_sq': 'ingest lanczos h smem48 ph1 v crop_t cw256 sq',
    'mat_512x513_512': 'ingest lanczos h smem48 cbpart rowstep rowblk ph0 v crop_l',
    'mat_512x513_224': 'ingest lanczos h smem48 cbpart rowstep rowblk ph0 v s224',
    'mat_512x513_512_sq': 'ingest lanczos h smem48 cbpart rowstep rowblk ph0 v crop_l sq',
    'mat_1027x33_512': 'ingest lanczos h smem48 rowstep rowblk lastword ph3 v cw256',
    'mat_1027x33_224': 'ingest bicubic h smem48 cbpart rowstep rowblk lastword ph3 v crop_l s224',
    'mat_1027x33_512_sq': 'ingest lanczos h smem48 rowstep rowblk lastword ph3 v cw256 sq',
    'mat_1026x61_512': 'ingest lanczos h smem48 rowstep rowblk lastword ph2 v crop_t cw256',
    'mat_1026x61_224': 'ingest bicubic h smem48 cbpart rowstep rowblk lastword ph2 v crop_l s224',
    'mat_1026x61_512_sq': 'ingest lanczos h smem48 rowstep rowblk lastword ph2 v crop_t cw256 sq',
    'mat_1025x47_512': 'ingest lanczos h smem48 rowstep rowblk lastword ph1 v crop_t cw256',
    'mat_1025x47_224': 'ingest bicubic h smem48 cbpart rowstep rowblk lastword ph1 v crop_l s224',
    'mat_1025x47_512_sq': 'ingest lanczos h smem48 rowstep rowblk lastword ph1 v crop_t cw256 sq',
    'mat_1024x1029_512': 'ingest lanczos h smem48 cbpart rowstep rowblk ph0 v crop_l',
    'mat_1024x1029_224': 'ingest lanczos h smem48 cbpart rowstep rowblk ph0 v s224',
    'mat_1024x1029_512_sq': 'ingest lanczos h smem48 cbpart rowstep rowblk ph0 v crop_l sq',
    'mat_640x481_512': 'ingest lanczos h smem48 rowstep rowblk ph0 v cw256',
    'mat_640x481_224': 'ingest lanczos h smem48 cbpart rowstep rowblk ph0 v crop_l s224',
    'mat_640x481_512_sq': 'ingest lanczos h smem48 rowstep rowblk ph0 v cw256 sq',
    'mat_700x29_512': 'ingest lanczos h smem48 rowstep rowblk ph0 v crop_t cw256',
    'mat_700x29_224': 'ingest bicubic h smem48 cbpart rowstep rowblk ph0 v crop_l s224',
    'mat_700x29_512_sq': 'ingest lanczos h smem48 rowstep rowblk ph0 v crop_t cw256 sq',
    'mat_64x600_512': 'ingest lanczos h smem48 cb1 cbpart rowblk ph0 v crop_l',
    'mat_64x600_224': 'ingest bicubic h smem48 cbpart rowblk ph0 v crop_t s224',
    'mat_64x600_512_sq': 'ingest lanczos h smem48 cb1 cbpart rowblk ph0 v crop_l sq',
    'mat_5000x170_512': 'ingest lanczos h smem48 rowstep rowblk ph0 v cw256',
    'mat_5000x170_224': 'ingest bicubic h smem48 cbpart rowstep rowblk ph0 v crop_l s224',
    'mat_5000x170_512_sq': 'ingest lanczos h smem48 rowstep rowblk ph0 v cw256 sq',
    'mat_200x4097_512': 'ingest lanczos h smem48 cb1 cbpart rowstep rowblk ph0 v crop_l',
    'mat_200x4097_224': 'ingest bicubic h smem48 cbpart rowstep rowblk ph0 v crop_t s224',
    'mat_200x4097_512_sq': 'ingest lanczos h smem48 cb1 cbpart rowstep rowblk ph0 v crop_l sq',
    'mat_2000x350_512': 'ingest lanczos h smem48 rowstep rowblk ph0 v crop_t cw256',
    'mat_2000x350_224': 'ingest lanczos h smem48 rowstep rowblk ph0 v crop_l s224',
    'mat_2000x350_512_sq': 'ingest lanczos h smem48 rowstep rowblk ph0 v crop_t cw256 sq',
    'mat_1000x1000_512': 'ingest lanczos h smem48 rowblk ph0 v crop_t cw256',
    'mat_1000x1000_224': 'ingest lanczos h smem48 cbpart rowblk ph0 v s224',
    'mat_1000x1000_512_sq': 'ingest lanczos h smem48 rowblk ph0 v cw256 sq',
    'pano_32000x1000': 'ingest lanczos h optin rowblk ph0 v cw256',
    'pano_33000x1000': 'ingest lanczos h direct ph0 v cw256',
    'pano_40000x2000': 'ingest lanczos h direct ph0 v crop_t cw256',
    'pano_40000x2000_224': 'ingest lanczos h smem48 rowblk ph0 v crop_l s224',
    'pano_2000x40000': 'ingest lanczos h optin cb1 cbpart ph0 v crop_l',
    'offset1_501x301': 'ingest bicubic h smem48 rowstep rowblk lastword ph1 v crop_t cw256',
    'offset2_501x301': 'ingest bicubic h smem48 rowstep rowblk lastword ph1 v crop_t cw256',
    'offset3_333x201': 'ingest bicubic h smem48 rowstep rowblk lastword ph1 v crop_t cw256',
    'copy_512x384_512': 'ingest copy cw256',
    'copy_512x512_512_sq': 'ingest copy cw256 sq',
}
for _c in CASES:
    _c["key"] = DECLARED[_c["name"]]


# ------------------------------------------------------------------------------------------------------- stream builder
def _photo(w, h, seed):
    import importlib.util
    import os
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg", "make_fixtures.py")
    spec = importlib.util.spec_from_file_location("jpeg_fixture_gen", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.photo(w, h, seed=seed)


def _place(kind, boundary, samp, seed):
    """A stream with restart markers every MCU whose first stuffed FF (kind "ff00") or first RST FF (kind "rst") past
    `boundary` - 1 is moved onto the last byte of a `boundary`-byte span by fill bytes before the RST ahead of it."""
    from tests import jpeg_streams as J
    rng = np.random.default_rng(seed)
    w = 200 if boundary == UNSTUFF_BYTES else 640
    spec = J.make_spec(w, 120, samp, rng, dri=1, tables="short", density=0.6)
    scan = J.scan_bytes(spec)
    stuffed, rst, _, _, _ = scan_markers(scan)
    target = [m for m in (stuffed if kind == "ff00" else rst) if m >= boundary - 1][0]
    j = max(i for i, r in enumerate(rst) if r < target) if kind == "ff00" else rst.index(target)
    shift = (boundary - 1 - target) % boundary
    spec.fill = {j: shift if shift else boundary}
    return J.encode(spec)


def _segsub(samp, seed):
    """dri = 1 and the first seed whose unstuffed restart segments include one starting on a 1024-bit boundary."""
    from tests import jpeg_streams as J
    for s in range(seed, seed + 200):
        spec = J.make_spec(256, 256, samp, np.random.default_rng(s), dri=1, tables="short")
        data = J.encode(spec)
        if any(x * 8 % SUB_BITS == 0 for x in scan_markers(parse_headers(data)["scan"])[3]):
            return data
    raise AssertionError("no seed puts a segment on a subsequence boundary")


def build_stream(case) -> bytes:
    """The bytes of a decode case (deterministic)."""
    import io
    from tests import jpeg_streams as J
    kind, a = case["recipe"]
    o = case["orientation"]
    if kind == "pil":
        import PIL.Image
        w, h, q, ss, rows = a
        im = _photo(w, h, seed=w + h)
        kw = dict(quality=q, subsampling=ss)
        if rows:
            kw["restart_marker_rows"] = rows
        if o != 1:
            ex = PIL.Image.Exif()
            ex[0x0112] = o
            kw["exif"] = ex.tobytes()
        buf = io.BytesIO()
        im.save(buf, "JPEG", **kw)
        return buf.getvalue()
    if kind == "spec":
        w, h, samp, seed, kw = a
        spec = J.make_spec(w, h, samp, np.random.default_rng(seed), **kw)
        spec.orientation = o if o != 1 else 0
        return J.encode(spec)
    if kind == "place":
        return _place(*a)
    if kind == "segsub":
        return _segsub(*a)
    if kind == "sync":
        return J.sync_stream(a)
    raise KeyError(kind)
