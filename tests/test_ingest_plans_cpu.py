"""Image ingest without a GPU.

- The real callers (load_images, decode_jpeg, ingest_rgb8) run with the library's CUDA calls replaced by recorders:
  f3r_jpeg_decode answers with the host decoder (tests/jpeg_host_decoder.cpp) through the orientation map, and
  f3r_ingest_rgb8 with oracle/ingest_oracle.c.  Each recorder records the launch key of its call
  (tests/ingest_plans.py) from the arguments the caller passed.  Every case must reach the key it declares, every key
  the callers reach at their geometries (photos at EXIF 1/6/8 with rotate and crop, sizes 512 and 224, bench.py's
  call) must be a declared key, and every axis of the keys must have a case.
- The header probe agrees with Pillow on every stream tests/ingest_plans.py builds (supported => Pillow decodes it to
  the host decoder's pixels; Pillow raises => the probe does not say supported), including the Huffman tables libjpeg
  rejects.
- The Python restatement of the decode workspace layout equals f3r_jpeg_info.workspace_bytes, and f3r_ingest_rgb8
  refuses a misaligned source before any CUDA call."""
import ctypes as C
import io

import numpy as np
import pytest

from tests import ingest_plans as IP
from oracle import ingest_oracle as ORC
from tests import jpeg_streams as J
from tests.test_jpeg_cpu import hostlib  # noqa: F401  (fixture)

SMALL = [c for c in IP.DECODE if c["recipe"][0] != "pil"]


def _pillow(data):
    import PIL.Image
    try:
        return np.asarray(PIL.Image.open(io.BytesIO(data)).convert("RGB"))
    except Exception:  # noqa: BLE001
        return None


def _host(lib, data):
    dims = np.zeros(3, np.int32)
    if lib.f3r_test_jpeg_parse(data, len(data), dims.ctypes.data) != 0:
        return None
    out = np.zeros((dims[1], dims[0], 3), np.uint8)
    assert lib.f3r_test_jpeg_decode(data, len(data), out.ctypes.data) == 0
    return out


def _check_probe_vs_pillow(lib, data):
    from fast3r_b200 import ingest, lib as L
    ref = _pillow(data)
    st = ingest.probe_jpeg(data).status
    if ref is None:
        assert st != L.JPEG_SUPPORTED, "the probe accepts a stream Pillow refuses"
    elif st == L.JPEG_SUPPORTED:
        np.testing.assert_array_equal(_host(lib, data), ref)


@pytest.mark.parametrize("case", SMALL, ids=[c["name"] for c in SMALL])
def test_probe_and_host_decoder_match_pillow(hostlib, case):  # noqa: F811
    data = IP.build_stream(case)
    assert _pillow(data) is not None
    _check_probe_vs_pillow(hostlib, data)


def _all_ones_table():
    """A DC table whose last code is all ones: lengths 1, 2 and 2 fill the code space exactly (0, 10, 11)."""
    rng = np.random.default_rng(4)
    spec = J.make_spec(16, 16, "gray", rng, tables="short")
    spec.coef[0][..., 0] = 0
    spec.dc[0] = J.Huff([1, 2] + [0] * 14, [0, 1, 2])
    return J.encode(spec)


def _unused_dc16():
    rng = np.random.default_rng(5)
    spec = J.make_spec(16, 16, "gray", rng, tables="short")
    spec.dc[0] = J.Huff(list(spec.dc[0].counts[:15]) + [1], list(spec.dc[0].symbols) + [16])
    return J.encode(spec)


def _unused_all_ones_slot1():
    """The all-ones table in DC slot 1, which the scan does not use: libjpeg validates only the tables a scan uses, so
    Pillow decodes; the probe may refuse it (the host path then decodes it)."""
    rng = np.random.default_rng(6)
    spec = J.make_spec(16, 16, "gray", rng, tables="short")
    spec.extra_dht = J.dht_payload(0, 1, J.Huff([1, 2] + [0] * 14, [0, 1, 2]))
    return J.encode(spec)


@pytest.mark.parametrize("build", [_all_ones_table, _unused_dc16, _unused_all_ones_slot1],
                         ids=["all_ones_code", "dc_symbol_16", "unused_slot_all_ones"])
def test_probe_follows_libjpeg_huffman_rules(hostlib, build):  # noqa: F811
    """jpeg_make_d_derived_tbl rejects a code of all ones and a DC symbol above 15; where Pillow raises the probe must not
    send the stream to the GPU."""
    data = build()
    _check_probe_vs_pillow(hostlib, data)
    if build is not _unused_all_ones_slot1:
        assert _pillow(data) is None, "Pillow decoded a table libjpeg should refuse"


class Recorder:
    """Stand-in for fast3r_b200.ops._call: records the launch key of every f3r_jpeg_decode / f3r_ingest_rgb8 call from
    its arguments and answers from the host decoder / the ingest oracle, so the callers go on as with the kernels.
    `ctx` holds what the ingest key needs beyond the arguments (the caller's size and square_ok)."""

    def __init__(self, hostlib):
        self.lib, self.keys, self.ctx = hostlib, [], dict(size=512, square_ok=False)

    def __call__(self, name, anchor, *args):
        getattr(self, name)(*args)

    def f3r_jpeg_decode(self, data_ptr, n, dev, orientation, rot, left, top, ow, oh, out, status, ws, nws):
        data = C.string_at(data_ptr, n)
        assert bytes(dev.numpy().tobytes()) == data and ws.numel() >= nws
        self.keys.append(IP.decode_key(data, orientation, bool(rot), left, top, ow, oh))
        src = _host(self.lib, data)
        m = np.zeros(6, np.int32)
        self.lib.f3r_test_jpeg_orient_map(src.shape[1], src.shape[0], orientation, rot, left, top, m.ctypes.data)
        oy, ox = np.mgrid[0:oh, 0:ow]
        out.numpy()[...] = src[m[3] * ox + m[4] * oy + m[5], m[0] * ox + m[1] * oy + m[2]]
        status.zero_()

    @staticmethod
    def _filter(n_in, n_out, bounds, taps):
        """The filter whose oracle tables equal the ones the caller passed (None when it passed none)."""
        if taps is None:
            return None
        for filt in (ORC.BICUBIC, ORC.LANCZOS):
            ks = ORC.lib().f3r_oracle_ksize(n_in, n_out, filt)
            if ks != taps.shape[1] if taps.dim() == 2 else ks * n_out != taps.numel():
                continue
            b, k = np.empty((n_out, 2), np.int32), np.empty((n_out, ks), np.int32)
            ORC.lib().f3r_oracle_coeffs(n_in, n_out, filt, C.c_void_p(b.ctypes.data), C.c_void_p(k.ctypes.data))
            if np.array_equal(b, bounds.numpy().reshape(n_out, 2)) and np.array_equal(k, taps.numpy().reshape(n_out, ks)):
                return filt
        raise AssertionError(f"tap tables {n_in} -> {n_out} are not the oracle's for either filter")

    def f3r_ingest_rgb8(self, src, h, w, oh, ow, hb, hk, hks, span, vb, vk, vks, tmp, left, top, cw, ch, out):
        assert src.data_ptr() % 4 == 0, "a misaligned source reached the library"
        assert src.is_contiguous() and tuple(src.shape) == (h, w, 3) and tuple(out.shape) == (3, ch, cw)
        fh, fv = self._filter(w, ow, hb, hk), self._filter(h, oh, vb, vk)
        assert fh is None or fv is None or fh == fv
        filt = fh if fh is not None else fv
        if hk is not None:
            assert tuple(tmp.shape) == (h, ow, 3)
        self.keys.append(IP.ingest_key(dict(h=h, w=w, oh=oh, ow=ow, filt=filt, hks=hks, span=span, left=left, top=top,
                                            cw=cw, ch=ch, **self.ctx)))
        img = src.numpy()
        r = img if filt is None else ORC.resize_rgb8(img, ow, oh, filt)
        out.numpy()[...] = ORC.crop_normalize(r, (left, top, left + cw, top + ch))


@pytest.fixture
def rec(monkeypatch, hostlib):  # noqa: F811
    import contextlib

    import torch
    import fast3r_b200.ops as O
    from fast3r_b200 import ingest as I
    r = Recorder(hostlib)
    monkeypatch.setattr(O, "_call", r)
    monkeypatch.setattr(O, "_ptr", lambda t: t)
    monkeypatch.setattr(I, "_need_cuda", lambda device, what: None)
    monkeypatch.setattr(I, "_h2d", lambda arr, device: torch.from_numpy(np.array(arr)))
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    return r


def _run_case(rec, case):
    """Runs one case through its real caller (decode_jpeg / ingest_rgb8) on the CPU; returns the keys recorded."""
    import torch
    from fast3r_b200 import ingest as I
    rec.keys.clear()
    if case["op"] == "decode":
        I.decode_jpeg(IP.build_stream(case), case["rot"], case["crop"], device="cpu")
    else:
        h, w, off = case["h"], case["w"], case["offset"]
        img = np.random.default_rng(h * 7 + w).integers(0, 256, (h, w, 3), dtype=np.uint8)
        flat = torch.zeros(h * w * 3 + 8, dtype=torch.uint8)
        base = (-flat.data_ptr()) % 4 + off
        src = flat[base:base + h * w * 3].view(h, w, 3)
        src.copy_(torch.from_numpy(img))
        assert src.data_ptr() % 4 == off
        rec.ctx = dict(size=case["size"], square_ok=case["square_ok"])
        I.ingest_rgb8(src, case["size"], case["square_ok"])
    return list(rec.keys)


@pytest.mark.parametrize("case", IP.CASES, ids=[c["name"] for c in IP.CASES])
def test_case_reaches_its_declared_key(rec, case):
    assert _run_case(rec, case) == [case["key"]]


PHOTOS = [c for c in IP.DECODE if c["recipe"][0] == "pil"]


@pytest.mark.parametrize("case", PHOTOS, ids=[c["name"] for c in PHOTOS])
def test_load_images_reaches_declared_keys(rec, case, tmp_path):
    """load_images on the callers' photos (EXIF 1 / 6 / 8, rotate, 4:3 crop) at sizes 512 and 224: the decode reaches
    the photo case's key and every resize of the decoded view a declared ingest key."""
    from fast3r_b200 import ingest as I
    path = tmp_path / "photo.jpg"
    path.write_bytes(IP.build_stream(case))
    declared = {c["key"] for c in IP.INGEST}
    for size in (512, 224):
        rec.keys.clear()
        rec.ctx = dict(size=size, square_ok=False)
        views = I.load_images([str(path)], size, verbose=False, rotate_clockwise_90=case["rot"],
                              crop_to_landscape=case["crop"], device="cpu")
        assert len(views) == 1 and rec.keys[0] == case["key"], rec.keys
        assert len(rec.keys) == 2 and rec.keys[1] in declared, (size, rec.keys[1])


def test_bench_ingest_call_is_declared(rec):
    """bench.py's ingest: a 4032 x 3024 image at size 512 into a preallocated output."""
    import torch
    from fast3r_b200 import ingest as I
    u8 = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (3024, 4032, 3), dtype=np.uint8))
    out = torch.empty(3, 384, 512, dtype=torch.float32)
    I.ingest_rgb8(u8, 512, out=out)
    assert rec.keys == [next(c["key"] for c in IP.INGEST if c["name"] == "call_4032x3024_512")]


def test_table_covers_every_axis():
    """Every axis the key functions can produce is declared by some case."""
    dec = set().union(*(IP.decode_axes(c["key"]) for c in IP.DECODE))
    want = {"gray", "444", "422", "420", "edge_r", "edge_b", "cw2", "chunks", "ff_span", "ff_chunk", "fill", "cta1",
            "cta2", "ctan", "seg_sub", "lutmiss", "slots", "dqt16", "rot", "crop", "wrap", "ri_none", "ri_1", "ri_div",
            "ri_nodiv"} | {f"o{o}" for o in range(1, 9)}
    assert want <= dec, sorted(want - dec)
    ing = set().union(*(set(c["key"].split()[1:]) for c in IP.INGEST))
    want = {"lanczos", "bicubic", "copy", "h", "v", "smem48", "optin", "direct", "cb1", "cbpart", "rowstep", "rowblk",
            "lastword", "ph0", "ph1", "ph2", "ph3", "crop_l", "crop_t", "cw256", "s224", "sq"}
    assert want <= ing, sorted(want - ing)
    assert {c["name"] for c in IP.CASES if " direct" in c["key"]} >= {"pano_33000x1000", "pano_40000x2000"}
    assert " optin" in next(c["key"] for c in IP.CASES if c["name"] == "pano_32000x1000")


def _layout(info, scan_bytes, segments, blocks, plane):
    """jpeg.cu:483-512 restated (DevTables 2 x 2 Huffman tables + 3 quant tables; Rec 24 bytes)."""
    a = lambda x: (x + 255) & ~255  # noqa: E731
    huff = 2 * 512 + 4 * 18 * 2 + 256
    tab = 4 * huff + 3 * 128
    nchunks = -(-scan_bytes // 4096)
    nsub = -(-scan_bytes * 8 // 1024)
    o = a(tab)
    o = a(o + scan_bytes + 16)
    o = a(o + (nchunks + 1) * 8)
    o = a(o + (segments + 1) * 4)
    o = a(o + (3 + IP.MAX_ROUNDS) * 4)
    o = a(o + (nsub + 2) * 8)
    o = a(o + (nsub + 2) * 8)
    o = a(o + (nsub + 1) * 24)
    o = a(o + (nsub + 1) * 24)
    o = a(o + blocks * 128)
    return a(o + plane)


@pytest.mark.parametrize("case", [c for c in SMALL if c["recipe"][0] in ("spec", "sync")][::5],
                         ids=lambda c: c["name"])
def test_workspace_layout_restated(case):
    from fast3r_b200 import ingest
    data = IP.build_stream(case)
    p = ingest.probe_jpeg(data)
    h = IP.parse_headers(data)
    comps = h["comps"] if len(h["comps"]) == 3 else [(1, 1, 0)]
    hm, vm = comps[0][0], comps[0][1]
    mcux, mcuy = -(-p.width // (8 * hm)), -(-p.height // (8 * vm))
    blocks = sum(mcux * c[0] * mcuy * c[1] for c in comps)
    assert p.info.workspace_bytes == _layout(p.info, p.info.scan_bytes, p.info.segments, blocks, blocks * 64)


def test_ingest_refuses_misaligned_source_first():
    """f3r_ingest_rgb8 reports a source 1 byte past a 4-byte boundary before it looks at anything else.  The pointers are
    made up and the shape is empty, so no version of the library can launch on them."""
    from fast3r_b200 import lib as L
    lib = L.load()
    fake = C.c_void_p(0x10001)
    rc = lib.f3r_ingest_rgb8(fake, 0, 5, 4, 3, fake, fake, 3, 5, None, None, 0, C.c_void_p(0x20000), 0, 0, 3, 4,
                             C.c_void_p(0x30000), None)
    assert rc != 0 and lib.f3r_last_error().decode() == "f3r_ingest_rgb8: src not 4-byte aligned"
