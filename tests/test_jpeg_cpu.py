"""Baseline JPEG decode without a GPU: the library's header probe classifies every fixture, and the per-sample math of
the GPU decoder (fast3r_b200/csrc/jpeg_math.h), compiled for the host around a plain sequential Huffman decoder
(tests/jpeg_host_decoder.cpp), reproduces Pillow bit-exactly - on the committed fixtures (tests/golden/jpeg) and on
seeded random images encoded here at every sampling layout."""
import ctypes as C
import hashlib
import io
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "fast3r_b200", "csrc")
FIX = os.path.join(HERE, "golden", "jpeg")
with open(os.path.join(FIX, "fixtures.json")) as _f:
    META = json.load(_f)
SUPPORTED = sorted(n for n, e in META["files"].items() if e["probe"] == 0)


def _read(name):
    with open(os.path.join(FIX, name), "rb") as f:
        return f.read()


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    so = str(tmp_path_factory.mktemp("jpeg") / "libjpeg_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", CSRC,
                           os.path.join(HERE, "jpeg_host_decoder.cpp"), "-o", so])
    lib = C.CDLL(so)
    lib.f3r_test_jpeg_parse.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p]
    lib.f3r_test_jpeg_decode.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p]
    lib.f3r_test_jpeg_orient_map.argtypes = [C.c_int] * 6 + [C.c_void_p]
    return lib


def host_decode(lib, data):
    dims = np.zeros(3, np.int32)
    assert lib.f3r_test_jpeg_parse(data, len(data), dims.ctypes.data) == 0
    out = np.zeros((dims[1], dims[0], 3), np.uint8)
    assert lib.f3r_test_jpeg_decode(data, len(data), out.ctypes.data) == 0
    return out


def pillow_rgb(data):
    import PIL.Image
    return np.asarray(PIL.Image.open(io.BytesIO(data)).convert("RGB"))


def test_fixture_versions_recorded():
    assert META["pillow"] and META["libjpeg_turbo"]


@pytest.mark.parametrize("name", sorted(META["files"]))
def test_probe_classifies_fixture(name):
    from fast3r_b200 import ingest
    data = _read(name)
    info = ingest.probe_jpeg(data)
    assert info.status == META["files"][name]["probe"], (name, info.why)
    if info.status == 0:
        w, h = pillow_rgb(data).shape[1::-1]
        assert (info.width, info.height) == (w, h)


def test_probe_rejects_non_jpeg_bytes():
    from fast3r_b200 import ingest
    assert ingest.probe_jpeg(b"\x89PNG\r\n\x1a\n" + b"\0" * 64).status == 1
    assert ingest.probe_jpeg(b"").status == 1
    assert ingest.probe_jpeg(b"\xff\xd8\xff").status == 2


@pytest.mark.parametrize("name", SUPPORTED)
def test_host_math_matches_pillow_on_fixture(hostlib, name):
    data = _read(name)
    np.testing.assert_array_equal(host_decode(hostlib, data), pillow_rgb(data))


@pytest.mark.parametrize("subsampling", [0, 1, 2, "gray"])
def test_host_math_matches_pillow_on_random_images(hostlib, subsampling):
    import PIL.Image
    rng = np.random.default_rng(17 if subsampling == "gray" else subsampling)
    for trial in range(12):
        w, h = int(rng.integers(1, 90)), int(rng.integers(1, 90))
        arr = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        if trial % 3 == 1:  # smooth content: long zero runs, EOB-heavy blocks
            arr = np.clip(np.cumsum(rng.integers(-3, 4, (h, w, 3)), 1) + 128, 0, 255).astype(np.uint8)
        im = PIL.Image.fromarray(arr, "RGB")
        kw = dict(quality=int(rng.choice([1, 30, 75, 95, 100])), optimize=bool(trial % 2))
        if trial % 4 == 3:
            kw["restart_marker_blocks"] = int(rng.integers(1, 5))
        buf = io.BytesIO()
        if subsampling == "gray":
            im.convert("L").save(buf, "JPEG", **kw)
        else:
            im.save(buf, "JPEG", subsampling=subsampling, **kw)
        data = buf.getvalue()
        np.testing.assert_array_equal(host_decode(hostlib, data), pillow_rgb(data), err_msg=f"{trial} {w}x{h} {kw}")


@pytest.mark.parametrize("rot", [0, 1])
@pytest.mark.parametrize("crop", [0, 1])
def test_orientation_map_matches_pillow(hostlib, rot, crop):
    """The store's index map (EXIF orientation, rotation, 4:3 crop) applied to the plain decode reproduces _decode."""
    from fast3r_b200 import ingest
    for o in range(1, 9):
        name = f"s420_45x29_exif{o}.jpg"
        data = _read(name)
        src = host_decode(hostlib, data)
        want = ingest._decode(os.path.join(FIX, name), bool(rot), bool(crop))
        h0, w0 = src.shape[:2]
        oh, ow, left, top = ingest._store_geometry(w0, h0, o, bool(rot), bool(crop))
        assert (oh, ow) == want.shape[:2]
        m = np.zeros(6, np.int32)
        hostlib.f3r_test_jpeg_orient_map(w0, h0, o, rot, left, top, m.ctypes.data)
        oy, ox = np.mgrid[0:oh, 0:ow]
        got = src[m[3] * ox + m[4] * oy + m[5], m[0] * ox + m[1] * oy + m[2]]
        np.testing.assert_array_equal(got, want, err_msg=name)


@pytest.mark.parametrize("name", sorted(META["files"]))
def test_golden_digests_match_runtime_pillow(name):
    """The committed digests still describe what this Pillow decodes (guards the fixtures against a Pillow change)."""
    from fast3r_b200 import ingest
    ent = META["files"][name]["decode"]["rot0_crop0"]
    if "error" in ent:
        with pytest.raises(Exception):
            ingest._decode(os.path.join(FIX, name), False, False)
        return
    arr = np.ascontiguousarray(ingest._decode(os.path.join(FIX, name), False, False))
    assert list(arr.shape) == ent["shape"] and hashlib.sha256(arr.tobytes()).hexdigest() == ent["sha256"]


def test_jpeg_info_struct_matches_header():
    from fast3r_b200 import lib as L
    from tests.test_cabi_bindings_cpu import _ctypes_kind, _struct_fields
    assert [(n, _ctypes_kind(t)) for n, t in L.JpegInfo._fields_] == _struct_fields("f3r_jpeg_info")


def test_decode_rejects_bad_arguments_before_any_cuda_call():
    from fast3r_b200 import lib as L
    lib = L.load()
    data = _read("s420_17x9_q75.jpg")
    assert lib.f3r_jpeg_decode(data, len(data), None, 1, 0, 0, 0, 17, 9, 8, 8, 256, 1 << 20, None) != 0
    assert lib.f3r_last_error().decode() == "f3r_jpeg_decode: null operand"
    assert lib.f3r_jpeg_probe(None, 0, None) != 0
