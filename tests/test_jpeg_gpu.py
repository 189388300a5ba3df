"""Baseline JPEG decode on the GPU (f3r_jpeg_decode through ingest.decode_jpeg / load_images) against Pillow: bit-exact on
every committed fixture (tests/golden/jpeg), on seeded 12-Mpixel photos with and without restart markers, and through
load_images on a folder that mixes GPU-decoded and host-decoded files.  Needs an H100."""
import hashlib
import importlib.util
import io
import json
import os
import shutil

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FIX = os.path.join(HERE, "golden", "jpeg")
with open(os.path.join(FIX, "fixtures.json")) as _f:
    META = json.load(_f)
COMBOS = [(r, c) for r in (False, True) for c in (False, True)]


def _gen():
    spec = importlib.util.spec_from_file_location("jpeg_fixture_gen", os.path.join(FIX, "make_fixtures.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _read(name):
    with open(os.path.join(FIX, name), "rb") as f:
        return f.read()


@pytest.mark.parametrize("name", sorted(n for n, e in META["files"].items() if e["probe"] == 0))
def test_decode_matches_digests_and_pillow(name):
    from fast3r_b200 import ingest
    data = _read(name)
    for rot, crop in COMBOS:
        want = META["files"][name]["decode"][f"rot{int(rot)}_crop{int(crop)}"]
        got = ingest.decode_jpeg(data, rot, crop).cpu().numpy()
        assert list(got.shape) == want["shape"], (name, rot, crop)
        assert hashlib.sha256(got.tobytes()).hexdigest() == want["sha256"], (name, rot, crop)
        np.testing.assert_array_equal(got, ingest._decode(os.path.join(FIX, name), rot, crop), err_msg=f"{name} {rot} {crop}")


def test_decode_refuses_what_the_gpu_does_not_decode():
    from fast3r_b200 import ingest
    for name, ent in META["files"].items():
        if ent["probe"] != 0:
            with pytest.raises(ValueError):
                ingest.decode_jpeg(_read(name))


@pytest.fixture(scope="module")
def big_photos():
    gen = _gen()
    im = gen.photo(4032, 3024, seed=123)
    out = {}
    for ss in (0, 2):
        out[(ss, None)] = gen.save(im, quality=90, subsampling=ss)
        out[(ss, "rows")] = gen.save(im, quality=90, subsampling=ss, restart_marker_rows=4)
    out[(2, "q100")] = gen.save(im, quality=100, subsampling=2, optimize=True)
    return out


def test_12mpix_photos_match_pillow(big_photos):
    from fast3r_b200 import ingest
    import PIL.Image
    for key, data in big_photos.items():
        ref = np.asarray(PIL.Image.open(io.BytesIO(data)).convert("RGB"))
        got = ingest.decode_jpeg(data).cpu().numpy()
        assert got.shape == ref.shape, key
        assert np.array_equal(got, ref), (key, int((got != ref).any(-1).sum()))


def test_restart_markers_do_not_change_pixels(big_photos):
    from fast3r_b200 import ingest
    for ss in (0, 2):
        a = ingest.decode_jpeg(big_photos[(ss, None)])
        b = ingest.decode_jpeg(big_photos[(ss, "rows")])
        assert torch.equal(a, b), ss


def test_load_images_mixed_folder_matches_host_path(tmp_path):
    """Every JPEG kind, a progressive JPEG, a CMYK JPEG, a PNG and a non-image file: the views equal the host path's
    (_decode + ingest_rgb8) exactly, in the same order."""
    import PIL.Image
    from fast3r_b200 import ingest
    names = [n for n, e in META["files"].items() if e["probe"] in (0, 1) and "1x1" not in n and "2x2" not in n]
    for n in names:
        shutil.copy(os.path.join(FIX, n), tmp_path / n)
    PIL.Image.fromarray(np.random.default_rng(0).integers(0, 256, (70, 90, 3), dtype=np.uint8)).save(tmp_path / "x.png")
    (tmp_path / "notes.txt").write_text("not an image")
    for size, rot, crop in ((512, False, False), (224, True, True)):
        views = ingest.load_images(str(tmp_path), size, verbose=False, rotate_clockwise_90=rot, crop_to_landscape=crop)
        paths = sorted(p for p in os.listdir(tmp_path) if p.lower().endswith((".jpg", ".png")))
        assert len(views) == len(paths)
        for v, p in zip(views, paths):
            arr = ingest._decode(str(tmp_path / p), rot, crop)
            ref, (h, w) = ingest.ingest_rgb8(torch.from_numpy(np.ascontiguousarray(arr)).cuda(), size)
            assert torch.equal(v["img"][0], ref), p
            assert v["true_shape"].tolist() == [[h, w]]


def test_truncated_jpeg_behaves_as_before(tmp_path):
    from fast3r_b200 import ingest
    name = "truncated_s420_331x211.jpg"
    shutil.copy(os.path.join(FIX, name), tmp_path / name)
    with pytest.raises(Exception) as want:
        ingest._decode(str(tmp_path / name), False, False)
    with pytest.raises(type(want.value)):
        ingest.load_images(str(tmp_path), 512, verbose=False)


def test_corrupt_entropy_data_is_a_status_not_a_fault(tmp_path):
    """Bytes flipped inside the scan: the device reports an inconsistent stream (or decodes what libjpeg decodes), and
    load_images returns what the host path returns."""
    from fast3r_b200 import ingest
    data = bytearray(_read("s420_331x211_q100.jpg"))
    probe = ingest.probe_jpeg(bytes(data))
    off = probe.info.scan_offset + probe.info.scan_bytes // 2
    data[off:off + 16] = bytes(np.random.default_rng(1).integers(0, 255, 16, dtype=np.uint8))  # no 0xFF: stays parseable
    (tmp_path / "c.jpg").write_bytes(bytes(data))
    views = ingest.load_images(str(tmp_path), 512, verbose=False)
    arr = ingest._decode(str(tmp_path / "c.jpg"), False, False)
    ref, _ = ingest.ingest_rgb8(torch.from_numpy(np.ascontiguousarray(arr)).cuda(), 512)
    assert torch.equal(views[0]["img"][0], ref)
