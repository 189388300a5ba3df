"""Writes the JPEG fixtures of tests/test_jpeg_cpu.py / tests/test_jpeg_gpu.py with Pillow's encoder (seeded) and
fixtures.json: for every file its expected probe class and, for every (rotate_clockwise_90, crop_to_landscape), the shape
and SHA-256 of what fast3r_b200.ingest._decode (Pillow) returns.  Run from the repository root:

    python tests/golden/jpeg/make_fixtures.py

Written with Pillow 12.2.0 / libjpeg-turbo 3.1.4.1 (recorded in fixtures.json)."""
import hashlib
import io
import json
import os
import sys

import numpy as np
import PIL
import PIL.Image
import PIL.features

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "..", ".."))

SUPPORTED, UNSUPPORTED, MALFORMED = 0, 1, 2


def photo(w, h, seed):
    """Smooth colour fields, hard edges and grain: exercises every coefficient band at a modest file size."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.empty((h, w, 3))
    for c in range(3):
        fx, fy, ph = rng.uniform(0.5, 6, 2).tolist() + [rng.uniform(0, 6.3)]
        img[..., c] = 128 + 90 * np.sin(2 * np.pi * (fx * x / max(w, 1) + fy * y / max(h, 1)) + ph)
    for _ in range(6):  # rectangles with hard edges
        x0, y0 = rng.integers(0, max(w, 1)), rng.integers(0, max(h, 1))
        img[y0:y0 + rng.integers(1, max(h // 3, 2)), x0:x0 + rng.integers(1, max(w // 3, 2))] = rng.uniform(0, 255, 3)
    img += rng.normal(0, 4, img.shape)
    return PIL.Image.fromarray(np.clip(img, 0, 255).astype(np.uint8), "RGB")


def checkerboard(w, h):
    y, x = np.mgrid[0:h, 0:w]
    a = np.where((x + y) % 2 == 0, 255, 0).astype(np.uint8)
    rgb = np.stack([a, 255 - a, np.where((x // 2 + y) % 2 == 0, 255, 0).astype(np.uint8)], -1)
    return PIL.Image.fromarray(rgb, "RGB")


def save(img, **kw):
    buf = io.BytesIO()
    img.save(buf, "JPEG", **kw)
    return buf.getvalue()


def exif_bytes(orientation):
    e = PIL.Image.Exif()
    e[0x0112] = orientation
    return e.tobytes()


def cases():
    """name -> (bytes, expected probe class)"""
    out = {}
    layouts = {"444": 0, "422": 1, "420": 2}
    for wh in ((1, 1), (2, 2), (3, 5), (5, 7), (17, 9), (97, 131)):
        im = photo(*wh, seed=wh[0] * 1000 + wh[1])
        for name, ss in layouts.items():
            out[f"s{name}_{wh[0]}x{wh[1]}_q75.jpg"] = (save(im, quality=75, subsampling=ss), SUPPORTED)
        out[f"gray_{wh[0]}x{wh[1]}_q75.jpg"] = (save(im.convert("L"), quality=75), SUPPORTED)
    im = photo(331, 211, seed=5)
    for name, ss in layouts.items():
        for q in (1, 100):
            out[f"s{name}_331x211_q{q}.jpg"] = (save(im, quality=q, subsampling=ss), SUPPORTED)
        out[f"s{name}_331x211_opt.jpg"] = (save(im, quality=85, subsampling=ss, optimize=True), SUPPORTED)
        out[f"s{name}_331x211_rstblk3.jpg"] = (save(im, quality=80, subsampling=ss, restart_marker_blocks=3), SUPPORTED)
        out[f"s{name}_331x211_rstrow1.jpg"] = (save(im, quality=80, subsampling=ss, restart_marker_rows=1), SUPPORTED)
        out[f"s{name}_331x211_rstblk1.jpg"] = (save(im, quality=60, subsampling=ss, restart_marker_blocks=1), SUPPORTED)
    out["gray_331x211_q100_opt.jpg"] = (save(im.convert("L"), quality=100, optimize=True), SUPPORTED)
    out["gray_331x211_rstrow2.jpg"] = (save(im.convert("L"), quality=70, restart_marker_rows=2), SUPPORTED)
    # 16-bit quantisation tables (SOF1)
    qt = [[min(300 + 37 * i, 32000) for i in range(64)], [min(400 + 53 * i, 32000) for i in range(64)]]
    out["s420_331x211_sof1.jpg"] = (save(im, qtables=qt, subsampling=2), SUPPORTED)
    out["s444_331x211_sof1_small.jpg"] = (save(im, qtables=[[1] * 63 + [256]] * 2, subsampling=0), SUPPORTED)
    # saturated, high-contrast content at quality 100
    for name, ss in layouts.items():
        out[f"s{name}_checker_83x61_q100.jpg"] = (save(checkerboard(83, 61), quality=100, subsampling=ss), SUPPORTED)
    out["gray_checker_83x61_q100.jpg"] = (save(checkerboard(83, 61).convert("L"), quality=100), SUPPORTED)
    # EXIF orientation 1..8 on a non-square image (and one at 4:2:2 with restart markers)
    small = photo(45, 29, seed=9)
    for o in range(1, 9):
        out[f"s420_45x29_exif{o}.jpg"] = (save(small, quality=90, subsampling=2, exif=exif_bytes(o)), SUPPORTED)
    out["s422_45x29_exif6_rst.jpg"] = (save(small, quality=90, subsampling=1, exif=exif_bytes(6),
                                            restart_marker_blocks=2), SUPPORTED)
    out["s420_1001x751_q90.jpg"] = (save(photo(1001, 751, seed=11), quality=90, subsampling=2), SUPPORTED)
    # Pillow keeps these
    out["progressive_97x131.jpg"] = (save(photo(97, 131, seed=3), quality=80, progressive=True), UNSUPPORTED)
    out["cmyk_33x21.jpg"] = (save(photo(33, 21, seed=4).convert("CMYK"), quality=80), UNSUPPORTED)
    full = out["s420_331x211_q100.jpg"][0]
    out["truncated_s420_331x211.jpg"] = (full[: len(full) * 2 // 3], MALFORMED)
    return out


def main():
    from fast3r_b200.ingest import _decode
    meta = {"pillow": PIL.__version__, "libjpeg_turbo": PIL.features.version("libjpeg_turbo"), "files": {}}
    for name, (data, cls) in sorted(cases().items()):
        path = os.path.join(HERE, name)
        with open(path, "wb") as f:
            f.write(data)
        ent = {"probe": cls, "decode": {}}
        for rot in (False, True):
            for crop in (False, True):
                key = f"rot{int(rot)}_crop{int(crop)}"
                try:
                    arr = np.ascontiguousarray(_decode(path, rot, crop))
                    ent["decode"][key] = {"shape": list(arr.shape), "sha256": hashlib.sha256(arr.tobytes()).hexdigest()}
                except Exception as e:  # noqa: BLE001 - the truncated file: record what Pillow raises
                    ent["decode"][key] = {"error": type(e).__name__}
        meta["files"][name] = ent
    with open(os.path.join(HERE, "fixtures.json"), "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True)
    total = sum(os.path.getsize(os.path.join(HERE, n)) for n in meta["files"])
    print(f"{len(meta['files'])} files, {total / 1e3:.0f} kB")


if __name__ == "__main__":
    main()
