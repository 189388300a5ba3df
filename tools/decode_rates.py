"""Ingest decode rates: the GPU JPEG decode (f3r_jpeg_decode) against the host path it replaces, on 32 seeded
4032x3024 q90 4:2:0 photos written by this script.  In one process it reports the card, its power limit and the host core
count, then, alternating the two paths:
  * host path per image on one thread: PIL _decode + pinned copy + H2D + ingest_rgb8, to a device synchronise;
  * load_images wall clock with the default thread pool, host path (the pre-GPU-decode loop) and GPU-decode path;
  * the device decode per image (CUDA events), per stage from torch.profiler kernel times, compressed MB/s, Mpixel/s.

    python tools/decode_rates.py [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

STAGES = {"unstuff/split": ("jpeg_unstuff", "jpeg_chunk_scan"), "sync": ("jpeg_sync",),
          "write": ("jpeg_rec_scan", "jpeg_write"), "idct": ("jpeg_idct",), "upsample+colour": ("jpeg_color", "jpeg_finish")}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"unknown ({e})"
    return q


def write_photos(d, n=32):
    import importlib.util
    import PIL.Image
    spec = importlib.util.spec_from_file_location("gen", os.path.join(ROOT, "tests", "golden", "jpeg", "make_fixtures.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    base = np.asarray(gen.photo(4032, 3024, seed=2024)).astype(np.int16)
    paths = []
    for i in range(n):
        rng = np.random.default_rng(i)
        a = np.roll(base, (int(rng.integers(0, 3024)), int(rng.integers(0, 4032))), (0, 1))
        a = np.clip(a + rng.integers(-6, 7, a.shape, dtype=np.int16), 0, 255).astype(np.uint8)
        p = os.path.join(d, f"photo_{i:02d}.jpg")
        PIL.Image.fromarray(a).save(p, quality=90, subsampling=2)
        paths.append(p)
    return paths


def old_load_images(paths, size=512):
    """load_images before the GPU decode: PIL on the default pool, pinned H2D of the decoded image, ingest_rgb8."""
    from fast3r_b200 import ingest
    out = []
    with ThreadPoolExecutor(max_workers=min(32, os.cpu_count() or 4)) as pool:
        for arr in pool.map(lambda p: ingest._decode(p, False, False), paths):
            u8 = torch.from_numpy(np.ascontiguousarray(arr)).pin_memory().to("cuda", non_blocking=True)
            out.append(ingest.ingest_rgb8(u8, size)[0])
    torch.cuda.synchronize()
    return out


def new_load_images(paths, size=512):
    from fast3r_b200 import ingest
    v = ingest.load_images(paths, size, verbose=False)
    torch.cuda.synchronize()
    return v


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    from fast3r_b200 import ingest
    assert torch.cuda.is_available(), "decode_rates needs a GPU"
    res = {"card": card(), "host_cores": os.cpu_count()}
    with tempfile.TemporaryDirectory() as d:
        paths = write_photos(d)
        datas = []
        for p in paths:
            with open(p, "rb") as f:
                datas.append(f.read())
        res["compressed_MB_mean"] = float(np.mean([len(x) for x in datas]) / 1e6)
        mpix = 4032 * 3024 / 1e6
        # warm-up both paths
        old_load_images(paths[:2])
        new_load_images(paths[:2])
        # host path per image, one thread
        t_host = []
        for p in paths[:8]:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            arr = ingest._decode(p, False, False)
            u8 = torch.from_numpy(np.ascontiguousarray(arr)).pin_memory().to("cuda", non_blocking=True)
            ingest.ingest_rgb8(u8, 512)
            torch.cuda.synchronize()
            t_host.append(time.perf_counter() - t0)
        res["host_path_per_image_ms"] = 1e3 * float(np.median(t_host))
        # device decode per image (events around the decode only; compressed bytes already probed)
        probes = [ingest.probe_jpeg(x) for x in datas]
        t_dev = []
        for x, pr in zip(datas, probes):
            out, st = ingest._decode_jpeg_async(x, pr, 1, False, False, "cuda")  # uploads, allocates
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out, st = ingest._decode_jpeg_async(x, pr, 1, False, False, "cuda")
            e1.record()
            torch.cuda.synchronize()
            assert int(st.item()) == 0
            t_dev.append(e0.elapsed_time(e1))
        ms = float(np.median(t_dev))
        res["device_decode_per_image_ms"] = ms  # includes the compressed H2D copy issued inside the timed window
        res["device_decode_MBps_compressed"] = res["compressed_MB_mean"] / (ms / 1e3)
        res["device_decode_Mpixps"] = mpix / (ms / 1e3)
        # per stage
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for x, pr in zip(datas[:8], probes[:8]):
                ingest._decode_jpeg_async(x, pr, 1, False, False, "cuda")
            torch.cuda.synchronize()
        per = {k: 0.0 for k in STAGES}
        other = {}
        for ev in prof.key_averages():
            us = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            hit = [k for k, pre in STAGES.items() if any(pr_ in ev.key for pr_ in pre)]
            if hit:
                per[hit[0]] += us / 8
            elif us > 0:
                other[ev.key[:60]] = us / 8
        res["device_stage_us_per_image"] = per
        res["device_other_us_per_image"] = other
        # load_images wall clock, alternating
        for rep in range(2):
            for name, fn in (("host_path", old_load_images), ("gpu_decode", new_load_images)):
                t0 = time.perf_counter()
                fn(paths)
                res.setdefault(f"load_images_32_s_{name}", []).append(time.perf_counter() - t0)
        # same views
        a, b = old_load_images(paths[:4]), new_load_images(paths[:4])
        res["views_equal"] = all(torch.equal(x, y["img"][0]) for x, y in zip(a, b))
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
