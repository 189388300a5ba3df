"""Throughput of fast3r_b200.views.prepare_views: CUDA-event time of a call on 32 raw views from 1920x1440 and from
640x480 photos to 512x384, from host inputs (the time includes the pinned uploads over PCIe) and from inputs already on
the device (a loader that decodes on the GPU), the bytes the device work moves and their share of the H100's 3.35 TB/s, and the PIL + cv2 + numpy restatement of the reference's pipeline
(tests/views_reference.py) on the same inputs, on one host thread and on a thread pool.  Prints the card's name and
power limit with the numbers.  Needs a GPU.
Run: python tools/view_rates.py [--views 32] [--reps 5] [--out rates.json]"""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from fast3r_b200 import views  # noqa: E402
from tests import views_cases as VC  # noqa: E402
from tests import views_reference as R  # noqa: E402

HBM = 3.35e12


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else torch.cuda.get_device_name()


def inputs(n, w, h):
    rng = np.random.default_rng(w)
    return [[VC.raw_view(rng, w, h) for _ in range(n)]]


def device_bytes(samples, plans, uploads=True):
    """Bytes the device work reads and writes: each image's principal-point crop (read by the resampler, plus the
    copy of a crop narrower than its image), the 8-bit intermediate of the horizontal pass, the float32 image, and per
    output pixel one depth read, 12 + 1 + 4 bytes of points, mask and depth; the uploads of the source arrays."""
    total = 0
    for raw, ps in zip(samples, plans):
        for v, p in zip(raw, ps):
            h, w = v["depthmap"].shape
            l, t, r, b = p.crop
            cw, ch = r - l, b - t
            oh, ow = p.shape
            total += h * w * (3 + 4) if uploads else 0    # uploads land in device memory
            total += (2 if cw != w else 1) * ch * cw * 3   # crop copy (if strided) and the resampler's read
            total += 2 * ch * p.size[0] * 3                # horizontal pass: write and read of the intermediate
            total += oh * ow * (3 * 4 + 4 + 12 + 1 + 4)    # image, depth gather, points, mask, depth
    return total


def time_device(samples, res, reps, on_device=False):
    plans = [views._plan_sample(s, res, None, False) for s in samples]
    if on_device:
        samples = [[dict(v, img=torch.from_numpy(v["img"]).cuda(), depthmap=torch.from_numpy(v["depthmap"]).cuda())
                    for v in s] for s in samples]
    for _ in range(2):
        views.prepare_views(samples, plans=plans)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ms = []
    for _ in range(reps):
        ev[0].record()
        views.prepare_views(samples, plans=plans)
        ev[1].record()
        torch.cuda.synchronize()
        ms.append(ev[0].elapsed_time(ev[1]))
    return float(np.median(ms)), device_bytes(samples, plans, not on_device), plans


def time_host(samples, plans, threads):
    jobs = [(v, p) for raw, ps in zip(samples, plans) for v, p in zip(raw, ps)]
    t0 = time.perf_counter()
    if threads == 1:
        for v, p in jobs:
            R.host_view(v, p)
    else:
        with ThreadPoolExecutor(threads) as pool:
            list(pool.map(lambda j: R.host_view(*j), jobs))
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=32)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("view_rates needs a GPU")
    rows = []
    threads = min(32, os.cpu_count() or 4)
    for w, h in ((1920, 1440), (640, 480)):
        samples = inputs(a.views, w, h)
        ms, nbytes, plans = time_device(samples, (512, 384), a.reps)
        dms, dbytes, _ = time_device(samples, (512, 384), a.reps, on_device=True)
        row = dict(source=f"{w}x{h}", views=a.views, host_inputs_ms=ms, host_inputs_bytes=nbytes,
                   host_inputs_tbps=nbytes / ms / 1e9, device_inputs_ms=dms, device_inputs_bytes=dbytes,
                   device_inputs_tbps=dbytes / dms / 1e9, device_inputs_hbm_fraction=dbytes / dms / 1e9 / (HBM / 1e12),
                   host_1thread_ms=time_host(samples, plans, 1),
                   host_threads=threads, host_pool_ms=time_host(samples, plans, threads))
        rows.append(row)
        print(json.dumps(row))
    res = dict(card=card(), rows=rows)
    print(json.dumps(dict(card=res["card"])))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
