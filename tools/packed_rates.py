"""Scenes per second of (a) a loop of inference() over K scenes and (b) one inference_many() over the same scenes,
alternated in one process, with the largest difference between the two over all views (relative L2 per view and output).

Scenes are seeded and synthetic: view counts drawn from 1..8 and one shape per scene from 368x512, 384x512 and 512x384,
random-init ViT-L, bf16.  Every shape is warmed up by one untimed pass of each path.  Prints one JSON line (the card,
its power limit and SM clock are read in the same run) and writes it to --out if given.

    python tools/packed_rates.py --scenes 32 --rounds 3
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = [(368, 512), (384, 512), (512, 384)]


def card():
    info = {"name": torch.cuda.get_device_name()}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        info["power_limit"], info["sm_clock"], info["sm_clock_max"] = [s.strip() for s in q.stdout.split(",")]
    except Exception as e:  # noqa: BLE001 - report what could not be read rather than fail the measurement
        info["nvidia_smi"] = f"unavailable: {e}"
    return info


def make_scenes(k, seed):
    import numpy as np
    from tests.golden.synth import synth_images
    rnd = random.Random(seed)
    scenes = []
    for s in range(k):
        n, (h, w) = rnd.randint(1, 8), rnd.choice(SHAPES)
        imgs = synth_images(n, 1, h, w, seed0=10000 + 100 * s)
        scenes.append([dict(img=im.pin_memory(), true_shape=np.int32([[h, w]]), idx=i, instance=str(i))
                       for i, im in enumerate(imgs)])
    return scenes


def fresh(scenes):
    """inference() adds keys to the view dicts: every call gets its own dicts over the same image tensors."""
    return [[dict(v) for v in views] for views in scenes]


def rel_l2(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("packed_rates.py measures on the GPU; no CUDA device found")
    from fast3r_b200 import Fast3R, inference, inference_many, vit_large_args
    torch.manual_seed(0)
    with torch.device("cuda"):
        model = Fast3R(*vit_large_args()).eval()
    scenes = make_scenes(args.scenes, args.seed)
    dev, dt = torch.device("cuda"), torch.bfloat16

    def loop():
        return [inference(v, model, dev, dt, verbose=False) for v in fresh(scenes)]

    def packed():
        return inference_many(fresh(scenes), model, dev, dt, verbose=False)

    def timed(fn):
        torch.manual_seed(1)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, out

    timed(loop)
    timed(packed)  # warm-up: every shape, both paths
    t_loop, t_packed = [], []
    for _ in range(args.rounds):
        t, a = timed(loop)
        t_loop.append(t)
        t, b = timed(packed)
        t_packed.append(t)
    worst = {}
    for ra, rb in zip(a, b):
        for pa, pb in zip(ra["preds"], rb["preds"]):
            for k in pa:
                worst[k] = max(worst.get(k, 0.0), rel_l2(pb[k], pa[k]))
    views = sum(len(s) for s in scenes)
    res = dict(
        card=card(), scenes=args.scenes, views=views, rounds=args.rounds, precision="bf16",
        view_counts=[len(s) for s in scenes], shapes={f"{h}x{w}": sum(1 for s in scenes if tuple(s[0]["img"].shape[-2:]) == (h, w))
                                                     for h, w in SHAPES},
        loop_s=t_loop, packed_s=t_packed,
        loop_scenes_per_s=[args.scenes / t for t in t_loop], packed_scenes_per_s=[args.scenes / t for t in t_packed],
        speedup_median=sorted(t_loop)[len(t_loop) // 2] / sorted(t_packed)[len(t_packed) // 2],
        max_view_rel_l2_packed_vs_loop=worst)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
