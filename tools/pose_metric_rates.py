"""Times the camera-pose metric on one GPU and compares it with the reference's formula restated in torch
(tests/pose_metric_torch.py) on the host CPU and on cuda.  Prints the card and its power limit, then per size: the
kernel time (the device time torch.profiler records for the pm_* kernels of one ops.pose_metric call, counts only), the
per-call time of back-to-back ops.pose_metric calls (CUDA events; at these sizes bound by host dispatch: allocations, the
ctypes call, a memset and two launches), the wall time of cam_pose_metric.pose_counts with its
host copies (ending in a synchronise), the torch restatement's wall time on the CPU and on cuda, and how many counts
(of the PM_COUNTS row per item) the cuda restatement gets different from the CPU one.  With --out the rows also go to
that JSON file.

Run: python tools/pose_metric_rates.py [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from fast3r_b200 import cam_pose_metric as M  # noqa: E402
from fast3r_b200 import ops  # noqa: E402
from tests import pose_metric_cases as PC  # noqa: E402
from tests import pose_metric_torch as T  # noqa: E402

SIZES = [(1, 10), (1, 32), (1, 320), (1, 1000), (8, 32)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def wall(fn, reps):
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


def torch_counts(pred, gt):
    return torch.stack([T.counts(*(lambda e: (e["r"], e["t"], e["bad"]))(T.errors(p, g))) for p, g in zip(pred, gt)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "pose_metric_rates needs a GPU"
    rows = []
    info = {"card": card()}
    print(info)
    for items, n in SIZES:
        pred, gt = PC.pose_set(n, torch.float32)
        pred, gt = pred[None].repeat(items, 1, 1, 1).contiguous(), gt[None].repeat(items, 1, 1, 1).contiguous()
        pd, gd = pred.cuda(), gt.cuda()
        reps = 200 if n <= 320 else 50
        ops.pose_metric(pd, gd)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            ops.pose_metric(pd, gd)
        e1.record()
        torch.cuda.synchronize()
        per_call_ms = e0.elapsed_time(e1) / reps
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(20):
                ops.pose_metric(pd, gd)
            torch.cuda.synchronize()
        kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "pm_" in e.name]
        assert len(kern) == 40, [e.name for e in kern]
        kernel_us = sum(e.device_time for e in kern) / 20
        ours_host = wall(lambda: M.pose_counts(pred, gt), reps)
        ours_dev = wall(lambda: M.pose_counts(pd, gd), reps)
        cpu_reps = 3 if n >= 320 else 20
        t0 = time.perf_counter()
        for _ in range(cpu_reps):
            c_cpu = torch_counts(pred, gt)
        torch_cpu = (time.perf_counter() - t0) / cpu_reps
        torch_cuda = wall(lambda: torch_counts(pd, gd), cpu_reps)
        c_cuda = torch_counts(pd, gd)
        ours = M.pose_counts(pd, gd)[0]
        row = dict(items=items, views=n, pairs=items * n * (n - 1) // 2, kernel_us=kernel_us, per_call_ms=per_call_ms,
                   pose_counts_host_inputs_ms=ours_host * 1e3, pose_counts_device_inputs_ms=ours_dev * 1e3,
                   torch_cpu_ms=torch_cpu * 1e3, torch_cuda_ms=torch_cuda * 1e3,
                   ours_equal_torch_cpu=bool(torch.equal(ours, c_cpu)),
                   torch_cuda_counts_differing=int((c_cuda != c_cpu).sum()))
        rows.append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
