"""Times the validation criterion on one GPU and compares it with the reference's formula restated in torch
(tests/val_loss_torch.py, float32) on the same device.  Prints the card and its power limit, then per size (one item of
N views of 368x512, with and without the local head):
  * kernel: the device time torch.profiler records for the three vl_* kernels of one ops.val_loss call;
  * bytes moved over that time, against the H100 SXM's 3.35 TB/s: pass 1 reads points, validity and predictions, pass 2
    reads them again with the confidences (37 + 45 bytes per pixel with the local head, 25 + 29 without);
  * call: CUDA events around back-to-back ops.val_loss calls on stacked maps; dispatch: the host time of one call;
  * criterion: ConfLossMultiviewV2 on device preds, wall clock ending in its one synchronise (stacking included);
  * torch: the restated formula on cuda, wall clock with a synchronise.
With --out the rows also go to that JSON file.

Run: python tools/val_loss_rates.py [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from fast3r_b200 import losses as LS  # noqa: E402
from fast3r_b200 import ops  # noqa: E402
from tests import val_loss_cases as VC  # noqa: E402
from tests import val_loss_torch as VT  # noqa: E402

H, W = 368, 512
PEAK = 3.35e12


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


def device_inputs(views, local):
    """Seeded inputs made on the device (the host generator of tests/val_loss_cases is slow at 320 views)."""
    base_v, base_p = VC.make(1, 2, H, W, local, seed=5)
    views_out, preds_out = [], []
    for i in range(views):
        v, p = base_v[i % 2], base_p[i % 2]
        s = 1 + 0.01 * i
        views_out.append({k: (t * s if t.is_floating_point() and k == "pts3d" else t).cuda() for k, t in v.items()})
        preds_out.append({k: (t * s if k.startswith("pts3d") else t).cuda() for k, t in p.items()})
    return views_out, preds_out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    print("card:", card())
    crit = LS.ConfLossMultiviewV2(LS.Regr3DMultiviewV4(LS.L21Loss(), norm_mode="avg_dis"), alpha=VC.ALPHA)
    rows = []
    for views in (32, 320):
        for local in (True, False):
            gts, preds = device_inputs(views, local)
            m = LS.stack_maps(gts, preds, torch.device("cuda"))
            call = lambda: ops.val_loss(**m, alpha=VC.ALPHA)  # noqa: E731
            call()
            torch.cuda.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    call()
                torch.cuda.synchronize()
            kern = sum(e.device_time_total for e in prof.key_averages() if "vl_" in e.key) / 5 * 1e-6
            reps = 50
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                call()
            e1.record()
            torch.cuda.synchronize()
            per_call = e0.elapsed_time(e1) / reps * 1e-3
            t0 = time.perf_counter()
            for _ in range(reps):
                call()
            dispatch = (time.perf_counter() - t0) / reps
            torch.cuda.synchronize()
            crit_t = wall(lambda: crit(gts, preds), 10)
            torch_t = wall(lambda: VT.view_sums(gts, preds, VC.ALPHA, dtype=torch.float32), 3)
            pixels = views * H * W
            nbytes = pixels * ((37 + 45) if local else (25 + 29))
            row = dict(views=views, local=local, kernel_ms=kern * 1e3, gbytes=nbytes / 1e9,
                       tb_per_s=nbytes / kern / 1e12, of_peak=nbytes / kern / PEAK, call_ms=per_call * 1e3,
                       dispatch_us=dispatch * 1e6, criterion_ms=crit_t * 1e3, torch_cuda_ms=torch_t * 1e3)
            print(json.dumps(row))
            rows.append(row)
            del gts, preds, m
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=card(), rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
