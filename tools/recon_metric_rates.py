"""Times the reconstruction metrics on the GPU (fast3r_b200.recon_metric) against scipy's cKDTree (workers = all host
cores) in the same process, on the same seeded depth-map clouds: N views of 512x368 for the ground truth and for the
reconstruction (N = 8 / 32 / 320 by default).  Prints one JSON document (with the card's name, power limit and SM clock
read in the same run); writes a file only with --out.

    python tools/recon_metric_rates.py [--views 8 32 320] [--scipy-max-views 320] [--repeats 3] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def clouds(views: int, seed: int, h: int = 368, w: int = 512):
    """Two depth-map-like clouds (ground truth, reconstruction) of `views` back-projected wavy surfaces, fp32."""
    rng = np.random.default_rng(seed)
    v, u = np.meshgrid(np.linspace(-0.75, 0.75, h, dtype=np.float32), np.linspace(-1, 1, w, dtype=np.float32),
                       indexing="ij")
    out = []
    for side in range(2):
        pts = np.empty((views, h * w, 3), np.float32)
        for k in range(views):
            z = 2 + 0.3 * np.sin(3 * u + 0.37 * k) * np.cos(2 * v) + 0.01 * rng.standard_normal((h, w), dtype=np.float32)
            ang = 0.05 * k
            x = u * z
            pts[k, :, 0] = (np.cos(ang) * x + np.sin(ang) * z).reshape(-1)
            pts[k, :, 1] = (v * z).reshape(-1)
            pts[k, :, 2] = (-np.sin(ang) * x + np.cos(ang) * z).reshape(-1) + 0.002 * side
        out.append(pts.reshape(-1, 3))
    return out


def gpu_time(fn, repeats):
    ts = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return min(ts), r


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, nargs="+", default=[8, 32, 320])
    ap.add_argument("--scipy-max-views", type=int, default=320)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from scipy.spatial import cKDTree
    from fast3r_b200 import ops, recon_metric as rm
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    rows = []
    for views in a.views:
        gt_h, rec_h = clouds(views, seed=views)
        gt, rec = torch.from_numpy(gt_h).to(dev), torch.from_numpy(rec_h).to(dev)
        row = {"views": views, "points_per_cloud": int(gt.shape[0])}
        rm.accuracy(gt, rec)  # warm-up of every kernel at this size
        t_build, ix = gpu_time(lambda: ops.pc_index(gt), a.repeats)
        t_query, (d_acc, _) = gpu_time(lambda: ops.pc_nearest(ix, rec), a.repeats)
        t_comp, _ = gpu_time(lambda: ops.pc_nearest(ops.pc_index(rec), gt), a.repeats)
        t_metrics, acc = gpu_time(lambda: (rm.accuracy(gt, rec), rm.completion(gt, rec)), a.repeats)
        t_normals, _ = gpu_time(lambda: (rm.estimate_normals(gt), rm.estimate_normals(rec)), 1)
        row["gpu_s"] = {"index_build": t_build, "accuracy_query": t_query, "completion_build_query": t_comp,
                        "accuracy_plus_completion_with_reductions": t_metrics, "normals_both_clouds_k30": t_normals}
        del ix
        if views <= a.scipy_max_views:
            t0 = time.perf_counter()
            tree = cKDTree(gt_h)
            t1 = time.perf_counter()
            d_ref, _ = tree.query(rec_h, workers=-1)
            t2 = time.perf_counter()
            cKDTree(rec_h).query(gt_h, workers=-1)
            t3 = time.perf_counter()
            row["scipy_s"] = {"index_build": t1 - t0, "accuracy_query": t2 - t1, "completion_build_query": t3 - t2,
                              "total": t3 - t0}
            row["distances_bit_equal"] = bool(np.array_equal(d_acc.cpu().numpy(), d_ref))
            row["speedup_total"] = (t3 - t0) / (t_build + t_query + t_comp)
            del tree
        rows.append(row)
        print(json.dumps(row), file=sys.stderr)
        del gt, rec
        torch.cuda.empty_cache()
    doc = {"card": card(), "host_cores": os.cpu_count(), "rows": rows}
    s = json.dumps(doc, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
