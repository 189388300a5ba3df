"""Wall time of estimate_camera_poses on 32 seeded views of 512x368 (tests/pose_plans.synth_preds(11, 32, 1, 368, 512),
the views of the goldens), two ways, alternated in one process:

  * cv2: fast_pnp's loop around cv2.solvePnPRansac (fast3r/dust3r/cloud_opt/init_im_poses.py:300-350) per view, the
    views on a thread pool as estimate_cam_pose_one_sample runs them - OpenCV on the host's cores;
  * gpu: fast3r_b200.poses.estimate_camera_poses (scoring and compaction on the GPU, EPnP / SQPnP on the host).

For `individual` with niter_PnP=10 and `first_view_from_global_head` with niter_PnP=100 it prints one JSON line per
run: wall seconds of each, the GPU time of the pnp_score launches (CUDA events), the host thread-seconds spent in the
EPnP hypotheses, in the SQPnP refits and in the RANSAC bookkeeping, whether both give the same poses, how many views
got a pose, and the card name, power limit and host core count read in the same run.
Run: python tools/pose_rates.py [--reps 2]
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from fast3r_b200 import ops  # noqa: E402
from fast3r_b200 import poses as PS  # noqa: E402
from fast3r_b200.postprocess import estimate_focal  # noqa: E402
from tests import pose_plans as PP  # noqa: E402


class Clock:
    """Thread-seconds per label, summed over the threads of the pool."""

    def __init__(self):
        self.t, self.lock = {}, threading.Lock()

    def wrap(self, label, fn):
        def timed(*a, **k):
            t0 = time.perf_counter()
            try:
                return fn(*a, **k)
            finally:
                with self.lock:
                    self.t[label] = self.t.get(label, 0.0) + time.perf_counter() - t0
        return timed


def cv2_poses(preds, niter, mode):
    """The host way: per view fast_pnp's loop around cv2.solvePnPRansac, views on a thread pool."""
    focal = None
    if mode == "first_view_from_global_head":
        focal = estimate_focal(preds[0]["pts3d_in_other_view"][0:1], preds[0]["conf"][0:1], min_conf_thr_percentile=10)
    H, W = preds[0]["conf"].shape[1:]
    pixels = np.mgrid[:W, :H].T.astype(np.float32)

    def view(p):
        msk = p["conf"][0].numpy() > 1.0
        job = PS._Job(PS._tentative_focals(focal, H, W, 100), (W / 2, H / 2), niter)
        return PS._reference_loop(p["pts3d_in_other_view"][0].numpy()[msk], pixels[msk], job, "cpu")

    with ThreadPoolExecutor() as ex:
        return list(ex.map(view, preds))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "pose_rates measures the GPU path: no CUDA device"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    preds = PP.synth_preds(11, 32, 1, 368, 512)

    clock = Clock()
    events = []
    score = ops.pnp_score

    def timed_score(*a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = score(*a, **k)
        e1.record()
        events.append((e0, e1))
        return out

    ops.pnp_score = timed_score
    PS._epnp = clock.wrap("epnp", PS._epnp)
    PS.ransac_replay = clock.wrap("bookkeeping", PS.ransac_replay)
    cv2 = PS._cv2()

    class Cv2:  # cv2 with the SQPnP refits timed
        def __getattr__(self, name):
            return getattr(cv2, name)

        def solvePnP(self, *a, flags=None, **k):
            f = cv2.solvePnP if flags != cv2.SOLVEPNP_SQPNP else clock.wrap("sqpnp", cv2.solvePnP)
            return f(*a, flags=flags, **k)

    proxy = Cv2()
    PS._cv2 = lambda: proxy

    PS.estimate_camera_poses([dict(p) for p in preds], niter_PnP=1)  # warm-up: library load, allocator
    for mode, niter in (("individual", 10), ("first_view_from_global_head", 100)):
        for rep in range(args.reps):
            t0 = time.perf_counter()
            want = cv2_poses(preds, niter, mode)
            t_cv2 = time.perf_counter() - t0
            clock.t.clear()
            events.clear()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            poses, focals = PS.estimate_camera_poses([dict(p) for p in preds], niter_PnP=niter,
                                                     focal_length_estimation_method=mode)
            torch.cuda.synchronize()
            t_gpu = time.perf_counter() - t0
            same = all((w[1] is None and f is None) or (w[0] == f and np.array_equal(w[1].numpy(), p))
                       for w, p, f in zip(want, poses[0], focals[0]))
            print(json.dumps({
                "mode": mode, "niter_PnP": niter, "rep": rep, "views": len(preds), "hw": [368, 512],
                "cv2_wall_s": round(t_cv2, 3), "gpu_wall_s": round(t_gpu, 3),
                "pnp_score_gpu_ms": round(sum(a.elapsed_time(b) for a, b in events), 3),
                "host_thread_s": {k: round(v, 3) for k, v in sorted(clock.t.items())},
                "same_poses": same, "views_posed": sum(f is not None for f in focals[0]),
                "focal": None if mode == "individual" else focals[0][0], "card": smi, "host_cores": os.cpu_count(),
                "cv2": cv2.__version__}), flush=True)


if __name__ == "__main__":
    main()
