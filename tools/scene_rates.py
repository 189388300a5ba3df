"""Times the viewer scene: fast3r_b200.scene.prepare_scene plus the launch state's visible points and PLY bytes, against
the numpy / cv2 / scipy host loop of the reference viewer (restated in tests/scene_oracle.py) on the same seeded frames
of 512 x 368, and checks that both give the same PLY bytes.

    python tools/scene_rates.py [--frames 32 320] [--repeats 3]

GPU times are a host clock around work that ends in a device synchronise (inputs already on the device); the card
and its power limit are printed with them."""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from fast3r_b200 import scene as S  # noqa: E402
from tests import scene_cases as SC  # noqa: E402
from tests import scene_oracle as O  # noqa: E402


def card() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def gpu_path(out):
    """PLY bytes of the launch state, and the seconds of each stage (each ends in a device synchronise)."""
    t0 = time.perf_counter()
    sc = S.prepare_scene(out)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    pts, cols = sc.visible_points()
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    ply = S.ply_bytes(pts, cols)
    t3 = time.perf_counter()
    return ply, (t1 - t0, t2 - t1, t3 - t2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[32, 320])
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "scene_rates needs a GPU"
    print(f"card: {card()}")
    for n in a.frames:
        host = SC.synth_output(0, [(368, 512)] * n)
        dev = {k: [{kk: vv.cuda() for kk, vv in d.items()} for d in v] for k, v in host.items()}
        torch.cuda.synchronize()
        gpu_path(dev)  # warm-up of every shape
        times, stages = [], []
        for _ in range(a.repeats):
            torch.cuda.synchronize()
            t = time.perf_counter()
            ply, st = gpu_path(dev)
            times.append(time.perf_counter() - t)
            stages.append(st)
        t = time.perf_counter()
        ref = O.prepare_scene(host)
        rp, rc = O.visible_points(ref)
        ref_ply = O.ply_bytes(rp, rc)
        host_s = time.perf_counter() - t
        assert ply == ref_ply, f"N={n}: the GPU and host PLY bytes differ"
        best = stages[int(np.argmin(times))]
        print(f"N={n} 512x368: GPU prepare_scene + launch-state ply_bytes min {min(times) * 1e3:.1f} ms "
              f"(runs {', '.join(f'{x * 1e3:.1f}' for x in times)} ms; fastest run: prepare_scene {best[0] * 1e3:.1f}, "
              f"visible_points {best[1] * 1e3:.1f}, ply_bytes {best[2] * 1e3:.1f} ms); host loop {host_s:.2f} s; "
              f"PLY {len(ply) / 1e6:.1f} MB, identical")


if __name__ == "__main__":
    main()
