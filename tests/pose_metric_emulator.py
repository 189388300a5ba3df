"""CPU emulator of the camera-pose metric entry points of fast3r_b200.ops (pose_metric, pose_metric_counts), TEST
INFRASTRUCTURE ONLY: the same arguments and results, computed by a host build of the kernels' own math
(fast3r_b200/csrc/pose_metric_math.h through tests/pose_metric_host.cpp, g++ -ffp-contract=off), so the host side of
fast3r_b200.cam_pose_metric / postprocess.evaluate_camera_poses runs without a GPU and the GPU tests have a host answer
for every launch."""
import ctypes as C
import functools
import os
import subprocess
import tempfile

import torch

from fast3r_b200 import lib as L
from tests.conftest import ROOT

CSRC = os.path.join(ROOT, "fast3r_b200", "csrc")


@functools.lru_cache(maxsize=1)
def host_lib():
    so = os.path.join(tempfile.mkdtemp(prefix="f3r_pose_metric_"), "pose_metric_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I", CSRC,
                           os.path.join(ROOT, "tests", "pose_metric_host.cpp"), "-o", so])
    lib = C.CDLL(so)
    P = C.c_void_p
    lib.f3r_test_pose_metric.argtypes = [C.c_int, P, P, C.c_int, C.c_int, C.c_int, P, P, P, P, P]
    lib.f3r_test_pose_counts.argtypes = [C.c_int, P, P, C.c_longlong, C.c_int, P]
    lib.f3r_test_acos.argtypes = [C.c_int, P, C.c_longlong, P]
    return lib


def _host(t):
    return t.detach().cpu().contiguous()


def run(pred, gt, hist_max=30, angles=True, intermediates=False):
    """(counts int64 (items, PM_COUNTS), r, t, trace, acos argument of the translation angle), each (items, P) or None."""
    pred, gt = _host(pred), _host(gt)
    assert pred.dtype == gt.dtype and pred.dtype in (torch.float32, torch.float64)
    items, n = pred.shape[0], pred.shape[1]
    assert pred.shape == (items, n, 4, 4) == gt.shape and n >= 2
    pairs = n * (n - 1) // 2
    out = [torch.empty(items, pairs, dtype=pred.dtype) if on else None
           for on in (angles, angles, intermediates, intermediates)]
    counts = torch.empty(items, L.PM_COUNTS, dtype=torch.int64)
    ptr = lambda x: None if x is None else x.data_ptr()  # noqa: E731
    host_lib().f3r_test_pose_metric(int(pred.dtype == torch.float64), ptr(pred), ptr(gt), items, n, int(hist_max),
                                    *[ptr(x) for x in out], ptr(counts))
    return (counts, *out)


def pose_metric(pred, gt, hist_max=30, angles=False):
    counts, r, t, _, _ = run(pred, gt, hist_max, angles)
    return counts, r, t


def pose_metric_counts(r, t, hist_max=30):
    r, t = _host(r).reshape(-1), _host(t).reshape(-1)
    assert r.dtype == t.dtype and r.shape == t.shape
    counts = torch.empty(L.PM_COUNTS, dtype=torch.int64)
    host_lib().f3r_test_pose_counts(int(r.dtype == torch.float64), r.data_ptr(), t.data_ptr(), r.numel(), int(hist_max),
                                    counts.data_ptr())
    return counts


def acos(x):
    x = _host(x)
    out = torch.empty_like(x)
    host_lib().f3r_test_acos(int(x.dtype == torch.float64), x.data_ptr(), x.numel(), out.data_ptr())
    return out
