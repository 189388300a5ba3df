"""CPU emulator of fast3r_b200.ops.val_loss, TEST INFRASTRUCTURE ONLY: the same arguments and result, computed by a host
build of the kernels' own per-pixel math (fast3r_b200/csrc/val_loss_math.h through tests/val_loss_host.cpp), so
fast3r_b200.losses runs without a GPU and the GPU tests have a host answer for every launch.  The float64 sums are
taken sequentially here and in a fixed tree order on the GPU, and logf / log1pf come from different libraries, so the
two agree to rounding, not bit for bit."""
import ctypes as C
import functools
import os
import subprocess
import tempfile

import torch

from tests.conftest import ROOT

CSRC = os.path.join(ROOT, "fast3r_b200", "csrc")
SUMS = 5


@functools.lru_cache(maxsize=1)
def host_lib():
    so = os.path.join(tempfile.mkdtemp(prefix="f3r_val_loss_"), "val_loss_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", CSRC,
                           os.path.join(ROOT, "tests", "val_loss_host.cpp"), "-o", so])
    lib = C.CDLL(so)
    P, I = C.c_void_p, C.c_int
    lib.f3r_test_val_loss.argtypes = [P, P, P, P, P, P, P, I, I, I, C.c_float, I, I, I, P, P]
    lib.f3r_test_val_loss_inverse.argtypes = [P, C.c_longlong, P]
    return lib


def _host(t):
    return None if t is None else t.detach().cpu().contiguous()


def run(gt, valid, pr, conf, poses, pr_local=None, conf_local=None, alpha=1.0, log1p=False, gt_scale=False,
        local_scale_consistent=False):
    """(sums float64 [views, items, 5] as ops.val_loss returns them, [views, items, 4] sums of |d| and
    |d c - alpha log c| of the global and the local term)."""
    gt, valid, pr, conf, poses, pr_local, conf_local = map(_host, (gt, valid, pr, conf, poses, pr_local, conf_local))
    views, items, n = valid.shape
    assert valid.dtype == torch.uint8 and gt.shape == pr.shape == (views, items, n, 3) and conf.shape == valid.shape
    assert poses.shape == (views, items, 4, 4) and (pr_local is None) == (conf_local is None)
    out = torch.empty(views, items, SUMS, dtype=torch.float64)
    mags = torch.empty(views, items, 4, dtype=torch.float64)
    ptr = lambda x: None if x is None else x.data_ptr()  # noqa: E731
    host_lib().f3r_test_val_loss(ptr(gt), ptr(valid), ptr(pr), ptr(pr_local), ptr(conf), ptr(conf_local), ptr(poses),
                                 views, items, n, float(alpha), int(log1p), int(gt_scale), int(local_scale_consistent),
                                 ptr(out), ptr(mags))
    return out, mags


def val_loss(gt, valid, pr, conf, poses, pr_local=None, conf_local=None, alpha=1.0, log1p=False, gt_scale=False,
             local_scale_consistent=False):
    return run(gt, valid, pr, conf, poses, pr_local, conf_local, alpha, log1p, gt_scale, local_scale_consistent)[0]


def inverse(m):
    m = _host(m).float()
    out = torch.empty_like(m)
    host_lib().f3r_test_val_loss_inverse(m.data_ptr(), m.numel() // 16, out.data_ptr())
    return out
