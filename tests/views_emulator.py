"""CPU emulator of the device side of fast3r_b200.views, TEST INFRASTRUCTURE ONLY: ``view_geometry`` is
fast3r_b200.ops.view_geometry computed by a host build of the kernel's own per-pixel code
(fast3r_b200/csrc/views_math.h through tests/views_math_host.cpp), and ``resize_crop_rgb8`` is
fast3r_b200.ingest.resize_crop_rgb8 computed by the C restatement of Pillow's resampler (oracle/ingest_oracle.c).
``patch(monkeypatch)`` lets prepare_views run on host tensors, and the GPU tests have a host answer for every launch."""
import ctypes as C
import functools
import os
import subprocess
import tempfile

import numpy as np
import torch

from oracle import ingest_oracle
from tests.conftest import ROOT

CSRC = os.path.join(ROOT, "fast3r_b200", "csrc")


@functools.lru_cache(maxsize=1)
def host_lib():
    so = os.path.join(tempfile.mkdtemp(prefix="f3r_views_"), "views_math_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I", CSRC,
                           os.path.join(ROOT, "tests", "views_math_host.cpp"), "-o", so])
    lib = C.CDLL(so)
    P, I = C.c_void_p, C.c_int
    lib.f3r_test_nearest.argtypes = [I, I, P]
    lib.f3r_test_points.argtypes = [P, P, P, C.c_longlong, P, P, P, P, P]
    lib.f3r_test_view_geometry.argtypes = [P, I, P, P, P]
    lib.f3r_test_view_param_layout.argtypes = [P]
    return lib


def nearest(ssize, dsize):
    out = np.empty(dsize, np.int32)
    host_lib().f3r_test_nearest(ssize, dsize, out.ctypes.data)
    return out


def points(u, v, z, k4, pose):
    """(camera points, world points, valid) of pixels (u, v) at depths z, as the kernel computes them."""
    u, v = np.ascontiguousarray(u, np.int32), np.ascontiguousarray(v, np.int32)
    z = np.ascontiguousarray(z, np.float32)
    k4, pose = np.ascontiguousarray(k4, np.float32), np.ascontiguousarray(pose, np.float32)
    n = z.size
    cam, world, valid = np.empty((n, 3), np.float32), np.empty((n, 3), np.float32), np.empty(n, np.uint8)
    host_lib().f3r_test_points(u.ctypes.data, v.ctypes.data, z.ctypes.data, n, k4.ctypes.data, pose.ctypes.data,
                               cam.ctypes.data, world.ctypes.data, valid.ctypes.data)
    return cam, world, valid.astype(bool)


def param_layout():
    out = np.empty(19, np.int64)
    host_lib().f3r_test_view_param_layout(out.ctypes.data)
    return out


def view_geometry(params, out_pts, out_valid, out_depth):
    """ops.view_geometry on host tensors; the records' depth pointers point into host memory."""
    for t in (out_pts, out_valid, out_depth):
        assert t.device.type == "cpu" and t.is_contiguous()
    host_lib().f3r_test_view_geometry(params.ctypes.data, len(params), out_pts.data_ptr(), out_valid.data_ptr(),
                                      out_depth.data_ptr())


def resize_crop_rgb8(img_u8, nw, nh, filt, box, out=None):
    img = np.ascontiguousarray(img_u8.cpu().numpy())
    res = torch.from_numpy(ingest_oracle.crop_normalize(ingest_oracle.resize_rgb8(img, nw, nh, filt), box))
    if out is None:
        return res
    out.copy_(res)
    return out


def patch(monkeypatch):
    """Runs fast3r_b200.views.prepare_views(..., device="cpu") on this emulator."""
    from fast3r_b200 import ingest, ops, views
    monkeypatch.setattr(views, "_need_cuda", lambda device: None)
    monkeypatch.setattr(views, "_upload", lambda arr, device: torch.from_numpy(np.array(arr)))
    monkeypatch.setattr(ops, "view_geometry", view_geometry)
    monkeypatch.setattr(ingest, "resize_crop_rgb8", resize_crop_rgb8)
