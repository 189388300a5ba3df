"""Reconstruction metrics without a GPU: fast3r_b200/csrc/pointcloud_math.h compiled for the host against scipy's cKDTree
(bit-exact distances) and numpy's eigh, the golden digests against the installed scipy, and the argument checks of the
new C-ABI entry points (which run before any CUDA call)."""
import ctypes as C
import hashlib
import json
import os
import shutil
import subprocess

import numpy as np
import pytest
from scipy.spatial import cKDTree

from tests.golden.recon_clouds import CASES, make_case

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "fast3r_b200", "csrc")
GOLDEN = os.path.join(HERE, "golden", "recon_metric.json")


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    so = str(tmp_path_factory.mktemp("pc") / "libpc_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I", CSRC,
                           os.path.join(HERE, "pointcloud_math_host.cpp"), "-o", so])
    lib = C.CDLL(so)
    lib.f3r_test_nearest.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    lib.f3r_test_normal.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    lib.f3r_test_morton.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_void_p]
    lib.f3r_test_dkey.argtypes, lib.f3r_test_dkey.restype = [C.c_double], C.c_uint64
    lib.f3r_test_dkey_inv.argtypes, lib.f3r_test_dkey_inv.restype = [C.c_uint64], C.c_double
    return lib


def nearest(lib, ref, query):
    ref = np.ascontiguousarray(ref, np.float64)
    query = np.ascontiguousarray(query, np.float64)
    d = np.empty(len(query))
    i = np.empty(len(query), np.int64)
    lib.f3r_test_nearest(ref.ctypes.data, len(ref), query.ctypes.data, len(query), d.ctypes.data, i.ctypes.data)
    return d, i


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_distance_rounding_is_scipys(hostlib, dtype):
    """The brute-force minimum of pc_dist2 is cKDTree.query's distance bit for bit, and its index wherever the nearest
    point is unique (scipy's k=2 query tells)."""
    rng = np.random.default_rng(5)
    for scale, offset in ((1.0, 0.0), (1e-3, 10.0), (50.0, -1e4)):
        ref = (rng.standard_normal((1500, 3)) * scale + offset).astype(dtype)
        query = (rng.standard_normal((3000, 3)) * scale * 1.2 + offset).astype(dtype)
        d, i = nearest(hostlib, ref, query)
        d2, i2 = cKDTree(ref).query(query, k=2)
        assert np.array_equal(d, d2[:, 0]), (scale, offset)
        unique = d2[:, 0] < d2[:, 1]
        assert np.array_equal(i[unique], i2[unique, 0])


def test_distance_rounding_on_fixture_clouds(hostlib):
    for kind, seed in CASES:
        gt, rec, _, _ = make_case(kind, seed)
        rec = rec[:2000]
        d, _ = nearest(hostlib, gt, rec)
        assert np.array_equal(d, cKDTree(gt).query(rec)[0]), kind


def test_eigen_solve_matches_eigh(hostlib):
    """Normal = smallest-eigenvalue eigenvector of the neighbourhood covariance: |dot| with numpy's >= 1 - 1e-12 where
    the gap to the middle eigenvalue is healthy."""
    rng = np.random.default_rng(6)
    checked = 0
    for trial in range(400):
        k = int(rng.integers(3, 33))
        a = rng.standard_normal((3, 3)) * np.array([1.0, rng.uniform(0.05, 1), rng.uniform(1e-4, 0.5)])
        pts = (rng.standard_normal((k, 3)) @ a + rng.standard_normal(3) * 10 ** rng.uniform(-2, 3))
        pts = np.ascontiguousarray(pts)
        n = np.empty(3)
        hostlib.f3r_test_normal(pts.ctypes.data, k, n.ctypes.data)
        c = np.cov(pts.T, bias=True)
        lam, vec = np.linalg.eigh(c)
        assert abs(np.linalg.norm(n) - 1) < 1e-12
        if lam[1] - lam[0] > 1e-3 * lam[2]:
            assert abs(n @ vec[:, 0]) >= 1 - 1e-12, (trial, n, vec[:, 0])
            checked += 1
    assert checked > 300
    for k in (0, 1, 2):
        n = np.empty(3)
        hostlib.f3r_test_normal(np.zeros(6).ctypes.data, k, n.ctypes.data)
        assert list(n) == [0.0, 0.0, 1.0]


def test_morton_keys_and_double_keys(hostlib):
    rng = np.random.default_rng(7)
    origin = np.zeros(3)
    hi, lo = C.c_uint64(), C.c_uint64()
    # the (hi, lo) order is the 33-bit-per-axis Morton order: compare with a direct interleave in Python
    for _ in range(200):
        p = np.ascontiguousarray(rng.random(3))
        hostlib.f3r_test_morton(p.ctypes.data, origin.ctypes.data, 1.0, C.byref(hi), C.byref(lo))
        c = [int(v * 2 ** 33) for v in p]
        code = 0
        for b in range(33):
            for a in range(3):
                code |= ((c[a] >> b) & 1) << (3 * b + 2 - a)
        assert (hi.value << 36 | lo.value) == code
    # clamped outside the cube, NaN to cell 0
    p = np.array([-5.0, 7.0, np.nan])
    hostlib.f3r_test_morton(p.ctypes.data, origin.ctypes.data, 1.0, C.byref(hi), C.byref(lo))
    assert hi.value == 0x1249249249249249 << 1 and lo.value == 0x249249249 << 1
    v = np.sort(np.concatenate([rng.standard_normal(500) * 10 ** rng.uniform(-300, 300, 500), [0.0, -0.0, np.inf, -np.inf]]))
    keys = [hostlib.f3r_test_dkey(float(x)) for x in v]
    assert all(a <= b for a, b in zip(keys, keys[1:]))
    assert all(hostlib.f3r_test_dkey_inv(k) == x for k, x in zip(keys, v))


def test_golden_digests_describe_installed_scipy():
    """The committed digests and metric values (written by the reference's recon_metric) are what scipy / numpy return
    here for the same seeded clouds."""
    with open(GOLDEN) as f:
        gold = json.load(f)
    assert [(c["kind"], c["seed"]) for c in gold["cases"]] == CASES
    for c in gold["cases"]:
        gt, rec, gn, rn = make_case(c["kind"], c["seed"])
        d_acc, i_acc = cKDTree(gt).query(rec)
        d_comp, i_comp = cKDTree(rec).query(gt)
        dig = lambda a: hashlib.sha256(np.ascontiguousarray(a, "<f8").tobytes()).hexdigest()  # noqa: E731
        assert dig(d_acc) == c["dist_accuracy_sha256"] and dig(d_comp) == c["dist_completion_sha256"], c["kind"]
        assert float(np.median(d_acc)) == c["accuracy"][1] and float(np.median(d_comp)) == c["completion"][1]
        assert float(np.mean((d_comp < 0.05).astype(np.float32))) == c["completion_ratio"]
        if gn is not None:
            nc1 = np.abs(np.sum(gn[i_acc] * rn, axis=-1))
            assert float(np.median(nc1)) == c["accuracy"][3]


def test_cabi_rejects_bad_arguments_before_any_cuda_call():
    from fast3r_b200 import lib as L
    lib = L.load()
    cases = [
        ("f3r_pc_index_build", (None, 0, 10, 256, 10 ** 9, None), "null operand"),
        ("f3r_pc_index_build", (256, 0, 0, 256, 10 ** 9, None), "bad size"),
        ("f3r_pc_index_build", (256, 0, 10, 256, 16, None), "index block too small"),
        ("f3r_pc_index_build", (256, 0, 10, 264, 10 ** 9, None), "not 256-byte aligned"),
        ("f3r_pc_nearest", (256, 10 ** 9, 10, None, 0, 5, 256, 256, 256, 10 ** 9, None), "null operand"),
        ("f3r_pc_nearest", (256, 10 ** 9, -1, 256, 0, 5, 256, 256, 256, 10 ** 9, None), "bad sizes"),
        ("f3r_pc_nearest", (256, 16, 10, 256, 0, 5, 256, 256, 256, 10 ** 9, None), "index block too small"),
        ("f3r_pc_nearest", (256, 10 ** 9, 10, 256, 0, 5, 256, 256, 256, 16, None), "workspace too small"),
        ("f3r_pc_nearest", (256, 10 ** 9, 10, 256, 0, 5, 256, 256, 260, 10 ** 9, None), "not 256-byte aligned"),
        ("f3r_pc_knn_normals", (256, 10 ** 9, 10, 33, 256, None), "must be in [1, 32]"),
        ("f3r_pc_knn_normals", (256, 10 ** 9, 10, 0, 256, None), "must be in [1, 32]"),
        ("f3r_pc_knn_normals", (None, 10 ** 9, 10, 30, 256, None), "null operand"),
        ("f3r_pc_knn_normals", (256, 16, 10, 30, 256, None), "index block too small"),
        ("f3r_pc_count_nonfinite", (256, 0, 10, None, None), "null operand"),
        ("f3r_pc_count_nonfinite", (256, 0, -1, 256, None), "bad size"),
        ("f3r_pc_abs_dot", (None, None, 256, None, 10, 256, None), "null operand"),
        ("f3r_pc_abs_dot", (256, None, 256, None, -2, 256, None), "bad size"),
        ("f3r_f64_mean", (256, 10, 256, None, 10 ** 6, None), "null operand"),
        ("f3r_f64_mean", (256, 0, 256, 256, 10 ** 6, None), "bad size"),
        ("f3r_f64_median", (256, 10, 256, 256, 8, None), "workspace too small"),
        ("f3r_f64_median", (256, 10, 256, 260, 10 ** 6, None), "not 256-byte aligned"),
        ("f3r_f64_count_below", (256, 10, None, 256, None), "null operand"),
        ("f3r_f64_count_below", (256, -3, 256, 256, None), "bad size"),
    ]
    for name, args, msg in cases:
        assert getattr(lib, name)(*args) != 0, name
        err = lib.f3r_last_error().decode()
        assert err.startswith(name) and msg in err, (name, err)
    # size queries are pure host functions
    assert lib.f3r_pc_index_workspace(0) == 0 and lib.f3r_pc_query_workspace(0) == 0
    assert lib.f3r_pc_index_workspace(1000) % 256 == 0 and lib.f3r_pc_index_workspace(2000) > lib.f3r_pc_index_workspace(1000)
    assert lib.f3r_f64_reduce_workspace() % 256 == 0


def test_python_entry_points_need_cuda_or_raise():
    """Without a CUDA device the drop-ins raise instead of computing on the host."""
    import torch
    from fast3r_b200 import recon_metric as rm
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    pts = np.zeros((4, 3))
    for fn in (lambda: rm.accuracy(pts, pts), lambda: rm.completion(pts, pts), lambda: rm.completion_ratio(pts, pts),
               lambda: rm.nearest_neighbors(pts, pts), lambda: rm.estimate_normals(pts)):
        with pytest.raises(RuntimeError, match="needs a CUDA device"):
            fn()
