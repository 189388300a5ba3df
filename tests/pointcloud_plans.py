"""Launch keys of the reconstruction metrics (fast3r_b200/csrc/pointcloud.cu), for the tests: which code runs for a call
of the index build, the nearest-neighbour query, the kNN normals and the reductions, the seeded clouds the cases run on,
and the table of GPU cases that tests/test_pointcloud_plans_gpu.py runs and tests/test_pointcloud_plans_cpu.py checks
the recon_metric callers against.

A call is a plain dict ("descriptor") with its op and what decides the code path; the descriptor of a call is read off
its operands by the functions `*_desc` below, so the CPU test, the GPU test and the case table all derive it the same
way.  Each key function restates the launcher's branches and cites the lines of pointcloud.cu it restates."""
import numpy as np

PC_LEAF = 32         # points per bucket: pointcloud.cu:19
PC_FAN = 8           # children per parent: :20
STILE = 256 * 16     # keys per radix-sort tile: :26-28
SCAN_T = 1024        # threads of the one-CTA scan: :220
BBOX_CAP = 1024      # bounding-box blocks of 256 threads: :733
RED = 256 * 256      # RED_BLOCKS x RED_T, the mean's grid: :561
RED_CAP = 1024 * 256  # blocks x threads of the capped reduction grids: :807, :821, :786
CELLS = 2.0 ** 33    # Morton cells per axis: pointcloud_math.h:47


def _flags(*pairs):
    return "".join(" " + f for f, on in pairs if on)


def tree_counts(n):
    """Nodes per level, buckets first (make_tree, :39-53)."""
    c, out = (n + PC_LEAF - 1) // PC_LEAF, []
    while True:
        out.append(c)
        if c <= 1:
            return out
        c = (c + PC_FAN - 1) // PC_FAN


def sort_tiles(n):
    return (n + STILE - 1) // STILE


# ------------------------------------------------------------------------------------------------ Morton keys (numpy)
def _spread3(v):
    v = v & np.uint64(0x1fffff)
    for s, m in ((32, 0x1f00000000ffff), (16, 0x1f0000ff0000ff), (8, 0x100f00f00f00f00f), (4, 0x10c30c30c30c30c3),
                 (2, 0x1249249249249249)):
        v = (v | (v << np.uint64(s))) & np.uint64(m)
    return v


def header(ref):
    """(origin, inv_extent, extents) of the index over ref (float64 (n, 3)), as pc_bbox_finish_kernel (:150-159)."""
    lo, hi = ref.min(0), ref.max(0)
    ext = hi - lo
    e = float(ext.max())
    return lo, (1.0 / e if e > 0.0 else 0.0), ext


def morton_hi(p, origin, inv_extent):
    """The 63-bit key of every point of p (pointcloud_math.h:45-58): cells clamped to the cube, NaN to cell 0."""
    h = np.zeros(len(p), np.uint64)
    with np.errstate(invalid="ignore", over="ignore"):
        for a in range(3):
            t = (p[:, a] - origin[a]) * inv_extent * CELLS
            c = np.zeros(len(p), np.uint64)
            top = t >= CELLS - 1.0
            mid = ~top & (t > 0.0)
            c[top] = np.uint64((1 << 33) - 1)
            c[mid] = t[mid].astype(np.uint64)
            h |= _spread3(c >> np.uint64(12)) << np.uint64(2 - a)
    return h


# ------------------------------------------------------------------------------------------------ descriptors
def index_desc(ref):
    ref = np.asarray(ref)
    r = ref.astype(np.float64)
    _, inv, ext = header(r)
    return dict(op="index", n=len(r), f64=ref.dtype == np.float64, flat=inv == 0.0,
                flat_axis=inv != 0.0 and bool((ext == 0.0).any()))


def nearest_desc(ref, query):
    ref, query = np.asarray(ref), np.asarray(query)
    d = dict(op="nearest", n_ref=len(ref), nq=len(query), f64_index=ref.dtype == np.float64,
             f64_query=query.dtype == np.float64, outside=False, past=False)
    if len(ref) and len(query):
        r, q = ref.astype(np.float64), query.astype(np.float64)
        origin, inv, ext = header(r)
        e = float(ext.max())
        d["outside"] = bool(((q < origin) | (q > origin + e)).any())
        d["past"] = bool(morton_hi(q, origin, inv).max() > morton_hi(r, origin, inv).max())
    return d


def knn_desc(n, k):
    return dict(op="knn", n=n, k=k)


def mean_desc(n):
    return dict(op="mean", n=n)


def median_desc(x):
    x = np.asarray(x, np.float64)
    n = len(x)
    s = np.sort(x[~np.isnan(x)])
    tie = n % 2 == 0 and not np.isnan(x).any() and s[n // 2 - 1] == s[n // 2]
    return dict(op="median", n=n, tie=bool(tie), nan=bool(np.isnan(x).any()))


def count_below_desc(n):
    return dict(op="count_below", n=n)


def nonfinite_desc(pts):
    pts = np.asarray(pts)
    return dict(op="nonfinite", n=len(pts), f64=pts.dtype == np.float64)


def abs_dot_desc(n, a_idx, b_idx):
    return dict(op="abs_dot", n=n, a_idx=a_idx, b_idx=b_idx)


# ------------------------------------------------------------------------------------------------ keys
def index_key(d):
    """launch_pc_index_build (:721-754): pc_bbox_kernel on min(ceil(n / 256), 1024) blocks (:733); the radix sorts run
    ceil(n / 4096) tiles (:311), and the one-CTA scan over 256 tiles digits loops per thread past 4 tiles (:226); the
    last bucket holds n % 32 points (:341), a level of c nodes ends in a partial parent when c % 8 != 0 (:360); a zero
    extent gives inv_extent = 0 and every key 0 (:158), a zero extent on some axes collapses those bits only."""
    n, cnt = d["n"], tree_counts(d["n"])
    ppart = any(c % PC_FAN for c in cnt[:-1])
    return f"index {'f64' if d['f64'] else 'f32'} L{len(cnt)}" + _flags(
        ("small", n < PC_LEAF), ("partial", n % PC_LEAF != 0), ("ppart", ppart), ("tiles", sort_tiles(n) > 1),
        ("scanloop", sort_tiles(n) * 256 > SCAN_T), ("bboxcap", (n + 255) // 256 > BBOX_CAP), ("flat", d["flat"]),
        ("flataxis", d["flat_axis"]))


def nearest_key(d):
    """launch_pc_nearest (:756-774): an empty reference fills inf / n_ref (:758, pc_fill_empty_kernel); else the queries
    are converted as their dtype (load_pt, :106-114) against an index of its own dtype, sorted in ceil(nq / 4096) tiles
    (:771), their keys clamped to the index cube (pointcloud_math.h:51-52), and a key past every index key clamps the
    bucket search to the last bucket (:482)."""
    if d["n_ref"] == 0:
        return "nearest empty"
    return f"nearest {'f64' if d['f64_index'] else 'f32'}x{'f64' if d['f64_query'] else 'f32'}" + _flags(
        ("tiles", sort_tiles(d["nq"]) > 1), ("outside", d["outside"]), ("past", d["past"]))


def knn_key(d):
    """launch_pc_knn_normals (:776-779) and pc_knn_normals_kernel (:510-558): the heap holds min(k, n) points (:519),
    fewer than 3 give (0, 0, 1) (pointcloud_math.h:92), k = 32 fills the 32-entry heap (:515-516); the first bucket
    scanned is the point's own (:549-550), and the last one holds n % 32 points, fewer than k when k > n % 32."""
    n, k = d["n"], d["k"]
    last = n - PC_LEAF * (tree_counts(n)[0] - 1)
    return "knn" + _flags(("k<3", k < 3), ("k32", k == 32), ("k>n", k > n), ("k=n", k == n), ("spill", last < k))


def mean_key(d):
    """launch_f64_mean (:796-801): a fixed grid of 256 x 256 threads, each striding past 65 536 elements (:566)."""
    return "mean" + _flags(("one", d["n"] == 1), ("stride", d["n"] > RED))


def median_key(d):
    """launch_f64_median (:803-816): odd n returns the selected key (:673); even n runs sel_succ_kernel (:814) and takes
    the selected key twice when more than n / 2 elements are <= it (:677); the grids cap at 1024 blocks (:807); a NaN
    anywhere makes the result NaN (flagged in sel_hist_kernel's first pass, :620 and :624, returned at :668-671)."""
    n = d["n"]
    return "median" + _flags(("odd", n % 2 == 1), ("even", n % 2 == 0), ("tie", d["tie"]), ("cap", n > RED_CAP),
                             ("nan", d["nan"]))


def count_below_key(d):
    """launch_f64_count_below (:818-822): min(ceil(n / 256), 1024) blocks (:821)."""
    return "count_below" + _flags(("cap", d["n"] > RED_CAP))


def nonfinite_key(d):
    """launch_pc_count_nonfinite (:781-788): 3n values on min(ceil(3n / 256), 1024) blocks, as their dtype."""
    return f"nonfinite {'f64' if d['f64'] else 'f32'}" + _flags(("cap", 3 * d["n"] > RED_CAP))


def abs_dot_key(d):
    """launch_pc_abs_dot (:790-794): a_idx / b_idx gather their row or take row i (:708-709); ceil(n / 256) blocks."""
    return "abs_dot" + _flags(("aidx", d["a_idx"]), ("bidx", d["b_idx"]), ("partial", d["n"] % 256 != 0))


KEYS = dict(index=index_key, nearest=nearest_key, knn=knn_key, mean=mean_key, median=median_key,
            count_below=count_below_key, nonfinite=nonfinite_key, abs_dot=abs_dot_key)


def key(d):
    return KEYS[d["op"]](d)


# ------------------------------------------------------------------------------------------------ seeded clouds
def cloud(geometry, n, seed):
    """float64 (n, 3) reference cloud of a geometry:
    gauss      standard normal
    plane      z = 0 exactly, x, y uniform
    line       collinear: t (1, 2, -0.5), t uniform
    lattice    integer lattice points (ties everywhere), n taken in raster order of a 64 x 64 x m block
    same       all points equal
    cluster    a unit cluster with 1 % of its points as outliers at 1e6 (the 36-bit low key decides the order)
    geo        georeferenced-style: 1e7 + uniform(-1e-3, 1e-3) per axis
    huge       coordinates near 1e160: squared distances overflow to inf
    tiny       coordinates near 1e-170: squared distances underflow to 0
    subnorm    coordinates near 1e-161: squared distances in the subnormal range"""
    rng = np.random.default_rng(seed)
    if geometry == "gauss":
        return rng.standard_normal((n, 3))
    if geometry == "plane":
        return np.concatenate([rng.uniform(-1, 1, (n, 2)), np.zeros((n, 1))], 1)
    if geometry == "line":
        return rng.uniform(-1, 1, (n, 1)) * np.array([1.0, 2.0, -0.5])
    if geometry == "lattice":
        i = np.arange(n)
        return np.stack([i % 64, (i // 64) % 64, i // 4096], 1).astype(np.float64)
    if geometry == "same":
        return np.tile(np.array([[0.25, -3.5, 7.0]]), (n, 1))
    if geometry == "cluster":
        p = rng.standard_normal((n, 3)) * 0.3
        m = rng.random(n) < 0.01
        p[m] = rng.uniform(-1e6, 1e6, (int(m.sum()), 3))
        return p
    if geometry == "geo":
        return 1e7 + rng.uniform(-1e-3, 1e-3, (n, 3))
    if geometry == "huge":
        return rng.standard_normal((n, 3)) * 1e160
    if geometry == "tiny":
        return rng.standard_normal((n, 3)) * 1e-170
    if geometry == "subnorm":
        return rng.standard_normal((n, 3)) * 1e-161
    raise ValueError(geometry)


def queries(ref, nq, mode, seed):
    """float64 (nq, 3) queries for a reference cloud: reference points jittered by 1 % of the cloud's spread, every
    eighth one on a reference point exactly.  "in" clips them to the index cube; "near" leaves them and puts the first
    just below the cube's low corner; "far" puts a quarter up to 10 spreads outside the cube on every side and one 10
    spreads past its high corner (clamped keys, and a key past every index key).  An empty cloud gets gaussian queries."""
    rng = np.random.default_rng(seed)
    if len(ref) == 0:
        return rng.standard_normal((nq, 3))
    lo, hi = ref.min(0), ref.max(0)
    spread = max(float((hi - lo).max()), float(np.abs(ref).max()) * 1e-3, np.finfo(np.float64).tiny)
    pick = rng.integers(0, len(ref), nq)
    q = ref[pick] + rng.standard_normal((nq, 3)) * (0.01 * spread)
    q[::8] = ref[pick[::8]]
    if mode == "in":  # a margin keeps the float32 rounding of a float64 cloud or query inside too
        q = np.clip(q, lo + 1e-4 * (hi - lo), hi - 1e-4 * (hi - lo))
    elif mode == "near":
        q[0] = lo - 0.01 * spread
    elif mode == "far":
        m = max(1, nq // 4)
        q[:m] = lo + rng.uniform(-10, 11, (m, 3)) * spread
        q[-1] = hi + 10 * spread  # past every key
    return q


def nearest_inputs(c):
    """(ref, query) of a nearest / index case, in the case's dtypes."""
    ref = cloud(c["geometry"], c["n"], c["seed"])
    if c["qmode"] == "in":  # the cube of either dtype
        ref = ref.astype(np.float32).astype(np.float64)
    q = queries(ref, c["nq"], c["qmode"], c["seed"] + 1)
    return ref.astype(c["index_dtype"]), q.astype(c["query_dtype"])


def knn_cloud(c):
    """The cloud of a knn case: its geometry, or for "dup" a cloud of n / k distinct points each repeated k + 1 times."""
    if c["geometry"] == "dup":
        base = cloud("gauss", max(1, c["n"] // (c["k"] + 1) + 1), c["seed"])
        return np.repeat(base, c["k"] + 1, 0)[:c["n"]].astype(c["dtype"])
    if c["geometry"] == "surface":
        rng = np.random.default_rng(c["seed"])
        u, v = rng.uniform(-1, 1, (2, c["n"]))
        return (np.stack([u, v, 0.3 * np.sin(2 * u) * np.cos(3 * v)], -1)
                + 0.002 * rng.standard_normal((c["n"], 3))).astype(c["dtype"])
    return cloud(c["geometry"], c["n"], c["seed"]).astype(c["dtype"])


# ------------------------------------------------------------------------------------------------ the case table
F32, F64 = np.float32, np.float64
VIEW = 368 * 512
CALLER_N = (32 * VIEW, 4 * VIEW)  # 6 029 312 and 753 664 points: evaluate_reconstruction at 32 and 4 views
SIZES = (1, 2, 3, 31, 32, 33, 255, 256, 257, 2047, 2048, 2049, 4095, 4096, 4097, 16385, 262143, 262144, 262145,
         (1 << 20) + 3)
GEOMETRIES = ("gauss", "plane", "line", "lattice", "same", "cluster", "geo", "huge", "tiny", "subnorm")
KS = (1, 2, 3, 4, 30, 32)

_nearest, _knn, _red = [], [], []


def _nq_for(n):
    return min(max(n, 64), 20000)


def expected_flags(c):
    """The flags a nearest case is built to reach (tests/test_pointcloud_plans_cpu.py checks that its data does): far
    queries leave the cube and pass every index key unless the cloud is a single point; "same" clouds and single points
    have zero extent, planes and small lattices a zero-extent axis; more than 4096 queries or points sort in tiles."""
    n, g = c["n"], c["geometry"]
    if n == 0:
        return set()
    flat = g == "same" or n == 1
    out = {"flat"} if flat else set()
    if c["qmode"] != "in":
        out.add("outside")
    if c["qmode"] == "far" and not flat:
        out.add("past")
    if not flat and (g == "plane" or (g == "lattice" and n <= 4096) or (g == "line" and n == 2)):
        out.add("flataxis")
    if c["nq"] > STILE:
        out.add("tiles")
    return out


def _add_nearest(name, geometry, n, nq, idt, qdt, qmode, seed=0):
    c = dict(name=name, op="nearest", geometry=geometry, n=n, nq=nq, index_dtype=idt, query_dtype=qdt, qmode=qmode,
             seed=seed)
    c["expect"] = sorted(expected_flags(c))
    _nearest.append(c)


# callers' shapes: the registered clouds are fp32; accuracy queries the reconstruction against the ground truth
for _n in CALLER_N:
    _add_nearest(f"call_nn_{_n}", "gauss", _n, _n, F32, F32, "near", 1)
# the size matrix, alternating dtypes, with queries near and far
for _i, _n in enumerate(SIZES):
    _dt = ((F32, F32), (F64, F64), (F32, F64), (F64, F32))[_i % 4]
    _add_nearest(f"nn_gauss_n{_n}", "gauss", _n, _nq_for(_n), *_dt, "far" if _i % 2 else "near", 10 + _i)
_add_nearest("nn_gauss_n4097_q4097", "gauss", 4097, 4097, F32, F32, "far", 40)
# every geometry at a few sizes (f64 where f32 cannot hold the coordinates: geo, huge, tiny, subnorm)
for _g in GEOMETRIES:
    _wide = _g in ("geo", "huge", "tiny", "subnorm")
    for _n in (33, 4097, 262145):
        for _qm in ("near", "far"):
            _add_nearest(f"nn_{_g}_n{_n}_{_qm}", _g, _n, _nq_for(_n), F64 if _wide else F32, F64 if _wide else F32, _qm,
                         100 + _n)
# every dtype pair with queries inside, near and far, one tile and several, against one point and 2049
for _idt in (F32, F64):
    for _qdt in (F32, F64):
        for _qm in ("in", "near", "far"):
            for _n in (1, 2049):
                for _nq in (33, 4097):
                    _add_nearest(f"nn_{np.dtype(_idt).name}x{np.dtype(_qdt).name}_{_qm}_n{_n}_q{_nq}", "gauss", _n, _nq,
                                 _idt, _qdt, _qm, 200 + _n)
_add_nearest("nn_empty", "gauss", 0, 100, F64, F64, "near")
_add_nearest("nn_cluster_1m", "cluster", (1 << 20) + 3, 20000, F32, F32, "near", 7)
_add_nearest("nn_geo_f32_query", "geo", 4097, 4097, F64, F32, "near", 8)
for _idt in (F32, F64):
    for _qdt in (F32, F64):
        _add_nearest(f"nn_lattice_{np.dtype(_idt).name}x{np.dtype(_qdt).name}", "lattice", 4096, 4096, _idt, _qdt,
                     "near", 9)

for _n, _k in ((CALLER_N[0], 30), (CALLER_N[1], 30)):
    _knn.append(dict(name=f"call_knn_{_n}", op="knn", geometry="surface", n=_n, k=_k, dtype=F32, seed=2,
                     sample=4000))
for _k in KS:
    for _n in (1, 2, 3, 4, 31, 33, 4097):
        _knn.append(dict(name=f"knn_surface_n{_n}_k{_k}", op="knn", geometry="surface", n=_n, k=_k, dtype=F64, seed=_n))
    for _g in ("dup", "lattice", "plane", "line", "same", "geo", "cluster"):
        _knn.append(dict(name=f"knn_{_g}_k{_k}", op="knn", geometry=_g, n=4096 if _g == "lattice" else 4097, k=_k,
                         dtype=F64 if _g in ("geo", "cluster") else F32, seed=_k))
_knn.append(dict(name="knn_surface_n32_k32", op="knn", geometry="surface", n=32, k=32, dtype=F64, seed=5))
_knn.append(dict(name="knn_surface_n262145_k30", op="knn", geometry="surface", n=262145, k=30, dtype=F32, seed=6,
                 sample=4000))

# reductions: n over the size matrix and the callers' sizes; the GPU test runs every input regime on each
RED_SIZES = (1, 2, 3, 4, 255, 256, 257, 65536, 65537, 262144, 262145, 262146, 1_000_003, CALLER_N[1], CALLER_N[0])
for _n in RED_SIZES:
    _red.append(dict(name=f"red_n{_n}", op="reductions", n=_n))
COMPLETION_RATIO_N = ((1 << 24) - 1, (1 << 24) + 3, 20_000_001)

NEAREST = _nearest
KNN = _knn
REDUCTIONS = _red


def case_descs(c):
    """Every descriptor a case reaches (the index build and query of a nearest case; the build and normals of a knn
    case; every reduction regime of a reduction case)."""
    if c["op"] == "nearest":
        ref, q = nearest_inputs(c)
        return ([index_desc(ref)] if len(ref) else []) + [nearest_desc(ref, q)]
    if c["op"] == "knn":
        return [index_desc(knn_cloud(c)), knn_desc(c["n"], c["k"])]
    n = c["n"]
    out = [mean_desc(n), count_below_desc(n), nonfinite_desc(np.zeros((n, 3), F32)),
           nonfinite_desc(np.zeros((n, 3), F64))]
    out += [median_desc(x) for x in reduction_inputs(n, 0).values()]
    out += [abs_dot_desc(n, a, b) for a, b in ((False, False), (True, False), (False, True))]
    return out


def reduction_inputs(n, seed):
    """float64 (n,) inputs of the median / mean / count regimes: random, a tie across the middle, +-inf, NaN of either
    sign (first, last and inside), negative and signed zeros."""
    rng = np.random.default_rng(seed)
    base = np.abs(rng.standard_normal(n)) * 10.0 ** rng.uniform(-3, 3)
    out = dict(random=base.copy())
    t = base.copy()
    if n >= 2:
        s = np.sort(t)
        t[(t >= s[max(0, n // 2 - 2)]) & (t <= s[min(n - 1, n // 2 + 1)])] = s[n // 2]
    out["tie"] = t
    t = rng.standard_normal(n)
    t[rng.random(n) < 0.2] = np.inf
    t[rng.random(n) < 0.2] = -np.inf
    out["inf"] = t
    for sign, tag in ((1, "pos"), (-1, "neg")):
        for where in ("first", "last", "inside"):
            t = base.copy()
            t[{"first": 0, "last": n - 1, "inside": n // 2}[where]] = np.copysign(np.nan, sign)
            out[f"{tag}_nan_{where}"] = t
    t = rng.standard_normal(n)
    t[rng.random(n) < 0.5] = np.copysign(0.0, -1) if n > 1 else 0.0
    t[rng.random(n) < 0.25] = 0.0
    out["zeros"] = t
    return out


CASES = NEAREST + KNN + REDUCTIONS
