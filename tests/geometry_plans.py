"""Launch keys of the geometry tail (fast3r_b200/csrc/geometry.cu), for the tests: which code runs for a call of the
confidence quantile, the similarity fit, the similarity apply and the Weiszfeld focal, and the table of GPU cases that
tests/test_geometry_plans_gpu.py runs and tests/test_geometry_plans_cpu.py checks the postprocess callers against.

A call is a plain dict ("descriptor") with its kernel and the arguments that decide the code path:
    quantile  views, n, q, aligned
    fit       views, n, conf, valid, aligned      (conf: conf and thr given; valid: a valid mask given)
    apply     views, n, aligned, alias            (alias: out is x)
    focal     views, H, W, conf, pp, iters        (conf: conf and thr given; pp: principal points given)
`aligned` is what the launchers test on the pointers: every float operand 16-byte aligned and the valid mask 4-byte
aligned.  The key restates the launchers' rules (each function cites the lines it restates)."""
import numpy as np

QC = 8           # CTAs (cluster slices) per view of the quantile: geometry.cu:29
FIT_CHUNKS = 32  # chunks per view of the moments: geometry.cu:166
FOC_CHUNKS = 256  # chunks per view of the Weiszfeld iteration: geometry.cu:338


def _flags(*pairs):
    return "".join(" " + f for f, on in pairs if on)


def quantile_per(n):
    """Elements per cluster slice, rounded up to 4 (geometry.cu:74-75)."""
    return ((n + QC - 1) // QC + 3) & ~3


def fit_per(n):
    """Pixels per chunk of the moments, rounded up to 4 (geometry.cu:204-205)."""
    return ((n + FIT_CHUNKS - 1) // FIT_CHUNKS + 3) & ~3


def focal_per(n):
    """Pixels per chunk of the Weiszfeld iteration (geometry.cu:385-386)."""
    return (n + FOC_CHUNKS - 1) // FOC_CHUNKS


def quantile_rank(n, q):
    """(lo, hi, w) of the order statistic: rank = q (n - 1) in fp32 like ATen (geometry.cu:76-79)."""
    rank = np.float32(q) * np.float32(n - 1)
    lo, hi = int(np.floor(rank)), int(np.ceil(rank))
    return lo, hi, np.float32(rank - np.float32(lo))


def quantile_key(d):
    """geometry.cu:449-452 picks the float4 loads from n % 4 and the base's alignment; :116 returns after the radix select
    when the rank is integral, else :123-159 run the successor pass and the lerp; slices past n are empty (:74-75)."""
    n = d["n"]
    lo, hi, _ = quantile_rank(n, d["q"])
    return "quantile" + _flags(("vec", n % 4 == 0 and d["aligned"]), ("interp", hi != lo),
                               ("empty", (QC - 1) * quantile_per(n) >= n))


def fit_key(d):
    """geometry.cu:460-476: float4 / uchar4 loads when n % 4 == 0 and x, y, conf are 16-byte and valid 4-byte aligned
    (:464-465); with conf and thr two passes (mode 0, then mode 1 for the views with fewer than 3 selected pixels, :466);
    chunks past n are empty (:204-205)."""
    n = d["n"]
    return "fit" + _flags(("vec", n % 4 == 0 and d["aligned"]), ("conf", d["conf"]), ("valid", d["valid"]),
                          ("empty", (FIT_CHUNKS - 1) * fit_per(n) >= n))


def apply_key(d):
    """geometry.cu:478-483: similarity_apply_kernel<true> when n % 4 == 0 and x, out are 16-byte aligned; out may be x."""
    return "apply" + _flags(("vec", d["n"] % 4 == 0 and d["aligned"]), ("alias", d["alias"]))


def focal_key(d):
    """geometry.cu:487-498: iters + 1 launches of weiszfeld_iter_kernel (the first with unit weights, :351) then the final
    kernel; conf/thr select pixels (:383-389), pp replaces the image centre (:379-380); chunks past n are empty
    (:385-386)."""
    n = d["H"] * d["W"]
    return "focal" + _flags(("conf", d["conf"]), ("pp", d["pp"]), ("iters0", d["iters"] == 0),
                            ("empty", (FOC_CHUNKS - 1) * focal_per(n) >= n))


KEYS = dict(quantile=quantile_key, fit=fit_key, apply=apply_key, focal=focal_key)


def key(d):
    return KEYS[d["op"]](d)


# ------------------------------------------------------------------------------------------------------ the case table
def _case(name, op, key_, **f):
    return dict(name=name, op=op, key=key_, **f)


def _q(name, k, views, n, q, aligned=True):
    return _case(name, "quantile", k, views=views, n=n, q=q, aligned=aligned)


def _fit(name, k, views, n, conf, valid, aligned=True):
    return _case(name, "fit", k, views=views, n=n, conf=conf, valid=valid, aligned=aligned)


def _apply(name, k, views, n, aligned=True, alias=False):
    return _case(name, "apply", k, views=views, n=n, aligned=aligned, alias=alias)


def _focal(name, k, views, H, W, conf, pp, iters):
    return _case(name, "focal", k, views=views, H=H, W=W, conf=conf, pp=pp, iters=iters)


LAND, PORT, FOUR3, CROP = 368 * 512, 512 * 368, 384 * 512, 224 * 224  # pixels per view of the callers' resolutions

# ---- one case per key the postprocess entry points reach (tests/test_geometry_plans_cpu.py records them), at their
# shapes: align_local_pts3d_to_global stacks up to 64 (view, batch) pairs (1, 2, 32, 64 and the 65th alone), estimate_focal
# runs one view, evaluate_reconstruction quantiles V views and fits / applies one "view" of V H W points (V = 4, 32)
CALLERS = [
    _q("call_q_align_p0_v1", "quantile vec", 1, LAND, 0.0),
    _q("call_q_align_p0_v2_port", "quantile vec", 2, PORT, 0.0),
    _q("call_q_align_p0_v32", "quantile vec", 32, LAND, 0.0),
    _q("call_q_align_p0_v64_crop", "quantile vec", 64, CROP, 0.0),
    _q("call_q_align_p0_v65", "quantile vec", 65, LAND, 0.0),
    _q("call_q_align_p30_v1_4x3", "quantile vec interp", 1, FOUR3, 0.3),
    _q("call_q_focal_p10", "quantile vec interp", 1, LAND, 0.1),
    _q("call_q_focal_p10_crop", "quantile vec interp", 1, CROP, 0.1),
    _fit("call_fit_align_v1", "fit vec conf", 1, LAND, True, False),
    _fit("call_fit_align_valid_v2", "fit vec conf valid", 2, PORT, True, True),
    _fit("call_fit_align_valid_v32", "fit vec conf valid", 32, LAND, True, True),
    _fit("call_fit_align_v64_crop", "fit vec conf", 64, CROP, True, False),
    _fit("call_fit_align_valid_v65", "fit vec conf valid", 65, FOUR3, True, True),
    _fit("call_fit_eval_v4", "fit vec valid", 1, 4 * LAND, False, True),
    _fit("call_fit_eval_v32", "fit vec valid", 1, 32 * LAND, False, True),
    _apply("call_apply_align_v1", "apply vec", 1, LAND),
    _apply("call_apply_align_v32", "apply vec", 32, PORT),
    _apply("call_apply_align_v65", "apply vec", 65, FOUR3),
    _apply("call_apply_eval_v4", "apply vec", 1, 4 * LAND),
    _apply("call_apply_eval_v32", "apply vec", 1, 32 * LAND),
    _focal("call_focal_p10", "focal conf", 1, 368, 512, True, False, 100),
    _focal("call_focal_p10_pp_port", "focal conf pp", 1, 512, 368, True, True, 100),
    _focal("call_focal_depth", "focal pp", 3, 368, 512, False, True, 10),
    _focal("call_focal_depth_crop", "focal pp", 2, 224, 224, False, True, 10),
]

# ---- the contract beyond the callers: n in {1, 2, 3, 5, 31, 32, 33, 4099} for every kernel (empty slices / chunks and
# scalar tails), the vectorisable kernels with n % 4 == 0 but a base 4 bytes off, in-place apply, every focal option
QS = (0.0, 1e-7, 0.1, 0.3, 0.5, 0.85, 0.999, 1.0)
NS = (1, 2, 3, 5, 31, 32, 33, 4099)
CONTRACT = []
for _n in NS:
    for _qv in QS:
        _d = dict(n=_n, q=_qv, aligned=True)
        CONTRACT.append(_q(f"q_n{_n}_q{_qv:g}", quantile_key(_d), 3, _n, _qv))
    CONTRACT.append(_q(f"q_n{_n}_q0.5_mis", quantile_key(dict(_d, q=0.5, aligned=False)), 2, _n, 0.5, aligned=False))
    for _conf, _valid in ((True, True), (True, False), (False, True), (False, False)):
        _d = dict(n=_n, conf=_conf, valid=_valid, aligned=True)
        CONTRACT.append(_fit(f"fit_n{_n}" + _flags(("conf", _conf), ("valid", _valid)).replace(" ", "_"), fit_key(_d),
                             6, _n, _conf, _valid))
    for _alias in (False, True):
        _d = dict(n=_n, aligned=True, alias=_alias)
        CONTRACT.append(_apply(f"apply_n{_n}" + ("_alias" if _alias else ""), apply_key(_d), 3, _n, alias=_alias))
CONTRACT += [
    _q("q_land_q0.5_mis", "quantile interp", 2, LAND, 0.5, aligned=False),
    _q("q_land_q1e-7", "quantile vec interp", 2, LAND, 1e-7),
    _q("q_land_q0.999", "quantile vec interp", 2, LAND, 0.999),
    _q("q_land_q1", "quantile vec", 2, LAND, 1.0),
    _fit("fit_n32_mis", "fit conf valid empty", 6, 32, True, True, aligned=False),
    _fit("fit_land_mis", "fit conf valid", 6, LAND, True, True, aligned=False),
    _fit("fit_n4096_mis_noconf", "fit valid", 6, 4096, False, True, aligned=False),
    _apply("apply_n32_mis", "apply", 3, 32, aligned=False),
    _apply("apply_land_mis", "apply", 2, LAND, aligned=False),
    _apply("apply_land_mis_alias", "apply alias", 2, LAND, aligned=False, alias=True),
    _apply("apply_land_alias", "apply vec alias", 2, LAND, alias=True),
]
_FOCAL_HW = ((1, 1), (1, 2), (1, 3), (1, 5), (1, 31), (4, 8), (3, 11), (1, 4099), (15, 15), (368, 512))
for _H, _W in _FOCAL_HW:
    for _conf, _pp in ((True, False), (False, True), (True, True), (False, False)):
        for _it in (0, 1, 100):
            _d = dict(H=_H, W=_W, conf=_conf, pp=_pp, iters=_it)
            _nm = f"focal_{_H}x{_W}" + _flags(("conf", _conf), ("pp", _pp)).replace(" ", "_") + f"_it{_it}"
            CONTRACT.append(_focal(_nm, focal_key(_d), 4, _H, _W, _conf, _pp, _it))

CASES = CALLERS + CONTRACT
