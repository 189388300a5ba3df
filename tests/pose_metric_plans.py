"""Launch keys of the camera-pose metric kernels (fast3r_b200/csrc/pose_metric.cu) and the table of GPU cases that
tests/test_pose_metric_gpu.py runs and tests/test_pose_metric_plans_cpu.py checks the callers against.

A call is a dict with its op ("pairs": f3r_pose_metric, "counts": f3r_pose_metric_counts) and the arguments that decide
the code path: dtype, angles (r / t stored), items and the pairs per item.  The pair kernel runs PT = 256 pairs per CTA
row and at most MAX_GX CTAs per item before it strides (pose_metric.cu:21-22)."""
PT = 256
MAX_GX = 1024


def pairs_of(views):
    return views * (views - 1) // 2


def _blocks(p):
    if p < PT:
        return "below-block"
    if p == PT:
        return "one-block"
    if p > PT * MAX_GX:
        return "strided"
    return "blocks" if p % PT == 0 else "blocks-tail"


def key(d):
    k = f"{d['op']} {d['dtype']} {_blocks(d['pairs'])}"
    if d["op"] == "pairs":
        k += (" angles" if d["angles"] else "") + (" many-items" if d["items"] > 1 else "")
    return k


# (name, op, dtype, angles, items, views or n)
CASES_SPEC = [
    ("p_f32_v2", "pairs", "float32", True, 1, 2),
    ("p_f32_v10_b8", "pairs", "float32", False, 8, 10),
    ("p_f32_v32_ang", "pairs", "float32", True, 1, 32),
    ("p_f32_v32_b8", "pairs", "float32", False, 8, 32),
    ("p_f32_v4_b2", "pairs", "float32", False, 2, 4),
    ("p_f32_v4_ang_b2", "pairs", "float32", True, 2, 4),
    ("p_f32_v10", "pairs", "float32", False, 1, 10),
    ("p_f32_v1000", "pairs", "float32", False, 1, 1000),
    ("p_f32_v1000_ang", "pairs", "float32", True, 1, 1000),
    ("p_f64_v320_ang", "pairs", "float64", True, 1, 320),
    ("p_f64_v8_b2", "pairs", "float64", False, 2, 8),
    ("p_f64_v3_ang", "pairs", "float64", True, 1, 3),
    ("p_f64_v32", "pairs", "float64", False, 1, 32),
    ("p_f32_v257_b3", "pairs", "float32", True, 3, 257),
    ("p_f32_v23_ang", "pairs", "float32", True, 1, 23),     # 253 pairs
    ("p_f32_v24", "pairs", "float32", False, 1, 24),        # 276
    ("c_f32_45", "counts", "float32", False, 1, 45),
    ("c_f64_496", "counts", "float64", False, 1, 496),
    ("c_f32_256", "counts", "float32", False, 1, 256),
    ("c_f32_big", "counts", "float32", False, 1, PT * MAX_GX + 77),
    ("c_f64_big", "counts", "float64", False, 1, 51040),
    ("c_f32_496", "counts", "float32", False, 1, 496),
    ("c_f64_45", "counts", "float64", False, 1, 45),
    ("c_f64_strided", "counts", "float64", False, 1, 499500),
    ("c_f32_512blocks", "counts", "float32", False, 1, 512 * PT),
    ("p_f64_v32_b8", "pairs", "float64", False, 8, 32),
    ("p_f64_v1000_ang", "pairs", "float64", True, 1, 1000),
    ("p_f32_v512", "pairs", "float32", False, 1, 512),      # 130816 pairs: 511 full blocks
]


def desc(c):
    name, op, dtype, angles, items, v = c
    return dict(name=name, op=op, dtype=dtype, angles=angles, items=items, views=v,
                pairs=pairs_of(v) if op == "pairs" else v)


CASES = [dict(key=key(desc(c)), **desc(c)) for c in CASES_SPEC]
