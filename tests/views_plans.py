"""Launch keys of the ground-truth view kernel (fast3r_b200/csrc/views.cu) and the cases that
tests/test_views_gpu.py runs and tests/test_views_plans_cpu.py checks the callers against.

A record's key is what decides its path through the kernel and through f3r_ingest_rgb8: the orientation (a portrait
view is stored transposed), the direction of the nearest-neighbour map per axis (down, up or the same size, which
f3r_ingest_rgb8 does not resample) and the resampling filter.  A call adds "many-views" when it has more than one
record and "tail" when a view's pixel count is not a multiple of the kernel's 256-thread CTA (views.cu VWT)."""
from tests import views_cases as VC

VWT = 256


def _dir(src, dst):
    return "same" if src == dst else "down" if dst < src else "up"


def record_key(p):
    """Key of one lib.VIEW_PARAM record and the filter its image is resampled with."""
    rec, filt = p
    return (f"{'portrait' if rec['transpose'] else 'landscape'} x-{_dir(rec['crop_w'], rec['rs_w'])} "
            f"y-{_dir(rec['crop_h'], rec['rs_h'])} {'lanczos' if filt else 'bicubic'}")


def call_keys(records):
    """Keys reached by one call: its records' keys plus the call-level ones."""
    keys = {record_key(p) for p in records}
    if len(records) > 1:
        keys.add("many-views")
    if any(int(r["out_w"]) * int(r["out_h"]) % VWT for r, _ in records):
        keys.add("tail")
    return keys


# the GPU cases: every case of tests/views_cases that the reference does not refuse, and the keys each reaches
CASES = [name for name, c in VC.CASES.items() if not c[6].get("raises")]
KEYS = {
    "sevenscenes_640x480": {"landscape x-down y-down lanczos", "many-views"},
    "photo_1920x1440": {"landscape x-down y-down lanczos"},
    "photo_1600x1200": {"landscape x-down y-down lanczos", "many-views"},
    "re10k_640x360": {"landscape x-down y-down lanczos", "many-views"},
    "re10k_portrait_360x640": {"portrait x-down y-down lanczos"},
    "portrait_480x640": {"portrait x-down y-down lanczos", "many-views"},
    "near_square_aug_crop": {"landscape x-up y-up bicubic", "portrait x-up y-up bicubic", "many-views"},
    "near_square_square_res": {"landscape x-down y-down lanczos", "many-views"},
    "upscale_320x240": {"landscape x-up y-up bicubic", "many-views"},
    "margin_just_inside": {"portrait x-up y-up bicubic"},
    "depth_specials": {"landscape x-down y-down lanczos", "many-views"},
    "missing_pose": {"landscape x-down y-down lanczos", "many-views"},
    "batch2_mixed": {"landscape x-down y-down lanczos", "many-views"},
    "exact_512x384": {"landscape x-same y-same bicubic", "many-views"},
    "odd_resolution_500x375": {"landscape x-down y-down lanczos", "tail"},
}
