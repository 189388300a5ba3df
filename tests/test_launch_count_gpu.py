"""f3r_launch_count() against the CUDA trace: for each call below, the number of kernels the library says it launched
equals the number of its kernels that torch.profiler (CUDA activity) records for the call.  Needs an H100."""
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

JPEG = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg")


def _launches(fn, tmp_path):
    """(launch-count delta, kernels of the library in the CUDA trace) of fn(), run to completion."""
    from fast3r_b200 import lib as L
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        n0 = L.launch_count()
        fn()
        torch.cuda.synchronize()
        n = L.launch_count() - n0
    trace = tmp_path / "trace.json"
    prof.export_chrome_trace(str(trace))
    events = json.loads(trace.read_text())["traceEvents"]
    # every kernel of the library is in namespace f3r; torch's own kernels (fills, copies) are not the library's
    return n, sum(1 for e in events if e.get("cat") == "kernel" and "f3r" in e.get("name", ""))


def _check(fn, tmp_path, expected=None):
    n, traced = _launches(fn, tmp_path)
    assert n == traced, (n, traced)
    if expected is not None:
        assert n == expected


def _pts(n, dtype=torch.float64, seed=0):
    return torch.randn(n, 3, generator=torch.Generator().manual_seed(seed), dtype=dtype).cuda()


def _tree_levels(n):
    """Levels of the index's bounding-box tree: buckets of 32 points, parents of 8 children, up to one root."""
    c, levels = (n + 31) // 32, 1
    while c > 1:
        c, levels = (c + 7) // 8, levels + 1
    return levels


@pytest.mark.parametrize("n,dtype", [(1, torch.float64), (100, torch.float32), (5000, torch.float64),
                                     (70000, torch.float32)])
def test_pc_index(n, dtype, tmp_path):
    from fast3r_b200 import ops
    pts = _pts(n, dtype)
    # bbox init, bbox, bbox finish, codes, gather keys, gather points; 13 sort passes of 3; one kernel per tree level
    _check(lambda: ops.pc_index(pts), tmp_path, expected=6 + 13 * 3 + _tree_levels(n))


def test_empty_inputs_launch_nothing(tmp_path):
    from fast3r_b200 import ops
    empty_pts = torch.empty(0, 3, dtype=torch.float64, device="cuda")
    empty = torch.empty(0, dtype=torch.float64, device="cuda")
    _check(lambda: ops.pc_count_nonfinite(empty_pts), tmp_path, expected=0)
    _check(lambda: ops.f64_count_below(empty, 0.5), tmp_path, expected=0)


def test_pc_nearest(tmp_path):
    from fast3r_b200 import ops
    index, empty_index = ops.pc_index(_pts(3000)), ops.pc_index(_pts(0))
    query = _pts(1000, seed=1)
    _check(lambda: ops.pc_nearest(index, query), tmp_path)
    _check(lambda: ops.pc_nearest(empty_index, query), tmp_path)


@pytest.mark.parametrize("n", [1001, 1000])
def test_f64_median(n, tmp_path):
    from fast3r_b200 import ops
    x = torch.randn(n, dtype=torch.float64, generator=torch.Generator().manual_seed(n)).cuda()
    _check(lambda: ops.f64_median(x), tmp_path)


@pytest.mark.parametrize("with_conf", [False, True])
def test_similarity_fit(with_conf, tmp_path):
    from fast3r_b200 import ops
    g = torch.Generator().manual_seed(3)
    x, y = (torch.randn(3, 500, 3, generator=g).cuda() for _ in range(2))
    conf = torch.rand(3, 500, generator=g).cuda() if with_conf else None
    thr = torch.full((3,), 0.3).cuda() if with_conf else None
    _check(lambda: ops.similarity_fit(x, y, conf, thr), tmp_path)


def test_focal_weiszfeld(tmp_path):
    from fast3r_b200 import ops
    pts = torch.randn(2, 16, 24, 3, generator=torch.Generator().manual_seed(4)).cuda()
    _check(lambda: ops.focal_weiszfeld(pts, iters=10), tmp_path)


@pytest.mark.parametrize("name", ["s420_331x211_rstblk1.jpg", "s420_97x131_q75.jpg"])
def test_decode_jpeg(name, tmp_path):
    from fast3r_b200 import ingest
    with open(os.path.join(JPEG, name), "rb") as f:
        data = f.read()
    _check(lambda: ingest.decode_jpeg(data), tmp_path)


@pytest.mark.parametrize("w,h", [(640, 480), (512, 384)])  # resized to 512 x 384, and already that size
def test_ingest_rgb8(w, h, tmp_path):
    from fast3r_b200.ingest import ingest_rgb8
    img = torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(5)).cuda()
    _check(lambda: ingest_rgb8(img, 512), tmp_path)


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_tiny_forward(precision, tmp_path):
    from fast3r_b200 import Fast3R, tiny_args
    from tests.golden.synth import synth_state_dict, synth_images
    enc, dec, head = tiny_args()
    model = Fast3R(enc, dec, head).eval()
    model.load_state_dict(synth_state_dict({k: tuple(v.shape) for k, v in model.state_dict().items()}, seed=0))
    model = model.cuda()
    model.set_precision(precision)
    views = [dict(img=im.cuda()) for im in synth_images(2, 1, 64, 96)]
    with torch.no_grad():
        _check(lambda: model(views), tmp_path)
