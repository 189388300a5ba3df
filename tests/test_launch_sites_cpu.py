"""Every kernel of the library is launched through f3r::launch (csrc/f3r_kernels.h), which counts the launches that
f3r_launch_count() reports.  A launch written anywhere else would run uncounted, so the sources are checked here: no
triple-chevron launch, cudaLaunchKernelEx, cudaFuncSetAttribute or cudaGetLastError outside f3r::launch, and no hand
counting in capi.cu."""
import glob
import os
import re

from tests.conftest import ROOT

CSRC = os.path.join(ROOT, "fast3r_b200", "csrc")


def _code(path: str) -> str:
    """Source without comments."""
    with open(path) as f:
        return re.sub(r"/\*.*?\*/|//[^\n]*", "", f.read(), flags=re.S)


def _launch_body(src: str) -> str:
    """The body of the f3r::launch template in f3r_kernels.h."""
    start = src.index("{", re.search(r"\bcudaError_t launch\(", src).end())
    depth = 0
    for i in range(start, len(src)):
        depth += {"{": 1, "}": -1}.get(src[i], 0)
        if depth == 0:
            return src[start:i + 1]
    raise AssertionError("unbalanced braces in f3r::launch")


def test_every_launch_goes_through_f3r_launch():
    header = _code(os.path.join(CSRC, "f3r_kernels.h"))
    body = _launch_body(header)
    assert body.count("cudaLaunchKernelEx(") == 1 and "++g_launch_count" in body
    sources = sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh")) +
                     glob.glob(os.path.join(CSRC, "*.h")))
    assert len(sources) >= 10
    for path in sources:
        src = _code(path)
        if path.endswith("f3r_kernels.h"):
            src = src.replace(body, "")
        for pattern in ("<<<", "cudaLaunchKernelEx", "cudaLaunchKernel(", "cudaFuncSetAttribute", "cudaGetLastError"):
            assert pattern not in src, (os.path.basename(path), pattern)


def test_capi_does_not_count_by_hand():
    src = _code(os.path.join(CSRC, "capi.cu"))
    assert not re.search(r"\b(g_launches|launches)\b", src)
    assert re.findall(r"\bg_launch_count\b[^;]*", src) == ["g_launch_count.load()"]
