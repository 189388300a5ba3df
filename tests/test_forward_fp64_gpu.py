"""The whole forward at the view counts this project runs at, every view, row, column, patch, pixel phase and channel
checked against a float64 oracle (oracle/forward_slices.py).

The cases (tests/forward_cases.py) reach the host code that only runs above a handful of views: DPT-head chunks of 25
(8 on the parity path) including a chunk boundary between the two batch elements of one view, the host sink that
streams each head chunk to pinned memory inside inference(), two encoder chunks at N=320, views of two shapes packed
into one decoder sequence, and several scenes in one forward_many.  The reference is oracle/fast3r_oracle.py in
float64 on the GPU (torch, cuBLAS and cuDNN only: none of the kernels under test), computed once per case and held on
the host; every precision of the case is checked against it.  The global torch RNG is seeded identically before the
model and before the oracle, so both draw the same image ids."""
import time

import numpy as np
import pytest
import torch

from oracle import forward_slices as FS
from tests.forward_cases import CASES, scene_images, state_dict

pytestmark = pytest.mark.gpu

SEED = 7
HEAD_CHUNK = 8  # oracle images per DPT-head call: bounds the float64 feature maps, same result


class _Case:
    def __init__(self, name):
        from oracle import fast3r_oracle as O
        from fast3r_b200 import Fast3R
        c = CASES[name]
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        self.name, self.c = name, c
        cfg, sd = state_dict(c["model"], c["gain"])
        self.scenes = scene_images(c["scenes"], c["B"])
        torch.manual_seed(SEED)
        ref = []
        for imgs in self.scenes:  # one oracle forward per scene, in scene order: the model draws one id set per scene
            out = O.forward(sd, *cfg, imgs, dtype=torch.float64, device="cuda", head_chunk=HEAD_CHUNK)
            ref += [{k: v.cpu() for k, v in p.items()} for p in out]
            del out
        torch.cuda.synchronize()
        self.ref = ref
        self.oracle_s = time.perf_counter() - t0
        self.oracle_peak = torch.cuda.max_memory_allocated()
        model = Fast3R(*cfg).eval()
        model.load_state_dict(sd)
        self.model = model.cuda()

    def run(self, precision):
        from fast3r_b200 import inference, inference_many
        c, model = self.c, self.model
        model.set_precision(precision)
        dtype = "32" if precision == "fp32" else torch.bfloat16  # a model set to fp16 keeps fp16 on the fast path
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        torch.manual_seed(SEED)
        if c["entry"] == "forward":
            preds, = [model([dict(img=im.cuda()) for im in imgs]) for imgs in self.scenes]
        else:
            samples = [[dict(img=im, true_shape=np.int32([list(im.shape[-2:])] * im.shape[0]), idx=i, instance=str(i))
                        for i, im in enumerate(imgs)] for imgs in self.scenes]
            if c["entry"] == "inference":
                preds = inference(samples[0], model, torch.device("cuda"), dtype=dtype, verbose=False)["preds"]
            else:
                res = inference_many(samples, model, torch.device("cuda"), dtype=dtype, verbose=False)
                preds = [p for r in res for p in r["preds"]]
        torch.cuda.synchronize()
        secs, peak = time.perf_counter() - t0, torch.cuda.max_memory_allocated()
        assert len(preds) == len(self.ref)
        for p, q in zip(preds, self.ref):
            assert sorted(p) == sorted(q)
            for k in q:
                assert p[k].shape == q[k].shape and p[k].dtype == torch.float32, (k, p[k].shape, q[k].shape)
        return preds, secs, peak


@pytest.fixture(scope="module")
def case_cache():
    cache = {}
    yield cache
    cache.clear()


def _get(cache, name):
    if name not in cache:
        cache.clear()  # hold one case's float64 reference at a time
        torch.cuda.empty_cache()
        cache[name] = _Case(name)
    return cache[name]


PARAMS = [(n, p) for n, c in CASES.items() for p in c["precisions"]]


@pytest.mark.parametrize("case,precision", PARAMS, ids=[f"{n}-{p}" for n, p in PARAMS])
def test_forward_vs_fp64_per_slice(case_cache, case, precision):
    cs = _get(case_cache, case)
    preds, secs, peak = cs.run(precision)
    print(f"\n{case} [{precision}]: forward {secs:.2f} s, max_memory_allocated {peak / 2**30:.2f} GiB; fp64 oracle "
          f"{cs.oracle_s:.1f} s, {cs.oracle_peak / 2**30:.2f} GiB; {torch.cuda.get_device_name()}")
    FS.check_all(FS.by_shape(preds, cs.ref), precision, case)
