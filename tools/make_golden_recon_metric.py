"""Writes tests/golden/recon_metric.json: the reference's own fast3r.eval.recon_metric (imported unmodified from a
checkout of facebookresearch/fast3r; it needs scipy and scikit-learn) run on the seeded clouds of
tests/golden/recon_clouds.py.  Stores per case the seed, the metric values and SHA-256 digests of the fp64 distance
arrays of both directions (cKDTree(gt).query(rec) for accuracy, cKDTree(rec).query(gt) for completion).

    python tools/make_golden_recon_metric.py --reference /path/to/fast3r [--out tests/golden/recon_metric.json]
"""
import argparse
import hashlib
import importlib.util
import json
import os
import sys

import numpy as np
import scipy
from scipy.spatial import cKDTree

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.golden.recon_clouds import CASES, make_case  # noqa: E402


def digest(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a, dtype="<f8").tobytes()).hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", required=True, help="root of a fast3r checkout")
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "recon_metric.json"))
    a = ap.parse_args()
    spec = importlib.util.spec_from_file_location("recon_metric", os.path.join(a.reference, "fast3r", "eval", "recon_metric.py"))
    rm = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(rm)
    cases = []
    for kind, seed in CASES:
        gt, rec, gn, rn = make_case(kind, seed)
        acc = rm.accuracy(gt, rec, gn, rn)
        comp = rm.completion(gt, rec, gn, rn)
        ratio = rm.completion_ratio(gt, rec)
        d_acc = cKDTree(gt).query(rec)[0]
        d_comp = cKDTree(rec).query(gt)[0]
        cases.append({"kind": kind, "seed": seed, "n_gt": len(gt), "n_rec": len(rec),
                      "accuracy": [float(v) for v in acc], "completion": [float(v) for v in comp],
                      "completion_ratio": float(ratio),
                      "dist_accuracy_sha256": digest(d_acc), "dist_completion_sha256": digest(d_comp)})
        print(kind, acc, comp, ratio)
    with open(a.out, "w") as f:
        json.dump({"generator": "tools/make_golden_recon_metric.py", "scipy": scipy.__version__, "numpy": np.__version__,
                   "cases": cases}, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
