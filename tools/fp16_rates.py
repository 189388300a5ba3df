"""ms per forward of precision="bf16" and precision="fp16" on one model, alternated in one process, with the relative L2
distance of the fp16 predictions to the bf16 ones (per output key, over all views).

Random-init ViT-L (seeded), synthetic 368x512 views already on the device; N views per forward for each N of --views.
Every (N, precision) is warmed up by one untimed forward.  Prints one JSON line (the card, its power limit and SM clock
are read in the same run) and writes it to --out if given.

    python tools/fp16_rates.py --views 32,320 --rounds 3
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.packed_rates import card, rel_l2  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", default="32,320", help="comma-separated view counts")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp16_rates.py measures on the GPU; no CUDA device found")
    from fast3r_b200 import Fast3R, vit_large_args
    from tests.golden.synth import synth_images
    torch.manual_seed(0)
    with torch.device("cuda"):
        model = Fast3R(*vit_large_args()).eval()
    res = dict(card=card(), rounds=args.rounds, shape="368x512", sizes={})
    for n in [int(v) for v in args.views.split(",")]:
        views = [dict(img=im.cuda()) for im in synth_images(n, 1, 368, 512)]

        def timed(precision):
            model.set_precision(precision)
            torch.manual_seed(1)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = model(views)
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e3, out

        timed("bf16")
        timed("fp16")  # warm-up: packs the weights of both precisions
        ms = {"bf16": [], "fp16": []}
        for _ in range(args.rounds):
            for p in ("bf16", "fp16"):
                t, out = timed(p)
                ms[p].append(t)
                if p == "bf16":
                    ref = out
                else:
                    got = out
        dist = {k: rel_l2(torch.cat([g[k].flatten() for g in got]), torch.cat([r[k].flatten() for r in ref]))
                for k in ref[0]}
        med = {p: sorted(v)[len(v) // 2] for p, v in ms.items()}
        res["sizes"][str(n)] = dict(ms_bf16=ms["bf16"], ms_fp16=ms["fp16"], ms_median_bf16=med["bf16"],
                                    ms_median_fp16=med["fp16"], fp16_over_bf16=med["fp16"] / med["bf16"],
                                    rel_l2_fp16_vs_bf16=dist)
        del views, ref, got
        torch.cuda.empty_cache()
    model.set_precision("bf16")
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
