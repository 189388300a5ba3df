"""Generates tests/golden/views.pt by running the REFERENCE's unmodified dataset pipeline on the raw views of
tests/views_cases.CASES, on the CPU:
  - BaseStereoViewDataset._crop_resize_if_necessary / __getitem__ / transpose_to_landscape
    (fast3r/dust3r/datasets/base/base_stereo_view_dataset.py) with cropping.py and geometry.py, through a minimal
    dataset whose _get_views crops the case's raw views in order, one generator per item, then default_collate;
  - the RE10K benchmark's crop_resize_if_necessary (scripts/fast3r_re10k_pose_eval.py:84-134), taken from the script
    by its syntax tree (the script itself imports the whole training stack).
The datasets package's __init__ imports every loader, so its packages are stood in for by empty modules whose __path__
is the real directory: the modules above load from the reference's files, unmodified.

Stored per case: the geometry of every raw view (both crop boxes, the resized size and filter, the float32 intrinsics),
each generator's state after the case, and per collated view the small arrays in full and a sha256 digest of each pixel
array's bytes (img, depthmap, pts3d, valid_mask).  Inputs are regenerated from the seeds.
Run: python tools/make_golden_views.py
"""
import ast
import hashlib
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_harness  # noqa: E402
from tests import views_cases as VC  # noqa: E402

PIXEL_KEYS = ("img", "depthmap", "pts3d", "valid_mask")
SMALL_KEYS = ("camera_intrinsics", "camera_pose", "true_shape", "rng")


def digest(t):
    t = t.contiguous()
    return f"{t.dtype}:{tuple(t.shape)}:" + hashlib.sha256(t.numpy().tobytes()).hexdigest()


def reference_modules():
    """(base_stereo_view_dataset, cropping, the RE10K crop function) from the reference's files."""
    root = ref_harness.REFERENCE_ROOT
    for name in ("fast3r", "fast3r.dust3r", "fast3r.dust3r.utils", "fast3r.dust3r.datasets",
                 "fast3r.dust3r.datasets.base", "fast3r.dust3r.datasets.utils"):
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(root, *name.split("."))]
        sys.modules[name] = m
    if root not in sys.path:
        sys.path.insert(0, root)
    import fast3r.dust3r.datasets.base.base_stereo_view_dataset as base
    import fast3r.dust3r.datasets.utils.cropping as cropping
    from PIL import Image
    path = os.path.join(root, "scripts", "fast3r_re10k_pose_eval.py")
    tree = ast.parse(open(path).read())
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "crop_resize_if_necessary")
    ns = dict(np=np, Image=Image, cropping=cropping)
    exec(compile(ast.Module(body=[fn], type_ignores=[]), path, "exec"), ns)
    return base, cropping, ns["crop_resize_if_necessary"]


class Recorder:
    """Wraps the cropping functions and PIL's resize to record each raw view's geometry as the reference computes it."""

    def __init__(self, cropping):
        import PIL.Image
        self.events = []
        crop, resize = cropping.crop_image_depthmap, PIL.Image.Image.resize

        def crop_rec(image, depthmap, K, bbox):
            out = crop(image, depthmap, K, bbox)
            self.events.append(("crop", tuple(int(v) for v in bbox), out[2].copy()))
            return out

        def resize_rec(im, size, resample=None, *a, **k):
            self.events.append(("resize", tuple(int(v) for v in size), int(resample)))
            return resize(im, size, resample, *a, **k)

        cropping.crop_image_depthmap = crop_rec
        PIL.Image.Image.resize = resize_rec

    def take(self):
        """The plans of the views recorded since the last call: crop, resize, crop per view."""
        ev, self.events = self.events, []
        plans = []
        for i in range(0, len(ev), 3):
            (_, crop, _), (_, size, filt), (_, box, K) = ev[i:i + 3]
            plans.append(dict(crop=crop, size=size, filt=1 if filt == 1 else 0, box=box, intrinsics=K))
        return plans


def run_dataset_case(base, rec, name):
    kind, B, N, _, res, aug, sp = VC.CASES[name]

    class Views(base.BaseStereoViewDataset):
        def __init__(self, raw):
            super().__init__(split="test", resolution=res, aug_crop=aug)
            self.raw = raw

        def _get_views(self, idx, resolution, rng):
            out = []
            for v in self.raw:
                img, depth, K = self._crop_resize_if_necessary(v["img"], v["depthmap"], v["camera_intrinsics"],
                                                               resolution, rng=rng, info=v["instance"])
                view = dict(img=img, depthmap=depth, camera_intrinsics=K, dataset=v["dataset"], label=v["label"],
                            instance=v["instance"])
                if "camera_pose" in v:
                    view["camera_pose"] = v["camera_pose"]
                out.append(view)
            return out

    items, plans, states = [], [], []
    for b, (raw, seed) in enumerate(zip(VC.samples(name), VC.rng_seeds(name))):
        ds = Views(raw)
        ds._rng = np.random.default_rng(seed)
        try:
            items.append(ds[0])
        except AssertionError as e:
            return dict(raises="AssertionError", message=str(e))
        plans.append(rec.take())
        states.append(ds._rng.bit_generator.state)
    views = torch.utils.data.default_collate(items)
    out = []
    for v in views:
        out.append({**{k: digest(v[k]) for k in PIXEL_KEYS}, **{k: v[k].clone() for k in SMALL_KEYS}})
    return dict(plans=plans, rng_states=states, views=out)


def run_re10k_case(crop_fn, rec, name):
    from fast3r.dust3r.utils.image import ImgNorm  # what the benchmark applies to the crop
    plans, imgs = [], []
    for raw in VC.samples(name):
        ps, ims = [], []
        for v in raw:
            image, K = crop_fn(v["img"], v["camera_intrinsics"])
            ps.extend(rec.take())
            ims.append(dict(img=digest(ImgNorm(image)), intrinsics=K.copy()))
        plans.append(ps)
        imgs.append(ims)
    return dict(plans=plans, images=imgs)


def main():
    base, cropping, crop_fn = reference_modules()
    rec = Recorder(cropping)
    out = {"what": "reference outputs, see tools/make_golden_views.py", "cases": {}}
    for name, (kind, *_rest) in VC.CASES.items():
        r = run_dataset_case(base, rec, name) if kind == "dataset" else run_re10k_case(crop_fn, rec, name)
        rec.take()
        out["cases"][name] = r
        print(name, "raises" if "raises" in r else "ok")
    path = os.path.join(ROOT, "tests", "golden", "views.pt")
    torch.save(out, path)
    print("wrote", path)


if __name__ == "__main__":
    main()
