"""GPU image ingest: drop-in for ``fast3r.dust3r.utils.image.load_images`` (fast3r/dust3r/utils/image.py:76-159).

Same signature (plus ``device``), same list of view dicts, same pixels: file decoding, EXIF transposition, the optional
90-degree rotation and the 4:3 landscape crop stay PIL calls on a pool of host threads (cheap, lossless index
operations); the expensive part - PIL's LANCZOS / BICUBIC resize of the full-resolution photo, the center crop and the
ToTensor + Normalize - runs in ``libfast3r_b200.so`` (``f3r_ingest_rgb8``), bit-exact with Pillow's 8-bit resampler, and the
views come back already on the device, so ``inference()`` has nothing to upload.  No CPU fallback: without the library /
a CUDA device this raises.
"""
from __future__ import annotations

import ctypes as C
import os
from concurrent.futures import ThreadPoolExecutor
from typing import Dict, Tuple

import numpy as np
import torch

from . import lib as L, ops

BICUBIC, LANCZOS = 0, 1
_TABLES: Dict[Tuple, Tuple] = {}


def resize_plan(w1: int, h1: int, long_edge: int):
    """_resize_pil_image (image.py:68-75): long side -> long_edge; LANCZOS when shrinking, BICUBIC otherwise."""
    s = max(w1, h1)
    filt = LANCZOS if s > long_edge else BICUBIC
    return int(round(w1 * long_edge / s)), int(round(h1 * long_edge / s)), filt


def crop_box(w: int, h: int, size: int, square_ok: bool = False):
    """Center crop of load_images (image.py:126-137) as (left, top, right, bottom)."""
    cx, cy = w // 2, h // 2
    if size == 224:
        half = min(cx, cy)
        return cx - half, cy - half, cx + half, cy + half
    halfw, halfh = ((2 * cx) // 16) * 8, ((2 * cy) // 16) * 8
    if not square_ok and w == h:
        halfh = 3 * halfw / 4
    return cx - halfw, int(cy - halfh), cx + halfw, int(cy + halfh)


def _tables(in_size: int, out_size: int, filt: int, device):
    """Device copies of Pillow's tap tables for one dimension (cached per geometry)."""
    key = (in_size, out_size, filt, str(device))
    if key not in _TABLES:
        lib = L.load()
        ks = lib.f3r_resample_ksize(in_size, out_size, filt)
        bounds = np.empty((out_size, 2), np.int32)
        kk = np.empty((out_size, ks), np.int32)
        span = lib.f3r_resample_coeffs(in_size, out_size, filt, bounds.ctypes.data_as(C.c_void_p),
                                       kk.ctypes.data_as(C.c_void_p))
        if span < 0:
            raise RuntimeError("f3r_resample_coeffs failed: " + lib.f3r_last_error().decode())
        if len(_TABLES) >= 256:   # photo collections have a handful of geometries; bound the cache anyway
            _TABLES.pop(next(iter(_TABLES)))
        _TABLES[key] = (torch.from_numpy(bounds).to(device), torch.from_numpy(kk).to(device), ks, span)
    return _TABLES[key]


def ingest_rgb8(img_u8: torch.Tensor, size: int = 512, square_ok: bool = False, out: torch.Tensor = None):
    """img_u8: CUDA uint8 (h, w, 3) RGB.  Returns (fp32 (3, H, W) in [-1, 1], (H, W)): resize + crop + normalise of
    load_images()."""
    if not img_u8.is_cuda or img_u8.dtype != torch.uint8 or img_u8.dim() != 3 or img_u8.shape[2] != 3:
        raise RuntimeError("ingest_rgb8 needs a CUDA uint8 (h, w, 3) tensor (there is no CPU path)")
    img_u8 = img_u8.contiguous()
    h1, w1, _ = img_u8.shape
    if size == 224:
        nw, nh, filt = resize_plan(w1, h1, round(size * max(w1 / h1, h1 / w1)))
    else:
        nw, nh, filt = resize_plan(w1, h1, size)
    left, top, right, bottom = crop_box(nw, nh, size, square_ok)
    cw, ch = right - left, bottom - top
    dev = img_u8.device
    if out is None:
        out = torch.empty(3, ch, cw, dtype=torch.float32, device=dev)
    assert out.shape == (3, ch, cw) and out.is_contiguous()
    hb = hk = vb = vk = tmp = None
    hks = vks = span = 0
    if nw != w1:
        hb, hk, hks, span = _tables(w1, nw, filt, dev)
        tmp = torch.empty(h1, nw, 3, dtype=torch.uint8, device=dev)
    if nh != h1:
        vb, vk, vks, _ = _tables(h1, nh, filt, dev)
    p = ops._ptr
    ops._call("f3r_ingest_rgb8", img_u8, p(img_u8), h1, w1, nh, nw, p(hb), p(hk), hks, span, p(vb), p(vk), vks, p(tmp),
              left, top, cw, ch, p(out))
    return out, (ch, cw)


def _decode(path, rotate_clockwise_90, crop_to_landscape):
    """Host part of load_images (image.py:103-124): open, EXIF transpose, RGB, optional rotation / 4:3 crop."""
    import PIL.Image
    from PIL.ImageOps import exif_transpose
    img = exif_transpose(PIL.Image.open(path)).convert("RGB")
    if rotate_clockwise_90:
        img = img.rotate(-90, expand=True)
    if crop_to_landscape:
        desired = 4 / 3
        width, height = img.size
        if width / height > desired:
            new_width = int(height * desired)
            left = (width - new_width) // 2
            img = img.crop((left, 0, left + new_width, height))
        else:
            new_height = int(width / desired)
            top = (height - new_height) // 2
            img = img.crop((0, top, width, top + new_height))
    return np.asarray(img)


def load_images(folder_or_list, size, square_ok=False, verbose=True, rotate_clockwise_90=False, crop_to_landscape=False,
                device="cuda", num_threads=None):
    """open and convert all images in a list or folder to proper input format for DUSt3R (views on `device`)."""
    if isinstance(folder_or_list, str):
        if verbose:
            print(f">> Loading images from {folder_or_list}")
        root, folder_content = folder_or_list, sorted(os.listdir(folder_or_list))
    elif isinstance(folder_or_list, list):
        if verbose:
            print(f">> Loading a list of {len(folder_or_list)} images")
        root, folder_content = "", folder_or_list
    else:
        raise ValueError(f"bad {folder_or_list=} ({type(folder_or_list)})")
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("fast3r_b200.ingest.load_images produces CUDA views (no CPU path); use the reference's "
                           "load_images for host tensors")
    L.load()
    exts = (".jpg", ".jpeg", ".png", ".heic", ".heif")
    paths = [os.path.join(root, p) for p in folder_content if p.lower().endswith(exts)]
    assert paths, "no images foud at " + root
    imgs = []
    with ThreadPoolExecutor(max_workers=num_threads or min(32, os.cpu_count() or 4)) as pool:
        for path, arr in zip(paths, pool.map(lambda p: _decode(p, rotate_clockwise_90, crop_to_landscape), paths)):
            h1, w1 = arr.shape[:2]
            u8 = torch.from_numpy(np.ascontiguousarray(arr)).pin_memory().to(device, non_blocking=True)
            out, (H2, W2) = ingest_rgb8(u8, size, square_ok)
            if verbose:
                print(f" - adding {path} with resolution {w1}x{h1} --> {W2}x{H2}")
            imgs.append(dict(img=out[None], true_shape=np.int32([[H2, W2]]), idx=len(imgs), instance=str(len(imgs))))
    if verbose:
        print(f" (Found {len(imgs)} images)")
    return imgs
