"""GPU image ingest: drop-in for ``fast3r.dust3r.utils.image.load_images`` (fast3r/dust3r/utils/image.py:76-159).

Same signature (plus ``device``), same list of view dicts, same pixels.  Baseline JPEGs - the files phones and cameras
write: Huffman-coded 8-bit sequential, grayscale or YCbCr at 4:4:4 / 4:2:2 / 4:2:0 - are decoded on the GPU
(``f3r_jpeg_decode``, bit-exact with Pillow/libjpeg-turbo), with the EXIF orientation, the optional 90-degree rotation and
the 4:3 landscape crop applied as an index map when the pixels are stored; host threads only read the file, probe its
header and read its EXIF orientation, and the compressed bytes are what crosses PCIe.  Every other file (progressive,
CMYK, PNG, HEIC, ...) keeps the PIL path on the host threads, as does a JPEG whose entropy-coded data the device reports
as inconsistent.  The expensive part after decoding - PIL's LANCZOS / BICUBIC resize of the full-resolution photo, the
center crop and the ToTensor + Normalize - runs in ``libfast3r_b200.so`` (``f3r_ingest_rgb8``), bit-exact with Pillow's
8-bit resampler, and the views come back already on the device, so ``inference()`` has nothing to upload.  No CPU
fallback: without the library / a CUDA device this raises.
"""
from __future__ import annotations

import ctypes as C
import io
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


def _need_cuda(device, what: str):
    """Raises unless `device` is a CUDA device: the library has no CPU path."""
    if torch.device(device).type != "cuda":
        raise RuntimeError(what)


def _h2d(arr: np.ndarray, device) -> torch.Tensor:
    """Copies a host uint8 array to `device` through a pinned staging buffer (asynchronous on the current stream)."""
    host = torch.empty(arr.shape, dtype=torch.uint8, pin_memory=True)
    host.numpy()[...] = arr
    return host.to(device, non_blocking=True)


def ingest_rgb8(img_u8: torch.Tensor, size: int = 512, square_ok: bool = False, out: torch.Tensor = None):
    """img_u8: CUDA uint8 (h, w, 3) RGB.  Returns (fp32 (3, H, W) in [-1, 1], (H, W)): resize + crop + normalise of
    load_images()."""
    _check_rgb8(img_u8)
    h1, w1, _ = img_u8.shape
    if size == 224:
        nw, nh, filt = resize_plan(w1, h1, round(size * max(w1 / h1, h1 / w1)))
    else:
        nw, nh, filt = resize_plan(w1, h1, size)
    left, top, right, bottom = crop_box(nw, nh, size, square_ok)
    out = resize_crop_rgb8(img_u8, nw, nh, filt, (left, top, right, bottom), out)
    return out, (bottom - top, right - left)


def _check_rgb8(img_u8: torch.Tensor):
    if img_u8.dtype != torch.uint8 or img_u8.dim() != 3 or img_u8.shape[2] != 3:
        raise RuntimeError("ingest_rgb8 needs a CUDA uint8 (h, w, 3) tensor (there is no CPU path)")
    _need_cuda(img_u8.device, "ingest_rgb8 needs a CUDA uint8 (h, w, 3) tensor (there is no CPU path)")


def resize_crop_rgb8(img_u8: torch.Tensor, nw: int, nh: int, filt: int, box, out: torch.Tensor = None) -> torch.Tensor:
    """PIL ``Image.resize((nw, nh), LANCZOS | BICUBIC)`` of the CUDA uint8 (h, w, 3) RGB image, then ``crop(box)`` (box =
    (left, top, right, bottom) inside the resized image) and ToTensor + Normalize(0.5, 0.5): fp32 (3, bottom - top,
    right - left) in [-1, 1], into `out` when given.  A dimension that keeps its size is not resampled, as in Pillow."""
    _check_rgb8(img_u8)
    img_u8 = img_u8.contiguous()
    if img_u8.data_ptr() % 4:  # e.g. a row slice of an image whose width is not a multiple of 4; the library needs 4
        img_u8 = img_u8.clone()
    h1, w1, _ = img_u8.shape
    left, top, right, bottom = box
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
    return out


def _landscape_crop(width: int, height: int):
    """The 4:3 crop box of load_images (image.py:111-124) as (left, top, right, bottom)."""
    desired = 4 / 3
    if width / height > desired:
        new_width = int(height * desired)
        left = (width - new_width) // 2
        return left, 0, left + new_width, height
    new_height = int(width / desired)
    top = (height - new_height) // 2
    return 0, top, width, top + new_height


def _decode(path, rotate_clockwise_90, crop_to_landscape):
    """Host part of load_images (image.py:103-124): open, EXIF transpose, RGB, optional rotation / 4:3 crop."""
    import PIL.Image
    from PIL.ImageOps import exif_transpose
    img = exif_transpose(PIL.Image.open(path)).convert("RGB")
    if rotate_clockwise_90:
        img = img.rotate(-90, expand=True)
    if crop_to_landscape:
        img = img.crop(_landscape_crop(*img.size))
    return np.asarray(img)


class JpegProbe:
    """What the library's header probe says about a file: status (lib.JPEG_SUPPORTED / JPEG_UNSUPPORTED /
    JPEG_MALFORMED), width, height, components, the reason when not supported, and the raw f3r_jpeg_info."""

    def __init__(self, info: L.JpegInfo, why: str):
        self.info, self.why = info, why
        self.status, self.width, self.height, self.components = info.status, info.width, info.height, info.components


def probe_jpeg(data) -> JpegProbe:
    """Classifies the bytes of a file from its headers (no pixel is decoded; no CUDA call)."""
    buf = np.frombuffer(data, np.uint8) if len(data) else np.zeros(1, np.uint8)
    lib = L.load()
    info = L.JpegInfo()
    L.check(lib.f3r_jpeg_probe(buf.ctypes.data, len(data), C.byref(info)), "f3r_jpeg_probe")
    why = lib.f3r_last_error().decode() if info.status != L.JPEG_SUPPORTED else ""
    return JpegProbe(info, why)


_ORIENTATIONS = (2, 3, 4, 5, 6, 7, 8)


def _exif_orientation(fp) -> int:
    """The orientation ImageOps.exif_transpose acts on (EXIF, or XMP through getexif()); reads no pixel data."""
    import PIL.Image
    with PIL.Image.open(fp) as im:
        o = im.getexif().get(0x0112, 1)
    return int(o) if o in _ORIENTATIONS else 1


def _store_geometry(w: int, h: int, orientation: int, rotate_clockwise_90: bool, crop_to_landscape: bool):
    """Shape (oh, ow) and crop offset (left, top) of _decode's output for a w x h decoded image."""
    if orientation >= 5:
        w, h = h, w
    if rotate_clockwise_90:
        w, h = h, w
    left, top, right, bottom = _landscape_crop(w, h) if crop_to_landscape else (0, 0, w, h)
    return bottom - top, right - left, left, top


def _decode_jpeg_async(data, probe: JpegProbe, orientation: int, rotate_clockwise_90: bool, crop_to_landscape: bool,
                       device):
    """Enqueues the device decode of a supported JPEG on the current stream.  Returns the uint8 (h, w, 3) image and a
    device int32 status (0: decoded; non-zero: the entropy-coded data is inconsistent and the image is undefined)."""
    buf = np.frombuffer(data, np.uint8)
    dev = _h2d(buf, device)
    oh, ow, left, top = _store_geometry(probe.width, probe.height, orientation, rotate_clockwise_90, crop_to_landscape)
    out = torch.empty(oh, ow, 3, dtype=torch.uint8, device=device)
    status = torch.zeros(1, dtype=torch.int32, device=device)
    if oh == 0 or ow == 0:  # the 4:3 crop of a 1-pixel-high image is empty, as with PIL
        return out, status
    ws = ops._scratch(probe.info.workspace_bytes, device)
    p = ops._ptr
    ops._call("f3r_jpeg_decode", out, buf.ctypes.data, len(buf), p(dev), orientation, int(bool(rotate_clockwise_90)), left,
              top, ow, oh, p(out), p(status), p(ws), probe.info.workspace_bytes)
    return out, status


def decode_jpeg(data, rotate_clockwise_90: bool = False, crop_to_landscape: bool = False, device="cuda") -> torch.Tensor:
    """Decodes the bytes of a baseline JPEG on the GPU into a CUDA uint8 (h, w, 3) RGB tensor equal to what load_images'
    host path (``_decode``: PIL open, ImageOps.exif_transpose, convert("RGB"), optional rotate(-90, expand=True) and
    4:3 crop) returns for the same file.  Raises ValueError for a file the GPU does not decode (progressive, CMYK,
    non-JPEG, ...; see probe_jpeg) and RuntimeError when the entropy-coded data is inconsistent.  Synchronises."""
    device = torch.device(device)
    _need_cuda(device, "decode_jpeg decodes on a CUDA device (there is no CPU path)")
    probe = probe_jpeg(data)
    if probe.status != L.JPEG_SUPPORTED:
        raise ValueError(f"not a JPEG the GPU decodes: {probe.why}")
    orientation = _exif_orientation(io.BytesIO(bytes(data)))
    out, status = _decode_jpeg_async(data, probe, orientation, rotate_clockwise_90, crop_to_landscape, device)
    code = int(status.item())
    if code:
        raise RuntimeError(f"f3r_jpeg_decode: inconsistent entropy-coded data (status {code})")
    return out


def _read(path, rotate_clockwise_90, crop_to_landscape):
    """Host-thread part of load_images: (bytes, probe, orientation) for a JPEG the GPU decodes, else (None, None, the
    decoded image) from _decode."""
    with open(path, "rb") as f:
        data = f.read()
    probe = probe_jpeg(data)
    if probe.status == L.JPEG_SUPPORTED:
        try:
            return data, probe, _exif_orientation(path)
        except Exception:  # noqa: BLE001 - let _decode raise (or not) exactly as it does for this file
            pass
    return None, None, _decode(path, rotate_clockwise_90, crop_to_landscape)


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
    _need_cuda(device, "fast3r_b200.ingest.load_images produces CUDA views (no CPU path); use the reference's "
                       "load_images for host tensors")
    L.load()
    exts = (".jpg", ".jpeg", ".png", ".heic", ".heif")
    paths = [os.path.join(root, p) for p in folder_content if p.lower().endswith(exts)]
    assert paths, "no images foud at " + root
    imgs = []

    def upload(arr):
        return _h2d(np.ascontiguousarray(arr), device)

    with ThreadPoolExecutor(max_workers=num_threads or min(32, os.cpu_count() or 4)) as pool:
        for path, (data, probe, payload) in zip(paths, pool.map(
                lambda p: _read(p, rotate_clockwise_90, crop_to_landscape), paths)):
            if data is not None:
                with torch.cuda.device(device):
                    u8, status = _decode_jpeg_async(data, probe, payload, rotate_clockwise_90, crop_to_landscape,
                                                    device)
                    out, (H2, W2) = ingest_rgb8(u8, size, square_ok)
                    if int(status.item()):  # inconsistent entropy-coded data: this file takes the host path
                        u8 = upload(_decode(path, rotate_clockwise_90, crop_to_landscape))
                        out, (H2, W2) = ingest_rgb8(u8, size, square_ok)
            else:
                u8 = upload(payload)
                out, (H2, W2) = ingest_rgb8(u8, size, square_ok)
            h1, w1 = u8.shape[:2]
            if verbose:
                print(f" - adding {path} with resolution {w1}x{h1} --> {W2}x{H2}")
            imgs.append(dict(img=out[None], true_shape=np.int32([[H2, W2]]), idx=len(imgs), instance=str(len(imgs))))
    if verbose:
        print(f" (Found {len(imgs)} images)")
    return imgs
