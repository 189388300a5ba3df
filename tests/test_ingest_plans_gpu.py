"""Every case of tests/ingest_plans.CASES on the GPU, bit-exact against Pillow itself.  Needs an H100.

Decode cases run f3r_jpeg_decode with canaries: 4 KB of a sentinel before and after the output image, and the byte
past `workspace_bytes` of the workspace.  The image must equal ingest._decode (Pillow open, exif_transpose, RGB,
rotate, 4:3 crop) of the same bytes, and the status word must be the one the case declares: 0 for every stream Pillow
decodes below the sync limit, F3R_JPEG_ERR_SYNC at and above it (derivation: tests/jpeg_streams.sync_stream), in which
case load_images must still return the host path's view.  Ingest cases run ingest_rgb8 into an output with canaries,
with the resize intermediate swapped for one with canaries, and must equal Pillow's resize + crop + torchvision
ToTensor / Normalize.  The cases whose source sits 1-3 bytes past a 4-byte boundary first establish, without a launch,
that the library refuses such a source and that ingest_rgb8 hands the library an aligned copy."""
import io

import numpy as np
import pytest
import torch

from tests import ingest_plans as IP

pytestmark = pytest.mark.gpu

PAD = 4096
SENT = 0xA5


def _pillow_decode(data, case):
    from fast3r_b200 import ingest
    return ingest._decode(io.BytesIO(data), case["rot"], case["crop"])


@pytest.mark.parametrize("case", IP.DECODE, ids=[c["name"] for c in IP.DECODE])
def test_decode_case(case):
    from fast3r_b200 import ingest, lib as L, ops
    data = IP.build_stream(case)
    probe = ingest.probe_jpeg(data)
    assert probe.status == L.JPEG_SUPPORTED, probe.why
    o = ingest._exif_orientation(io.BytesIO(data))
    assert o == case["orientation"]
    oh, ow, left, top = ingest._store_geometry(probe.width, probe.height, o, case["rot"], case["crop"])
    buf = torch.full((oh * ow * 3 + 2 * PAD,), SENT, dtype=torch.uint8, device="cuda")
    out = buf[PAD:PAD + oh * ow * 3].view(oh, ow, 3)
    nws = probe.info.workspace_bytes
    ws = torch.full((nws + 256,), SENT, dtype=torch.uint8, device="cuda")
    status = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    host = np.frombuffer(data, np.uint8)
    dev = torch.from_numpy(host.copy()).cuda()
    ops._call("f3r_jpeg_decode", out, host.ctypes.data, len(host), dev.data_ptr(), o, int(case["rot"]), left, top, ow,
              oh, out.data_ptr(), status.data_ptr(), ws.data_ptr(), nws)
    torch.cuda.synchronize()
    st = int(status.item())
    assert bool((buf[:PAD] == SENT).all()) and bool((buf[PAD + oh * ow * 3:] == SENT).all()), "write outside the image"
    assert bool((ws[nws:] == SENT).all()), "write past workspace_bytes"
    if case["status"]:
        assert st & case["status"], st
        from fast3r_b200.ingest import ingest_rgb8
        import tempfile, os
        with tempfile.TemporaryDirectory() as d:
            p = os.path.join(d, "s.jpg")
            open(p, "wb").write(data)
            views = ingest.load_images([p], 512, verbose=False)
            ref, _ = ingest_rgb8(torch.from_numpy(np.ascontiguousarray(ingest._decode(p, False, False))).cuda(), 512)
            assert torch.equal(views[0]["img"][0], ref)
        return
    assert st == 0, st
    want = _pillow_decode(data, case)
    got = out.cpu().numpy()
    assert got.shape == want.shape
    bad = np.argwhere((got != want).any(-1))
    assert len(bad) == 0, f"{len(bad)} pixels differ, first at {bad[:4].tolist()}"


def _pillow_ingest(img, size, square_ok):
    import torchvision.transforms as tvf
    from PIL import Image
    norm = tvf.Compose([tvf.ToTensor(), tvf.Normalize((0.5, 0.5, 0.5), (0.5, 0.5, 0.5))])
    pil = Image.fromarray(img)
    W1, H1 = pil.size
    S = max(pil.size)
    le = round(size * max(W1 / H1, H1 / W1)) if size == 224 else size
    pil = pil.resize(tuple(int(round(x * le / S)) for x in pil.size), Image.LANCZOS if S > le else Image.BICUBIC)
    W, H = pil.size
    cx, cy = W // 2, H // 2
    if size == 224:
        half = min(cx, cy)
        pil = pil.crop((cx - half, cy - half, cx + half, cy + half))
    else:
        halfw, halfh = ((2 * cx) // 16) * 8, ((2 * cy) // 16) * 8
        if not square_ok and W == H:
            halfh = 3 * halfw / 4
        pil = pil.crop((cx - halfw, cy - halfh, cx + halfw, cy + halfh))
    return norm(pil).numpy()


def _library_refuses_misaligned(dev_ptr):
    """f3r_ingest_rgb8 on a real device address 1 byte past a 4-byte boundary, with an empty shape so no version of the
    library can launch: the call must report the alignment."""
    import ctypes as C
    from fast3r_b200 import lib as L
    lib = L.load()
    p = C.c_void_p(dev_ptr + (1 - dev_ptr % 4) % 4)
    rc = lib.f3r_ingest_rgb8(p, 0, 5, 4, 3, p, p, 3, 5, None, None, 0, p, 0, 0, 3, 4, p, None)
    return rc != 0 and lib.f3r_last_error().decode() == "f3r_ingest_rgb8: src not 4-byte aligned"


class _GuardedCall:
    """Wraps ops._call for f3r_ingest_rgb8: refuses (as a test failure, before any launch) a source that is not 4-byte
    aligned, and swaps the resize intermediate for one with canaries on both sides, checked after the call."""

    def __init__(self, real):
        self.real, self.tmp = real, None

    def __call__(self, name, anchor, *args):
        assert name == "f3r_ingest_rgb8"
        args = list(args)
        if args[0] % 4:
            pytest.fail("ingest_rgb8 handed the library a source that is not 4-byte aligned")
        if args[12] is not None:
            h, ow = args[1], args[4]
            n = h * ow * 3
            self.tmp = (torch.full((n + 2 * PAD,), SENT, dtype=torch.uint8, device="cuda"), n)
            args[12] = self.tmp[0].data_ptr() + PAD
        self.real(name, anchor, *args)

    def check(self):
        if self.tmp is not None:
            buf, n = self.tmp
            assert bool((buf[:PAD] == SENT).all()) and bool((buf[PAD + n:] == SENT).all()), "write outside tmp"


@pytest.mark.parametrize("case", IP.INGEST, ids=[c["name"] for c in IP.INGEST])
def test_ingest_case(case):
    from fast3r_b200.ingest import ingest_rgb8
    h, w, off = case["h"], case["w"], case["offset"]
    rng = np.random.default_rng(h * 7 + w)
    img = rng.integers(0, 256, (h + 1, w, 3), dtype=np.uint8)[1:] if off else rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if off:  # a flat buffer holding the image `off` bytes past a 4-byte boundary
        flat = torch.zeros(h * w * 3 + 8, dtype=torch.uint8, device="cuda")
        assert _library_refuses_misaligned(flat.data_ptr()), "the library would load words from a misaligned source"
        src = flat[off:off + h * w * 3].view(h, w, 3)
        src.copy_(torch.from_numpy(np.ascontiguousarray(img)))
        assert src.data_ptr() % 4 == off
    else:
        src = torch.from_numpy(img).cuda()
    ref = _pillow_ingest(img, case["size"], case["square_ok"])
    n = ref.size
    buf = torch.full((n + 2 * 1024,), -1234.5, dtype=torch.float32, device="cuda")
    out = buf[1024:1024 + n].view(ref.shape)
    from fast3r_b200 import ops
    guard = _GuardedCall(ops._call)
    ops._call = guard
    try:
        got, shape = ingest_rgb8(src, case["size"], case["square_ok"], out=out)
        torch.cuda.synchronize()
    finally:
        ops._call = guard.real
    guard.check()
    assert got.data_ptr() == out.data_ptr() and tuple(shape) == ref.shape[1:]
    assert bool((buf[:1024] == -1234.5).all()) and bool((buf[1024 + n:] == -1234.5).all()), "write outside out"
    g = out.cpu().numpy()
    assert np.array_equal(g, ref), (int((g != ref).sum()), float(np.abs(g - ref).max()))
