"""Image ingest kernels (f3r_ingest_rgb8) against the CPU oracle (oracle/ingest_oracle.c, pinned against Pillow /
torchvision / the reference's load_images by tests/test_ingest_cpu.py): bit-exact.  Needs an H100."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SIZES = [(640, 480), (4032, 3024), (3024, 4032), (300, 200), (1000, 1000), (97, 131), (512, 384), (513, 384), (2000, 350),
         (1920, 1080), (5000, 170), (64, 64), (4000, 3000), (200, 4097)]


def _img(w, h, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize("w,h", SIZES)
def test_ingest_bit_exact_vs_oracle(w, h):
    from fast3r_b200.ingest import ingest_rgb8
    from oracle import ingest_oracle as O
    img = _img(w, h, 11 * w + h)
    for size, square_ok in ((512, False), (512, True), (224, False)):
        ref, shape = O.ingest(img, size, square_ok)
        out, shp = ingest_rgb8(torch.from_numpy(img).cuda(), size, square_ok)
        torch.cuda.synchronize()
        assert tuple(shp) == tuple(shape) and out.dtype == torch.float32
        assert np.array_equal(out.cpu().numpy(), ref), (w, h, size, float(np.abs(out.cpu().numpy() - ref).max()))


def test_extreme_values_and_constant_images():
    """Saturation (clip8) and exact reproduction of constant images (weights sum to 1 after fixed-point rounding?  Pillow
    does not guarantee it - the oracle defines the answer)."""
    from fast3r_b200.ingest import ingest_rgb8
    from oracle import ingest_oracle as O
    for fill in (0, 255):
        img = np.full((777, 1234, 3), fill, np.uint8)
        img[::7, ::5] = 255 - fill
        ref, _ = O.ingest(img, 512)
        out, _ = ingest_rgb8(torch.from_numpy(img).cuda(), 512)
        assert np.array_equal(out.cpu().numpy(), ref)


def test_load_images_from_files(tmp_path):
    """fast3r_b200.ingest.load_images (same signature as the reference's) on PNG files: same view dicts, pixels equal to the
    oracle pipeline, tensors already on the device; the views run through the model's inference() unchanged."""
    from PIL import Image
    from fast3r_b200.ingest import load_images
    from oracle import ingest_oracle as O
    arrs = []
    for i, (w, h) in enumerate([(800, 600), (600, 800), (1024, 1024), (321, 123)]):
        a = _img(w, h, 100 + i)
        Image.fromarray(a).save(tmp_path / f"im{i}.png")
        arrs.append(a)
    (tmp_path / "notes.txt").write_text("not an image")
    views = load_images(str(tmp_path), size=512, verbose=False)
    assert len(views) == len(arrs)
    for i, (v, a) in enumerate(zip(views, arrs)):
        ref, shape = O.ingest(a, 512)
        assert v["img"].is_cuda and v["img"].shape == (1, 3) + tuple(shape)
        assert tuple(v["true_shape"][0]) == tuple(shape) and v["idx"] == i and v["instance"] == str(i)
        assert np.array_equal(v["img"][0].cpu().numpy(), ref)
    with pytest.raises(RuntimeError):
        load_images(str(tmp_path), size=512, verbose=False, device="cpu")
