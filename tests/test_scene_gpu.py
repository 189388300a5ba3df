"""fast3r_b200.scene on the GPU equals the numpy / cv2 / scipy oracle (tests/scene_oracle.py) bit for bit: sky masks,
the confidence order, the frame arrays, is_outdoor, max_extent, the visible points of the viewer's states and the PLY
bytes."""
import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from fast3r_b200 import ops, scene as S  # noqa: E402
from tests import scene_cases as SC  # noqa: E402
from tests import scene_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name,img", SC.quirk_images(), ids=[n for n, _ in SC.quirk_images()])
def test_sky_mask_quirks(name, img):
    got = S.detect_sky_mask(img)
    assert got.dtype == np.int8 and got.shape == img.shape[:2]
    np.testing.assert_array_equal(got, O.detect_sky_mask(img))


def test_sky_mask_all_triplets():
    img = SC.all_triplets()
    np.testing.assert_array_equal(S.detect_sky_mask(img), O.detect_sky_mask(img))


def test_sky_mask_batch_32_views():
    rng = np.random.default_rng(3)
    imgs = [SC.outdoor(rng, 368, 512) if k % 3 else SC.indoor(rng, 368, 512) for k in range(32)]
    batch = torch.stack([torch.from_numpy(i).permute(2, 0, 1) for i in imgs]).cuda().contiguous()
    got, counts = ops.sky_mask(batch)
    ref = np.stack([O.detect_sky_mask(i).reshape(-1) for i in imgs])
    np.testing.assert_array_equal(got.cpu().numpy(), ref)
    np.testing.assert_array_equal(counts.cpu().numpy(), ref.astype(np.int64).sum(1))


ORDER_CASES = [("specials_odd", [(7, 9)]), ("size1", [(1, 1)]), ("size2", [(1, 2)]), ("all_equal", [(5, 7)]),
               ("512x512", [(512, 512)]), ("mixed", [(17, 23), (1, 1), (40, 8), (9, 31)])]


@pytest.mark.parametrize("name,shapes", ORDER_CASES, ids=[c[0] for c in ORDER_CASES])
def test_order_is_stable_argsort(name, shapes):
    out = SC.synth_output(11, shapes)
    rng = np.random.default_rng(5)
    for p in out["preds"]:
        for ck in ("conf", "conf_local"):
            n = p[ck].numel()
            if name == "all_equal":
                c = np.full(n, 2.0, np.float32)
            elif name == "512x512":
                c = rng.integers(0, 50, n).astype(np.float32)  # many ties
            else:
                c = rng.choice(np.array([np.nan, 0.0, -0.0, np.inf, -np.inf, 1.5, -2.0, 3.0], np.float32), n)
            p[ck] = torch.from_numpy(c.reshape(p[ck].shape))
        h, w = p["conf"].shape[1:]
        idx = np.arange(h * w, dtype=np.float32)
        p["pts3d_in_other_view"] = torch.from_numpy(np.repeat(idx, 3).reshape(1, h, w, 3))
        p["pts3d_local_aligned_to_global"] = p["pts3d_in_other_view"].clone()
    sc = S.prepare_scene(out)
    for i, p in enumerate(out["preds"]):
        a, b = sc.offsets[i], sc.offsets[i + 1]
        for head, ck in (("global", "conf"), ("local", "conf_local")):
            got = getattr(sc, f"pts_{head}")[a:b, 0].cpu().numpy().astype(np.int64)
            np.testing.assert_array_equal(got, O.order(p[ck].numpy().reshape(-1)))
        conf = p["conf"].numpy().reshape(-1)
        np.testing.assert_array_equal(sc.max_conf_global[i], conf.max())


def _check_scene(out, sc, ref):
    n = len(out["preds"])
    assert sc.is_outdoor == ref["is_outdoor"]
    assert np.float32(sc.max_extent) == ref["max_extent"] or (np.isnan(sc.max_extent) and np.isnan(ref["max_extent"]))
    for i in range(n):
        fd = ref["frames"][i]
        a, b = sc.offsets[i], sc.offsets[i + 1]
        for head in ("global", "local"):
            np.testing.assert_array_equal(getattr(sc, f"pts_{head}")[a:b].cpu().numpy(), fd[f"pts_{head}"])
            np.testing.assert_array_equal(getattr(sc, f"rgb_{head}")[a:b].cpu().numpy(), fd[f"rgb_{head}"])
            np.testing.assert_array_equal(getattr(sc, f"not_sky_{head}")[a:b].cpu().numpy(), fd[f"not_sky_{head}"])
        assert sc.max_conf_global[i] == fd["max_conf_global"]
        assert sc.is_high_confidence[i] == fd["is_high_confidence"]
        np.testing.assert_array_equal(sc.view_colors[i], fd["view_color"])
    for st in SC.viewer_states(n):
        t, p, sky, g, l, drop, color = st
        pts, cols = sc.visible_points(timestep=t, min_conf_thr_percentile=p, mask_sky=sky, show_global=g, show_local=l,
                                      drop_low_conf_views=drop, color=color)
        rp, rc = O.visible_points(ref, t, p, sky, g, l, drop, color)
        np.testing.assert_array_equal(pts.cpu().numpy(), rp, err_msg=str(st))
        np.testing.assert_array_equal(cols.cpu().numpy(), rc, err_msg=str(st))
        assert S.ply_bytes(pts, cols) == O.ply_bytes(rp, rc), st


@pytest.mark.parametrize("on_device", [False, True], ids=["host_preds", "device_preds"])
@pytest.mark.parametrize("shapes", [[(368, 512)] * 32, [(368, 512), (64, 96), (1, 5), (368, 512)]],
                         ids=["v32_512x368", "mixed4"])
def test_prepare_scene_matches_oracle(shapes, on_device):
    out = SC.synth_output(1, shapes)
    ref = O.prepare_scene(out)
    if on_device:
        out = {k: [{kk: vv.cuda() for kk, vv in d.items()} for d in v] for k, v in out.items()}
    sc = S.prepare_scene(out)
    assert sc.pts_global.is_cuda
    _check_scene(out, sc, ref)


def test_extent_percentiles_nan_and_sizes():
    rng = np.random.default_rng(9)
    for n in (1, 2, 3, 5, 1000, 1 << 20):
        p = (rng.normal(size=(n, 3)) * 10 ** rng.uniform(-3, 3)).astype(np.float32)
        if n >= 5:
            p[rng.integers(0, n), 1] = np.nan
            p[rng.integers(0, n), 2] = np.inf
        got = ops.extent_percentiles(torch.from_numpy(p).cuda()).cpu().numpy()
        lo, hi = np.percentile(p, 20, axis=0), np.percentile(p, 80, axis=0)
        np.testing.assert_array_equal(got[:3], lo)
        np.testing.assert_array_equal(got[3:6], hi)
        np.testing.assert_array_equal(got[6], np.max(hi - lo))


def test_save_ply(tmp_path):
    out = SC.synth_output(2, [(20, 30), (20, 30)])
    sc = S.prepare_scene(out)
    pts, cols = sc.visible_points()
    S.save_ply(tmp_path / "a.ply", pts, cols)
    assert (tmp_path / "a.ply").read_bytes() == S.ply_bytes(pts, cols)


def test_rejects_bad_inputs():
    out = SC.synth_output(2, [(20, 30)])
    del out["preds"][0]["pts3d_local_aligned_to_global"]
    with pytest.raises(KeyError, match="align_local_pts3d_to_global"):
        S.prepare_scene(out)
    out = SC.synth_output(2, [(20, 30)])
    out["views"][0]["img"] = out["views"][0]["img"].repeat(2, 1, 1, 1)
    with pytest.raises(ValueError):
        S.prepare_scene(out)


# ------------------------------------------------------------------- reference goldens, launch-key table, canaries
from tests import scene_emulator as E  # noqa: E402
from tests import scene_golden as G  # noqa: E402
from tests import scene_plans as SP  # noqa: E402



@pytest.mark.parametrize("on_device", [False, True], ids=["host_preds", "device_preds"])
@pytest.mark.parametrize("name", ["outdoor", "indoor"])
def test_prepare_scene_equals_reference_goldens(name, on_device):
    g = G.load()[name]
    G.check_scene(S, S.prepare_scene(G.output(g, "cuda" if on_device else None)), g)


def test_several_sort_groups():
    """70 frames: the frame order is sorted in two groups (64 + 6 frames)."""
    out = SC.synth_output(3, [(12, 16)] * 70)
    _check_scene(out, S.prepare_scene(out), O.prepare_scene(out))


GUARD = 4096
CANARY = 0xA5


class _Guarded:
    """Stands in for torch inside fast3r_b200.ops: every torch.empty (outputs and workspaces) gets GUARD canary bytes
    behind it, checked after the call."""

    def __init__(self):
        self.tails = []

    def __getattr__(self, name):
        return getattr(torch, name)

    def empty(self, *shape, dtype=torch.float32, device=None):
        shape = tuple(shape[0]) if len(shape) == 1 and isinstance(shape[0], (tuple, list, torch.Size)) else shape
        n = int(np.prod(shape)) * torch.empty(0, dtype=dtype).element_size()
        buf = torch.full((n + GUARD,), CANARY, dtype=torch.uint8, device=device)
        self.tails.append(buf[n:])
        return buf[:n].view(dtype).reshape(shape)

    def check(self):
        torch.cuda.synchronize()
        for t in self.tails:
            assert bool((t == CANARY).all()), "a kernel wrote past an output or workspace"


def _guarded_out(shape, dtype):
    """A caller-owned output with GUARD canary bytes on both sides."""
    n = int(np.prod(shape)) * torch.empty(0, dtype=dtype).element_size()
    buf = torch.full((n + 2 * GUARD,), CANARY, dtype=torch.uint8, device="cuda")
    return buf, buf[GUARD:GUARD + n].view(dtype).reshape(shape)


def _check_guards(*bufs):
    for buf in bufs:
        assert bool((buf[:GUARD] == CANARY).all()) and bool((buf[-GUARD:] == CANARY).all())


@pytest.mark.parametrize("case", SP.CASES, ids=[c["name"] for c in SP.CASES])
def test_launch_key_case(case, monkeypatch):
    g = _Guarded()
    monkeypatch.setattr(ops, "torch", g)
    rng = np.random.default_rng(abs(hash(case["name"])) % 2 ** 32)
    op = case["op"]
    if op == "sky":
        imgs = [SC.outdoor(rng, case["h"], case["w"]) for _ in range(case["frames"])]
        img = torch.stack([torch.from_numpy(i).permute(2, 0, 1) for i in imgs]).contiguous()
        buf, out = _guarded_out((case["frames"], case["h"] * case["w"]), torch.int8)
        got, counts = ops.sky_mask(img.cuda(), out=out)
        want, want_counts = E.sky_mask(img)
        g.check(); _check_guards(buf)
        np.testing.assert_array_equal(got.cpu().numpy(), want.numpy())
        np.testing.assert_array_equal(counts.cpu().numpy(), want_counts.numpy())
    elif op == "sort":
        sizes = case["sizes"]
        n = sum(sizes)
        off = torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64))
        conf = torch.from_numpy(rng.choice(np.array([np.nan, -0.0, 0.0, 1.5, np.inf], np.float32), n)
                                if n < 5000 else (1 + np.exp(rng.normal(size=n))).astype(np.float32))
        pts = torch.from_numpy(rng.normal(size=(n, 3)).astype(np.float32))
        img = torch.from_numpy(rng.uniform(-1, 1, 3 * n).astype(np.float32))
        ns = torch.from_numpy(rng.integers(0, 2, n).astype(np.int8))
        outs = [_guarded_out(s, d) for s, d in (((n, 3), torch.float32), ((n, 3), torch.uint8), ((n,), torch.int8),
                                                ((len(sizes),), torch.float32))]
        ops.scene_sort(conf.cuda(), pts.cuda(), img.cuda(), ns.cuda(), off.cuda(), *[o for _, o in outs])
        want = [torch.empty(n, 3), torch.empty(n, 3, dtype=torch.uint8), torch.empty(n, dtype=torch.int8),
                torch.empty(len(sizes))]
        E.scene_sort(conf, pts, img, ns, off, *want)
        g.check(); _check_guards(*[b for b, _ in outs])
        for (_, o), w in zip(outs, want):
            np.testing.assert_array_equal(o.cpu().numpy(), w.numpy())
    elif op == "visible":
        lens = case["lens"]
        rows = sum(lens) + 10
        pts_g, pts_l = (torch.from_numpy(rng.normal(size=(rows, 3)).astype(np.float32)) for _ in range(2))
        rgb_g, rgb_l = (torch.from_numpy(rng.integers(0, 256, (rows, 3)).astype(np.uint8)) for _ in range(2))
        ns_g, ns_l = (torch.from_numpy(rng.integers(0, 2, rows).astype(np.int8)) for _ in range(2))
        segs, start = [], 0
        for k, ln in enumerate(lens):
            segs.append((k % 2, start, ln, 0x12ab34 if (case["view"] and k % 2 == 0) else -1))
            start += ln
        segs = np.array(segs, np.int64)
        dev = [t.cuda() for t in (pts_g, pts_l, rgb_g, rgb_l, ns_g, ns_l)]
        p, c = ops.scene_visible(segs, *dev, case["mask_sky"])
        wp, wc = E.scene_visible(segs, pts_g, pts_l, rgb_g, rgb_l, ns_g, ns_l, case["mask_sky"])
        g.check()
        np.testing.assert_array_equal(p.cpu().numpy(), wp.numpy())
        np.testing.assert_array_equal(c.cpu().numpy(), wc.numpy())
    elif op == "ply":
        pts = torch.from_numpy(rng.normal(size=(case["n"], 3)).astype(np.float32))
        col = torch.from_numpy(rng.integers(0, 256, (case["n"], 3)).astype(np.uint8))
        got = ops.ply_pack(pts.cuda(), col.cuda())
        g.check()
        np.testing.assert_array_equal(got.cpu().numpy(), E.ply_pack(pts, col).numpy())
    else:
        pts = torch.from_numpy(rng.normal(size=(case["n"], 3)).astype(np.float32))
        got = ops.extent_percentiles(pts.cuda())
        g.check()
        np.testing.assert_array_equal(got.cpu().numpy(), E.extent_percentiles(pts).numpy())
