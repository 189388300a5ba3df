"""Launch keys of the viewer-scene kernels (fast3r_b200/csrc/scene.cu) and the table of GPU cases that
tests/test_scene_gpu.py runs and tests/test_scene_plans_cpu.py checks the fast3r_b200.scene callers against.

A call is a plain dict ("descriptor") with its op and the arguments that decide the code path:
    sky      frames, h, w
    sort     sizes (the frames' pixel counts)
    visible  lens (segment row counts), mask_sky, view (a segment has a frame colour)
    ply      n
    extent   n
The key restates the launchers' rules (each function cites what it restates)."""
VT = 2048       # rows per compaction tile: scene.cu
STILE = 4096    # keys per radix-sort tile: pointcloud.cu ST * SI


def _flags(*pairs):
    return "".join(" " + f for f, on in pairs if on)


def sky_key(d):
    """launch_sky_mask: several frames per launch; a morphology window clipped on both sides (h or w < 7); one row
    (the upper-rows rule covers no row when int(h * 0.4) = 0)."""
    return "sky" + _flags(("batch", d["frames"] > 1), ("narrow", min(d["h"], d["w"]) < 7), ("one_row", d["h"] == 1))


def sort_key(d):
    """launch_scene_sort: the frame index adds a fifth radix pass past one frame; frames of different sizes; a partial
    last sort tile; one tile only."""
    s = d["sizes"]
    return "sort" + _flags(("frames", len(s) > 1), ("ragged", len(set(s)) > 1), ("tail", sum(s) % STILE != 0),
                           ("multitile", sum(s) > STILE))


def visible_key(d):
    """launch_scene_visible: sky filter, frame colours, segments longer than one tile, segments of different lengths."""
    lens = d["lens"]
    return "visible" + _flags(("sky", d["mask_sky"]), ("view", d["view"]), ("multitile", max(lens) > VT),
                              ("ragged", len(set(lens)) > 1))


def ply_key(d):
    return "ply" + _flags(("empty", d["n"] == 0))


def extent_key(d):
    """launch_extent_percentiles: n = 1 (both ranks are the last one) or more."""
    return "extent" + _flags(("single", d["n"] == 1))


KEYS = dict(sky=sky_key, sort=sort_key, visible=visible_key, ply=ply_key, extent=extent_key)


def key(d):
    return KEYS[d["op"]](d)


# ------------------------------------------------------------------------------------------------------ the case table
SKY = [("sky_v32", 32, 368, 512), ("sky_one", 1, 368, 512), ("sky_narrow", 3, 5, 3), ("sky_one_row", 1, 1, 5),
       ("sky_one_row_batch", 2, 1, 5), ("sky_narrow_one", 1, 6, 40)]
SORT = [("sort_v32", [188416] * 32), ("sort_one", [188416]), ("sort_small_one", [7 * 9]), ("sort_exact_tile", [4096]),
        ("sort_mixed", [188416, 64 * 96, 5, 188416]), ("sort_mixed_small", [15, 3, 1000]),
        ("sort_same_small", [100, 100]), ("sort_same_tiles", [4096, 4096])]
VISIBLE = [("vis_sky", [188416] * 4, True, False), ("vis_plain_view", [188416, 188416], False, True),
           ("vis_sky_view_ragged", [188416, 1, 18841, 5], True, True), ("vis_small", [30, 30], False, False),
           ("vis_small_sky_ragged", [1, 600], True, False), ("vis_one_tile_view", [100], False, True),
           ("vis_ragged", [5000, 3], False, False), ("vis_sky_view", [5000, 5000], True, True),
           ("vis_sky_small_view_ragged", [3, 7], True, True), ("vis_view_ragged", [3, 7000], False, True),
           ("vis_plain_tiles", [5000, 5000], False, False), ("vis_sky_small", [20, 20], True, False),
           ("vis_small_view", [20, 20], False, True), ("vis_ragged_small", [20, 7], False, False),
           ("vis_sky_tiles_ragged", [188416, 1], True, False), ("vis_sky_view_small", [50], True, True)]
PLY = [("ply_n", 1000), ("ply_empty", 0)]
EXTENT = [("extent_n", 100000), ("extent_single", 1)]


def _d(op, **kw):
    d = dict(op=op, **kw)
    d["key"] = key(d)
    return d


CASES = ([dict(name=c[0], **_d("sky", frames=c[1], h=c[2], w=c[3])) for c in SKY]
         + [dict(name=c[0], **_d("sort", sizes=c[1])) for c in SORT]
         + [dict(name=c[0], **_d("visible", lens=c[1], mask_sky=c[2], view=c[3])) for c in VISIBLE]
         + [dict(name=c[0], **_d("ply", n=c[1])) for c in PLY]
         + [dict(name=c[0], **_d("extent", n=c[1])) for c in EXTENT])
