"""Launch keys of the element-wise kernels, for the tests: which code runs for a call of LayerNorm, patch im2col, the
stride-2 3x3 im2col, the bilinear x2 upsample, the fp32 -> 16-bit casts (fast3r_b200/csrc/elementwise.cu) and the
parity path's split3 / add_f32 (fast3r_b200/csrc/attention_x3.cu), and the table of GPU cases that
tests/test_elementwise_plans_gpu.py runs and tests/test_elementwise_plans_cpu.py checks the forward against.

A call is a plain dict ("descriptor") with its op and the arguments that decide the code path:
    layernorm     rows, dim, out ("bf16" | "f16" | "f32"), eps
    im2col_patch  n, H, W, out
    im2col3x3s2   n, H, W, C, Ho, Wo          (the kernel copies 16-byte groups: the 16-bit type is not in the key)
    upsample2x    n, H, W, C, Ho, Wo, dt      (dt: "bf16" | "f16" | "f32", input and output)
    cast          n, out ("bf16" | "f16")
    split3        rows, k, relu
    add_f32       n
The key restates the launchers' rules (each function cites the lines it restates); its flags name the tails:
"multi" a grid-stride loop that runs more than one pass (every grid-stride launcher caps its grid at 132 * 16 blocks
of 256 threads), "tail" a partial last block of such a loop."""
GRID_CAP = 132 * 16   # blocks of a grid-stride launch: elementwise.cu:133,164,285, attention_x3.cu:254,273
THREADS = 256
LN_DIMS = (128, 256, 384, 512, 768, 1024)  # the VEC = dim / 128 instances of layernorm_kernel (elementwise.cu:77-85)
UPS_ROWS = 8          # output rows per block of the 16-bit upsample (elementwise.cu:173)


def _flags(*pairs):
    return "".join(" " + f for f, on in pairs if on)


def _stride(total):
    """Flags of a grid-stride loop over `total` items (elementwise.cu:105-106 and the grid rule of its launcher)."""
    return _flags(("multi", total > GRID_CAP * THREADS), ("tail", total % THREADS != 0))


def layernorm_key(d):
    """elementwise.cu:77-93: dim picks the VEC instance, the output type the store, a warp per row and 8 rows per block
    (rows % 8: the last block has idle warps)."""
    assert d["dim"] in LN_DIMS and d["out"] in ("bf16", "f16", "f32"), d
    return f"layernorm d{d['dim']} {d['out']}" + _flags(("ptail", d["rows"] % 8 != 0))


def im2col_patch_key(d):
    """elementwise.cu:103-137: 96 vectors of 8 elements per 16x16 patch, grid-stride."""
    total = d["n"] * (d["H"] // 16) * (d["W"] // 16) * 96
    return f"im2col_patch {d['out']}" + _flags(("multi", total > GRID_CAP * THREADS))


def im2col3x3s2_key(d):
    """elementwise.cu:145-166: tap (ky, kx) of output (oy, ox) reads input (2 oy - 1 + ky, 2 ox - 1 + kx); the top and
    left zero padding are always read, the bottom / right padding only when 2 Ho - 1 >= H / 2 Wo - 1 >= W."""
    total = d["n"] * d["Ho"] * d["Wo"] * 9 * (d["C"] // 8)
    return "im2col3x3s2" + _flags(("pad_b", 2 * d["Ho"] - 1 >= d["H"]), ("pad_r", 2 * d["Wo"] - 1 >= d["W"]),
                                  ("multi", total > GRID_CAP * THREADS))


def upsample2x_key(d):
    """elementwise.cu:241-268: fp32 runs upsample2x_f32_kernel (4 channels per thread, one output row per block), bf16 /
    fp16 upsample2x_kernel<T> (8 channels per thread, UPS_ROWS rows per block); C sets the channel shift; Ho < 2H / Wo <
    2W crop the x2 output; H = 1 / W = 1 give the scale 0 (every output reads row / column 0)."""
    H, W, C, Ho, Wo, dt = (d[f] for f in ("H", "W", "C", "Ho", "Wo", "dt"))
    per = 4 if dt == "f32" else 8
    return f"upsample2x {dt} c{C}" + _flags(("cropy", Ho < 2 * H), ("cropx", Wo < 2 * W), ("sy0", H == 1),
                                            ("sx0", W == 1), ("rtail", dt != "f32" and Ho % UPS_ROWS != 0),
                                            ("xtail", Wo * (C // per) % THREADS != 0))


def cast_key(d):
    """elementwise.cu:272-293: one float4 per thread, grid-stride."""
    return f"cast {d['out']}" + _stride(d["n"] // 4)


def split3_key(d):
    """attention_x3.cu:236-257: one float4 per thread, grid-stride; relu folds fmaxf(x, 0) in before the split."""
    return "split3" + _flags(("relu", bool(d["relu"]))) + _stride(d["rows"] * d["k"] // 4)


def add_f32_key(d):
    """attention_x3.cu:260-275: one float4 per thread, grid-stride."""
    return "add_f32" + _flags(("multi", d["n"] // 4 > GRID_CAP * THREADS))


KEYS = dict(layernorm=layernorm_key, im2col_patch=im2col_patch_key, im2col3x3s2=im2col3x3s2_key,
            upsample2x=upsample2x_key, cast=cast_key, split3=split3_key, add_f32=add_f32_key)


def key(d):
    return KEYS[d["op"]](d)


# ------------------------------------------------------------------------------------------------------ the case table
def _case(name, op, key_, **f):
    return dict(name=name, op=op, key=key_, **f)


def _ln(name, k, dim, rows, out, eps=1e-6):
    return _case(name, "layernorm", k, dim=dim, rows=rows, out=out, eps=eps)


def _ups(name, k, H, W, C, Ho, Wo, dt, n=1):
    return _case(name, "upsample2x", k, n=n, H=H, W=W, C=C, Ho=Ho, Wo=Wo, dt=dt)


def _i3(name, k, n, H, W, C):
    return _case(name, "im2col3x3s2", k, n=n, H=H, W=W, C=C, Ho=(H + 1) // 2, Wo=(W + 1) // 2)


# ---- one case per key of the forward, reduced to the fewest rows / images that reach it: ViT-L at 368x512 (N=32 and
# N=4 in bf16, fp16 and fp32, one portrait view, forward_many of mixed resolution, N=320) and the fusion decoder of N=32
# sharded over 2, 4 and 8 ranks (tests/test_elementwise_plans_cpu.py records them).  The upsample's n only sets grid.z.
FORWARD = [
    # every LayerNorm of the forward: 1024 channels, 736 rows per view
    _ln("fwd_ln_bf16", "layernorm d1024 bf16", 1024, 736, "bf16"),
    _ln("fwd_ln_f16", "layernorm d1024 f16", 1024, 736, "f16", eps=1e-5),
    _ln("fwd_ln_f32", "layernorm d1024 f32", 1024, 736, "f32"),
    # patch im2col: one view (one pass) and N=32 (2.26 M vectors; 8 views already loop)
    _case("fwd_patch_bf16", "im2col_patch", "im2col_patch bf16", n=1, H=368, W=512, out="bf16"),
    _case("fwd_patch_f16", "im2col_patch", "im2col_patch f16", n=1, H=512, W=368, out="f16"),
    _case("fwd_patch_f32", "im2col_patch", "im2col_patch f32", n=1, H=368, W=512, out="f32"),
    _case("fwd_patch_bf16_multi", "im2col_patch", "im2col_patch bf16 multi", n=8, H=368, W=512, out="bf16"),
    _case("fwd_patch_f16_multi", "im2col_patch", "im2col_patch f16 multi", n=8, H=368, W=512, out="f16"),
    _case("fwd_patch_f32_multi", "im2col_patch", "im2col_patch f32 multi", n=8, H=368, W=512, out="f32"),
    # act_postprocess[3]'s stride-2 conv: landscape 23x32 (bottom padding; the parity forward's split operand, 3 * 768
    # channels) and portrait 32x23 (right padding, one pass)
    _i3("fwd_i3s2_land_x3", "im2col3x3s2 pad_b multi", 2, 23, 32, 3 * 768),
    _i3("fwd_i3s2_port", "im2col3x3s2 pad_r", 1, 32, 23, 768),
    _i3("fwd_i3s2_512x384_x3", "im2col3x3s2 multi", 2, 32, 24, 3 * 768),  # forward_many's 512x384 views: no padding
    # the hook casts: N=32 (6 M vectors) and one view
    _case("fwd_cast_bf16_multi", "cast", "cast bf16 multi", n=4 * 3 * GRID_CAP * THREADS, out="bf16"),
    _case("fwd_cast_f16_multi", "cast", "cast f16 multi", n=4 * 3 * GRID_CAP * THREADS, out="f16"),
    _case("fwd_cast_bf16", "cast", "cast bf16", n=736 * 1024, out="bf16"),
    _case("fwd_cast_f16", "cast", "cast f16", n=736 * 1024, out="f16"),
    # the parity forward's operand splits (relu: the residual units' first conv) and the fusion blocks' second residual
    _case("fwd_split3", "split3", "split3", rows=1536, k=256, relu=False),
    _case("fwd_split3_relu", "split3", "split3 relu", rows=1536, k=256, relu=True),
    _case("fwd_split3_multi", "split3", "split3 multi", rows=5888, k=384, relu=False),
    _case("fwd_split3_relu_multi", "split3", "split3 relu multi", rows=9000, k=256, relu=True),
    _case("fwd_add_f32", "add_f32", "add_f32", n=8 * 12 * 16 * 256 * 4),
    _case("fwd_add_f32_multi", "add_f32", "add_f32 multi", n=8 * 46 * 64 * 256),
]

# the five DPT upsamples of a landscape (368x512) and a portrait (512x368) view: refinenet4 (cropped to the layer-3 map),
# refinenet3..1 and the head, in every type
_UPS_FWD = [
    # (name, H, W, C, Ho, Wo, flags of the 16-bit kernel, flags of the fp32 kernel)
    ("r4_land", 12, 16, 256, 23, 32, " cropy rtail", " cropy"),
    ("r3_land", 23, 32, 256, 46, 64, " rtail", ""),
    ("r2_land", 46, 64, 256, 92, 128, " rtail", ""),
    ("r1_land", 92, 128, 256, 184, 256, "", ""),
    ("head_land", 184, 256, 128, 368, 512, "", ""),
    ("r4_port", 16, 12, 256, 32, 23, " cropx xtail", " cropx xtail"),
    ("r3_port", 32, 23, 256, 64, 46, " xtail", " xtail"),
    ("r2_port", 64, 46, 256, 128, 92, " xtail", ""),
    ("r1_port", 128, 92, 256, 256, 184, "", ""),
    ("head_port", 256, 184, 128, 512, 368, "", ""),
]
_seen = set()
for _n, _H, _W, _C, _Ho, _Wo, _f16, _f32 in _UPS_FWD:
    for _dt in ("bf16", "f16", "f32"):
        _k = f"upsample2x {_dt} c{_C}" + (_f32 if _dt == "f32" else _f16)
        if _k not in _seen:  # one case per key
            _seen.add(_k)
            FORWARD.append(_ups(f"fwd_ups_{_n}_{_dt}", _k, _H, _W, _C, _Ho, _Wo, _dt))

# ---- the contract beyond the forward
CONTRACT = []
for _dim in LN_DIMS:  # every VEC instance and output type, with a partial last block of 1, 7 and 1 of 8 rows
    for _out in ("bf16", "f16", "f32"):
        for _rows in (1, 7, 9):
            CONTRACT.append(_ln(f"ln_d{_dim}_{_out}_r{_rows}", f"layernorm d{_dim} {_out} ptail", _dim, _rows, _out,
                                eps=1e-5 if _rows == 7 else 1e-6))
for _dt in ("bf16", "f16", "f32"):
    _tail = "" if _dt == "f32" else " rtail"
    CONTRACT += [
        _ups(f"ups_h1_{_dt}", f"upsample2x {_dt} c64 sy0{_tail} xtail", 1, 5, 64, 2, 10, _dt, n=2),
        _ups(f"ups_w1_{_dt}", f"upsample2x {_dt} c64 sx0{_tail} xtail", 6, 1, 64, 12, 2, _dt, n=2),
        _ups(f"ups_c8_{_dt}", f"upsample2x {_dt} c8 cropy cropx{_tail} xtail", 7, 9, 8, 13, 17, _dt, n=3),
        _ups(f"ups_ho1_{_dt}", f"upsample2x {_dt} c16 cropy{_tail} xtail", 3, 4, 16, 1, 8, _dt),
        _ups(f"ups_cropx_{_dt}", f"upsample2x {_dt} c32 cropx xtail", 8, 5, 32, 16, 9, _dt),
        _ups(f"ups_cropy_{_dt}", f"upsample2x {_dt} c32 cropy{_tail} xtail", 6, 5, 32, 11, 10, _dt),
    ]
CONTRACT += [
    _i3("i3s2_1x1", "im2col3x3s2 pad_b pad_r", 3, 1, 1, 8),
    _i3("i3s2_2x2", "im2col3x3s2", 2, 2, 2, 16),
    _i3("i3s2_c768_multi", "im2col3x3s2 pad_b multi", 4, 23, 32, 768),
    _case("cast_bf16_n4", "cast", "cast bf16 tail", n=4, out="bf16"),
    _case("cast_f16_n4", "cast", "cast f16 tail", n=4, out="f16"),
    _case("cast_bf16_multi_tail", "cast", "cast bf16 multi tail", n=4 * (GRID_CAP * THREADS + 1000), out="bf16"),
    _case("split3_relu_tail", "split3", "split3 relu tail", rows=7, k=40, relu=True),
    _case("split3_multi_tail", "split3", "split3 multi tail", rows=3001, k=728, relu=False),
]

# ---- the hand-picked shapes of the earlier per-kernel checks (tests/kernel_checks.py runs them under these names)
KERNEL_CHECKS = [
    _case("x3_split3", "split3", "split3 relu tail", rows=300, k=200, relu=True),
    _ups("x3_upsample_f32", "upsample2x f32 c256 cropy", 12, 16, 256, 23, 32, "f32", n=2),
    _case("x3_im2col_patch_f32", "im2col_patch", "im2col_patch f32", n=2, H=32, W=48, out="f32"),
    _case("x3_add_f32", "add_f32", "add_f32", n=4096 * 5),
    _case("cast", "cast", "cast bf16", n=4096 * 3, out="bf16"),
    _ln("layernorm_1024", "layernorm d1024 bf16", 1024, 1000, "bf16", eps=1e-5),
    _ln("layernorm_128", "layernorm d128 bf16 ptail", 128, 77, "bf16"),
    _case("im2col_patch", "im2col_patch", "im2col_patch bf16", n=3, H=64, W=96, out="bf16"),
    _i3("im2col3x3s2", "im2col3x3s2 pad_b", 2, 5, 6, 64),
    _ups("upsample_crop", "upsample2x bf16 c64 cropy rtail", 12, 16, 64, 23, 32, "bf16", n=2),
    _ups("upsample_full", "upsample2x bf16 c128 rtail", 23, 32, 128, 46, 64, "bf16", n=2),
]

CASES = FORWARD + CONTRACT + KERNEL_CHECKS
