"""The element-wise kernels per element against float64, one case per launch key (tests/elementwise_plans.CASES), in
every type the key allows.  Needs an H100.

Every output sits between canaries (tests/canaries.py) that must keep their values.  u = 2^-24 is the fp32 unit
roundoff; r is the half-ulp of the stored type: 2^-8 (bf16), 2^-11 (fp16, plus 2^-25, half the spacing of its
subnormals, as absolute slack: SUB) or 0 (fp32).

LayerNorm.  The reference is float64 on the kernel's fp32 inputs: mu = mean(x), d = x - mu, var = mean(d^2), rstd =
1 / sqrt(var + eps) with eps rounded to fp32 as the kernel gets it, ref = d rstd w + b.  The kernel (one warp per row,
VEC = dim / 128 float4 per lane) sums each element through at most VEC + 7 additions (2 inside the float4, VEC - 1
across the lane's float4, 5 shuffle levels), then multiplies by the fp32 1/DIM (rounded for 384 and 768) - so
    |mu_k - mu| <= E_mu = 1.01 ((VEC + 7) u mean|x| + 2 u |mu|).
The variance is two-pass: sum (x - mu_k)^2 = sum d^2 + DIM (mu - mu_k)^2 (the cross term is DIM (mu - mu_k) sum d = 0),
so E_mu enters rstd only at second order; the squares, the VEC + 7 additions, the 1/DIM, + eps and rsqrtf (2 ulp = 4u)
give |rstd_k / rstd - 1| <= dr = (VEC/2 + 12) u + 0.51 rstd^2 E_mu^2.  The output (x - mu_k) rstd_k w + b takes 4 more
roundings:
    |y - ref| <= (1 + r) [((VEC/2 + 16) u + dr) |d| rstd |w| + 1.01 rstd |w| E_mu + u |b|] + r |ref| (+ SUB).
An E[x^2] - mu^2 variance fails the offset regime (300 + randn: cancellation of ~10^5 in fp32); 1/(DIM-1) fails the
fp32 outputs by 1/(2 DIM) relative.  Four regimes per case: random rows, a common offset of 300, a few outlier
channels at +-1e3, constant rows (variance 0, rstd = 1/sqrt(eps)).

Upsample.  The reference is the exact bilinear x2 with align_corners=True on the kernel's own (16-bit or fp32) inputs:
fy = oy (H-1)/(2H-1), y0 = floor(fy), y1 = min(y0+1, H-1), ly = fy - y0, the same in x, the four-term sum in float64
(cross-checked against F.interpolate once).  The kernel's scale is the fp32 quotient and fl(sy oy) adds a second
rounding, so its position is off by at most 2.01 u fy; bilinear interpolation is continuous in fy with slope at most the
largest neighbour difference Dy of the rows it may read (y0-1 .. y0+2 at columns x0, x1), so the position costs
2.01 u (fy Dy + fx Dx) whichever cell the rounded position lands in.  The weights (1-ly)(1-lx) ... carry 3 roundings,
the products and the 4-term sum 4 more, relative to sum w |v| <= M4 (the largest of the four neighbours):
    |out - ref| <= E = 8 u M4 + 2.01 u (fy Dy + fx Dx),   then   E + r (|ref| + E) (+ SUB).
The align_corners=False scale H/(2H) fails by up to half a pixel.

Exact kernels.  Patch im2col, the stride-2 im2col, the casts, split3 and add_f32 are compared with torch doing the same
roundings: .to(dtype) rounds to nearest even (overflow to inf), split3 is hi = bf16(x), lo = bf16(x - hi) laid out
[hi | lo | hi], add_f32 is one fp32 addition.  Values are compared, not bits: a NaN is 0x7FC0 in torch and 0x7FFF from
cvt.rn.bf16x2, and fmaxf(-0, 0) may give either zero.  split3's ReLU is fmaxf, which maps NaN to 0 where torch.relu keeps
it; the split3 inputs are finite.

Each bounded output also passes a relative L2 check (REL_L2) against a systematic drift that stays inside the per-element
bound (fp32 LayerNorm outputs: in the random and outlier regimes only, see run_layernorm)."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests import elementwise_plans as EP
from tests.canaries import PAD, buffer, check_elements, untouched

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SUB = 2.0 ** -25
R = {"bf16": 2.0 ** -8, "f16": 2.0 ** -11, "f32": 0.0}
DT = {"bf16": torch.bfloat16, "f16": torch.float16, "f32": torch.float32}
REL_L2 = {"bf16": 4e-3, "f16": 1e-3, "f32": 3e-5}
LN_REGIMES = ("random", "offset", "outliers", "constant")


def _bound_check(name, out, ref, bound, dt, l2=True):
    """Per element within `bound`, and (l2) the relative L2 error within REL_L2[dt]; returns the largest error / bound."""
    check_elements(name, out, ref, bound)
    out = out.double()
    ratio = float(((out - ref).abs() / bound.clamp_min(1e-300)).max())
    n = float(ref.norm())
    if l2 and n > 0:
        rel = float((out - ref).norm()) / n
        assert rel <= REL_L2[dt], f"{name}: relative L2 error {rel:.3g} > {REL_L2[dt]}"
    return ratio


def _same_values(name, out, ref):
    """out == ref value by value (NaN matches NaN, -0 matches 0)."""
    a, b = out.double(), ref.double()
    ok = (a == b) | (a.isnan() & b.isnan())
    if not bool(ok.all()):
        idx = (~ok).nonzero()[:5].tolist()
        raise AssertionError(f"{name}: {int((~ok).sum())} of {a.numel()} elements differ; first at {idx}: out "
                             f"{[float(a[tuple(i)]) for i in idx]} ref {[float(b[tuple(i)]) for i in idx]}")


def _out(shape, dt, fill=None):
    buf, view = buffer(shape, dt, fill)
    return buf, view, buf.clone()


def _canaries(name, buf, before):
    n = buf.numel() - 2 * PAD
    written = torch.zeros_like(buf, dtype=torch.bool)
    written[PAD:PAD + n] = True
    untouched(name, buf, before, written)


# ------------------------------------------------------------------ LayerNorm
def layernorm_input(rows, dim, regime, g):
    rnd = lambda *s: torch.randn(*s, generator=g, device="cuda")  # noqa: E731
    if regime == "random":
        return rnd(rows, dim) * 2 + 0.5
    if regime == "offset":
        return rnd(rows, dim) + 300
    if regime == "outliers":
        x = rnd(rows, dim)
        idx = torch.randint(0, dim, (rows, 3), generator=g, device="cuda")
        x.scatter_(1, idx, torch.where(rnd(rows, 3) > 0, 1e3, -1e3))
        return x
    return rnd(rows, 1).expand(rows, dim).contiguous() * 4


def layernorm_bound(x, w, b, eps, dt):
    """(ref, bound) in float64 (module docstring)."""
    dim = x.shape[-1]
    vec = dim // 128
    x64, w64, b64 = x.double(), w.double(), b.double()
    mu = x64.mean(-1, keepdim=True)
    d = x64 - mu
    rstd = 1.0 / torch.sqrt((d * d).mean(-1, keepdim=True) + torch.tensor(eps, dtype=torch.float32).item())
    ref = d * rstd * w64 + b64
    e_mu = 1.01 * ((vec + 7) * U * x64.abs().mean(-1, keepdim=True) + 2 * U * mu.abs())
    dr = (vec / 2 + 12) * U + 0.51 * rstd ** 2 * e_mu ** 2
    r = R[dt]
    core = ((vec / 2 + 16) * U + dr) * d.abs() * rstd * w64.abs() + 1.01 * rstd * w64.abs() * e_mu + U * b64.abs()
    return ref, (1 + r) * core + r * ref.abs() + (SUB if dt == "f16" else 0.0)


def run_layernorm(c, regime, seed):
    from fast3r_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    rows, dim, dt = c["rows"], c["dim"], c["out"]
    x = layernorm_input(rows, dim, regime, g)
    w = torch.randn(dim, generator=g, device="cuda")
    b = torch.randn(dim, generator=g, device="cuda") * 0.5
    buf, out, before = _out((rows, dim), DT[dt])
    ops.layernorm(x, w, b, c["eps"], out)
    torch.cuda.synchronize()
    name = f"{c['name']} {regime}"
    _canaries(name, buf, before)
    ref, bound = layernorm_bound(x, w, b, c["eps"], dt)
    # the offset and constant regimes stress the mean: their error is the bound's E_mu term, a per-row offset that
    # the relative L2 of a few rows measures as drift (constant rows: 1/sqrt(eps) times the mean's rounding, against
    # ref = b); the per-element bound checks them
    return _bound_check(name, out, ref, bound, dt, l2=regime in ("random", "outliers") or dt != "f32")


# ------------------------------------------------------------------ upsample
def upsample_ref(x, Ho, Wo):
    """(ref, bound without the output rounding) in float64 for x (n, H, W, C) of the kernel's input type."""
    n, H, W, C = x.shape
    x64 = x.double()
    dev = x.device

    def axis(size, out):
        f = torch.arange(out, dtype=torch.float64, device=dev) * (size - 1) / (2 * size - 1)
        i0 = f.floor().long().clamp_max(size - 1)
        return f, i0, (i0 + 1).clamp_max(size - 1), f - i0

    fy, y0, y1, ly = axis(H, Ho)
    fx, x0, x1, lx = axis(W, Wo)
    ly, fy = ly[:, None, None], fy[:, None, None]
    lx, fx = lx[None, :, None], fx[None, :, None]
    rows0, rows1 = x64[:, y0], x64[:, y1]
    a, b, d, e = rows0[:, :, x0], rows0[:, :, x1], rows1[:, :, x0], rows1[:, :, x1]
    ref = (1 - ly) * (1 - lx) * a + (1 - ly) * lx * b + ly * (1 - lx) * d + ly * lx * e
    m4 = torch.maximum(torch.maximum(a.abs(), b.abs()), torch.maximum(d.abs(), e.abs()))
    del a, b, d, e, rows0, rows1
    # the largest neighbour differences the rounded position can reach: y pairs (y0-1 .. y0+2) at columns x0 and x1,
    # x pairs (x0-1 .. x0+2) at rows y0 and y1
    bound = 8 * U * m4
    del m4
    if H > 1:
        dy = (x64[:, 1:] - x64[:, :-1]).abs()
        dyr = torch.stack([dy[:, (y0 + k).clamp(0, H - 2)] for k in (-1, 0, 1)]).amax(0)
        bound += 2.01 * U * fy * torch.maximum(dyr[:, :, x0], dyr[:, :, x1])
        del dy, dyr
    if W > 1:
        dx = (x64[:, :, 1:] - x64[:, :, :-1]).abs()
        dxc = torch.stack([dx[:, :, (x0 + k).clamp(0, W - 2)] for k in (-1, 0, 1)]).amax(0)
        bound += 2.01 * U * fx * torch.maximum(dxc[:, y0], dxc[:, y1])
    return ref, bound


def run_upsample(c, seed):
    from fast3r_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    n, H, W, C, Ho, Wo, dt = (c[f] for f in ("n", "H", "W", "C", "Ho", "Wo", "dt"))
    x = (torch.randn(n, H, W, C, generator=g, device="cuda") * 50).to(DT[dt])
    buf, out, before = _out((n, Ho, Wo, C), DT[dt])
    ops.upsample2x(x, out, n, H, W, C, Ho, Wo)
    torch.cuda.synchronize()
    _canaries(c["name"], buf, before)
    ref, E = upsample_ref(x, Ho, Wo)
    r = R[dt]
    return _bound_check(c["name"], out, ref, E + r * (ref.abs() + E) + (SUB if dt == "f16" else 0.0), dt)


# ------------------------------------------------------------------ the exact kernels
def run_im2col_patch(c, seed):
    from fast3r_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    n, H, W, dt = c["n"], c["H"], c["W"], c["out"]
    img = torch.randn(n, 3, H, W, generator=g, device="cuda") * 100
    rows = n * (H // 16) * (W // 16)
    buf, out, before = _out((rows, 768), DT[dt])
    ops.im2col_patch(img, out)
    torch.cuda.synchronize()
    _canaries(c["name"], buf, before)
    ref = F.unfold(img, kernel_size=16, stride=16).transpose(1, 2).reshape(-1, 768).to(DT[dt])
    _same_values(c["name"], out, ref)


def run_im2col3x3s2(c, dt, seed):
    from fast3r_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    n, H, W, C, Ho, Wo = (c[f] for f in ("n", "H", "W", "C", "Ho", "Wo"))
    x = (torch.randn(n, H, W, C, generator=g, device="cuda") * 1000).to(DT[dt])
    buf, out, before = _out((n * Ho * Wo, 9 * C), DT[dt])
    ops.im2col3x3s2(x, out, n, H, W, C, Ho, Wo)
    torch.cuda.synchronize()
    name = f"{c['name']} {dt}"
    _canaries(name, buf, before)
    u = F.unfold(x.float().permute(0, 3, 1, 2), kernel_size=3, stride=2, padding=1)  # (n, C*9, L), channel-major
    ref = u.reshape(n, C, 9, Ho * Wo).permute(0, 3, 2, 1).reshape(n * Ho * Wo, 9 * C)
    _same_values(name, out, ref)


F32_MAX = torch.finfo(torch.float32).max
CAST_EDGES = {
    # fp16: max, rounds to inf, overflows, the 2^-25 tie to 0, 3 * 2^-26 up to 2^-24, the smallest subnormal, ties to even
    "f16": [65504.0, 65520.0, -1e6, 2.0 ** -25, 3 * 2.0 ** -26, 2.0 ** -24, 1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11,
            -(1 + 2.0 ** -11), 1e-40, -0.0, float("inf"), float("-inf"), float("nan")],
    # bf16: ties to even, the largest finite, fp32 max (rounds to inf), fp32 subnormals
    "bf16": [1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8, -(1 + 2.0 ** -8), 3.3895313892515355e38, F32_MAX, 1e-40, 2.0 ** -149,
             -(2.0 ** -149), 2.0 ** -133 + 2.0 ** -141, -0.0, float("inf"), float("-inf"), float("nan")],
}


def _with_edges(x, edges):
    """x with the edge values at its start and end (the first and the last pass of a grid-stride loop)."""
    e = torch.tensor(edges, dtype=torch.float32, device=x.device)[:x.numel()]
    x[:e.numel()] = e
    if x.numel() >= 2 * e.numel():
        x[-e.numel():] = e
    return x


def run_cast(c, seed):
    from fast3r_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    n, dt = c["n"], c["out"]
    lo, hi = (-9, 4.8) if dt == "f16" else (-40, 38)
    x = torch.randn(n, generator=g, device="cuda") * torch.logspace(lo, hi, n, device="cuda")
    x = _with_edges(x, CAST_EDGES[dt])
    buf, out, before = _out((n,), DT[dt])
    (ops.cast_f16 if dt == "f16" else ops.cast_bf16)(x, out)
    torch.cuda.synchronize()
    _canaries(c["name"], buf, before)
    _same_values(c["name"], out, x.to(DT[dt]))


SPLIT_EDGES = [1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8, -(1 + 2.0 ** -8), 1 + 2.0 ** -8 + 2.0 ** -16 + 2.0 ** -17, 1e-40,
               -1e-40, 2.0 ** -149, -0.0, 0.0, 3e38, -3e38, 1.2e-38]


def run_split3(c, seed):
    from fast3r_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    rows, k = c["rows"], c["k"]
    x = torch.randn(rows * k, generator=g, device="cuda") * 3
    x = _with_edges(x, SPLIT_EDGES).view(rows, k)
    buf, out, before = _out((rows, 3 * k), torch.bfloat16)
    ops.split3(x, out, relu=c["relu"])
    torch.cuda.synchronize()
    _canaries(c["name"], buf, before)
    v = x.clamp_min(0) if c["relu"] else x
    hi = v.to(torch.bfloat16)
    lo = (v - hi.float()).to(torch.bfloat16)
    _same_values(c["name"], out, torch.cat([hi, lo, hi], -1))


def run_add_f32(c, seed):
    from fast3r_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(c["n"], generator=g, device="cuda")
    b = torch.randn(c["n"], generator=g, device="cuda") * torch.logspace(-8, 8, c["n"], device="cuda")
    buf, dst, before = _out((c["n"],), torch.float32, fill=a)
    ops.add_f32(dst, b)
    torch.cuda.synchronize()
    _canaries(c["name"], buf, before)
    _same_values(c["name"], dst, a + b)


def run_case(c, variant, seed):
    """Runs one table case (variant: the LayerNorm regime or the stride-2 im2col's 16-bit type); raises on a failure.
    Returns the largest error / bound of the bounded ops (None for the exact ones)."""
    op = c["op"]
    if op == "layernorm":
        return run_layernorm(c, variant, seed)
    if op == "upsample2x":
        return run_upsample(c, seed)
    if op == "im2col3x3s2":
        return run_im2col3x3s2(c, variant, seed)
    return dict(im2col_patch=run_im2col_patch, cast=run_cast, split3=run_split3, add_f32=run_add_f32)[op](c, seed)


def variants(c):
    return {"layernorm": LN_REGIMES, "im2col3x3s2": ("bf16", "f16")}.get(c["op"], (None,))


PARAMS = [pytest.param(c, v, id=c["name"] + (f"-{v}" if v else "")) for c in EP.CASES for v in variants(c)]


@pytest.mark.parametrize("case,variant", PARAMS)
def test_elementwise_case(case, variant):
    assert EP.key(case) == case["key"], f"{case['name']} reaches {EP.key(case)!r}, not its declared {case['key']!r}"
    i = EP.CASES.index(case)
    ratio = run_case(case, variant, seed=3000 + 8 * i + (LN_REGIMES.index(variant) if case["op"] == "layernorm" else 0))
    if ratio is not None:
        print(f"\nERROR/BOUND {case['op']} {case.get('out') or case.get('dt')} {case['name']} {variant or ''}: "
              f"{ratio:.3g}")


def test_upsample_reference_is_interpolate():
    """The float64 reference of the upsample checks is F.interpolate(scale_factor=2, bilinear, align_corners=True)."""
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(2, 7, 9, 16, generator=g, device="cuda", dtype=torch.float64)
    ref, _ = upsample_ref(x, 14, 18)
    t = F.interpolate(x.permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=True).permute(0, 2, 3, 1)
    assert float((ref - t).abs().max()) <= 1e-12 * float(x.abs().max())
    assert math.isclose(float(ref[0, -1, -1, 0]), float(x[0, -1, -1, 0]), rel_tol=1e-12)
