"""The geometry tail per element against float64, one case per launch key (tests/geometry_plans.CASES).  Needs an H100.

Every output sits between canaries (tests/canaries.py) that must keep their values; inputs that the table marks as not
aligned start 4 bytes (the valid mask: 1 byte) past an aligned address.  u = 2^-24 is the fp32 unit roundoff, e = 2^-53
the fp64 one, gamma_k = k e / (1 - k e).  Reference sums are taken in numpy's long double (unit roundoff e_L = 2^-64 on
x86-64) over the float64 terms, so a reference sum of m terms is off by at most (m - 1) e_L sum|t|; that is added to
every bound below.

Quantile.  Bit-exact against torch.quantile on the same tensor and on its CPU copy, value by value (NaN matches NaN, -0
matches +0: ATen's sort does not order the two zeros).  A view holding a NaN gives NaN, whatever its sign.  torch.quantile
on a CUDA tensor sorts a NaN with the sign bit set below -inf and then returns the view's largest element instead (seen
with torch 2.11 on an H100); its CPU path returns NaN for either sign, as documented, so views with a negative NaN are
compared with the CPU result only.  (NaNs made by GPU arithmetic are positive; x86 makes negative ones.)  Regimes: random, a third of the view tied at the order statistic, +-inf at the
order statistic and next to it, one NaN of either sign (first, last or inside the view; every fourth view has none),
subnormals, -0/+0 mixes, constant views.  q runs over the table's value; the contract part crosses n with every q in
geometry_plans.QS.

Fit, the partials.  f3r_similarity_fit through the C ABI with a caller-owned workspace: partial[v][c][j] is the sum over
chunk c (geometry_plans.fit_per pixels) of moment j of the selected pixels.  Each term is exact in fp64 (a product of two
fp32 values has 48 significant bits) except sum|x|^2, which adds its three squares with two roundings.  A term passes
through at most 4 ceil(per / 1024) additions in its thread (four pixels per iteration, 1024 pixels per block iteration),
5 shuffle levels and 8 per-warp additions, so
    |partial - ref| <= gamma_K sum|t|,   K = 4 ceil(per / 1024) + 13 (+ 2 for sum|x|^2).
After the call, flagged views (fewer than 3 pixels with conf >= thr & valid) hold the valid-only moments of mode 1; the
flags themselves are checked exactly.

Fit, the solve.  rts against the host-compiled umeyama_from_moments (geometry_math.h, CPU-tested against numpy's SVD) on
the reference moments, and against geometry_oracle.umeyama of the selected points.  The kernel's totals add 32 partials
more, so they are off by gamma_{K + 32} of sum|t|.  The moment form centres by subtraction, var = sum|x|^2 - n |x_m|^2,
which amplifies that relative error by kappa = sum|x|^2 / var (1 for a centred cloud, 10^4 - 10^6 for the far clouds of
offset / spread 10^2 - 10^3); the solve's own rounding (Jacobi sweeps, normalisations) adds at most 64 e, and the
singular values of the test clouds' cross-covariance (axis ratio 3:2:1) amplify a relative perturbation of M by at most
16 in the rotation.  So the fp64 solve is off by E = 16 (K + 32 + 64) e kappa, and after the fp32 rounding of both sides
    |R - R_ref| <= u (|R| + |R_ref|) + E,   |s - s_ref| <= u (|s| + |s_ref|) + E s,
    |t - t_ref| <= u (|t| + |t_ref|) + E (|y_m| + 3 s |x_m|)   (t = y_m - s R x_m).
Views left with fewer than 3 pixels must hold the exact identity.

Apply.  out = fma(s, fma(r2, x2, fma(r1, x1, r0 x0)), t) per row: the inner dot product takes 3 roundings relative to
S = sum_j |r_j x_j|, the outer fma one more relative to the result, so with the kernel's own fp32 rts
    |out - ref| <= (1 + u) gamma3(u) |s| S + u |ref|.
Vector, scalar, misaligned and in-place paths; every element outside `out` keeps its bits.

Focal, first pass (iters = 0).  weiszfeld_iter_kernel's per-pixel terms use _rn intrinsics, so numpy float32 reproduces
x/z, y/z (non-finite -> 0), dpx = fl(fl(xz u) + fl(yz v)) and dxx exactly; each chunk (geometry_plans.focal_per pixels)
sums them in fp64 through at most ceil(per / 256) + 13 additions: |partial - ref| <= gamma_K sum|t|, count exact.  The
focal of the final kernel is fl(num / den) of the 256 partials: within u |f| + |f| (dnum / |num| + dden / den).

Focal, later iterations (iters = 1, 100) against geometry_oracle.focal_weiszfeld (fp64 throughout).  One kernel step
evaluates g(f) = sum w dpx / sum w dxx with w = 1 / max(|px - f xz|, 1e-8) in fp32 at the fp32 focal; du, dv may be
contracted to fma.  Rounding du, dv, the sum of squares, sqrt, the reciprocal and w dpx costs each weight a relative
    delta_i = u ((|f xz| + |f yz|) / dis_i + 8),
so a step is off by e_step = (sum w |dpx| delta + |f| sum w dxx delta) / sum w dxx (+ gamma_600 for the fp64 sums).  With
L_k = |g'(f_k)| along the oracle's trajectory (central difference), the error obeys
    err_{k+1} <= L_k (err_k + u |f_k|) + e_step(f_k),   err_0 = gamma_600 |f_0|,
and the result adds u |f| for its own rounding.  A view whose every z is 0 has num = den = 0: the reference
(torch, post_process.py) divides 0 / 0 and keeps the NaN through every iteration and the clip; the kernel and the oracle
return NaN too.  An empty selection returns max(H, W) / (2 tan 30 deg).

End to end.  align_local_pts3d_to_global and estimate_focal on predictions with a NaN confidence against the oracle
pipeline: a NaN threshold selects nothing, so the alignment falls back to the valid pixels and the focal to its default.
The alignment is compared at 1e-5 of the cloud's magnitude (E and the apply bound are below 1e-6 for these well
conditioned clouds), and the fit over the finite-confidence pixels, which the quantile gave before it returned NaN, is
shown to lie well outside that."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import geometry_oracle as go
from tests import geometry_plans as GP
from tests.canaries import PAD, buffer, check_elements, untouched

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
E64 = 2.0 ** -53
EL = float(np.finfo(np.longdouble).eps) / 2
MOM = 17
QREGIMES = ("random", "ties", "inf", "pos_nan", "neg_nan", "subnormal", "zeros", "constant")
FIT_REGIMES = ("random", "far100", "far1000", "mode1_solve", "mode1_identity", "three")
HERE = os.path.dirname(os.path.abspath(__file__))


def gamma(k, u=E64):
    return k * u / (1 - k * u)


def _ops():
    from fast3r_b200 import ops
    return ops


def _call(name, anchor, *args):
    ops = _ops()
    ops._call(name, anchor, *[ops._ptr(a) if isinstance(a, torch.Tensor) or a is None else a for a in args])


def _inp(a, dtype, aligned):
    """A contiguous CUDA copy of numpy array `a`: at an aligned base, or one element (4 bytes; 1 byte for uint8) past."""
    t = torch.from_numpy(np.ascontiguousarray(a)).to(dtype)
    flat = torch.empty(t.numel() + 16, dtype=dtype, device="cuda")
    off = 0 if aligned else 1
    v = flat[off:off + t.numel()].view(t.shape)
    v.copy_(t)
    assert (v.data_ptr() % 16 == 0) == aligned or v.numel() == 0
    return v


def _canaries(name, buf, before):
    written = torch.zeros_like(buf, dtype=torch.bool)
    written[PAD:buf.numel() - PAD] = True
    untouched(name, buf, before, written)


def _ratio(err, bound):
    return float((np.asarray(err, np.float64) / np.maximum(np.asarray(bound, np.float64), 1e-300)).max(initial=0.0))


def _check(name, got, ref, bound):
    """Per element on the CPU in float64; returns the largest error / bound."""
    g, r, b = (torch.as_tensor(np.asarray(a, np.float64)) for a in (got, ref, bound))
    check_elements(name, g, r, b)
    return _ratio((g - r).abs().numpy(), b.numpy())


def _report(kind, name, ratio):
    print(f"\nERROR/BOUND {kind} {name}: {ratio:.3g}")


# ------------------------------------------------------------------ quantile
def quantile_input(views, n, q, regime, rng):
    f = np.float32
    lo, hi, _ = GP.quantile_rank(n, q)
    c = (1 + np.exp(rng.standard_normal((views, n)))).astype(f)
    for v in range(views):
        row = c[v]
        if regime == "ties":
            row[rng.permutation(n)[:max(1, n // 3)]] = np.sort(row)[lo]
        elif regime == "inf":
            s = np.sort(row)
            j = v % 4
            if j == 0:
                s[lo:] = np.inf        # the order statistic is +inf
            elif j == 1:
                s[lo + 1:] = np.inf    # the order statistic finite, its successor +inf
            elif j == 2:
                s[:lo + 1] = -np.inf   # the order statistic -inf, its successor finite
            else:
                s[:lo + 2] = -np.inf   # both -inf
            row[:] = rng.permutation(s)
        elif regime in ("pos_nan", "neg_nan") and v % 4 != 3:
            pos = (0, n - 1, int(rng.integers(n)))[v % 3]
            row[pos] = np.array([0x7FC00000 if regime == "pos_nan" else 0xFFC00001], np.uint32).view(f)[0]
        elif regime == "subnormal":
            row[:] = (rng.standard_normal(n) * 1e-39).astype(f)
            row[rng.permutation(n)[:max(1, n // 7)]] = f(2.0 ** -149)
        elif regime == "zeros":
            r = rng.random(n)
            row[:] = np.where(r < 0.45, f(-0.0), np.where(r < 0.9, f(0.0), rng.standard_normal(n).astype(f)))
        elif regime == "constant":
            row[:] = (f(2.5), f(-0.0), f(3e-39), f(-7.0))[v % 4]
    return c


def run_quantile(c, regime, seed):
    views, n, q = c["views"], c["n"], c["q"]
    rng = np.random.default_rng(seed)
    conf = _inp(quantile_input(views, n, q, regime, rng), torch.float32, c["aligned"])
    buf, thr = buffer((views,), torch.float32)
    before = buf.clone()
    _call("f3r_conf_quantile", conf, conf, views, n, float(q), thr)
    torch.cuda.synchronize()
    name = f"{c['name']} {regime}"
    _canaries(name, buf, before)
    got = thr.cpu()
    wants = [("cpu", torch.stack([torch.quantile(conf[v].cpu(), q) for v in range(views)]))]
    if regime != "neg_nan":
        wants.append(("cuda", torch.stack([torch.quantile(conf[v], q) for v in range(views)]).cpu()))
    for where, want in wants:
        same = (got == want) | (got.isnan() & want.isnan())
        if not bool(same.all()):
            bad = (~same).nonzero().flatten()[:5].tolist()
            raise AssertionError(f"{name}: {int((~same).sum())} of {views} views differ from torch.quantile on the {where}; "
                                 f"views {bad}: got {[float(got[i]) for i in bad]} want {[float(want[i]) for i in bad]}")


# ------------------------------------------------------------------ similarity fit
def _rot(rng):
    q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
    return q * np.sign(np.linalg.det(q))


def fit_input(views, n, with_conf, with_valid, rng):
    """x, y (views, n, 3) fp32, conf (views, n), thr (views,), valid (views, n) bool - per-view regimes FIT_REGIMES."""
    f = np.float32
    x = np.empty((views, n, 3), f)
    y = np.empty((views, n, 3), f)
    conf = (1 + rng.random((views, n))).astype(f)
    thr = np.empty(views, f)
    valid = np.ones((views, n), bool)
    tri = np.array([[2.0, 0, 0], [0, 1.0, 0], [0, 0, 0.5]])
    for v in range(views):
        reg = FIT_REGIMES[v % len(FIT_REGIMES)]
        off = {"far100": 1e2, "far1000": 1e3}.get(reg, 0.0)
        xv = rng.standard_normal((n, 3)) * np.array([3.0, 2.0, 1.0]) @ _rot(rng).T + off * _rot(rng)[0]
        if with_valid:
            valid[v] = rng.random(n) > 0.2
        three = None
        if reg == "mode1_identity" and with_valid and n >= 2:
            valid[v] = False
            valid[v, rng.permutation(n)[:2]] = True
        if reg == "three" and not with_conf and with_valid and n >= 3:  # without conf: exactly 3 valid pixels
            three = rng.permutation(n)[:3]
            valid[v] = False
            valid[v, three] = True
        cv, vm = conf[v], valid[v]
        ranked = np.sort(cv[vm])[::-1]
        if reg == "mode1_solve":
            thr[v] = ranked[1] if ranked.size >= 2 else f(3.0)   # 2 selected (or none): mode 1 over >= 3 valid
        elif reg == "three" and with_conf and ranked.size >= 3:
            thr[v] = ranked[2]                                      # exactly 3 selected
            three = np.nonzero(vm & (cv >= thr[v]))[0]
        else:
            thr[v] = np.quantile(cv, 0.3).astype(f)
        if three is not None and len(three) == 3:  # a well-conditioned triangle (planar: the third singular value is 0)
            xv[three] = tri @ _rot(rng).T + off * _rot(rng)[0]
        x[v] = xv
        s = rng.uniform(0.5, 2.0)
        y[v] = s * xv @ _rot(rng).T + rng.standard_normal(3) * (1 + off) + 0.01 * rng.standard_normal((n, 3))
    return x, y, conf, thr, valid


def moment_terms(xv, yv):
    """The 17 per-pixel moment terms in float64 (x, y fp32 -> exact products)."""
    a, b = xv.astype(np.float64), yv.astype(np.float64)
    yield np.ones(len(a))
    for i in range(3):
        yield a[:, i]
    for i in range(3):
        yield b[:, i]
    yield (a * a).sum(1)
    for i in range(3):
        for j in range(3):
            yield b[:, i] * a[:, j]


def chunk_sums(term, sel, per, chunks):
    """(long-double sums, float64 sums of |term|) of term over the selected pixels of each chunk."""
    n = len(term)
    pad = np.zeros(per * chunks, np.float64)
    pad[:n] = np.where(sel, term, 0.0)
    pad = pad.reshape(chunks, per)
    return pad.astype(np.longdouble).sum(1), np.abs(pad).sum(1)


def fit_reference(x, y, conf, thr, valid, with_conf):
    """Per view: (selection, flagged, partial ref [32][17] long double, abs sums [32][17])."""
    views, n = x.shape[0], x.shape[1]
    per = GP.fit_per(n)
    out = []
    for v in range(views):
        sel = valid[v] & (conf[v] >= thr[v]) if with_conf else valid[v].copy()
        flagged = with_conf and int(sel.sum()) < 3
        if flagged:
            sel = valid[v].copy()
        ref = np.zeros((GP.FIT_CHUNKS, MOM), np.longdouble)
        ab = np.zeros((GP.FIT_CHUNKS, MOM))
        for j, t in enumerate(moment_terms(x[v], y[v])):
            ref[:, j], ab[:, j] = chunk_sums(t, sel, per, GP.FIT_CHUNKS)
        out.append((sel, flagged, ref, ab))
    return out


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    """geometry_math.h compiled for the host, as tests/test_geometry_math_cpu.py builds it."""
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    so = str(tmp_path_factory.mktemp("geom") / "libgeom_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I",
                           os.path.join(HERE, "..", "fast3r_b200", "csrc"), os.path.join(HERE, "geometry_math_host.cpp"),
                           "-o", so])
    lib = C.CDLL(so)
    lib.f3r_test_umeyama_from_moments.argtypes = [C.c_void_p, C.c_void_p]
    return lib


def _host_solve(lib, m):
    m = np.ascontiguousarray(m, np.float64)
    out = np.zeros(13, np.float32)
    lib.f3r_test_umeyama_from_moments(m.ctypes.data, out.ctypes.data)
    return out


def _rts_bound(got, ref, E, xm, ym, s):
    b = U * (np.abs(got) + np.abs(ref))
    b[:9] += E
    b[9:12] += E * (np.abs(ym).max() + 3 * abs(s) * np.abs(xm).max())
    b[12] += E * abs(s)
    return b


def run_fit(c, seed, hostlib):
    from fast3r_b200 import lib as L
    views, n, wc, wv, al = c["views"], c["n"], c["conf"], c["valid"], c["aligned"]
    rng = np.random.default_rng(seed)
    x, y, conf, thr, valid = fit_input(views, n, wc, wv, rng)
    xt, yt = _inp(x, torch.float32, al), _inp(y, torch.float32, al)
    ct = _inp(conf, torch.float32, al) if wc else None
    tt = torch.from_numpy(thr).cuda() if wc else None
    vt = _inp(valid.astype(np.uint8), torch.uint8, al) if wv else None
    nbytes = L.load().f3r_similarity_fit_workspace(views)
    ws = torch.full((nbytes // 8,), float("nan"), dtype=torch.float64, device="cuda")
    buf, rts = buffer((views, 13), torch.float32)
    before = buf.clone()
    _call("f3r_similarity_fit", xt, xt, yt, ct, tt, vt, views, n, rts, ws.data_ptr(), nbytes)
    torch.cuda.synchronize()
    name = c["name"]
    _canaries(name, buf, before)
    part = ws[:views * GP.FIT_CHUNKS * MOM].view(views, GP.FIT_CHUNKS, MOM).cpu().numpy()
    flags = ws[views * GP.FIT_CHUNKS * MOM:].view(torch.int32)[:views].cpu().numpy()
    rts = rts.cpu().numpy()
    if not wv:
        valid[:] = True
    per = GP.fit_per(n)
    k = 4 * math.ceil(per / 1024) + 13
    kk = np.full(MOM, k)
    kk[7] += 2
    worst = dict(partial=0.0, solve=0.0, oracle=0.0)
    for v, (sel, flagged, ref, ab) in enumerate(fit_reference(x, y, conf, thr, valid, wc)):
        if wc:
            assert flags[v] == int(flagged), (name, v, flags[v], flagged)
        bound = np.array([gamma(kj) for kj in kk])[None, :] * ab + (per - 1) * EL * ab
        worst["partial"] = max(worst["partial"], _check(f"{name} view {v} partials", part[v], ref.astype(np.float64),
                                                        bound))
        tot = ref.sum(0)
        cnt = int(sel.sum())
        if cnt < 3:
            assert np.array_equal(rts[v], np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0, 1], np.float32)), (name, v, rts[v])
            continue
        xs, ys = x[v][sel].astype(np.float64), y[v][sel].astype(np.float64)
        xm, ym = xs.mean(0), ys.mean(0)
        kappa = float((xs * xs).sum() / ((xs - xm) ** 2).sum())
        E = 16 * (kk.max() + 32 + 64) * E64 * kappa
        want = _host_solve(hostlib, tot.astype(np.float64))
        s = float(want[12])
        worst["solve"] = max(worst["solve"], _check(f"{name} view {v} rts vs umeyama_from_moments", rts[v], want,
                                                    _rts_bound(rts[v], want, E, xm, ym, s)))
        r0, t0, s0 = go.umeyama(xs, ys)
        o = np.concatenate([r0.reshape(-1), t0, [s0]])
        worst["oracle"] = max(worst["oracle"], _check(f"{name} view {v} rts vs oracle", rts[v], o,
                                                      _rts_bound(rts[v], o, E, xm, ym, s0)))
    return worst


# ------------------------------------------------------------------ similarity apply
def run_apply(c, seed):
    views, n, al, alias = c["views"], c["n"], c["aligned"], c["alias"]
    rng = np.random.default_rng(seed)
    f = np.float32
    x = (rng.standard_normal((views, n, 3)) * 10 + rng.standard_normal((views, 1, 3)) * 100).astype(f)
    rts = np.concatenate([np.stack([_rot(rng).reshape(-1) for _ in range(views)]),
                          rng.standard_normal((views, 3)) * 50, rng.uniform(0.1, 5, (views, 1))], 1).astype(f)
    total = views * n * 3
    off = 0 if al else 1
    xbuf, xwhole = buffer((total + 1,), torch.float32)
    xt = xwhole[off:off + total].view(views, n, 3)
    xt.copy_(torch.from_numpy(x))
    if alias:
        obuf, ot = xbuf, xt
    else:
        obuf, owhole = buffer((total + 1,), torch.float32)
        ot = owhole[off:off + total].view(views, n, 3)
    xbefore, obefore = xbuf.clone(), obuf.clone()
    rt = torch.from_numpy(rts).cuda()
    _call("f3r_similarity_apply", xt, xt, rt, ot, views, n)
    torch.cuda.synchronize()
    name = c["name"]
    written = torch.zeros_like(obuf, dtype=torch.bool)
    written[PAD + off:PAD + off + total] = True
    untouched(name, obuf, obefore, written)
    if not alias:
        assert torch.equal(xbuf, xbefore), f"{name}: the input changed"
    r = rts[:, :9].astype(np.float64).reshape(views, 1, 3, 3)
    s = rts[:, 12].astype(np.float64).reshape(views, 1, 1)
    x64 = x.astype(np.float64)
    ref = s * np.einsum("vnij,vkj->vki", r, x64) + rts[:, 9:12].astype(np.float64).reshape(views, 1, 3)
    S = np.einsum("vnij,vkj->vki", np.abs(r), np.abs(x64))
    bound = (1 + U) * gamma(3, U) * np.abs(s) * S + U * np.abs(ref)
    return _check(name, ot.cpu().numpy(), ref, bound)


# ------------------------------------------------------------------ focal
def focal_input(views, H, W, with_conf, with_pp, rng):
    """pts (views, H, W, 3), conf (views, H, W), thr (views,), pp (views, 2) - per-view regimes: noisy pinhole, z = 0 and
    NaN pixels, every z = 0, an empty selection (with conf; else another pinhole)."""
    f = np.float32
    pts = np.empty((views, H, W, 3), f)
    conf = (1 + rng.random((views, H, W))).astype(f)
    thr = np.empty(views, f)
    pp = np.empty((views, 2), f)
    vv, uu = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    for v in range(views):
        pp[v] = (W / 2 + 1.5 * (v + 1), H / 2 - 2.0 * v) if with_pp else (W / 2, H / 2)
        foc = 0.8 * max(H, W) + 37.0 * v + 5
        z = 2 + np.sin(uu / 50 + v) * np.cos(vv / 40) + rng.random((H, W)) * 0.1
        px = uu - pp[v, 0] + rng.standard_normal((H, W)) * 0.5
        py = vv - pp[v, 1] + rng.standard_normal((H, W)) * 0.5
        p = np.stack([px * z / foc, py * z / foc, z], -1)
        j = v % 4
        if j == 1:
            p.reshape(-1, 3)[::7, 2] = 0.0                  # x / 0 -> +-inf -> 0
            p.reshape(-1, 3)[3::11] = 0.0                   # 0 / 0 -> NaN -> 0
            p.reshape(-1, 3)[5::13, 0] = np.nan             # NaN / z -> 0
        elif j == 2:
            p[..., 2] = 0.0
        pts[v] = p
        thr[v] = np.quantile(conf[v], 0.1).astype(f)
        if j == 3 and with_conf:
            thr[v] = conf[v].max() + 1
    return pts, conf, thr, pp


def focal_terms(pts, pp, H, W):
    """Per pixel (xz, yz, u, v, dpx, dxx) in float32 exactly as weiszfeld_iter_kernel computes them."""
    f = np.float32
    p = pts.reshape(-1, 3)
    with np.errstate(divide="ignore", invalid="ignore"):
        xz, yz = p[:, 0] / p[:, 2], p[:, 1] / p[:, 2]
    xz = np.where(np.isfinite(xz), xz, f(0)).astype(f)
    yz = np.where(np.isfinite(yz), yz, f(0)).astype(f)
    i = np.arange(H * W)
    u = ((i % W).astype(f) - f(pp[0])).astype(f)
    v = ((i // W).astype(f) - f(pp[1])).astype(f)
    dpx = (xz * u + yz * v).astype(f)  # numpy float32: each product and the sum rounded once
    dxx = (xz * xz + yz * yz).astype(f)
    return xz, yz, u, v, dpx, dxx


def _g(f, xz, yz, u, v, dpx, dxx):
    dis = np.sqrt((u - f * xz) ** 2 + (v - f * yz) ** 2)
    w = 1.0 / np.maximum(dis, 1e-8)
    return (w * dpx).sum() / (w * dxx).sum(), w, dis


def focal_bound(terms, iters):
    """(oracle focal, bound) from the error recurrence of the module docstring, in float64."""
    xz, yz, u, v, dpx, dxx = (t.astype(np.float64) for t in terms)
    f = dpx.sum() / dxx.sum()
    err = gamma(600) * abs(f)
    for _ in range(iters):
        h = 1e-6 * abs(f)
        gp, _, _ = _g(f + h, xz, yz, u, v, dpx, dxx)
        gm, _, _ = _g(f - h, xz, yz, u, v, dpx, dxx)
        L = 1.01 * abs(gp - gm) / (2 * h)
        g, w, dis = _g(f, xz, yz, u, v, dpx, dxx)
        delta = U * ((np.abs(f * xz) + np.abs(f * yz)) / np.maximum(dis, 1e-8) + 8)
        den = (w * dxx).sum()
        e_step = ((w * np.abs(dpx) * delta).sum() + abs(f) * (w * dxx * delta).sum()) / den + gamma(600) * abs(g)
        err = L * (err + U * abs(f)) + e_step
        f = g
    return max(f, 0.0), err + U * abs(f)


def run_focal(c, seed):
    from fast3r_b200 import lib as L
    views, H, W, wc, wp, iters = c["views"], c["H"], c["W"], c["conf"], c["pp"], c["iters"]
    n = H * W
    rng = np.random.default_rng(seed)
    pts, conf, thr, pp = focal_input(views, H, W, wc, wp, rng)
    pt = _inp(pts, torch.float32, True)
    ct = _inp(conf, torch.float32, True) if wc else None
    tt = torch.from_numpy(thr).cuda() if wc else None
    ppt = torch.from_numpy(pp).cuda() if wp else None
    nbytes = L.load().f3r_focal_workspace(views)
    ws = torch.full((nbytes // 8,), float("nan"), dtype=torch.float64, device="cuda")
    buf, foc = buffer((views,), torch.float32)
    before = buf.clone()
    _call("f3r_focal_weiszfeld", pt, pt, ct, tt, ppt, views, H, W, iters, foc, ws.data_ptr(), nbytes)
    torch.cuda.synchronize()
    name = c["name"]
    _canaries(name, buf, before)
    got = foc.cpu().numpy().astype(np.float64)
    default = float(np.float32(max(H, W) / (2 * math.tan(math.pi / 6))))
    per = GP.focal_per(n)
    kind = "first-pass" if iters == 0 else "iterated"
    part = ws[:views * GP.FOC_CHUNKS * 3].view(views, GP.FOC_CHUNKS, 3).cpu().numpy()
    worst = {"partial": 0.0, kind: 0.0} if iters == 0 else {kind: 0.0}
    for v in range(views):
        terms = focal_terms(pts[v], pp[v], H, W)
        sel = (conf[v].reshape(-1) >= thr[v]) if wc else np.ones(n, bool)
        tag = f"{name} view {v}"
        if iters == 0:
            k = math.ceil(per / 256) + 13
            ref = np.zeros((GP.FOC_CHUNKS, 3))
            bnd = np.zeros((GP.FOC_CHUNKS, 3))
            sums = []
            for j, t in enumerate((terms[4], terms[5], np.ones(n, np.float32))):
                s, ab = chunk_sums(t.astype(np.float64), sel, per, GP.FOC_CHUNKS)
                ref[:, j], bnd[:, j] = s.astype(np.float64), (gamma(k) + (per - 1) * EL) * ab
                sums.append((s.sum(), ab.sum()))
            worst["partial"] = max(worst["partial"], _check(f"{tag} partials", part[v], ref, bnd))
            (num, anum), (den, aden), (cnt, _) = sums
            if cnt == 0:
                assert got[v] == default, (tag, got[v], default)
                continue
            with np.errstate(invalid="ignore", divide="ignore"):
                want = max(float(num / den), 0.0) if not np.isnan(float(num / den)) else float("nan")
            if np.isnan(want):
                assert np.isnan(got[v]), (tag, got[v])
                continue
            rel = gamma(k + 256) * (anum / abs(float(num)) + aden / float(den))
            worst[kind] = max(worst[kind], _check(f"{tag} focal", [got[v]], [want],
                                                  [U * abs(want) + abs(want) * rel * 1.01]))
            continue
        with np.errstate(invalid="ignore", divide="ignore"):
            want = go.focal_weiszfeld(pts[v], pp[v], sel.reshape(H, W) if wc else None, iters)
        if not sel.any():
            assert got[v] == np.float32(want), (tag, got[v], want)
            continue
        if np.isnan(want):
            assert np.isnan(got[v]), (tag, got[v], want)
            continue
        sub = tuple(t[sel] for t in terms)
        f_ref, bound = focal_bound(sub, iters)
        assert abs(f_ref - want) <= 1e-9 * abs(want), (tag, f_ref, want)  # the bound's trajectory is the oracle's
        worst[kind] = max(worst[kind], _check(f"{tag} focal", [got[v]], [want], [bound]))
    return worst


# ------------------------------------------------------------------ the table
def _params():
    out = []
    for c in GP.CASES:
        for r in (QREGIMES if c["op"] == "quantile" else (None,)):
            out.append(pytest.param(c, r, id=c["name"] + (f"-{r}" if r else "")))
    return out


@pytest.mark.parametrize("case,regime", _params())
def test_geometry_case(case, regime, request):
    assert GP.key(case) == case["key"], f"{case['name']} reaches {GP.key(case)!r}, not its declared {case['key']!r}"
    i = GP.CASES.index(case)
    seed = 5000 + 16 * i + (QREGIMES.index(regime) if regime else 0)
    op = case["op"]
    if op == "quantile":
        run_quantile(case, regime, seed)
    elif op == "fit":
        for k, r in run_fit(case, seed, request.getfixturevalue("hostlib")).items():
            _report(f"fit {k}", case["name"], r)
    elif op == "apply":
        _report("apply", case["name"], run_apply(case, seed))
    else:
        for k, r in run_focal(case, seed).items():
            _report(f"focal {k}", case["name"], r)


# ------------------------------------------------------------------ end to end with a NaN confidence
def _nan_preds(rng, h, w):
    f = np.float32
    preds, views = [], []
    for i in range(3):
        x = rng.standard_normal((1, h, w, 3)) * np.array([3.0, 2.0, 1.0])
        conf = (1 + np.exp(rng.standard_normal((1, h, w)))).astype(f)
        noise = rng.standard_normal((1, h, w, 3)) / conf[..., None].astype(np.float64) ** 2  # confident pixels fit best
        y = 1.3 * x @ _rot(rng).T + np.array([1.0, -2.0, 0.5]) + noise
        if i < 2:
            conf.reshape(-1)[int(rng.integers(h * w))] = np.nan if i == 0 else -np.nan
        preds.append(dict(pts3d_local=torch.from_numpy(x.astype(f)), pts3d_in_other_view=torch.from_numpy(y.astype(f)),
                          conf=torch.from_numpy(conf), conf_local=torch.from_numpy(conf.copy())))
        views.append(dict(valid_mask=torch.from_numpy(rng.random((1, h, w)) > 0.3)))
    return preds, views


def test_nan_confidence_end_to_end():
    from fast3r_b200 import postprocess
    rng = np.random.default_rng(11)
    h, w = 48, 64
    preds, views = _nan_preds(rng, h, w)
    postprocess.align_local_pts3d_to_global(preds, views, min_conf_thr_percentile=30)
    for i, (p, v) in enumerate(zip(preds, views)):
        xl, c, yg, vm = (t[0].numpy() for t in (p["pts3d_local"], p["conf"], p["pts3d_in_other_view"], v["valid_mask"]))
        with np.errstate(invalid="ignore"):
            want, _, _, _ = go.align_local_to_global(xl, c, yg, vm, 30.0)
        got = p["pts3d_local_aligned_to_global"][0].cpu().numpy()
        tol = 1e-5 * np.abs(want).max()
        assert np.abs(got - want).max() <= tol, (i, np.abs(got - want).max(), tol)
        if i < 2:  # what the finite-confidence pixels would have given: far outside the tolerance
            fin = np.isfinite(c)
            thr = go.conf_quantile(c[fin], 0.3)
            sel = (c >= thr) & vm
            r, t, s = go.umeyama(xl.reshape(-1, 3)[sel.reshape(-1)], yg.reshape(-1, 3)[sel.reshape(-1)])
            other = s * xl.astype(np.float64) @ r.T + t
            assert np.abs(other - want).max() > 100 * tol, i
    for i in range(2):
        p = preds[i]
        got = postprocess.estimate_focal(p["pts3d_local"].cuda(), p["conf_local"].cuda())
        with np.errstate(invalid="ignore"):
            want = go.estimate_focal(p["pts3d_local"][0].numpy(), p["conf_local"][0].numpy())
        assert want == max(h, w) / (2 * np.tan(np.deg2rad(60) / 2))  # nothing selected: the 60-degree default
        assert abs(got - want) <= U * want, (got, want)
