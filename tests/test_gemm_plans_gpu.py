"""f3r_gemm per element against float64, one case per launch plan (tests/gemm_plans.CASES).  Needs an H100.

Reference.  The operands are rounded to bf16 first (A, W), so the reference is the exact result on the kernel's own
inputs: acc = unfold(A) @ W^T in float64 (3x3 taps by explicit shifts with zero padding), then the epilogue in float64 -
bias, RoPE on (acc + bias) with the kernel's fp32 cos/sin tables, the image-index embedding row, res0, res1, the
activation, the ConvTranspose scatter, and for FINAL relu -> 128x4 conv1x1 -> pts = xyz / |xyz| * expm1(|xyz|),
conf = 1 + exp(c).  The magnitude S = |unfold(A)| @ |W|^T (+ |bias| + |emb| + |res0| + |res1|, RoPE applied as
|cos| S_a + |sin| S_b) is computed the same way.

Bound, per element.  Products of bf16 values are exact in fp32, so the only error of the fp32 accumulator is the
rounding of K_eff = taps * K additions, each at most one unit of 2^-23 relative to a partial sum bounded by S (2^-22
allows for tensor-core accumulation that truncates instead of rounding), and at most 4 more roundings in the epilogue
(bias, embedding or RoPE, res0, res1, and the reduce-add of each K slice, which the slack of K_eff covers):
    |v - ref| <= E = (K_eff + 4) * 2^-22 * S.
The output is act(v) rounded to its type: relu is 1-Lipschitz; exact GELU has |gelu'| <= 1.13, and gelu_fast's erf
approximation adds at most 1.5e-7 * |x| / 2 plus a few roundings, so E_gelu = 1.2 E + 2e-7 |v|.  Rounding to bf16 adds
at most half a bf16 ulp, covered by r |ref| with r = 2^-8 (r = 0 for fp32 outputs):
    |out - ref| <= E_act + r |ref|.
FINAL propagates E through the epilogue to first order with derivatives taken in float64: the 4 outputs o_i = w4_i .
relu(v) + b4_i carry E_o,i = |w4_i| . E + (128 + 4) 2^-22 (|w4_i| . relu|v| + |b4_i|) + 2^-20 |o_i| (the last term: the
kernel's fp32 norm and exp); with d = |o_xyz| and g(d) = expm1(d) / d,
    |dpts_j| <= g E_o,j + |o_j| |g'(d)| |E_o,xyz| + 2^-20 (1 + d) |pts_j|,   |dconf| <= e^c E_o,c + 2^-20 (1 + |c|) conf.

Parity composition (run_case(..., x3=True), the cases with x3 set).  A and W are fp32; W is packed by the model's own
packing (fast3r_b200.model._Packed("fp32")._lin / _conv3 / _convt: [Whi | Whi | Wlo] along K) and A is split by
ops.gemm_x3 (split3: [hi | lo | hi], of relu(A) with a_relu).  The reference is the float64 product of the unsplit fp32
operands through the same epilogue reference, with S taken over the unsplit operands.  With hi = bf16(x) and lo =
bf16(x - hi) (x - hi is exact in fp32), |x - hi| <= 2^-9 |x|, |lo| <= 2^-9 |x| (1 + 2^-8) and the residual
|x - hi - lo| <= 2^-18 |x|; so a w - (ah wh + al wh + ah wl) = al wl + ra w + (ah + al) rw is at most
(2^-18 (1 + 2^-8)^2 + 2^-18 + 2^-18 (1 + 2^-9)) |a| |w| < 2^-16 |a| |w| per product, and
    |v - ref| <= E + 2^-16 S,
E as above with K_eff = taps * 3 k0 (the accumulator sees three products per element of K).  The stride-2 case
(x3="stride2") runs the parity forward's act_postprocess[3] conv: split3 of the map, im2col3x3s2 of the split operand
and ops.gemm over K = 27 k0 against the weight packed per tap by _conv3, compared with F.conv2d(stride 2, padding 1)
in float64.

The relative L2 error over each output is checked as well: the per-element bound catches a wrong element or tile, the
L2 check a systematic drift that stays inside the bound.  Every element outside the region a call may write (canaries
before and after each output, the columns beyond n for ldo > n, the other side of a column split) must keep its value."""
import os

import pytest
import torch
import torch.nn.functional as F

from tests import gemm_plans as GP
from fast3r_b200 import lib as L_
from tests.canaries import buffer as _buffer, check_elements, untouched as _untouched, region as _region

pytestmark = pytest.mark.gpu

REL_L2 = {"bf16": 6e-3, "f32": 3e-5, "final": 2e-3}


def _unfold(a, taps):
    """a (nb, h, w, k) float64 -> (nb*h*w, taps*k), tap-major like the packed weights [n, tap, k]."""
    nb, h, w, k = a.shape
    if taps == 1:
        return a.reshape(-1, k)
    p = F.pad(a, (0, 0, 1, 1, 1, 1))
    return torch.cat([p[:, 1 + dy:1 + dy + h, 1 + dx:1 + dx + w, :] for dy in (-1, 0, 1) for dx in (-1, 0, 1)],
                     dim=-1).reshape(-1, taps * k)


def _rope_tables(max_pos=256, base=100.0):
    j = torch.arange(16, dtype=torch.float32)
    ang = torch.arange(max_pos, dtype=torch.float32)[:, None] * (1.0 / (base ** (j / 16.0)))[None]
    return ang.cos().contiguous().cuda(), ang.sin().contiguous().cuda()


def _check(name, out, ref, bound, kind):
    check_elements(name, out, ref, bound)
    out = out.double()
    rel = float((out - ref).norm() / ref.norm().clamp_min(1e-30))
    assert rel <= REL_L2[kind], f"{name}: relative L2 error {rel:.3g} > {REL_L2[kind]}"


def _x3_weight(c, rnd):
    """fp32 weight of an x3 case in its module layout, packed by the model's own packing, and the float64 (n, taps * k0)
    matrix the reference multiplies (tap-major like _unfold), stated from the layer definitions."""
    from types import SimpleNamespace
    from fast3r_b200.model import _Packed
    P = _Packed("fp32")
    n, taps, k0 = c["n"], c["taps"], c["k"] // 3
    scale = (taps * k0) ** -0.5
    if c["epi"] == L_.EPI_CONVT:  # ConvTranspose2d (in, out, k, k): column (i*k + j)*out + o of pixel -> (i, j, o)
        kk, co = c["ct_k"], c["ct_cout"]
        wm = rnd(k0, co, kk, kk, scale=scale)
        col = torch.arange(n, device="cuda")
        return P._convt(SimpleNamespace(weight=wm)), wm.double()[:, col % co, col // (kk * co), (col // co) % kk].T
    if taps == 9:  # Conv2d (out, in, 3, 3): tap t = ky*3 + kx
        wm = rnd(n, k0, 3, 3, scale=scale)
        t = torch.arange(9, device="cuda")
        return P._conv3(SimpleNamespace(weight=wm)), wm.double()[:, :, t // 3, t % 3].transpose(1, 2).reshape(n, 9 * k0)
    wm = rnd(n, k0, scale=scale)  # Linear (out, in)
    return P._lin(SimpleNamespace(weight=wm)), wm.double()


def run_stride2_x3(c, seed):
    """The parity forward's stride-2 conv (x3="stride2"), per element against float64 (module docstring)."""
    from types import SimpleNamespace
    from fast3r_b200 import ops
    from fast3r_b200.model import _Packed
    g = torch.Generator(device="cuda").manual_seed(seed)
    k0, n = c["k"] // 27, c["n"]
    nv = c["w"] // (12 * 16)
    gh, gw, h3, w3 = 23, 32, 12, 16
    a = torch.randn(nv, gh, gw, k0, generator=g, device="cuda")
    wm = torch.randn(n, k0, 3, 3, generator=g, device="cuda") * (9 * k0) ** -0.5
    bias = torch.randn(n, generator=g, device="cuda")
    w31 = _Packed("fp32")._conv3(SimpleNamespace(weight=wm))
    a3 = torch.empty(nv, gh, gw, 3 * k0, dtype=torch.bfloat16, device="cuda")
    ops.split3(a, a3)
    col = torch.empty(nv * h3 * w3, 27 * k0, dtype=torch.bfloat16, device="cuda")
    ops.im2col3x3s2(a3, col, nv, gh, gw, 3 * k0, h3, w3)
    buf, out = _buffer((nv * h3 * w3, n), torch.float32)
    before = buf.clone()
    ops.gemm(col, w31.reshape(n, 1, -1), w=nv * h3 * w3, bias=bias, out0=out)
    torch.cuda.synchronize()
    _untouched(f"{c['name']} out0", buf, before, _region(buf.numel(), nv * h3 * w3, n, n))
    conv = lambda x, wt: F.conv2d(x.permute(0, 3, 1, 2), wt, stride=2, padding=1).permute(0, 2, 3, 1).reshape(-1, n)  # noqa: E731,E501
    ref = conv(a.double(), wm.double()) + bias.double()
    S = conv(a.double().abs(), wm.double().abs()) + bias.double().abs()
    _check(f"{c['name']} out0", out, ref, ((c["k"] + 4) * 2.0 ** -22 + 2.0 ** -16) * S, "f32")


def run_case(c, seed, x3=False):
    """Runs one table case through ops.gemm (x3: from fp32 operands through ops.gemm_x3, module docstring) and checks every
    output element; returns nothing (raises on failure)."""
    from fast3r_b200 import ops, lib as L
    if x3 and c["x3"] == "stride2":
        return run_stride2_x3(c, seed)
    g = torch.Generator(device="cuda").manual_seed(seed)
    bf, f32 = torch.bfloat16, torch.float32
    rnd = lambda *s, scale=1.0: torch.randn(*s, generator=g, device="cuda") * scale  # noqa: E731
    n, k, taps, w, h, nb, epi, act = (c[f] for f in ("n", "k", "taps", "w", "h", "nb", "epi", "act"))
    M, keff = nb * h * w, taps * k
    final, convt = epi == L.EPI_FINAL, epi == L.EPI_CONVT
    if x3:
        assert c["x3"] and k % 3 == 0 and not c["out1"] and not c["res1"], c["name"]
        a = rnd(nb, h, w, k // 3)
        wt, w64 = _x3_weight(c, rnd)
        a_ref = a.clamp_min(0) if c["a_relu"] else a
    else:
        a = rnd(nb, h, w, k).to(bf)
        wt = rnd(n, taps, k, scale=keff ** -0.5).to(bf)
        a_ref, w64 = a, wt.double().reshape(n, keff)
    nbias = c["ct_cout"] if convt else n
    bias = rnd(nbias, scale=0.5 if final else 1.0) if c["bias"] else None
    split = c["split_col"]
    ncols0 = split or n
    ldo = c["ldo"] or (c["ct_cout"] if convt else ncols0)
    kw = dict(w=w, h=h, nb=nb, taps=taps, bias=bias, act=act, epi=epi, ldo=ldo, ct_k=c["ct_k"], ct_cout=c["ct_cout"])
    outs = []  # (name, flat buffer, its old contents, written mask, values to check, reference key, dtype kind)

    # ---- float64 reference (acc, magnitude), before the outputs are written (res0 may alias out0)
    cols = _unfold(a_ref.double(), taps)
    acc = cols @ w64.T
    mag = cols.abs() @ w64.abs().T
    del cols
    if bias is not None:
        b = bias.double()[(torch.arange(n, device="cuda") % c["ct_cout"]) if convt else slice(None)]
        acc, mag = acc + b, mag + b.abs()
    if epi == L.EPI_ROPE:
        cos, sin = _rope_tables()
        kw.update(tok_per_img=c["tok_per_img"], grid_w=c["grid_w"], rope_cols=c["rope_cols"], rope_cos=cos, rope_sin=sin)
        t = torch.arange(M, device="cuda") % c["tok_per_img"]
        pos = torch.stack((t // c["grid_w"], t % c["grid_w"]))  # rows: y for the first 32 columns of 64, x for the rest
        for c0 in range(0, c["rope_cols"], 32):
            p = pos[(c0 >> 5) & 1]
            cc, ss = cos[p].double(), sin[p].double()
            x, y = acc[:, c0:c0 + 16].clone(), acc[:, c0 + 16:c0 + 32].clone()
            mx, my = mag[:, c0:c0 + 16].clone(), mag[:, c0 + 16:c0 + 32].clone()
            acc[:, c0:c0 + 16], acc[:, c0 + 16:c0 + 32] = x * cc - y * ss, y * cc + x * ss
            mag[:, c0:c0 + 16] = mx * cc.abs() + my * ss.abs()
            mag[:, c0 + 16:c0 + 32] = my * cc.abs() + mx * ss.abs()
    if epi == L.EPI_IDXEMB:
        table = rnd(1000, n)
        per = c["tok_per_img"]
        nid = -(-M // per) if per else M
        ids = torch.randint(0, 1000, (nid,), generator=g, device="cuda", dtype=torch.int32)
        ids[0], ids[-1] = 999, 0  # the table's last and first rows
        kw.update(tok_per_img=per, emb_table=table, emb_ids=ids)
        rows = ids.long().repeat_interleave(per)[:M] if per else ids.long()
        emb = table.double()[rows]
        acc, mag = acc + emb, mag + emb.abs()

    res0 = c["res0"]
    if res0:
        r0 = rnd(M, ldo)
        if res0 == "bf16":
            r0 = r0.to(bf)
        acc, mag = acc + r0.double()[:, :n], mag + r0.double()[:, :n].abs()
    if c["res1"]:
        r1 = rnd(M, ldo).to(bf)
        kw["res1"] = r1
        acc, mag = acc + r1.double()[:, :n], mag + r1.double()[:, :n].abs()
    E = ((keff + 4) * 2.0 ** -22 + (2.0 ** -16 if x3 else 0.0)) * mag

    # ---- outputs
    if final:
        w4, b4 = rnd(4, n, scale=n ** -0.5), rnd(4, scale=0.5)
        pts_buf, pts = _buffer((M, 3), f32)
        conf_buf, conf = _buffer((M,), f32)
        kw.update(w4=w4, b4=b4, pts=pts, conf=conf)
        outs += [("pts", pts_buf, pts_buf.clone(), _region(pts_buf.numel(), M, 3, 3)),
                 ("conf", conf_buf, conf_buf.clone(), _region(conf_buf.numel(), M, 1, 1))]
    elif c["out0"]:
        dt = f32 if c["out0"] == "f32" else bf
        rows_out, cols_out = (M * c["ct_k"] ** 2, c["ct_cout"]) if convt else (M, ncols0)
        buf0, out0 = _buffer((rows_out, ldo), dt, fill=r0 if res0 == "f32_inplace" else None)
        kw["out0"] = out0
        outs.append(("out0", buf0, buf0.clone(), _region(buf0.numel(), rows_out, ldo, cols_out)))
        if split:
            bufb, out0b = _buffer((M, c["ldo_b"]), dt)
            kw.update(split_col=split, out0b=out0b, ldo_b=c["ldo_b"])
            outs.append(("out0b", bufb, bufb.clone(), _region(bufb.numel(), M, c["ldo_b"], n - split)))
    if res0:
        kw["res0"] = kw["out0"] if res0 == "f32_inplace" else r0
    if c["out1"]:
        buf1, out1 = _buffer((M, ldo), bf)
        kw["out1"] = out1
        outs.append(("out1", buf1, buf1.clone(), _region(buf1.numel(), M, ldo, n)))

    if x3:
        ops.gemm_x3(a, wt, a_relu=c["a_relu"], **kw)
    else:
        ops.gemm(a, wt, **kw)
    torch.cuda.synchronize()

    # ---- checks
    for name, buf, before, written in outs:
        _untouched(f"{c['name']} {name}", buf, before, written)
    if final:
        y = acc.clamp_min(0)
        w4d, b4d = w4.double(), b4.double()
        o = y @ w4d.T + b4d
        Eo = E @ w4d.abs().T + (n + 4) * 2.0 ** -22 * (y @ w4d.abs().T + b4d.abs()) + 2.0 ** -20 * o.abs()
        xyz, d = o[:, :3], o[:, :3].norm(dim=-1, keepdim=True)
        gd = torch.expm1(d) / d
        dg = (d * torch.exp(d) - torch.expm1(d)) / (d * d)
        ref_pts = xyz * gd
        b_pts = gd * Eo[:, :3] + xyz.abs() * dg.abs() * Eo[:, :3].norm(dim=-1, keepdim=True) \
            + 2.0 ** -20 * (1 + d) * ref_pts.abs()
        cc = o[:, 3]
        ref_conf = 1 + torch.exp(cc)
        b_conf = torch.exp(cc) * Eo[:, 3] + 2.0 ** -20 * (1 + cc.abs()) * ref_conf
        _check(f"{c['name']} pts", pts, ref_pts, b_pts, "final")
        _check(f"{c['name']} conf", conf, ref_conf, b_conf, "final")
        return
    if c["out1"]:
        ref1 = acc.clamp_min(0)
        _check(f"{c['name']} out1", out1[:, :n], ref1, E + 2.0 ** -8 * ref1.abs(), "bf16")
    if not c["out0"]:
        return
    if act == L.ACT_RELU:
        ref0, E0 = acc.clamp_min(0), E
    elif act == L.ACT_GELU:
        ref0, E0 = F.gelu(acc), 1.2 * E + 2e-7 * acc.abs()
    else:
        ref0, E0 = acc, E
    kind = c["out0"]
    r = 2.0 ** -8 if kind == "bf16" else 0.0
    if convt:  # column (i*k + j)*cout + o of pixel (img, py, px) -> output pixel (py*k + i, px*k + j), channel o
        kk, co = c["ct_k"], c["ct_cout"]
        ref0 = ref0.reshape(nb, h, w, kk, kk, co).permute(0, 1, 3, 2, 4, 5).reshape(-1, co)
        E0 = E0.reshape(nb, h, w, kk, kk, co).permute(0, 1, 3, 2, 4, 5).reshape(-1, co)
        _check(f"{c['name']} out0", out0, ref0, E0 + r * ref0.abs(), kind)
        return
    _check(f"{c['name']} out0", out0[:, :ncols0], ref0[:, :ncols0], E0[:, :ncols0] + r * ref0[:, :ncols0].abs(), kind)
    if split:
        _check(f"{c['name']} out0b", out0b[:, :n - split], ref0[:, split:], E0[:, split:] + r * ref0[:, split:].abs(),
               kind)


@pytest.fixture(scope="module")
def num_sms():
    env = sorted(v for v in os.environ if v.startswith("F3R_GEMM_"))
    if env:
        pytest.skip(f"{', '.join(env)} set: the launch plans differ from the library's defaults")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if sms != GP.H100_SMS:
        pytest.skip(f"the case table's plan keys are those of a {GP.H100_SMS}-SM H100 SXM; this device has {sms} SMs")
    return sms


@pytest.mark.parametrize("case", GP.CASES, ids=[c["name"] for c in GP.CASES])
def test_gemm_case(case, num_sms):
    key = GP.plan_key(case, num_sms)
    assert key == case["key"], f"{case['name']} reaches plan {key!r}, not its declared {case['key']!r}"
    run_case(case, seed=1000 + GP.CASES.index(case))


X3_CASES = [c for c in GP.CASES if c["x3"]]


@pytest.mark.parametrize("case", X3_CASES, ids=[c["name"] for c in X3_CASES])
def test_gemm_case_x3(case, num_sms):
    """The case from fp32 operands as the parity forward computes it (module docstring)."""
    key = GP.plan_key(case, num_sms)
    assert key == case["key"], f"{case['name']} reaches plan {key!r}, not its declared {case['key']!r}"
    run_case(case, seed=4000 + GP.CASES.index(case), x3=True)
