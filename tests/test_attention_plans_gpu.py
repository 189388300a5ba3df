"""The attention kernels per element against float64, one case per plan key (tests/attention_plans.CASES), each in two
input regimes.  Needs an H100.

Reference.  Float64 on the kernel's own inputs (bf16 q/k/v for attention_kernel, fp32 for attention_x3_kernel) with the
scale the kernel applies, sl2 = fp32(fp32(scale) * fp32(log2 e)): t_j = sl2 (q . k_j), w_j = 2^(t_j - max t) / sum,
out = sum_j w_j v_j, lse = ln 2 * log2 sum_j 2^t_j.  A key-slice partial is referred to the keys of its own slice (the
kernel's partition j0 = s * nkv / n_split of the range's key blocks); the merge output to all keys of the merged ranges.
Per row: A = max_j sum_d |q_d k_jd|, T = max_j |t_j|, the spread max t - min t, and M_i = sum_j w_j |v_ji|.

Bound of attention_kernel (bf16), per element, nkv = key blocks of the slice, u = 2^-24:
  * S in the fp32 wgmma accumulator (the GEMM test's model, K = 64): |dS_j| <= 68 * 2^-22 * A; in the exponent's
    argument (log2 units) sl2 * |dS_j|.  The reference max m the kernel subtracts cancels in O / l and in the LSE, so only
    the roundings of its use count:
  * argument fma(S, sl2, -m sl2): one rounding of |x| <= 8 + spread (the lazy reference lags the max by at most 8) and
    one of -m sl2, |m sl2| <= T: u (8 + spread + T);
  * ex2.approx.ftz.f32: 2 ulp of its result, taken as 2^-21 relative; its flush of results below 2^-126 loses at most
    nkv * 128 * 2^-126 * max|v| against a row sum >= 1;
  * each of at most nkv - 1 moves of the reference multiplies O and l of the earlier blocks by alpha = ex2((m_old - m_new)
    sl2): 2^-21 + ln2 * 6u T.
  Together every weight carries a relative error ew <= 1.01 ln2 (sl2 dS + u (8 + spread + T)) + 2^-21 + (nkv - 1)(2^-21 +
  6 ln2 u T).  The numerator O = sum P_j v_j also carries P rounded to bf16 (2^-8 relative) and its fp32 accumulation,
  128 products per key block plus one rounding per block and per rescale: (128 nkv + nkv + 4) 2^-22 of sum |P v|, so
  c = ew + 2^-8 + (129 nkv + 4) 2^-22 (1 + 2^-8).  The row sum l adds the unrounded fp32 P, 32 nkv + 4 positive
  additions per thread with 2 shuffles and nkv rescales: eL = ew + (33 nkv + 4) u.  O / l then gives
      E_i = (c M_i + eL |ref_i|) / (1 - eL) + 1.01 * 2^-23 |ref_i| (the reciprocal and the product) + the flush term,
  and the output rounding to bf16 (2^-8, not for the fp32 partials): |out_i - ref_i| <= E_i + r (|ref_i| + E_i).
  LSE = m sl2 ln2 + logf(l): ln(l) is off by eL / (1 - eL); logf (1 ulp) and the three roundings of the first term and the
  sum stay below 2^-21 (|lse| + ln2 T + 1).
attention_x3_kernel: products of hi/lo-split operands miss lo*lo and the split remainders, 3 * 2^-16 relative per product
(bf16 keeps 8 bits: |x - hi - lo| <= 2^-16 |x|), taken as 3.1 * 2^-16; S is one chain of K_eff = 192 products, dS <=
(3.1 * 2^-16 + 196 * 1.02 * 2^-22) A; exp2f is 2 ulp; P splits into Phi + Plo with the same 3.1 * 2^-16 per product in
place of the bf16 rounding of P, and the three PV chains make 384 products per key block.  The output is fp32 (r = 0).
attention_merge_kernel: w_p = __expf(lse_p - max) (2 + 1.2 |x| ulp, plus the rounding of the difference) on partial
LSEs off by at most D = max_p E_lse,p; the normalised weights are off by eta = expm1(2 D + 2.01 e_exp) relative, so
      |out - ref| <= 1.01 [(1 + eta) sum_p W_p E_p + eta sum_p W_p |O_p - ref| + (2 n + 2) u (1 + eta) sum_p W_p (|O_p| +
      E_p) + (n + 2) u |ref|] (+ the bf16 rounding),
with W_p the exact slice weights and E_p the partials' bounds; partials with LSE = -inf have weight 0.

The per-element bound grows with the key count, so a dropped or repeated key block in a long flat row can stay inside
it.  Next to it, the relative L2 error of every (batch, head, query tile, key slice) is checked against REL_L2, set from
the largest values measured on an H100 over this table (printed at the end of the module's run) with a margin of 2x.

Input regimes: "flat" (standard normal q, k, v, q scaled by the case's qscale), and "grow": dimension 0 of every head
holds +-2 in q (alternating rows) and, in k, a level that rises by more than 8 log2 units per key block over the first
seven blocks of every key range, one more in its last 64 keys and one more in its last key.  Rows with +2 then move the
lazy reference after the first block of a slice, and their maximum sits in the range's last key (in the partial last
block when there is one); rows with -2 keep theirs in the first block.  The test asserts both from the float64 scores.
Every element outside what a call may write (canaries, columns past heads * 64 for a wider ldo, slots outside [part_base,
part_base + n_split)) must keep its value, and key rows outside every range of a call are NaN."""
import math

import pytest
import torch

from tests import attention_plans as AP
from tests.canaries import PAD, buffer, check_elements, untouched, region

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
LN2 = math.log(2.0)
# largest values measured on an H100 80GB HBM3 (700 W power limit) over this table: bf16 outputs 3.1e-3, fp32 partials
# 3.0e-3, attention_x3 7.2e-5; the tolerances are twice those
REL_L2 = {"bf16": 6.2e-3, "f32": 6e-3, "x3": 1.5e-4}
MEASURED = {k: 0.0 for k in REL_L2}


def _sl2(scale):
    return float(torch.tensor(scale, dtype=torch.float32) * torch.tensor(1.4426950408889634, dtype=torch.float32))


def _ref(q, k, v, sl2):
    """float64 softmax attention of rows q (n, 64) over keys k, v (m, 64), with the quantities the bound needs."""
    t = (q @ k.T) * sl2
    tmax = t.amax(1, keepdim=True)
    p = torch.exp2(t - tmax)
    L = p.sum(1, keepdim=True)
    w = p / L
    R = dict(ref=w @ v, M=w @ v.abs(), lse=LN2 * (tmax[:, 0] + torch.log2(L[:, 0])), T=t.abs().amax(1),
             spread=tmax[:, 0] - t.amin(1), A=(q.abs() @ k.abs().T).amax(1), vmax=float(v.abs().max()))
    nb = -(-k.shape[0] // AP.KB)
    bm = torch.nn.functional.pad(t, (0, nb * AP.KB - k.shape[0]), value=-math.inf).view(-1, nb, AP.KB).amax(-1)
    ref_m, moved = bm[:, 0].clone(), torch.zeros(q.shape[0], dtype=torch.bool, device=q.device)
    for b in range(1, nb):  # the lazy reference: moves when a block's max exceeds it by more than 8 (log2 units)
        mv = bm[:, b] - ref_m > 8
        ref_m = torch.where(mv, bm[:, b], ref_m)
        moved |= mv
    R["moved"], R["max_in_last"] = bool(moved.any()), bool((bm.argmax(1) == nb - 1).any())
    return R


def _weight_err(R, nkv, sl2, x3):
    dS = (3.1 * 2.0 ** -16 + 196 * 1.02 * 2.0 ** -22) if x3 else 68 * 2.0 ** -22
    arg = sl2 * dS * R["A"] + U * (8 + R["spread"] + R["T"])
    return 1.01 * LN2 * arg + 2.0 ** -21 + (nkv - 1) * (2.0 ** -21 + 6 * LN2 * U * R["T"])


def _bounds(R, nkv, sl2, x3, r):
    """(bound of out, bound of lse) of one slice of nkv key blocks; r: relative rounding of the stored output."""
    ew = _weight_err(R, nkv, sl2, x3)
    pr, kb, f = (3.1 * 2.0 ** -16, 384, 1.02) if x3 else (2.0 ** -8, 128, 1.0)
    c = ew + pr + ((kb + 1) * nkv + 4) * 2.0 ** -22 * f * (1 + pr)
    eL = ew + (33 * nkv + 4) * U
    ref = R["ref"].abs()
    E = (c[:, None] * R["M"] + eL[:, None] * ref) / (1 - eL)[:, None] + 1.01 * 2.0 ** -23 * ref \
        + nkv * AP.KB * 2.0 ** -126 * R["vmax"]
    return E + r * (ref + E), 1.01 * eL + 2.0 ** -21 * (R["lse"].abs() + LN2 * R["T"] + 1)


def _merge_bound(parts, ref, r):
    """Bound of the merge of partials [(O_p, E_p, lse_p, Else_p)] (rows, 64) / (rows,) against ref."""
    O = torch.stack([p[0] for p in parts])
    E = torch.stack([p[1] for p in parts])
    lse = torch.stack([p[2] for p in parts])
    El = torch.stack([p[3] for p in parts])
    live = lse > -math.inf
    mx = torch.where(live, lse, -math.inf).amax(0)
    x = torch.where(live, lse - mx, torch.zeros_like(lse))
    W = torch.where(live, torch.exp(x), torch.zeros_like(x))
    W = W / W.sum(0)
    D = torch.where(live, El, torch.zeros_like(El)).amax(0)
    ee = torch.where(live, (2 + 1.2 * x.abs()) * 2.0 ** -23 + U * x.abs(), torch.zeros_like(x)).amax(0)
    eta = torch.expm1(2 * D + 2.01 * ee)[:, None]
    W, E = W[:, :, None], torch.where(live[:, :, None], E, torch.zeros_like(E))
    n = len(parts)
    s1, s2 = (W * E).sum(0), (W * (O - ref).abs()).sum(0)
    s3 = (W * (O.abs() + E)).sum(0)
    B = 1.01 * ((1 + eta) * s1 + eta * s2 + (2 * n + 2) * U * (1 + eta) * s3 + (n + 2) * U * ref.abs())
    return B + r * (ref.abs() + B)


def _rel_l2(name, kind, out, ref, tile):
    """Relative L2 error of every query tile of one (batch, head[, slice])."""
    for r0 in range(0, out.shape[0], tile):
        o, g = out[r0:r0 + tile].double(), ref[r0:r0 + tile]
        rel = float((o - g).norm() / g.norm().clamp_min(1e-30))
        MEASURED[kind] = max(MEASURED[kind], rel)
        assert rel <= REL_L2[kind], f"{name} rows {r0}..: relative L2 error {rel:.3g} > {REL_L2[kind]}"


class Growth:
    """Tracks, over a case in the "grow" regime, that the float64 scores move the lazy reference after the first block
    of some slice of >= 2 blocks and put some row's maximum in a partial last block."""

    def __init__(self):
        self.need_move = self.moved = self.need_last = self.last = False

    def add(self, R, nkv, last_partial):
        if nkv >= 2:
            self.need_move, self.moved = True, self.moved or R["moved"]
        if last_partial:
            self.need_last, self.last = True, self.last or R["max_in_last"]

    def check(self, name):
        assert self.moved or not self.need_move, f"{name}: the grow regime did not move the reference after block 0"
        assert self.last or not self.need_last, f"{name}: no row has its maximum in the partial last key block"


def _inputs(g, rows_q, rows_kv, heads, qscale, sl2, ranges, grow, dtype):
    """q (rows_q, D), kv (rows_kv, 2D) [K | V] in `dtype`; key rows outside `ranges` (first row, rows) are NaN."""
    D = heads * 64
    q = torch.randn(rows_q, D, generator=g, device="cuda") * qscale
    kv = torch.full((rows_kv, 2 * D), math.nan, device="cuda")
    step = 10 + 4 * sl2 * qscale * 8  # log2 units per level: above the lazy threshold and the scores' spread
    for r0, n in ranges:
        kv[r0:r0 + n] = torch.randn(n, 2 * D, generator=g, device="cuda")
        if grow:
            j = torch.arange(n, device="cuda")
            lev = torch.clamp(j // AP.KB, max=6).float()
            lev[-64:] = 7
            lev[-1] = 8
            for h in range(heads):
                kv[r0:r0 + n, h * 64] = lev * step / (2 * sl2)
    if grow:
        sign = torch.where(torch.arange(rows_q, device="cuda") % 2 == 0, 2.0, -2.0)
        for h in range(heads):
            q[:, h * 64] = sign
    return q.to(dtype), kv.to(dtype)


def _slot_checks(name, c, q, kv, sl2, part_o, part_lse, slot, row0, skv, b, nkv_all, j0, nkv, grow):
    """Checks slot `slot` of the partials (keys [row0, row0 + skv) of batch b, blocks j0 .. j0 + nkv) for every head;
    returns the per-head (O, E, lse, Else) for the merge bound."""
    sq, heads = c["sq"], c["heads"]
    out = []
    k0, k1 = row0 + j0 * AP.KB, row0 + min((j0 + nkv) * AP.KB, skv)
    for h in range(heads):
        qh = q[b * sq:(b + 1) * sq, h * 64:(h + 1) * 64].double()
        kh = kv[k0:k1, h * 64:(h + 1) * 64].double()
        vh = kv[k0:k1, heads * 64 + h * 64:heads * 64 + (h + 1) * 64].double()
        R = _ref(qh, kh, vh, sl2)
        Eo, El = _bounds(R, nkv, sl2, False, 0.0)
        o = part_o[slot, b * sq:(b + 1) * sq, h * 64:(h + 1) * 64]
        ls = part_lse[slot, b, h]
        tag = f"{name} slot {slot} b{b} h{h}"
        check_elements(f"{tag} part_o", o, R["ref"], Eo)
        check_elements(f"{tag} part_lse", ls, R["lse"], El)
        _rel_l2(f"{tag} part_o", "f32", o, R["ref"], AP.BF16_TILE)
        if grow is not None:
            grow.add(R, nkv, j0 + nkv == nkv_all and skv % AP.KB != 0)
        out.append((R["ref"], Eo, R["lse"], El))
    return out


def _full_checks(name, c, q, kv, sl2, out, lse, b, keys, nkv, x3, grow):
    """out / lse of one launch over the keys rows `keys` (a list of row ranges) of batch b, every head."""
    sq, heads = c["sq"], c["heads"]
    idx = torch.cat([torch.arange(r0, r0 + n, device="cuda") for r0, n in keys])
    for h in range(heads):
        qh = q[b * sq:(b + 1) * sq, h * 64:(h + 1) * 64].double()
        kh = kv[idx, h * 64:(h + 1) * 64].double()
        vh = kv[idx, heads * 64 + h * 64:heads * 64 + (h + 1) * 64].double()
        R = _ref(qh, kh, vh, sl2)
        Eo, El = _bounds(R, nkv, sl2, x3, 0.0 if x3 else 2.0 ** -8)
        o = out[b * sq:(b + 1) * sq, h * 64:(h + 1) * 64]
        tag = f"{name} b{b} h{h}"
        check_elements(f"{tag} out", o, R["ref"], Eo)
        _rel_l2(f"{tag} out", "x3" if x3 else "bf16", o, R["ref"], AP.X3_TILE if x3 else AP.BF16_TILE)
        if lse is not None:
            check_elements(f"{tag} lse", lse[b, h], R["lse"], El)
        if grow is not None:
            grow.add(R, nkv, keys[-1][1] % AP.KB != 0)


def _out_buffers(c, rows, dtype, lse):
    D = c["heads"] * 64
    ob, o = buffer((rows, c["ldo"]), dtype)
    res = [("out", ob, ob.clone(), region(ob.numel(), rows, c["ldo"], D))]
    lb = lv = None
    if lse:
        lb, lv = buffer((c["batch"], c["heads"], c["sq"]), torch.float32)
        res.append(("lse", lb, lb.clone(), region(lb.numel(), 1, lv.numel(), lv.numel())))
    return o, lv, res


def _part_buffers(slots, rows, heads, lse_shape):
    pb, po = buffer((slots, rows, heads * 64), torch.float32)
    lb, pl = buffer((slots,) + lse_shape, torch.float32)
    return pb, po, lb, pl


def _slot_region(buf, view, s0, s1):
    per = view[0].numel()
    return region(buf.numel(), 1, (s1 - s0) * per, (s1 - s0) * per, offset=PAD + s0 * per)


def run_case(c, regime, seed):
    from fast3r_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    grow = Growth() if regime == "grow" else None
    kind, heads, scale = c["kind"], c["heads"], c["scale"]
    sl2 = _sl2(scale)
    qscale = c.get("qscale", 1.0)
    D = heads * 64
    written = []
    if kind == "merge":
        return _run_merge(c, regime, g)
    if kind in ("attention", "x3"):
        B, sq, skv = c["batch"], c["sq"], c["skv"]
        x3 = kind == "x3"
        dt = torch.float32 if x3 else torch.bfloat16
        q, kv = _inputs(g, B * sq, B * skv, heads, qscale, sl2, [(b * skv, skv) for b in range(B)], grow is not None, dt)
        out, lse, written = _out_buffers(c, B * sq, dt, c["lse"])
        if x3:
            ops.attention_x3(q, kv, out, batch=B, heads=heads, sq=sq, skv=skv, scale=scale, lse=lse)
        else:
            ops.attention(q, kv, out, batch=B, heads=heads, sq=sq, skv=skv, scale=scale, lse=lse, kv_split=1)
        torch.cuda.synchronize()
        for nm, buf, before, mask in written:
            untouched(f"{c['name']} {nm}", buf, before, mask)
        for b in range(B):
            _full_checks(c["name"], c, q, kv, sl2, out, lse, b, [(b * skv, skv)], -(-skv // AP.KB), x3, grow)
    elif kind == "split":
        B, sq, total = c["batch"], c["sq"], c["kv_rows_total"]
        ranges = [(b * total + r0, n) for b in range(B) for r0, n, _ in c["ranges"]]
        q, kv = _inputs(g, B * sq, B * total, heads, qscale, sl2, ranges, grow is not None, torch.bfloat16)
        n_parts = sum(ns for _, _, ns in c["ranges"])
        slots = c["base"] + n_parts + 1
        pb, po, lb, pl = _part_buffers(slots, B * sq, heads, (B, heads, sq))
        pb0, lb0 = pb.clone(), lb.clone()
        base = c["base"]
        for r0, n, ns in c["ranges"]:
            ops.attention_partial(q, kv, po, pl, part_base=base, n_split=ns, batch=B, heads=heads, sq=sq,
                                  kv_rows_total=total, kv_row0=r0, skv=n, scale=scale)
            base += ns
        out, _, written = _out_buffers(c, B * sq, torch.bfloat16, False)
        s0 = c["base"]
        ops.attention_merge(po[s0:s0 + n_parts], pl[s0:s0 + n_parts], n_parts, out, batch=B, heads=heads, sq=sq)
        if c["direct"]:
            dout, dlse, w2 = _out_buffers(c, B * sq, torch.bfloat16, True)
            ops.attention(q, kv, dout, batch=B, heads=heads, sq=sq, skv=total, scale=scale, lse=dlse, kv_split=1)
            written += [("direct " + nm, *rest) for nm, *rest in w2]
        torch.cuda.synchronize()
        untouched(f"{c['name']} part_o", pb, pb0, _slot_region(pb, po, s0, s0 + n_parts))
        untouched(f"{c['name']} part_lse", lb, lb0, _slot_region(lb, pl, s0, s0 + n_parts))
        for nm, buf, before, mask in written:
            untouched(f"{c['name']} {nm}", buf, before, mask)
        for b in range(B):
            parts = [[] for _ in range(heads)]
            slot = s0
            for r0, n, ns in c["ranges"]:
                nkv_all = -(-n // AP.KB)
                for j0, nkv in AP.slices(nkv_all, ns):
                    got = _slot_checks(c["name"], c, q, kv, sl2, po, pl, slot, b * total + r0, n, b, nkv_all, j0, nkv,
                                       grow)
                    for h in range(heads):
                        parts[h].append(got[h])
                    slot += 1
            keys = [(b * total + r0, n) for r0, n, _ in c["ranges"]]
            idx = torch.cat([torch.arange(r0, r0 + n, device="cuda") for r0, n in keys])
            for h in range(heads):
                qh = q[b * sq:(b + 1) * sq, h * 64:(h + 1) * 64].double()
                R = _ref(qh, kv[idx, h * 64:(h + 1) * 64].double(), kv[idx, D + h * 64:D + (h + 1) * 64].double(), sl2)
                o = out[b * sq:(b + 1) * sq, h * 64:(h + 1) * 64]
                check_elements(f"{c['name']} merged b{b} h{h}", o, R["ref"], _merge_bound(parts[h], R["ref"], 2.0 ** -8))
                _rel_l2(f"{c['name']} merged b{b} h{h}", "bf16", o, R["ref"], AP.BF16_TILE)
            if c["direct"]:
                _full_checks(c["name"] + " direct", c, q, kv, sl2, dout, dlse, b, [(b * total, total)],
                             -(-total // AP.KB), False, None)
    else:
        _run_segments(c, g, sl2, grow)
    if grow is not None:
        grow.check(c["name"])


def _run_segments(c, g, sl2, grow):
    from fast3r_b200 import ops
    off, heads, ns, scale = c["offsets"], c["heads"], c["n_split"], c["scale"]
    rows, D = off[-1], heads * 64
    segs = [(a, b - a) for a, b in zip(off, off[1:]) if b > a]
    q, kv = _inputs(g, rows, rows, heads, c.get("qscale", 1.0), sl2, segs, grow is not None, torch.bfloat16)
    dev_off = torch.tensor(off, dtype=torch.int32, device="cuda")
    out, _, written = _out_buffers(dict(c, batch=1, sq=rows), rows, torch.bfloat16, False)
    if ns > 1:
        pb, po, lb, pl = _part_buffers(ns + 1, rows, heads, (heads, rows))
        pb0, lb0 = pb.clone(), lb.clone()
        ops._call("f3r_attention_segments", q, q.data_ptr(), D, kv.data_ptr(), 2 * D, None, 0, dev_off.data_ptr(),
                  len(off) - 1, rows, heads, float(scale), ns, po.data_ptr(), pl.data_ptr())
        ops.attention_merge(po[:ns], pl[:ns].reshape(ns, 1, heads, rows), ns, out, batch=1, heads=heads, sq=rows)
    else:
        ops._call("f3r_attention_segments", q, q.data_ptr(), D, kv.data_ptr(), 2 * D, out.data_ptr(), c["ldo"],
                  dev_off.data_ptr(), len(off) - 1, rows, heads, float(scale), 1, None, None)
    torch.cuda.synchronize()
    for nm, buf, before, mask in written:
        untouched(f"{c['name']} {nm}", buf, before, mask)
    if ns > 1:
        untouched(f"{c['name']} part_o", pb, pb0, _slot_region(pb, po, 0, ns))
        untouched(f"{c['name']} part_lse", lb, lb0, _slot_region(lb, pl, 0, ns))
    for a, n in segs:
        nkv_all = -(-n // AP.KB)
        nsg = min(ns, nkv_all)
        for h in range(heads):
            qh = q[a:a + n, h * 64:(h + 1) * 64].double()
            parts = []
            for s, (j0, nkv) in enumerate(AP.slices(nkv_all, nsg)):
                k0, k1 = a + j0 * AP.KB, a + min((j0 + nkv) * AP.KB, n)
                R = _ref(qh, kv[k0:k1, h * 64:(h + 1) * 64].double(), kv[k0:k1, D + h * 64:D + (h + 1) * 64].double(),
                         sl2)
                if grow is not None:
                    grow.add(R, nkv, j0 + nkv == nkv_all and n % AP.KB != 0)
                if ns == 1:
                    o = out[a:a + n, h * 64:(h + 1) * 64]
                    E, _ = _bounds(R, nkv, sl2, False, 2.0 ** -8)
                    check_elements(f"{c['name']} seg {a} h{h} out", o, R["ref"], E)
                    _rel_l2(f"{c['name']} seg {a} h{h} out", "bf16", o, R["ref"], AP.BF16_TILE)
                    continue
                Eo, El = _bounds(R, nkv, sl2, False, 0.0)
                tag = f"{c['name']} seg {a} slot {s} h{h}"
                check_elements(f"{tag} part_o", po[s, a:a + n, h * 64:(h + 1) * 64], R["ref"], Eo)
                check_elements(f"{tag} part_lse", pl[s, h, a:a + n], R["lse"], El)
                _rel_l2(f"{tag} part_o", "f32", po[s, a:a + n, h * 64:(h + 1) * 64], R["ref"], AP.BF16_TILE)
                parts.append((R["ref"], Eo, R["lse"], El))
            if ns == 1:
                continue
            for s in range(nsg, ns):  # neutral partials: O = 0, LSE = -inf exactly
                assert bool((po[s, a:a + n, h * 64:(h + 1) * 64] == 0).all()), f"{c['name']} seg {a} slot {s} part_o"
                assert bool((pl[s, h, a:a + n] == -math.inf).all()), f"{c['name']} seg {a} slot {s} part_lse"
                parts.append((torch.zeros(n, 64, dtype=torch.float64, device="cuda"),) * 2
                             + (torch.full((n,), -math.inf, dtype=torch.float64, device="cuda"),
                                torch.zeros(n, dtype=torch.float64, device="cuda")))
            R = _ref(qh, kv[a:a + n, h * 64:(h + 1) * 64].double(), kv[a:a + n, D + h * 64:D + (h + 1) * 64].double(), sl2)
            o = out[a:a + n, h * 64:(h + 1) * 64]
            check_elements(f"{c['name']} seg {a} h{h} merged", o, R["ref"], _merge_bound(parts, R["ref"], 2.0 ** -8))
            _rel_l2(f"{c['name']} seg {a} h{h} merged", "bf16", o, R["ref"], AP.BF16_TILE)


def _run_merge(c, regime, g):
    """f3r_attention_merge of given fp32 partials: slots in c["neutral"] hold O = 0, LSE = -inf; slots in c["holes"] do
    so in every other row.  "grow": the partial LSEs spread over +-40 instead of +-2."""
    from fast3r_b200 import ops
    n, B, heads, sq = c["n_parts"], c["batch"], c["heads"], c["sq"]
    spread = 40.0 if regime == "grow" else 2.0
    po = torch.randn(n, B * sq, heads * 64, generator=g, device="cuda")
    pl = torch.randn(n, B, heads, sq, generator=g, device="cuda") * spread
    for s in c["neutral"]:
        po[s], pl[s] = 0, -math.inf
    for s in c["holes"]:
        po.view(n, B, sq, -1)[s, :, ::2], pl[s, :, :, ::2] = 0, -math.inf
    out, _, written = _out_buffers(c, B * sq, torch.bfloat16, False)
    ops.attention_merge(po, pl, n, out, batch=B, heads=heads, sq=sq)
    torch.cuda.synchronize()
    for nm, buf, before, mask in written:
        untouched(f"{c['name']} {nm}", buf, before, mask)
    zero = torch.zeros(sq, 64, dtype=torch.float64, device="cuda")
    for b in range(B):
        for h in range(heads):
            O = [po[p, b * sq:(b + 1) * sq, h * 64:(h + 1) * 64].double() for p in range(n)]
            L = torch.stack([pl[p, b, h].double() for p in range(n)])
            W = torch.softmax(L, 0)
            ref = sum(W[p][:, None] * O[p] for p in range(n))
            parts = [(O[p], zero, L[p], torch.zeros(sq, dtype=torch.float64, device="cuda")) for p in range(n)]
            o = out[b * sq:(b + 1) * sq, h * 64:(h + 1) * 64]
            check_elements(f"{c['name']} b{b} h{h}", o, ref, _merge_bound(parts, ref, 2.0 ** -8))
            _rel_l2(f"{c['name']} b{b} h{h}", "bf16", o, ref, AP.BF16_TILE)


@pytest.fixture(scope="module", autouse=True)
def report_measured():
    yield
    print("\nlargest relative L2 error per (batch, head, query tile, key slice): "
          + ", ".join(f"{k} {v:.3g} (tolerance {REL_L2[k]:g})" for k, v in MEASURED.items()))


@pytest.mark.parametrize("regime", ["flat", "grow"])
@pytest.mark.parametrize("case", AP.CASES, ids=[c["name"] for c in AP.CASES])
def test_attention_case(case, regime):
    assert AP.case_keys(case) == case["keys"], f"{case['name']} reaches {AP.case_keys(case)}, not {case['keys']}"
    run_case(case, regime, seed=2000 + 2 * AP.CASES.index(case) + (regime == "grow"))
