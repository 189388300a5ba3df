"""CPU emulator of the fast3r_b200 C ABI (TEST INFRASTRUCTURE ONLY).

An executable specification of what each ``fast3r_b200.ops`` entry point computes, written with plain torch CPU
ops: same argument meaning, same layouts, same rounding points (bf16 operands, fp32 accumulation, bf16/fp32 outputs).
tests monkeypatch it over ``fast3r_b200.model.ops`` to run the HOST orchestration (view grouping, batch permutes,
head chunking, sequence-parallel sharding over gloo, result assembly) without a GPU and compare against the
reference-generated fixtures.  It is never imported by the product; the product has no CPU path.
"""
import math

import torch
import torch.nn.functional as F

from fast3r_b200 import lib as L

BF16, F32 = torch.bfloat16, torch.float32
KERNEL_TIMER = None


def _store(dst, val):
    dst.copy_(val.to(dst.dtype).reshape(dst.shape))


def gemm(a, wt, *, w, h=1, nb=1, taps=1, bias=None, out0=None, out1=None, res0=None, res1=None, act=L.ACT_NONE,
         epi=L.EPI_STORE, ldo=None, split_col=0, out0b=None, ldo_b=0, tok_per_img=0, grid_w=0, rope_cols=0,
         rope_cos=None, rope_sin=None, emb_table=None, emb_ids=None, ct_k=0, ct_cout=0, w4=None, b4=None, pts=None,
         conf=None):
    n, k = wt.shape[0], wt.shape[-1]
    M = nb * h * w
    A = a.reshape(nb, h, w, k).float()
    W = wt.reshape(n, taps, k).float()
    if taps == 1:
        acc = A.reshape(M, k) @ W[:, 0].T
    else:  # 3x3, stride 1, zero pad 1; weight layout (out, ky*3+kx, in)
        wc = W.reshape(n, 3, 3, k).permute(0, 3, 1, 2)
        acc = F.conv2d(A.permute(0, 3, 1, 2), wc, padding=1).permute(0, 2, 3, 1).reshape(M, n)
    v = acc
    if bias is not None:
        v = v + (bias.float().repeat(n // bias.numel()) if epi == L.EPI_CONVT else bias.float())
    if epi == L.EPI_ROPE:
        t = torch.arange(M) % tok_per_img
        py, px = t // grid_w, t % grid_w
        v = v.clone()
        for c0 in range(0, rope_cols, 32):
            pos = px if (c0 // 32) % 2 else py
            cs, sn = rope_cos.float()[pos], rope_sin.float()[pos]  # (M,16)
            x1, x2 = v[:, c0:c0 + 16].clone(), v[:, c0 + 16:c0 + 32].clone()
            v[:, c0:c0 + 16] = x1 * cs - x2 * sn
            v[:, c0 + 16:c0 + 32] = x2 * cs + x1 * sn
    if epi == L.EPI_IDXEMB:
        rows = emb_ids.long().reshape(-1)
        if tok_per_img > 0:
            rows = rows.repeat_interleave(tok_per_img)
        v = v + emb_table.float()[rows]
    if epi == L.EPI_FINAL:
        y = F.relu(v) @ w4.float().T + b4.float()
        d = y[:, :3].norm(dim=-1, keepdim=True)
        _store(pts, y[:, :3] / d.clip(min=1e-8) * torch.expm1(d))
        _store(conf, 1 + y[:, 3].exp())
        return
    if epi == L.EPI_CONVT:  # column (i*k+j)*cout + o of pixel (y, x) -> pixel (y*k+i, x*k+j), channel o
        kk = ct_k
        v = v.reshape(nb, h, w, kk, kk, ct_cout).permute(0, 1, 3, 2, 4, 5).reshape(nb * h * kk * w * kk, ct_cout)
    if res0 is not None:
        v = v + res0.float().reshape(v.shape)
    if res1 is not None:
        v = v + res1.float().reshape(v.shape)
    if out1 is not None:
        _store(out1, F.relu(v))
    if out0 is None:
        return
    if act == L.ACT_RELU:
        v = F.relu(v)
    elif act == L.ACT_GELU:
        v = F.gelu(v)
    if split_col > 0:
        _store(out0, v[:, :split_col])
        _store(out0b, v[:, split_col:])
    else:
        _store(out0, v)


def linear(a, wt, bias=None, **kw):
    return gemm(a, wt, w=a.numel() // a.shape[-1], bias=bias, **kw)


def _hi_lo(x):
    hi = x.float().to(BF16)
    return hi, (x.float() - hi.float()).to(BF16)


def split3(x, out, relu=False):
    v = F.relu(x.float()) if relu else x.float()
    hi, lo = _hi_lo(v)
    _store(out, torch.cat([hi, lo, hi], dim=-1))


def gemm_x3(a, wt3, *, a_relu=False, **kw):
    a3 = torch.empty(a.shape[:-1] + (3 * a.shape[-1],), dtype=BF16)
    split3(a, a3, relu=a_relu)
    return gemm(a3, wt3, **kw)


def add_f32(dst, src):
    dst.add_(src.reshape(dst.shape))


def attention_x3(q, kv, out, *, batch, heads, sq, skv, scale, lse=None):
    """hi/lo-split operands, products hi*hi + lo*hi + hi*lo, fp32 softmax, fp32 output."""
    D = heads * 64
    qh = q.reshape(batch, sq, heads, 64).transpose(1, 2)
    kh = kv[:, :D].reshape(batch, skv, heads, 64).transpose(1, 2)
    vh = kv[:, D:].reshape(batch, skv, heads, 64).transpose(1, 2)
    (q_hi, q_lo), (k_hi, k_lo), (v_hi, v_lo) = _hi_lo(qh), _hi_lo(kh), _hi_lo(vh)
    kt_hi, kt_lo = k_hi.float().transpose(-2, -1), k_lo.float().transpose(-2, -1)
    s = (q_hi.float() @ kt_hi + q_lo.float() @ kt_hi + q_hi.float() @ kt_lo) * scale
    m = s.amax(-1, keepdim=True)
    p = torch.exp(s - m)
    p_hi, p_lo = _hi_lo(p)
    o = (p_hi.float() @ v_hi.float() + p_lo.float() @ v_hi.float() + p_hi.float() @ v_lo.float()) / p.sum(-1, keepdim=True)
    _store(out, o.transpose(1, 2).reshape(batch * sq, D))
    if lse is not None:
        _store(lse, torch.logsumexp(s, -1))


def attention(q, kv, out, *, batch, heads, sq, skv, scale, lse=None, kv_split=None):
    D = heads * 64
    qh = q.reshape(batch, sq, heads, 64).transpose(1, 2).float()
    kh = kv[:, :D].reshape(batch, skv, heads, 64).transpose(1, 2).float()
    vh = kv[:, D:].reshape(batch, skv, heads, 64).transpose(1, 2).float()
    s = (qh @ kh.transpose(-2, -1)) * scale
    o = s.softmax(-1) @ vh
    _store(out, o.transpose(1, 2).reshape(batch * sq, D))
    if lse is not None:
        _store(lse, torch.logsumexp(s, -1))


def pick_kv_split(units, key_blocks, max_split=8):
    from fast3r_b200.ops import pick_kv_split as f
    return f(units, key_blocks, max_split)


def attention_partial(q, kv, part_o, part_lse, *, part_base, n_split, batch, heads, sq, kv_rows_total, kv_row0, skv,
                      scale):
    D = heads * 64
    qh = q.reshape(batch, sq, heads, 64).transpose(1, 2).float()
    kvb = kv.reshape(batch, kv_rows_total, -1)[:, kv_row0:kv_row0 + skv]
    nblk = (skv + 127) // 128
    for s_ in range(n_split):
        lo, hi = (s_ * nblk // n_split) * 128, min(((s_ + 1) * nblk // n_split) * 128, skv)
        kh = kvb[:, lo:hi, :D].reshape(batch, hi - lo, heads, 64).transpose(1, 2).float()
        vh = kvb[:, lo:hi, D:].reshape(batch, hi - lo, heads, 64).transpose(1, 2).float()
        sc = (qh @ kh.transpose(-2, -1)) * scale
        p_ = sc.softmax(-1).to(BF16).float()  # (the kernel rounds P to bf16)
        part_o[part_base + s_] = (p_ @ vh).transpose(1, 2).reshape(batch * sq, D)
        part_lse[part_base + s_] = torch.logsumexp(sc, -1)


def attention_merge(part_o, part_lse, n_parts, out, *, batch, heads, sq):
    lse = part_lse[:n_parts]                                  # (P, b, h, sq)
    w = torch.exp(lse - lse.amax(0, keepdim=True))
    w = (w / w.sum(0, keepdim=True)).permute(0, 1, 3, 2)      # (P, b, sq, h)
    o = part_o[:n_parts].reshape(n_parts, batch, sq, heads, 64)
    _store(out, (o * w[..., None]).sum(0).reshape(batch * sq, heads * 64))


def layernorm(x, w, b, eps, out):
    _store(out, F.layer_norm(x.float(), (x.shape[-1],), w.float(), b.float(), eps))


def im2col_patch(img, out):
    n = img.shape[0]
    _store(out, F.unfold(img.float(), kernel_size=16, stride=16).transpose(1, 2).reshape(-1, 768))


def im2col3x3s2(x, out, n, h, w, c, ho, wo):
    u = F.unfold(x.reshape(n, h, w, c).float().permute(0, 3, 1, 2), kernel_size=3, stride=2, padding=1)
    _store(out, u.reshape(n, c, 9, ho * wo).permute(0, 3, 2, 1).reshape(n * ho * wo, 9 * c))


def upsample2x(x, out, n, h, w, c, ho, wo):
    r = F.interpolate(x.reshape(n, h, w, c).float().permute(0, 3, 1, 2), scale_factor=2, mode="bilinear",
                      align_corners=True)
    _store(out, r[:, :, :ho, :wo].permute(0, 2, 3, 1))


def cast_bf16(x, out):
    _store(out, x)


# ------------------------------------------------------------------ geometry tail (csrc/geometry.cu)
def conf_quantile(conf, q):
    return torch.stack([torch.quantile(c, float(q)) for c in conf])


def similarity_fit(x, y, conf=None, thr=None, valid=None):
    """Same reduction the kernel does: 17 raw moments per point set in fp64, then Umeyama from the moments."""
    views, n, _ = x.shape
    rts = torch.zeros(views, 13, dtype=F32)
    for v in range(views):
        vm = torch.ones(n, dtype=torch.bool) if valid is None else valid[v].bool()
        sel = vm if conf is None else (vm & (conf[v] >= thr[v]))
        if sel.sum() < 3:
            sel = vm
        if sel.sum() < 3:
            rts[v, 0] = rts[v, 4] = rts[v, 8] = rts[v, 12] = 1.0
            continue
        a, b = x[v][sel].double(), y[v][sel].double()
        cnt = a.shape[0]
        xm, ym = a.sum(0) / cnt, b.sum(0) / cnt
        m = b.T @ a - cnt * torch.outer(ym, xm)
        var = (a * a).sum() - cnt * (xm * xm).sum()
        u, s, vt = torch.linalg.svd(m)
        d = torch.sign(torch.det(u @ vt))
        dd = torch.tensor([1.0, 1.0, float(d) if d != 0 else 1.0], dtype=torch.float64)
        r = (u * dd) @ vt
        sc = (s * dd).sum() / var
        rts[v, :9] = r.reshape(-1).float()
        rts[v, 9:12] = (ym - sc * (r @ xm)).float()
        rts[v, 12] = sc.float()
    return rts


def similarity_apply(x, rts, out=None):
    r = rts[:, :9].reshape(-1, 3, 3)
    res = rts[:, 12].reshape(-1, 1, 1) * (x @ r.transpose(1, 2)) + rts[:, 9:12].reshape(-1, 1, 3)
    if out is None:
        return res
    out.copy_(res)
    return out


def focal_weiszfeld(pts, conf=None, thr=None, pp=None, iters=100):
    views, h, w, _ = pts.shape
    out = torch.zeros(views, dtype=F32)
    vv, uu = torch.meshgrid(torch.arange(h, dtype=F32), torch.arange(w, dtype=F32), indexing="ij")
    for v in range(views):
        cx, cy = (w / 2, h / 2) if pp is None else (float(pp[v, 0]), float(pp[v, 1]))
        px = torch.stack([uu - cx, vv - cy], -1).reshape(-1, 2)
        p = pts[v].reshape(-1, 3)
        if conf is not None:
            sel = (conf[v] >= thr[v]).reshape(-1)
            p, px = p[sel], px[sel]
        if p.shape[0] == 0:
            out[v] = max(h, w) / (2 * math.tan(math.radians(30)))
            continue
        xyz = (p[:, :2] / p[:, 2:3]).nan_to_num(nan=0.0, posinf=0.0, neginf=0.0)
        dpx, dxx = (xyz * px).sum(-1).double(), (xyz * xyz).sum(-1).double()
        f = dpx.sum() / dxx.sum()
        for _ in range(iters):
            dis = (px - f.float() * xyz).norm(dim=-1)
            wgt = dis.clip(min=1e-8).reciprocal().double()
            f = (wgt * dpx).sum() / (wgt * dxx).sum()
        out[v] = max(float(f), 0.0)
    return out
