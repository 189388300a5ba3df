"""Torch-tensor wrappers over the C ABI.  torch is plumbing here (device memory + streams); every op below
is one call into libfast3r_b200.so on ``torch.cuda.current_stream()``.  No op has a PyTorch fallback."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np
import torch

from . import lib as L

BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
HALF = (BF16, F16)  # the 16-bit types of the tensor-core operands: the bf16 and the fp16 forward

# Optional per-launch CUDA-event timing of the dominant kernel (bench.py's live roofline measurement).
# When set to a list, attention() appends (batch, heads, sq, skv, start_event, end_event), recorded on the
# launching stream.
KERNEL_TIMER = None


def _call(name: str, anchor: torch.Tensor, *args) -> None:
    """Calls library entry point `name` with `args` followed by the current stream of the CUDA tensor `anchor`'s device,
    and raises if it fails.  CUDA runtime calls inside the library (cudaFuncSetAttribute, launches) act on the CURRENT
    device, so the anchor's device is made current for the duration of the call (callers need not have done so)."""
    idx = anchor.device.index
    prev = torch.cuda.current_device()
    if prev != idx:
        torch.cuda.set_device(idx)
    try:
        rc = getattr(L.load(), name)(*args, torch.cuda.current_stream(idx).cuda_stream)
    finally:
        if prev != idx:
            torch.cuda.set_device(prev)
    L.check(rc, name)


def _scratch(nbytes: int, device) -> torch.Tensor:
    """Device workspace for one call.  The caching allocator aligns every block to >= 512 bytes, which covers the
    256-byte and 8-byte alignment the library's workspace arguments require."""
    return torch.empty(nbytes, dtype=torch.uint8, device=device)


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError("fast3r_b200 ops need CUDA tensors (there is no CPU path)")
    return t.data_ptr()


def _chk(t: torch.Tensor, dtype, name: str):
    if t.dtype != dtype:
        raise TypeError(f"{name}: expected {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise ValueError(f"{name}: must be contiguous")


def _half(t: torch.Tensor, name: str):
    """dtype of a 16-bit operand (bf16 or fp16): the kernels of that type run the call."""
    if t.dtype not in HALF:
        raise TypeError(f"{name}: expected bfloat16 or float16, got {t.dtype}")
    return t.dtype


def _elt(t: torch.Tensor) -> int:
    """Element-type code (lib.ELT_*) of a bf16 / fp32 / fp16 tensor."""
    return {BF16: L.ELT_BF16, F32: L.ELT_F32, F16: L.ELT_F16}[t.dtype]


def _f16(name: str, t: torch.Tensor) -> str:
    """The fp16 twin of attention entry point `name` for fp16 operands."""
    return name + "_f16" if t.dtype == F16 else name


def gemm(a: torch.Tensor, wt: torch.Tensor, *, w: int, h: int = 1, nb: int = 1, taps: int = 1,
         bias: Optional[torch.Tensor] = None, out0: Optional[torch.Tensor] = None,
         out1: Optional[torch.Tensor] = None, res0: Optional[torch.Tensor] = None,
         res1: Optional[torch.Tensor] = None, act: int = L.ACT_NONE, epi: int = L.EPI_STORE,
         ldo: Optional[int] = None, split_col: int = 0, out0b: Optional[torch.Tensor] = None, ldo_b: int = 0,
         tok_per_img: int = 0, grid_w: int = 0, rope_cols: int = 0, rope_cos=None, rope_sin=None,
         emb_table=None, emb_ids=None, ct_k: int = 0, ct_cout: int = 0, w4=None, b4=None, pts=None, conf=None):
    """Fused GEMM / implicit conv (f3r_gemm).  a: bf16 (..., K) channels-last with nb*h*w pixels;
    wt: bf16 (N, taps, K).  With fp16 a and wt the call runs in fp16: every 16-bit output and residual is fp16 too
    (mixing bf16 and fp16 in one call raises)."""
    h16 = _half(a, "a")
    _chk(a, h16, "a"); _chk(wt, h16, "wt")
    n, k = wt.shape[0], wt.shape[-1]
    assert wt.numel() == n * taps * k
    assert a.shape[-1] == k and a.numel() == nb * h * w * k, (a.shape, nb, h, w, k)
    d = L.GemmDesc()
    d.a, d.wt = _ptr(a), _ptr(wt)
    d.n, d.k, d.taps = n, k, taps
    d.w, d.h, d.nb = w, h, nb
    d.a_ld = k
    d.epi, d.act = epi, act
    d.ldo = ldo if ldo is not None else (ct_cout if epi == L.EPI_CONVT else n)
    d.split_col, d.ldo_b = split_col, ldo_b
    d.tok_per_img, d.grid_w, d.rope_cols = tok_per_img, grid_w, rope_cols
    d.ct_k, d.ct_cout = ct_k, ct_cout
    if bias is not None:
        _chk(bias, F32, "bias")
    d.bias = _ptr(bias)
    d.f16 = int(h16 == F16)
    if res0 is not None:
        if res0.dtype != F32:
            _chk(res0, h16, "res0")
        assert res0.is_contiguous()
        d.res0_f32 = int(res0.dtype == F32)
    d.res0 = _ptr(res0)
    if res1 is not None:
        _chk(res1, h16, "res1")
    d.res1 = _ptr(res1)
    if out0 is not None:
        if out0.dtype != F32:
            _chk(out0, h16, "out0")
        assert out0.is_contiguous()
        d.out0_f32 = int(out0.dtype == F32)
    d.out0 = _ptr(out0)
    if out0b is not None:
        assert out0 is not None and out0b.dtype == out0.dtype
    d.out0b = _ptr(out0b)
    if out1 is not None:
        _chk(out1, h16, "out1")
    d.out1 = _ptr(out1)
    d.rope_cos, d.rope_sin = _ptr(rope_cos), _ptr(rope_sin)
    d.emb_table, d.emb_ids = _ptr(emb_table), _ptr(emb_ids)
    d.w4, d.b4, d.pts, d.conf = _ptr(w4), _ptr(b4), _ptr(pts), _ptr(conf)
    _call("f3r_gemm", a, C.byref(d))


def gemm_x3(a: torch.Tensor, wt3: torch.Tensor, *, a_relu: bool = False, **kw):
    """Parity-mode GEMM: a fp32 (..., K) is split into bf16 [hi | lo | hi] (optionally of relu(a)) and multiplied with
    wt3 = bf16 (N, taps, 3K) packed as [Whi | Whi | Wlo]: hi*hi + lo*hi + hi*lo accumulated in fp32."""
    _chk(a, F32, "a")
    k = a.shape[-1]
    assert wt3.shape[-1] == 3 * k, (wt3.shape, k)
    a3 = torch.empty(a.shape[:-1] + (3 * k,), dtype=BF16, device=a.device)
    split3(a, a3, relu=a_relu)
    return gemm(a3, wt3, **kw)


def split3(x: torch.Tensor, out: torch.Tensor, relu: bool = False):
    _chk(x, F32, "x"); _chk(out, BF16, "out")
    k = x.shape[-1]
    assert out.numel() == 3 * x.numel()
    _call("f3r_split3", x, _ptr(x), _ptr(out), x.numel() // k, k, int(relu))


def add_f32(dst: torch.Tensor, src: torch.Tensor):
    _chk(dst, F32, "dst"); _chk(src, F32, "src")
    assert dst.numel() == src.numel()
    _call("f3r_add_f32", dst, _ptr(dst), _ptr(src), dst.numel())


def linear(a: torch.Tensor, wt: torch.Tensor, bias=None, **kw):
    """y = a @ wt.T (+bias ...) for a bf16 (M, K), wt bf16 (N, K)."""
    return gemm(a, wt, w=a.numel() // a.shape[-1], bias=bias, **kw)


NUM_SMS = 132
ATT_Q_TILE = 192  # query rows per attention CTA (ATT_Q_TILE in csrc/f3r_kernels.h)


def attention_units(batch: int, heads: int, sq: int) -> int:
    """(batch, head, query tile) work units of one attention launch: its CTA count before key slicing."""
    return batch * heads * -(-sq // ATT_Q_TILE)


def pick_kv_split(units: int, key_blocks: int, max_split: int = 8) -> int:
    """Key slices per (batch, head, query tile) unit (attention_units) so that units * slices CTAs fill whole waves of
    the 132 SMs (one CTA per SM): minimises ceil(units*s / 132) / s; every slice keeps >= 16 key blocks (below that the extra
    prologues and the merge pass cost more than the idle SMs); 1 = no slicing."""
    if units >= 3 * NUM_SMS:
        return 1
    best, best_cost = 1, None
    for s_ in range(1, max_split + 1):
        if s_ > 1 and key_blocks // s_ < 16:
            break
        cost = -(-units * s_ // NUM_SMS) / s_ * (1.0 + 0.01 * (s_ - 1))  # (+1 % per extra slice: merge + prologues)
        if best_cost is None or cost < best_cost - 1e-9:
            best, best_cost = s_, cost
    return best


def attention_partial(q: torch.Tensor, kv: torch.Tensor, part_o: torch.Tensor, part_lse: torch.Tensor, *, part_base: int,
                      n_split: int, batch: int, heads: int, sq: int, kv_rows_total: int, kv_row0: int, skv: int,
                      scale: float):
    """Attends q to the keys [kv_row0, kv_row0 + skv) of kv (batch*kv_rows_total, ldkv), cut into n_split slices; slice s
    fills slot part_base + s of part_o (slots, batch*sq, heads*64) fp32 / part_lse (slots, batch, heads, sq) fp32.
    q and kv: both bf16 or both fp16."""
    h16 = _half(q, "q")
    _chk(q, h16, "q"); _chk(kv, h16, "kv"); _chk(part_o, F32, "part_o"); _chk(part_lse, F32, "part_lse")
    ldq, ldkv = q.shape[-1], kv.shape[-1]
    assert q.numel() == batch * sq * ldq and kv.numel() == batch * kv_rows_total * ldkv
    slots = part_o.shape[0]
    assert part_base + n_split <= slots and part_o.numel() == slots * batch * sq * heads * 64
    assert part_lse.numel() == slots * batch * heads * sq
    _call(_f16("f3r_attention_partial", q), q, _ptr(q), ldq, _ptr(kv), ldkv, kv_rows_total, kv_row0, skv, n_split, _ptr(part_o),
          _ptr(part_lse), part_base, batch, heads, sq, float(scale))


def attention_merge(part_o: torch.Tensor, part_lse: torch.Tensor, n_parts: int, out: torch.Tensor, *, batch: int,
                    heads: int, sq: int):
    _chk(part_o, F32, "part_o"); _chk(part_lse, F32, "part_lse"); _half(out, "out"); _chk(out, out.dtype, "out")
    assert out.numel() == batch * sq * out.shape[-1] and n_parts <= part_o.shape[0]
    _call(_f16("f3r_attention_merge", out), out, _ptr(part_o), _ptr(part_lse), n_parts, _ptr(out), out.shape[-1], batch, heads, sq)


def attention(q: torch.Tensor, kv: torch.Tensor, out: torch.Tensor, *, batch: int, heads: int, sq: int, skv: int,
              scale: float, lse: Optional[torch.Tensor] = None, kv_split: Optional[int] = None):
    """q (batch*sq, ldq) bf16, kv (batch*skv, ldkv) bf16 [K | V], out (batch*sq, ldo) bf16 (or all three fp16: the
    fp16 kernels).  When the launch would
    leave SMs idle (few query tiles), the keys are cut into slices (more CTAs) and merged (pick_kv_split).  lse (batch,
    heads, sq) fp32 receives the log-sum-exp of the scaled scores; it is written by the one-slice kernel only, so lse with
    kv_split > 1 is refused."""
    if lse is not None and kv_split is not None and kv_split > 1:
        raise ValueError("ops.attention: lse is only written without key slices (kv_split > 1 merges partials that "
                         "carry no log-sum-exp output)")
    h16 = _half(q, "q")
    _chk(q, h16, "q"); _chk(kv, h16, "kv"); _chk(out, h16, "out")
    ldq, ldkv, ldo = q.shape[-1], kv.shape[-1], out.shape[-1]
    assert q.numel() == batch * sq * ldq and kv.numel() == batch * skv * ldkv and out.numel() == batch * sq * ldo
    timer = KERNEL_TIMER
    if timer is not None:
        st = torch.cuda.current_stream(q.device)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
    ns = kv_split if kv_split is not None else (
        1 if lse is not None else pick_kv_split(attention_units(batch, heads, sq), (skv + 127) // 128))
    if ns > 1:
        part_o = torch.empty(ns, batch * sq, heads * 64, dtype=F32, device=q.device)
        part_lse = torch.empty(ns, batch, heads, sq, dtype=F32, device=q.device)
        attention_partial(q, kv, part_o, part_lse, part_base=0, n_split=ns, batch=batch, heads=heads, sq=sq,
                          kv_rows_total=skv, kv_row0=0, skv=skv, scale=scale)
        attention_merge(part_o, part_lse, ns, out, batch=batch, heads=heads, sq=sq)
    else:
        _call(_f16("f3r_attention", q), q, _ptr(q), ldq, _ptr(kv), ldkv, _ptr(out), ldo, _ptr(lse), batch, heads, sq, skv,
              float(scale))
    if timer is not None:
        e1.record(st)
        timer.append((batch, heads, sq, skv, e0, e1))


class Segments:
    """Segment boundaries of a packed sequence, for attention_segments: the host offsets (they size the launch and pick
    the key split) and their int32 device copy, uploaded once for every call that shares them."""

    def __init__(self, offsets, device):
        self.offsets = [int(v) for v in offsets]
        if len(self.offsets) < 2 or self.offsets[0] != 0 or any(b < a for a, b in zip(self.offsets, self.offsets[1:])):
            raise ValueError(f"segment offsets must start at 0 and not decrease, got {self.offsets}")
        self.device_offsets = torch.tensor(self.offsets, dtype=torch.int32).to(device)

    @property
    def rows(self) -> int:
        return self.offsets[-1]

    def lengths(self):
        return [b - a for a, b in zip(self.offsets, self.offsets[1:])]


def attention_segments(q: torch.Tensor, kv: torch.Tensor, out: torch.Tensor, seg_off, *, heads: int, scale: float,
                       kv_split: Optional[int] = None):
    """Block-diagonal attention in one launch (f3r_attention_segments): q (rows, ldq), kv (rows, ldkv) [K | V] and out
    (rows, ldo), all bf16 or all fp16; the rows [seg_off[s], seg_off[s+1]) attend to those rows only, each segment exactly as
    attention(batch=1) over it alone with the same key split.  seg_off: a Segments, or the offsets as a host sequence.
    kv_split: key slices per segment (a segment with fewer key blocks uses one per block); None picks it with
    pick_kv_split over all the launch's query tiles."""
    h16 = _half(q, "q")
    _chk(q, h16, "q"); _chk(kv, h16, "kv"); _chk(out, h16, "out")
    if not isinstance(seg_off, Segments):
        seg_off = Segments(seg_off, q.device)
    rows = seg_off.rows
    ldq, ldkv, ldo = q.shape[-1], kv.shape[-1], out.shape[-1]
    assert q.numel() == rows * ldq and kv.numel() == rows * ldkv and out.numel() == rows * ldo
    lens = seg_off.lengths()
    key_blocks = max(-(-n // 128) for n in lens)
    if kv_split is None:
        units = sum(attention_units(1, heads, n) for n in lens)
        kv_split = pick_kv_split(units, key_blocks)
    ns = max(1, min(kv_split, key_blocks))
    n_seg, dev_off = len(lens), _ptr(seg_off.device_offsets)
    name = _f16("f3r_attention_segments", q)
    if ns > 1:
        part_o = torch.empty(ns, rows, heads * 64, dtype=F32, device=q.device)
        part_lse = torch.empty(ns, heads, rows, dtype=F32, device=q.device)
        _call(name, q, _ptr(q), ldq, _ptr(kv), ldkv, None, 0, dev_off, n_seg, rows, heads,
              float(scale), ns, _ptr(part_o), _ptr(part_lse))
        attention_merge(part_o, part_lse, ns, out, batch=1, heads=heads, sq=rows)
    else:
        _call(name, q, _ptr(q), ldq, _ptr(kv), ldkv, _ptr(out), ldo, dev_off, n_seg, rows, heads,
              float(scale), 1, None, None)


def attention_x3(q: torch.Tensor, kv: torch.Tensor, out: torch.Tensor, *, batch: int, heads: int, sq: int, skv: int,
                 scale: float, lse: Optional[torch.Tensor] = None):
    """Parity-mode attention: q (batch*sq, ldq), kv (batch*skv, ldkv) [K | V], out (batch*sq, ldo), all fp32."""
    _chk(q, F32, "q"); _chk(kv, F32, "kv"); _chk(out, F32, "out")
    ldq, ldkv, ldo = q.shape[-1], kv.shape[-1], out.shape[-1]
    assert q.numel() == batch * sq * ldq and kv.numel() == batch * skv * ldkv and out.numel() == batch * sq * ldo
    nbytes = L.load().f3r_attention_x3_workspace(batch, heads, sq, skv)
    ws = _scratch(nbytes, q.device)
    _call("f3r_attention_x3", q, _ptr(q), ldq, _ptr(kv), ldkv, _ptr(out), ldo, _ptr(lse), _ptr(ws), nbytes, batch, heads,
          sq, skv, float(scale))


def layernorm(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, eps: float, out: torch.Tensor):
    _chk(x, F32, "x"); _chk(w, F32, "w"); _chk(b, F32, "b")
    assert out.dtype in (BF16, F32, F16) and out.is_contiguous() and out.numel() == x.numel()
    dim = x.shape[-1]
    _call("f3r_layernorm", x, _ptr(x), _ptr(w), _ptr(b), _ptr(out), _elt(out), x.numel() // dim, dim, float(eps))


def im2col_patch(img: torch.Tensor, out: torch.Tensor):
    _chk(img, F32, "img")
    assert out.dtype in (BF16, F32, F16) and out.is_contiguous()
    n, c, h, w = img.shape
    assert c == 3 and out.numel() == n * (h // 16) * (w // 16) * 768
    _call("f3r_im2col_patch", img, _ptr(img), _ptr(out), _elt(out), n, h, w)


def im2col3x3s2(x: torch.Tensor, out: torch.Tensor, n: int, h: int, w: int, c: int, ho: int, wo: int):
    """x (n, h, w, c) -> out (n*ho*wo, 9*c), both bf16 or both fp16 (the kernel copies 16-bit elements)."""
    h16 = _half(x, "x")
    _chk(x, h16, "x"); _chk(out, h16, "out")
    assert x.numel() == n * h * w * c and out.numel() == n * ho * wo * 9 * c
    _call("f3r_im2col3x3s2", x, _ptr(x), _ptr(out), n, h, w, c, ho, wo)


def upsample2x(x: torch.Tensor, out: torch.Tensor, n: int, h: int, w: int, c: int, ho: int, wo: int):
    assert x.dtype in (BF16, F32, F16) and x.dtype == out.dtype and x.is_contiguous() and out.is_contiguous()
    assert x.numel() == n * h * w * c and out.numel() == n * ho * wo * c
    _call("f3r_upsample2x", x, _ptr(x), _ptr(out), _elt(x), n, h, w, c, ho, wo)


def cast_bf16(x: torch.Tensor, out: torch.Tensor):
    _chk(x, F32, "x"); _chk(out, BF16, "out")
    assert x.numel() == out.numel()
    _call("f3r_cast_bf16", x, _ptr(x), _ptr(out), x.numel())


def cast_f16(x: torch.Tensor, out: torch.Tensor):
    _chk(x, F32, "x"); _chk(out, F16, "out")
    assert x.numel() == out.numel()
    _call("f3r_cast_f16", x, _ptr(x), _ptr(out), x.numel())


# ------------------------------------------------------------------ geometry tail (csrc/geometry.cu)
def conf_quantile(conf: torch.Tensor, q: float) -> torch.Tensor:
    """conf fp32 [views, n] -> thr fp32 [views] = torch.quantile(conf[v], q) (exact, linear interpolation)."""
    _chk(conf, F32, "conf")
    assert conf.dim() == 2
    thr = torch.empty(conf.shape[0], dtype=F32, device=conf.device)
    _call("f3r_conf_quantile", conf, _ptr(conf), conf.shape[0], conf.shape[1], float(q), _ptr(thr))
    return thr


def similarity_fit(x: torch.Tensor, y: torch.Tensor, conf: Optional[torch.Tensor] = None,
                   thr: Optional[torch.Tensor] = None, valid: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x, y fp32 [views, n, 3]; conf fp32 [views, n] with thr fp32 [views]; valid uint8 [views, n].  Returns rts
    fp32 [views, 13] (R row-major, t, s) with y ~ s R x + t over conf >= thr & valid (fallbacks as the reference)."""
    _chk(x, F32, "x"); _chk(y, F32, "y")
    views, n = x.shape[0], x.shape[1]
    assert x.shape == y.shape == (views, n, 3)
    if conf is not None:
        _chk(conf, F32, "conf"); _chk(thr, F32, "thr")
        assert conf.shape == (views, n) and thr.shape == (views,)
    if valid is not None:
        _chk(valid, torch.uint8, "valid")
        assert valid.shape == (views, n)
    nbytes = L.load().f3r_similarity_fit_workspace(views)
    ws = _scratch(nbytes, x.device)
    rts = torch.empty(views, 13, dtype=F32, device=x.device)
    _call("f3r_similarity_fit", x, _ptr(x), _ptr(y), _ptr(conf), _ptr(thr), _ptr(valid), views, n, _ptr(rts), _ptr(ws),
          nbytes)
    return rts


def similarity_apply(x: torch.Tensor, rts: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[v] = s_v (x[v] R_v^T) + t_v, fp32 [views, n, 3]."""
    _chk(x, F32, "x"); _chk(rts, F32, "rts")
    views, n = x.shape[0], x.shape[1]
    assert x.shape == (views, n, 3) and rts.shape == (views, 13)
    if out is None:
        out = torch.empty_like(x)
    _chk(out, F32, "out")
    assert out.shape == x.shape
    _call("f3r_similarity_apply", x, _ptr(x), _ptr(rts), _ptr(out), views, n)
    return out


def focal_weiszfeld(pts: torch.Tensor, conf: Optional[torch.Tensor] = None, thr: Optional[torch.Tensor] = None,
                    pp: Optional[torch.Tensor] = None, iters: int = 100) -> torch.Tensor:
    """pts fp32 [views, H, W, 3]; conf fp32 [views, H, W] with thr fp32 [views]; pp fp32 [views, 2] or None (image
    centre).  Returns focal fp32 [views]."""
    _chk(pts, F32, "pts")
    views, h, w = pts.shape[0], pts.shape[1], pts.shape[2]
    assert pts.shape == (views, h, w, 3)
    if conf is not None:
        _chk(conf, F32, "conf"); _chk(thr, F32, "thr")
        assert conf.shape == (views, h, w) and thr.shape == (views,)
    if pp is not None:
        _chk(pp, F32, "pp")
        assert pp.shape == (views, 2)
    nbytes = L.load().f3r_focal_workspace(views)
    ws = _scratch(nbytes, pts.device)
    focal = torch.empty(views, dtype=F32, device=pts.device)
    _call("f3r_focal_weiszfeld", pts, _ptr(pts), _ptr(conf), _ptr(thr), _ptr(pp), views, h, w, int(iters), _ptr(focal),
          _ptr(ws), nbytes)
    return focal


# ------------------------------------------------------------------ camera poses (csrc/pose.cu)
def pnp_gather(pts: torch.Tensor, conf: Optional[torch.Tensor] = None, mask: Optional[torch.Tensor] = None):
    """pts fp32 [views, H, W, 3] and either conf fp32 [views, H, W] (selects conf > 1) or mask uint8 [views, H, W].
    Returns (points fp32 [views, H W, 3], pixels fp32 [views, H W, 2], counts int32 [views]): the first counts[v] rows
    of view v are its selected pixels in raster order with their pixel_grid coordinates (x, y)."""
    _chk(pts, F32, "pts")
    views, h, w = pts.shape[0], pts.shape[1], pts.shape[2]
    assert pts.shape == (views, h, w, 3) and (conf is None) != (mask is None)
    if conf is not None:
        _chk(conf, F32, "conf")
        assert conf.shape == (views, h, w)
    else:
        _chk(mask, torch.uint8, "mask")
        assert mask.shape == (views, h, w)
    nbytes = L.load().f3r_pnp_gather_workspace(views, h, w)
    ws = _scratch(max(nbytes, 4), pts.device)
    out_pts = torch.empty(views, h * w, 3, dtype=F32, device=pts.device)
    out_pix = torch.empty(views, h * w, 2, dtype=F32, device=pts.device)
    counts = torch.empty(views, dtype=torch.int32, device=pts.device)
    _call("f3r_pnp_gather", pts, _ptr(pts), _ptr(conf), _ptr(mask), views, h, w, _ptr(out_pts), _ptr(out_pix), _ptr(counts),
          _ptr(ws), nbytes)
    return out_pts, out_pix, counts


def _pnp_tables(pts, pix, offsets, view_counts, hyps):
    _chk(pts, F32, "pts"); _chk(pix, F32, "pix")
    assert pts.dim() == 2 and pts.shape[1] == 3 and pix.shape == (pts.shape[0], 2)
    offsets = np.ascontiguousarray(offsets, dtype=np.int64)
    view_counts = np.ascontiguousarray(view_counts, dtype=np.int32)
    hyps = np.ascontiguousarray(hyps, dtype=L.PNP_HYP)
    assert offsets.shape == view_counts.shape and offsets.ndim == 1 and hyps.ndim == 1
    if len(offsets) and int((offsets + view_counts).max()) > pts.shape[0]:
        raise ValueError("pnp: a view reaches past the points")
    return offsets, view_counts, hyps


def pnp_score(pts: torch.Tensor, pix: torch.Tensor, offsets, view_counts, hyps, thr: float) -> torch.Tensor:
    """Inlier counts int32 [nh] (device) of the hypothesis table `hyps` (host records of lib.PNP_HYP): row r counts the
    points of view hyps[r]["view"] = pts/pix rows [offsets[v], offsets[v] + view_counts[v]) (host int arrays) whose
    reprojection error is <= thr (OpenCV's arithmetic, pose_math.h)."""
    offsets, view_counts, hyps = _pnp_tables(pts, pix, offsets, view_counts, hyps)
    nbytes = L.load().f3r_pnp_score_workspace(len(offsets), len(hyps))
    ws = _scratch(nbytes, pts.device)
    counts = torch.empty(len(hyps), dtype=torch.int32, device=pts.device)
    _call("f3r_pnp_score", pts, _ptr(pts), _ptr(pix), offsets.ctypes.data, view_counts.ctypes.data, len(offsets),
          hyps.ctypes.data, len(hyps), float(thr), _ptr(counts), _ptr(ws), nbytes)
    return counts


def pnp_inliers(pts: torch.Tensor, pix: torch.Tensor, offsets, view_counts, hyps, thr: float):
    """The inliers of each row r of `hyps` among the points of its view (the rule of pnp_score), in index order.  Returns
    (points fp32 [m, 3], pixels fp32 [m, 2], counts int32 [nh]) on the device: row r's inliers are the first counts[r]
    rows from slot sum_{s<r} view_counts[hyps[s]["view"]] on (m is the sum over all rows)."""
    offsets, view_counts, hyps = _pnp_tables(pts, pix, offsets, view_counts, hyps)
    m = int(view_counts[hyps["view"]].astype(np.int64).sum())
    nbytes = L.load().f3r_pnp_inliers_workspace(len(hyps), int(view_counts.max()))
    ws = _scratch(nbytes, pts.device)
    out_pts = torch.empty(max(m, 1), 3, dtype=F32, device=pts.device)
    out_pix = torch.empty(max(m, 1), 2, dtype=F32, device=pts.device)
    counts = torch.empty(len(hyps), dtype=torch.int32, device=pts.device)
    _call("f3r_pnp_inliers", pts, _ptr(pts), _ptr(pix), offsets.ctypes.data, view_counts.ctypes.data, len(offsets),
          hyps.ctypes.data, len(hyps), float(thr), _ptr(out_pts), _ptr(out_pix), _ptr(counts), _ptr(ws), nbytes)
    return out_pts[:m], out_pix[:m], counts


# ------------------------------------------------------------------ camera-pose metric (csrc/pose_metric.cu)
def pose_metric(pred: torch.Tensor, gt: torch.Tensor, hist_max: int = 30, angles: bool = False):
    """pred, gt [items, views, 4, 4] cam-to-world, both float32 or both float64.  Returns (counts int64 [items,
    lib.PM_COUNTS], r, t): the counts row of f3r_pose_metric per item and, with `angles`, the rotation and translation
    angles in degrees [items, views (views - 1) / 2] of every pair in torch.combinations order (else None, None)."""
    if pred.dtype not in (F32, torch.float64) or gt.dtype != pred.dtype:
        raise TypeError(f"pose_metric: pred and gt must both be float32 or both float64, got {pred.dtype} and {gt.dtype}")
    _chk(pred, pred.dtype, "pred"); _chk(gt, pred.dtype, "gt")
    items, views = pred.shape[0], pred.shape[1]
    assert pred.shape == (items, views, 4, 4) and gt.shape == pred.shape
    f64 = int(pred.dtype == torch.float64)
    nbytes = L.load().f3r_pose_metric_workspace(f64, items, views)
    ws = _scratch(nbytes, pred.device)
    counts = torch.empty(items, L.PM_COUNTS, dtype=torch.int64, device=pred.device)
    r = t = None
    if angles:
        r = torch.empty(items, views * (views - 1) // 2, dtype=pred.dtype, device=pred.device)
        t = torch.empty_like(r)
    _call("f3r_pose_metric", pred, f64, _ptr(pred), _ptr(gt), items, views, int(hist_max), _ptr(r), _ptr(t),
          _ptr(counts), _ptr(ws), nbytes)
    return counts, r, t


def pose_metric_counts(r: torch.Tensor, t: torch.Tensor, hist_max: int = 30) -> torch.Tensor:
    """The counts row (int64 [lib.PM_COUNTS]) of given angle vectors r, t [n] (both float32 or both float64)."""
    if r.dtype not in (F32, torch.float64) or t.dtype != r.dtype:
        raise TypeError(f"pose_metric_counts: r and t must both be float32 or both float64, got {r.dtype} and {t.dtype}")
    _chk(r, r.dtype, "r"); _chk(t, r.dtype, "t")
    assert r.dim() == 1 and t.shape == r.shape
    counts = torch.empty(L.PM_COUNTS, dtype=torch.int64, device=r.device)
    _call("f3r_pose_metric_counts", r, int(r.dtype == torch.float64), _ptr(r), _ptr(t), r.numel(), int(hist_max),
          _ptr(counts))
    return counts


# ------------------------------------------------------------------ validation criterion (csrc/val_loss.cu)
VL_SUMS = 5  # per (view, item): sum d and sum d c - alpha log c of the global term, the same of the local term, count


def val_loss(gt: torch.Tensor, valid: torch.Tensor, pr: torch.Tensor, conf: torch.Tensor, poses: torch.Tensor,
             pr_local: Optional[torch.Tensor] = None, conf_local: Optional[torch.Tensor] = None, alpha: float = 1.0,
             log1p: bool = False, gt_scale: bool = False, local_scale_consistent: bool = False) -> torch.Tensor:
    """The sums of f3r_val_loss (float64 [views, items, VL_SUMS], on the device) from maps stacked [views, items, n]:
    gt, pr, pr_local float32 [..., 3], valid uint8, conf, conf_local float32, poses float32 [views, items, 4, 4].  The
    local term runs when pr_local and conf_local are given."""
    views, items, n = valid.shape
    for t, name in ((gt, "gt"), (pr, "pr"), (pr_local, "pr_local")):
        if t is not None:
            _chk(t, F32, name)
            assert t.shape == (views, items, n, 3), (name, t.shape)
    for t, name in ((conf, "conf"), (conf_local, "conf_local")):
        if t is not None:
            _chk(t, F32, name)
            assert t.shape == (views, items, n), (name, t.shape)
    _chk(valid, torch.uint8, "valid"); _chk(poses, F32, "poses")
    assert poses.shape == (views, items, 4, 4)
    has_local = pr_local is not None
    if has_local != (conf_local is not None):
        raise ValueError("val_loss: give both of pr_local and conf_local or neither")
    nbytes = L.load().f3r_val_loss_workspace(views, items, n)
    ws = _scratch(nbytes, gt.device)
    out = torch.empty(views, items, VL_SUMS, dtype=torch.float64, device=gt.device)
    _call("f3r_val_loss", gt, _ptr(gt), _ptr(valid), _ptr(pr), _ptr(pr_local), _ptr(conf), _ptr(conf_local),
          _ptr(poses), views, items, n, float(alpha), int(log1p), int(gt_scale), int(local_scale_consistent),
          int(has_local), _ptr(out), _ptr(ws), nbytes)
    return out


# ------------------------------------------------------------------ ground-truth views (csrc/views.cu)
def view_geometry(params: np.ndarray, out_pts: torch.Tensor, out_valid: torch.Tensor, out_depth: torch.Tensor) -> None:
    """f3r_view_geometry over the records `params` (numpy lib.VIEW_PARAM, one per (view, item), depth pointers on the
    device): the depth map, world points and validity of every view into the flat outputs out_pts float32 [P, 3],
    out_valid uint8 [P] and out_depth float32 [P].  The records are checked on the host and uploaded through pinned
    staging."""
    if params.dtype != L.VIEW_PARAM or params.ndim != 1 or not params.flags.c_contiguous:
        raise TypeError("view_geometry: params must be a contiguous 1-d lib.VIEW_PARAM array")
    _chk(out_pts, F32, "out_pts"); _chk(out_valid, torch.uint8, "out_valid"); _chk(out_depth, F32, "out_depth")
    n = out_valid.numel()
    assert out_pts.shape == (n, 3) and out_depth.numel() == n
    host = torch.from_numpy(params.view(np.uint8)).pin_memory()
    dev = host.to(out_pts.device, non_blocking=True)
    _call("f3r_view_geometry", out_pts, params.ctypes.data, _ptr(dev), len(params), _ptr(out_pts), _ptr(out_valid),
          _ptr(out_depth), n)


# ------------------------------------------------------------------ viewer scene (csrc/scene.cu)
I8, U8 = torch.int8, torch.uint8


def sky_mask(img: torch.Tensor, out: Optional[torch.Tensor] = None):
    """detect_sky_mask of each image of img fp32 [frames, 3, H, W] in [-1, 1].  Returns (not_sky int8 [frames, H W],
    not-sky counts int32 [frames]); `out` (int8 [frames, H W]) receives the masks if given."""
    _chk(img, F32, "img")
    frames, three, h, w = img.shape
    assert three == 3
    if out is None:
        out = torch.empty(frames, h * w, dtype=I8, device=img.device)
    _chk(out, I8, "out")
    assert out.shape == (frames, h * w)
    counts = torch.empty(frames, dtype=torch.int32, device=img.device)
    nbytes = L.load().f3r_sky_mask_workspace(frames, h, w)
    ws = _scratch(nbytes, img.device)
    # the reference's Python doubles: rows < int(H * 0.4) take the upper-rows rule; sky components need > H W 0.01 pixels
    upper, min_sky = int(h * 0.4), int(np.floor(h * w * 0.01)) + 1
    _call("f3r_sky_mask", img, _ptr(img), frames, h, w, upper, min_sky, _ptr(out), _ptr(counts), _ptr(ws), nbytes)
    return out, counts


def scene_sort(conf: torch.Tensor, pts: torch.Tensor, img: torch.Tensor, not_sky: torch.Tensor, offsets: torch.Tensor,
               out_pts: torch.Tensor, out_rgb: torch.Tensor, out_not_sky: torch.Tensor, max_conf: torch.Tensor) -> None:
    """One group of frames (frame f = elements offsets[f]:offsets[f + 1], offsets int64 on the device): each frame in
    the order of np.argsort(-conf, kind="stable"), with its points fp32 [n, 3], u8 colours from the planar images img
    (frame f's [3, hw] at 3 offsets[f]) and not-sky int8 [n] gathered into out_pts / out_rgb [n, 3] / out_not_sky [n];
    max_conf fp32 [frames] gets each frame's conf.max()."""
    n, frames = conf.numel(), offsets.numel() - 1
    _chk(conf, F32, "conf"); _chk(pts, F32, "pts"); _chk(img, F32, "img"); _chk(not_sky, I8, "not_sky")
    _chk(offsets, torch.int64, "offsets"); _chk(out_pts, F32, "out_pts"); _chk(out_rgb, U8, "out_rgb")
    _chk(out_not_sky, I8, "out_not_sky"); _chk(max_conf, F32, "max_conf")
    assert pts.numel() == 3 * n and img.numel() == 3 * n and not_sky.numel() == n and frames >= 1
    assert out_pts.numel() == 3 * n and out_rgb.numel() == 3 * n and out_not_sky.numel() == n and max_conf.numel() == frames
    nbytes = L.load().f3r_scene_sort_workspace(n)
    ws = _scratch(nbytes, conf.device)
    _call("f3r_scene_sort", conf, _ptr(conf), _ptr(pts), _ptr(img), _ptr(not_sky), _ptr(offsets), frames, n,
          _ptr(out_pts), _ptr(out_rgb), _ptr(out_not_sky), _ptr(max_conf), _ptr(ws), nbytes)


def scene_visible(segs: np.ndarray, pts_g: torch.Tensor, pts_l: torch.Tensor, rgb_g: torch.Tensor, rgb_l: torch.Tensor,
                  not_sky_g: torch.Tensor, not_sky_l: torch.Tensor, mask_sky: bool):
    """The rows of the segments segs (host int64 [nseg, 4]: head 0 global / 1 local, first row, row count, colour -1 for
    the rows' own RGB or 0xRRGGBB) of the frame arrays, without the sky rows if mask_sky, segment after segment.
    Returns (points fp32 [m, 3], colours uint8 [m, 3]) on the device."""
    segs = np.ascontiguousarray(segs, dtype=np.int64).reshape(-1, 4)
    dev = pts_g.device
    if len(segs) == 0 or int(segs[:, 2].max()) == 0:
        return torch.empty(0, 3, dtype=F32, device=dev), torch.empty(0, 3, dtype=U8, device=dev)
    for t, dt, name in ((pts_g, F32, "pts_g"), (pts_l, F32, "pts_l"), (rgb_g, U8, "rgb_g"), (rgb_l, U8, "rgb_l"),
                        (not_sky_g, I8, "not_sky_g"), (not_sky_l, I8, "not_sky_l")):
        _chk(t, dt, name)
    rows = (pts_g.shape[0], pts_l.shape[0])
    if (segs[:, 1] < 0).any() or (segs[:, 2] < 0).any() or any(
            int(s[1] + s[2]) > rows[int(s[0])] for s in segs) or not np.isin(segs[:, 0], (0, 1)).all():
        raise ValueError("scene_visible: a segment reaches past its frame arrays")
    nseg, max_len = len(segs), int(segs[:, 2].max())
    nbytes = L.load().f3r_scene_visible_workspace(nseg, max_len)
    ws = _scratch(nbytes, dev)
    segs_d = torch.from_numpy(segs).to(dev)
    total = torch.empty(1, dtype=torch.int64, device=dev)
    args = (_ptr(pts_g), _ptr(pts_l), _ptr(rgb_g), _ptr(rgb_l), _ptr(not_sky_g), _ptr(not_sky_l), int(bool(mask_sky)))
    _call("f3r_scene_visible", pts_g, _ptr(segs_d), nseg, max_len, *args, _ptr(total), None, None, _ptr(ws), nbytes)
    m = int(total.item())
    out_pts = torch.empty(m, 3, dtype=F32, device=dev)
    out_rgb = torch.empty(m, 3, dtype=U8, device=dev)
    if m:
        _call("f3r_scene_visible", pts_g, _ptr(segs_d), nseg, max_len, *args, None, _ptr(out_pts), _ptr(out_rgb),
              _ptr(ws), nbytes)
    return out_pts, out_rgb


def ply_pack(points: torch.Tensor, colors: torch.Tensor) -> torch.Tensor:
    """uint8 [n * 15]: the little-endian PLY records (x, y, z float32, red, green, blue uint8) of the points."""
    _chk(points, F32, "points"); _chk(colors, U8, "colors")
    n = points.shape[0]
    assert points.shape == (n, 3) and colors.shape == (n, 3)
    out = torch.empty(15 * n, dtype=U8, device=points.device)
    if n:
        _call("f3r_ply_pack", points, _ptr(points), _ptr(colors), n, _ptr(out))
    return out


def percentile_plan(n: int, p: float):
    """(lower rank, float32 weight) of np.percentile(x, p) for n float32 values, as numpy 2 forms them for method
    "linear": q = p / float32(100) in float32, virtual index (n - 1) q in float32, the ranks floor and floor + 1 (both
    n - 1 past the end), weight = virtual index - lower rank as numpy returns it from its index rule."""
    q = np.true_divide(p, np.float32(100))
    v = np.float32(n - 1) * q
    prev = int(np.floor(v))
    if v >= n - 1:
        return n - 1, np.float32(v - np.float32(-1))  # numpy marks both ranks -1 there; the weight meets equal bounds
    return prev, np.float32(v - np.float32(prev))


def extent_percentiles(points: torch.Tensor, lo: float = 20, hi: float = 80) -> torch.Tensor:
    """fp32 [7] on the device: np.percentile(points, lo, axis=0), np.percentile(points, hi, axis=0) and the largest
    per-axis difference hi - lo (NaN for an axis holding a NaN), for points fp32 [n, 3], n >= 1."""
    _chk(points, F32, "points")
    n = points.shape[0]
    assert points.shape == (n, 3) and n >= 1
    (k0, g0), (k1, g1) = percentile_plan(n, lo), percentile_plan(n, hi)
    nbytes = L.load().f3r_extent_percentiles_workspace()
    ws = _scratch(nbytes, points.device)
    out = torch.empty(7, dtype=F32, device=points.device)
    _call("f3r_extent_percentiles", points, _ptr(points), n, k0, k1, float(g0), float(g1), _ptr(out), _ptr(ws), nbytes)
    return out


# ------------------------------------------------------------------ reconstruction metrics (csrc/pointcloud.cu)
F64 = torch.float64


def _points(x: torch.Tensor, name: str) -> int:
    if x.dtype not in (F32, F64):
        raise TypeError(f"{name}: expected float32 or float64, got {x.dtype}")
    if x.dim() != 2 or x.shape[1] != 3:
        raise ValueError(f"{name}: expected shape (n, 3), got {tuple(x.shape)}")
    if not x.is_contiguous():
        raise ValueError(f"{name}: must be contiguous")
    return int(x.dtype == F64)


class PointIndex:
    """Spatial index over a point cloud (f3r_pc_index_build): the caller-owned block and the cloud's size."""

    def __init__(self, block: Optional[torch.Tensor], n: int, device: torch.device):
        self.block, self.n, self.device = block, n, device


def pc_index(pts: torch.Tensor) -> PointIndex:
    """pts float32 / float64 (n, 3) on the device -> PointIndex (n == 0: an empty index that no query matches)."""
    f64 = _points(pts, "pts")
    n = pts.shape[0]
    if n == 0:
        return PointIndex(None, 0, pts.device)
    nbytes = L.load().f3r_pc_index_workspace(n)
    block = _scratch(nbytes, pts.device)
    _call("f3r_pc_index_build", pts, _ptr(pts), f64, n, _ptr(block), nbytes)
    return PointIndex(block, n, pts.device)


def pc_nearest(index: PointIndex, query: torch.Tensor):
    """Exact nearest indexed point of every query point: (dist float64 (nq,), idx int64 (nq,)), as cKDTree.query."""
    f64 = _points(query, "query")
    nq = query.shape[0]
    dist = torch.empty(nq, dtype=F64, device=query.device)
    idx = torch.empty(nq, dtype=torch.int64, device=query.device)
    if nq == 0:
        return dist, idx
    nbytes = L.load().f3r_pc_query_workspace(nq) if index.n else 0
    ws = _scratch(nbytes, query.device) if nbytes else None
    block = index.block
    _call("f3r_pc_nearest", query, _ptr(block), block.numel() if block is not None else 0, index.n, _ptr(query), f64, nq,
          _ptr(dist), _ptr(idx), _ptr(ws), nbytes)
    return dist, idx


def pc_knn_normals(index: PointIndex, k: int = 30) -> torch.Tensor:
    """float64 (n, 3) unit normals of the indexed cloud from its k nearest points (the point included)."""
    out = torch.empty(index.n, 3, dtype=F64, device=index.device)
    if index.n:
        _call("f3r_pc_knn_normals", out, _ptr(index.block), index.block.numel(), index.n, int(k), _ptr(out))
    return out


def pc_count_nonfinite(pts: torch.Tensor) -> torch.Tensor:
    """Number of non-finite coordinates of pts (n, 3), as a device int32 (1,) tensor."""
    f64 = _points(pts, "pts")
    count = torch.empty(1, dtype=torch.int32, device=pts.device)
    _call("f3r_pc_count_nonfinite", pts, _ptr(pts), f64, pts.shape[0], _ptr(count))
    return count


def pc_abs_dot(a: torch.Tensor, b: torch.Tensor, a_idx: Optional[torch.Tensor] = None,
               b_idx: Optional[torch.Tensor] = None) -> torch.Tensor:
    """|a[a_idx] . b[b_idx]| row by row (float64 (.., 3); int64 indices or None for the identity)."""
    _chk(a, F64, "a"); _chk(b, F64, "b")
    for t, name in ((a_idx, "a_idx"), (b_idx, "b_idx")):
        if t is not None:
            _chk(t, torch.int64, name)
    n = (a_idx if a_idx is not None else b_idx if b_idx is not None else a).shape[0]
    out = torch.empty(n, dtype=F64, device=a.device)
    _call("f3r_pc_abs_dot", out, _ptr(a), _ptr(a_idx), _ptr(b), _ptr(b_idx), n, _ptr(out))
    return out


def _reduce(name: str, x: torch.Tensor) -> torch.Tensor:
    _chk(x, F64, "x")
    nbytes = L.load().f3r_f64_reduce_workspace()
    ws = _scratch(nbytes, x.device)
    out = torch.empty((), dtype=F64, device=x.device)
    _call(name, x, _ptr(x), x.numel(), _ptr(out), _ptr(ws), nbytes)
    return out


def f64_mean(x: torch.Tensor) -> torch.Tensor:
    """Mean of a float64 tensor (n >= 1) in a fixed summation order, as a 0-d device tensor."""
    return _reduce("f3r_f64_mean", x)


def f64_median(x: torch.Tensor) -> torch.Tensor:
    """numpy.median of a float64 tensor (n >= 1), exactly, as a 0-d device tensor."""
    return _reduce("f3r_f64_median", x)


def f64_count_below(x: torch.Tensor, th: float) -> torch.Tensor:
    """Number of elements of a float64 tensor that are < th, as a device int64 (1,) tensor."""
    _chk(x, F64, "x")
    t = torch.tensor([float(th)], dtype=F64, device=x.device)
    count = torch.empty(1, dtype=torch.int64, device=x.device)
    _call("f3r_f64_count_below", x, _ptr(x), x.numel(), _ptr(t), _ptr(count))
    return count
