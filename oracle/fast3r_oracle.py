"""CPU fp32 restatement of the Fast3R single-forward-pass hot path.

TEST INFRASTRUCTURE ONLY — this is the parity checker, never the product path.  Only
``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` / ``--impl reference`` legs
of ``bench.py`` may import it.  The product (``fast3r_b200``) never imports ``oracle``.

It restates, in plain functional PyTorch on the CPU in fp32, what the reference computes on
the path  CroCo encoder -> fusion decoder -> DPT heads -> postprocess.  Every function cites
the reference file:line it follows (paths relative to /root/reference).  It takes a reference
``state_dict`` (SURVEY.md §8(b) key schema) so it can be checked against the real reference.

PINNING: the reference ships no tests / golden vectors for this path (SURVEY.md §4), so the
oracle is pinned against outputs of the reference ITSELF, run in the build container by
``tests/golden/make_golden.py`` (which imports /root/reference through
``oracle/ref_harness.py``); the resulting fixtures live in ``tests/golden/*.pt`` and
``tests/test_oracle_vs_golden.py`` checks this file against them (per-stage taps and final
preds, tiny model end-to-end, ViT-L-width single ops, and the full ViT-L/512 at N=4 views
512x368 = BASELINE configs[0], through the reference's own inference(dtype="32")).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

Tensor = torch.Tensor


# ----------------------------------------------------------------------------- configs
def vit_large_args(attn_implementation: str = "flash_attention"):
    """ViT-L/512 dicts: configs/model/fast3r.yaml:50-88 overridden by
    configs/experiment/super_long_training/super_long_training.yaml:52-66; inference callers
    force PatchEmbedDust3R + landscape_only=False (fast3r/utils/checkpoint_utils.py:37-38)."""
    enc = dict(encoder_type="croco", img_size=512, patch_size=16, patch_embed_cls="PatchEmbedDust3R",
               embed_dim=1024, num_heads=16, depth=24, mlp_ratio=4, pos_embed="RoPE100",
               attn_implementation=attn_implementation)
    dec = dict(decoder_type="fast3r", random_image_idx_embedding=True, enc_embed_dim=1024, embed_dim=1024,
               num_heads=16, depth=24, mlp_ratio=4.0, qkv_bias=True, drop=0.0, attn_drop=0.0,
               attn_implementation=attn_implementation)
    head = dict(head_type="dpt", output_mode="pts3d", landscape_only=False,
                depth_mode=["exp", float("-inf"), float("inf")], conf_mode=["exp", 1, float("inf")],
                patch_size=16, with_local_head=True)
    return enc, dec, head


def tiny_args(attn_implementation: str = "flash_attention", dec_depth: int = 12):
    """Tiny config of SURVEY.md §7 step 0: D=128, 2 heads (hd=64), encoder depth 2, decoder
    depth 12 (DPT factory asserts depth > 9, fast3r/models/fast3r.py:137)."""
    enc, dec, head = vit_large_args(attn_implementation)
    enc.update(embed_dim=128, num_heads=2, depth=2)
    dec.update(enc_embed_dim=128, embed_dim=128, num_heads=2, depth=dec_depth)
    return enc, dec, head


# ----------------------------------------------------------------------------- small ops
def layer_norm(x: Tensor, w: Tensor, b: Tensor, eps: float) -> Tensor:
    """nn.LayerNorm over the last dim, biased variance (SURVEY Appendix A notes)."""
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + eps) * w + b


def gelu_erf(x: Tensor) -> Tensor:
    """nn.GELU() exact erf form (fast3r/croco/models/blocks.py:83,95)."""
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def rope2d(t: Tensor, pos: Tensor, base: float = 100.0) -> Tensor:
    """RoPE2D.forward, fast3r/croco/models/pos_embed.py:141-183.
    t: (B, H, S, hd); pos: (B, S, 2) int (y, x).  First hd/2 dims rotate with y, last hd/2
    with x; inside each half pair (j, j+hd/4) with angle pos * base**(-j/(hd/4)).  Angles in t's dtype, on t's device."""
    hd = t.shape[-1]
    D = hd // 2
    inv_freq = 1.0 / (base ** (torch.arange(0, D, 2, device=t.device).to(t.dtype) / D))  # (D/2,)

    def rope1d(tok, p):
        ang = p[:, None, :, None].to(device=t.device, dtype=t.dtype) * inv_freq  # (B,1,S,D/2)
        ang = torch.cat((ang, ang), dim=-1)
        cos, sin = ang.cos(), ang.sin()
        x1, x2 = tok[..., : D // 2], tok[..., D // 2:]
        rot = torch.cat((-x2, x1), dim=-1)
        return tok * cos + rot * sin

    y, x = t[..., :D], t[..., D:]
    return torch.cat((rope1d(y, pos[:, :, 0]), rope1d(x, pos[:, :, 1])), dim=-1)


def attention(x: Tensor, p: Dict[str, Tensor], pre: str, num_heads: int, scale: float,
              pos: Optional[Tensor]) -> Tensor:
    """Attention.forward, fast3r/croco/models/blocks.py:135-194 (CPU fp32 semantics: the inner
    autocast("cuda") is a no-op on CPU, SURVEY Q9).  Softmax over keys, scale on the logits."""
    B, S, C = x.shape
    hd = C // num_heads
    qkv = F.linear(x, p[pre + "qkv.weight"], p[pre + "qkv.bias"])
    qkv = qkv.reshape(B, S, 3, num_heads, hd).permute(2, 0, 3, 1, 4)  # (3,B,H,S,hd)
    q, k, v = qkv[0], qkv[1], qkv[2]
    if pos is not None:
        q, k = rope2d(q, pos), rope2d(k, pos)
    out = torch.empty_like(q)
    # chunk over queries so the S x S matrix never needs > ~1 GB
    step = max(1, int(2 ** 28 // max(1, S * num_heads * B)))
    for s0 in range(0, S, step):
        a = (q[:, :, s0:s0 + step] @ k.transpose(-2, -1)) * scale
        out[:, :, s0:s0 + step] = a.softmax(dim=-1) @ v
    out = out.transpose(1, 2).reshape(B, S, C)
    return F.linear(out, p[pre + "proj.weight"], p[pre + "proj.bias"])


def block(x: Tensor, p: Dict[str, Tensor], pre: str, num_heads: int, eps: float, scale: float,
          pos: Optional[Tensor]) -> Tensor:
    """Block.forward, fast3r/croco/models/blocks.py:236-239 with Mlp :100-106."""
    h = layer_norm(x, p[pre + "norm1.weight"], p[pre + "norm1.bias"], eps)
    x = x + attention(h, p, pre + "attn.", num_heads, scale, pos)
    h = layer_norm(x, p[pre + "norm2.weight"], p[pre + "norm2.bias"], eps)
    h = gelu_erf(F.linear(h, p[pre + "mlp.fc1.weight"], p[pre + "mlp.fc1.bias"]))
    return x + F.linear(h, p[pre + "mlp.fc2.weight"], p[pre + "mlp.fc2.bias"])


# ----------------------------------------------------------------------------- encoder
def patch_embed(img: Tensor, p: Dict[str, Tensor], patch: int = 16):
    """PatchEmbedDust3R.forward, fast3r/dust3r/patch_embed.py:25-38; conv at
    fast3r/croco/models/blocks.py:412-414; positions blocks.py:382-388 (cartesian (y,x))."""
    x = F.conv2d(img, p["encoder.patch_embed.proj.weight"], p["encoder.patch_embed.proj.bias"], stride=patch)
    n, C, gh, gw = x.shape
    x = x.flatten(2).transpose(1, 2)
    yy, xx = torch.meshgrid(torch.arange(gh, device=img.device), torch.arange(gw, device=img.device), indexing="ij")
    pos = torch.stack((yy.reshape(-1), xx.reshape(-1)), dim=-1)[None].expand(n, -1, -1)
    return x, pos


def encoder(img: Tensor, p: Dict[str, Tensor], depth: int, num_heads: int, taps: Optional[dict] = None):
    """CroCoEncoder.forward, fast3r/models/fast3r.py:549-559 (LN eps 1e-6, :509; RoPE100;
    attention scale hd**-0.5, blocks.py:116,153)."""
    x, pos = patch_embed(img, p)
    if taps is not None:
        taps["patch_embed"] = x.clone()
    hd = x.shape[-1] // num_heads
    for i in range(depth):
        x = block(x, p, f"encoder.enc_blocks.{i}.", num_heads, 1e-6, hd ** -0.5, pos)
        if taps is not None:
            taps[f"enc_block{i}"] = x.clone()
    x = layer_norm(x, p["encoder.enc_norm.weight"], p["encoder.enc_norm.bias"], 1e-6)
    return x, pos


# ----------------------------------------------------------------------------- decoder
def image_idx_table(dim: int, n: int = 1000) -> Tensor:
    """get_1d_sincos_pos_embed_from_grid(dim, arange(1000)), fast3r/croco/models/pos_embed.py:58-76,
    used at fast3r/models/fast3r.py:691-697: row i = [sin(i*w) (dim/2), cos(i*w) (dim/2)],
    w_j = 10000**(-j/(dim/2)); computed in float64 then cast to float32."""
    omega = np.arange(dim // 2, dtype=float)
    omega /= dim / 2.0
    omega = 1.0 / 10000 ** omega
    out = np.einsum("m,d->md", np.arange(n, dtype=float), omega)
    return torch.from_numpy(np.concatenate([np.sin(out), np.cos(out)], axis=1)).float()


def draw_image_ids(batch: int, num_views: int, rank: int = 0, max_image_idx: int = 999) -> Tensor:
    """RNG side effects of Fast3RDecoder._get_random_image_pos / _generate_per_rank_generator,
    fast3r/models/fast3r.py:702-713, :738-745: one global-RNG randint, then per-sample randperm
    from a fresh generator seeded with it (+rank).  View 0 always gets id 0."""
    seed = torch.randint(0, 2 ** 32, (1,)).item() + rank
    g = torch.Generator()
    g.manual_seed(seed)
    ids = torch.zeros(batch, num_views, dtype=torch.long)
    for b in range(batch):
        ids[b, 1:] = torch.randperm(max_image_idx, generator=g)[: num_views - 1] + 1
    return ids


def attn_bias_scale(hd: int) -> float:
    """fast3r/croco/models/blocks.py:119-124."""
    return hd ** -0.5 * (1.0 * math.log(137) / math.log(20)) ** 0.5


def decoder(feats: Tensor, image_ids: Tensor, p: Dict[str, Tensor], depth: int, num_heads: int,
            training: bool = False, attn_bias_for_inference_enabled: bool = True,
            taps: Optional[dict] = None, keep: Optional[Sequence[int]] = None) -> List[Optional[Tensor]]:
    """Fast3RDecoder.forward, fast3r/models/fast3r.py:768-808.
    feats: (B, N, P, D) encoder outputs; image_ids: (B, N) embedding-table rows per view.
    Returns the 1+depth layer outputs (B, N*P, D); last one through dec_norm (eps 1e-6);
    decoder blocks use LN eps 1e-5 (:683), no RoPE, eval scale 0.16019 (blocks.py:151-154).
    ``keep``: the layer outputs to return (the others are None, so a large forward holds only the hooked ones)."""
    if feats.dim() == 4:
        B, N, P, D = feats.shape
        x = feats.reshape(B, N * P, D)
        tok_rows = image_ids[:, :, None].expand(B, N, P).reshape(B, N * P)
    else:  # (B, S, D) with one table row per token (views of different resolutions)
        x, tok_rows = feats, image_ids
    kept = lambda i, t: t if keep is None or i in keep else None  # noqa: E731
    outs = [kept(0, x)]
    x = F.linear(x, p["decoder.decoder_embed.weight"], p["decoder.decoder_embed.bias"])
    table = image_idx_table(x.shape[-1]).to(x)  # the model's fp32 buffer, in the dtype of the run
    x = x + table[tok_rows.to(x.device)]
    if taps is not None:
        taps["dec_embed"] = x.clone()
    hd = x.shape[-1] // num_heads
    scale = attn_bias_scale(hd) if (not training and attn_bias_for_inference_enabled) else hd ** -0.5
    for i in range(depth):
        x = block(x, p, f"decoder.dec_blocks.{i}.", num_heads, 1e-5, scale, None)
        outs.append(kept(i + 1, x))
        if taps is not None:
            taps[f"dec_block{i}"] = x.clone()
    outs[-1] = layer_norm(x, p["decoder.dec_norm.weight"], p["decoder.dec_norm.bias"], 1e-6)
    return outs


# ----------------------------------------------------------------------------- DPT head
def _rcu(x: Tensor, p: Dict[str, Tensor], pre: str) -> Tensor:
    """ResidualConvUnit_custom.forward, fast3r/croco/models/dpt_block.py:133-154 (ReLU not in place)."""
    out = F.conv2d(F.relu(x), p[pre + "conv1.weight"], p[pre + "conv1.bias"], padding=1)
    out = F.conv2d(F.relu(out), p[pre + "conv2.weight"], p[pre + "conv2.bias"], padding=1)
    return out + x


def _fusion(p: Dict[str, Tensor], pre: str, x0: Tensor, x1: Optional[Tensor] = None) -> Tensor:
    """FeatureFusionBlock_custom.forward, fast3r/croco/models/dpt_block.py:202-250."""
    out = x0
    if x1 is not None:
        out = out + _rcu(x1, p, pre + "resConfUnit1.")
    out = _rcu(out, p, pre + "resConfUnit2.")
    out = F.interpolate(out, scale_factor=2, mode="bilinear", align_corners=True)
    return F.conv2d(out, p[pre + "out_conv.weight"], p[pre + "out_conv.bias"])


def dpt_head(hooked: Sequence[Tensor], H: int, W: int, p: Dict[str, Tensor], pre: str,
             patch: int = 16, taps: Optional[dict] = None) -> Tensor:
    """DPTOutputAdapter_fix.forward, fast3r/dust3r/heads/dpt_head.py:42-90 with modules of
    fast3r/croco/models/dpt_block.py:350-382, 401-490.  hooked: 4 x (b, P, C) tokens of hooks
    [0, d/2, 3d/4, d].  Returns (b, 4, H, W)."""
    nh, nw = H // patch, W // patch
    L = [t.reshape(t.shape[0], nh, nw, t.shape[-1]).permute(0, 3, 1, 2) for t in hooked]
    ap = pre + "dpt.act_postprocess."
    L[0] = F.conv_transpose2d(F.conv2d(L[0], p[ap + "0.0.weight"], p[ap + "0.0.bias"]),
                              p[ap + "0.1.weight"], p[ap + "0.1.bias"], stride=4)
    L[1] = F.conv_transpose2d(F.conv2d(L[1], p[ap + "1.0.weight"], p[ap + "1.0.bias"]),
                              p[ap + "1.1.weight"], p[ap + "1.1.bias"], stride=2)
    L[2] = F.conv2d(L[2], p[ap + "2.0.weight"], p[ap + "2.0.bias"])
    L[3] = F.conv2d(F.conv2d(L[3], p[ap + "3.0.weight"], p[ap + "3.0.bias"]),
                    p[ap + "3.1.weight"], p[ap + "3.1.bias"], stride=2, padding=1)
    sc = pre + "dpt.scratch."
    L = [F.conv2d(l, p[sc + f"layer{i + 1}_rn.weight"], None, padding=1) for i, l in enumerate(L)]
    if taps is not None:
        for i, l in enumerate(L):
            taps[f"layer_rn{i}"] = l.clone()
    path4 = _fusion(p, sc + "refinenet4.", L[3])[:, :, : L[2].shape[2], : L[2].shape[3]]
    path3 = _fusion(p, sc + "refinenet3.", path4, L[2])
    path2 = _fusion(p, sc + "refinenet2.", path3, L[1])
    path1 = _fusion(p, sc + "refinenet1.", path2, L[0])
    if taps is not None:
        taps.update(path4=path4.clone(), path3=path3.clone(), path2=path2.clone(), path1=path1.clone())
    hd = pre + "dpt.head."
    out = F.conv2d(path1, p[hd + "0.weight"], p[hd + "0.bias"], padding=1)
    out = F.interpolate(out, scale_factor=patch / 8, mode="bilinear", align_corners=True)
    out = F.relu(F.conv2d(out, p[hd + "2.weight"], p[hd + "2.bias"], padding=1))
    return F.conv2d(out, p[hd + "4.weight"], p[hd + "4.bias"])


def postprocess(out: Tensor) -> Dict[str, Tensor]:
    """postprocess / reg_dense_depth('exp') / reg_dense_conf('exp',1,inf),
    fast3r/dust3r/heads/postprocess.py:16-64."""
    fmap = out.permute(0, 2, 3, 1)
    xyz = fmap[..., 0:3]
    d = xyz.norm(dim=-1, keepdim=True)
    pts = xyz / d.clip(min=1e-8) * torch.expm1(d)
    conf = 1 + fmap[..., 3].exp()
    return dict(pts3d=pts, conf=conf)


# ----------------------------------------------------------------------------- whole path
def _heads_in_chunks(hooked: Sequence[Tensor], H: int, W: int, p: Dict[str, Tensor], pre: str, patch: int,
                     head_chunk: Optional[int], taps: Optional[dict] = None) -> Dict[str, Tensor]:
    """postprocess(dpt_head(...)) over the (views*B) images of ``hooked``, ``head_chunk`` images at a time (None: all at
    once).  The head is per-image arithmetic, so chunking only bounds the memory of the full-resolution feature maps."""
    n = hooked[0].shape[0]
    step = n if head_chunk is None else max(1, int(head_chunk))
    parts = [postprocess(dpt_head([t[s:s + step] for t in hooked], H, W, p, pre, patch, taps)) for s in range(0, n, step)]
    return parts[0] if len(parts) == 1 else {k: torch.cat([r[k] for r in parts]) for k in parts[0]}


def forward(state_dict: Dict[str, Tensor], enc_args: dict, dec_args: dict, head_args: dict,
            imgs: Sequence[Tensor], image_ids: Optional[Tensor] = None, training: bool = False,
            rank: int = 0, taps: Optional[dict] = None, *, dtype: torch.dtype = torch.float32,
            device=None, head_chunk: Optional[int] = None) -> List[Dict[str, Tensor]]:
    """Fast3R.forward for same-size views, fast3r/models/fast3r.py:302-497.
    imgs: N tensors (B,3,H,W) fp32 in [-1,1].  If ``image_ids`` is None they are drawn from the
    global torch RNG exactly like the reference does (seed before calling).
    ``dtype`` / ``device``: the weights and inputs are cast to ``dtype`` and moved to ``device`` (None: the CPU), and
    every op runs there (torch.float64 on a GPU gives an independent high-precision reference: torch, cuBLAS and cuDNN
    only).  The image ids are still drawn on the CPU generator.  ``head_chunk``: images per DPT-head call (None: all).
    Predictions come back in ``dtype`` on ``device``."""
    device = torch.device("cpu") if device is None else torch.device(device)
    p = {k: v.detach().to(device=device, dtype=dtype) for k, v in state_dict.items()}
    N = len(imgs)
    if any(im.shape != imgs[0].shape for im in imgs):
        return _forward_mixed(p, enc_args, dec_args, head_args, imgs, image_ids, training, rank, dtype, device,
                              head_chunk)
    B, _, H, W = imgs[0].shape
    x = torch.cat(list(imgs), dim=0).to(device=device, dtype=dtype)  # (N*B,3,H,W), view-major (fast3r.py:258)
    feats, _pos = encoder(x, p, enc_args["depth"], enc_args["num_heads"], taps)
    if taps is not None:
        taps["enc_out"] = feats.clone()
    P, D = feats.shape[1], feats.shape[2]
    feats = feats.reshape(N, B, P, D).permute(1, 0, 2, 3)  # (B,N,P,D)
    if image_ids is None:
        if dec_args.get("random_image_idx_embedding", True):
            image_ids = draw_image_ids(B, N, rank)
        else:
            image_ids = torch.arange(N)[None].expand(B, N)
    d = dec_args["depth"]
    hooks = [0, d * 2 // 4, d * 3 // 4, d]
    outs = decoder(feats, image_ids.to(device), p, dec_args["depth"], dec_args["num_heads"], training,
                   dec_args.get("attn_bias_for_inference_enabled", True), taps, keep=hooks)
    # 'B (n p) D -> (n B) p D'  (fast3r.py:385-398)
    hooked = [outs[h].reshape(B, N, P, -1).permute(1, 0, 2, 3).reshape(N * B, P, -1) for h in hooks]
    if taps is not None:
        for i, h in enumerate(hooked):
            taps[f"hook{i}"] = h.clone()
    patch = head_args.get("patch_size", 16)
    res = _heads_in_chunks(hooked, H, W, p, "downstream_head.", patch, head_chunk, taps)
    preds = [dict() for _ in range(N)]
    for i in range(N):
        preds[i]["pts3d_in_other_view"] = res["pts3d"][i * B:(i + 1) * B]
        preds[i]["conf"] = res["conf"][i * B:(i + 1) * B]
    if head_args.get("with_local_head", False):
        res_l = _heads_in_chunks(hooked, H, W, p, "downstream_head_local.", patch, head_chunk)
        for i in range(N):
            preds[i]["pts3d_local"] = res_l["pts3d"][i * B:(i + 1) * B]
            preds[i]["conf_local"] = res_l["conf"][i * B:(i + 1) * B]
    return preds


def _forward_mixed(p, enc_args, dec_args, head_args, imgs, image_ids, training, rank, dtype, device, head_chunk):
    """Different resolutions per view: per-view encoder and heads, one decoder pass over all tokens in view order
    (fast3r/models/fast3r.py:276-294, 339-348, 364-376, 407-428)."""
    N = len(imgs)
    B = imgs[0].shape[0]
    feats = [encoder(im.to(device=device, dtype=dtype), p, enc_args["depth"], enc_args["num_heads"])[0]
             for im in imgs]  # (B, P_i, D)
    if image_ids is None:
        image_ids = draw_image_ids(B, N, rank) if dec_args.get("random_image_idx_embedding", True) \
            else torch.arange(N)[None].expand(B, N)
    x = torch.cat(feats, dim=1)
    image_ids = image_ids.to(device)
    tok_rows = torch.cat([image_ids[:, i:i + 1].expand(B, f.shape[1]) for i, f in enumerate(feats)], dim=1)
    d = dec_args["depth"]
    hooks = [0, d * 2 // 4, d * 3 // 4, d]
    outs = decoder(x, tok_rows, p, dec_args["depth"], dec_args["num_heads"], training,
                   dec_args.get("attn_bias_for_inference_enabled", True), keep=hooks)
    preds = []
    off = 0
    for i, im in enumerate(imgs):
        P_i = feats[i].shape[1]
        hooked = [outs[h][:, off:off + P_i] for h in hooks]
        off += P_i
        H, W = im.shape[-2:]
        r = _heads_in_chunks(hooked, H, W, p, "downstream_head.", head_args.get("patch_size", 16), head_chunk)
        pr = dict(pts3d_in_other_view=r["pts3d"], conf=r["conf"])
        if head_args.get("with_local_head", False):
            rl = _heads_in_chunks(hooked, H, W, p, "downstream_head_local.", head_args.get("patch_size", 16), head_chunk)
            pr.update(pts3d_local=rl["pts3d"], conf_local=rl["conf"])
        preds.append(pr)
    return preds


def synthetic_views(n: int, H: int = 368, W: int = 512, seed0: int = 1234):
    """Synthetic inputs of SURVEY.md §8(d): uniform [-1,1] images, generator seed 1234+i."""
    views = []
    for i in range(n):
        g = torch.Generator().manual_seed(seed0 + i)
        views.append(dict(img=torch.rand(1, 3, H, W, generator=g) * 2 - 1,
                          true_shape=np.int32([[H, W]]), idx=i, instance=str(i),
                          dataset="synthetic", label=f"v{i}"))
    return views
