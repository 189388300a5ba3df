"""H100-native drop-in for ``fast3r.models.fast3r.Fast3R`` (reference: fast3r/models/fast3r.py:45-497).

Same constructor dicts, same ``state_dict`` key schema (SURVEY.md §8(b)), same
``forward(views, profiling=False) -> list[dict]`` contract and the same host-side RNG consumption for the random
image-index embedding — but every tensor op of the path runs in hand-written sm_90a kernels behind the C ABI
(``libfast3r_b200.so``).  torch.nn modules below are parameter containers only (so checkpoints load unchanged);
their ``forward`` is never called.  There is no PyTorch/CPU fallback: without the CUDA library this raises.

Numerics: bf16 tensor-core operands, fp32 accumulation, fp32 residual stream, fp32 LayerNorm/softmax
statistics, fp32 outputs — closer to the reference's fp32 path than the reference's own bf16-autocast path
(SURVEY.md Appendix B).  ``set_precision("fp16")`` runs the same kernels on fp16 operands and ``"fp32"`` the parity
path (Fast3R docstring).
"""
from __future__ import annotations

import math
import time
from copy import deepcopy
from itertools import accumulate
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn as nn

from . import lib as L
from . import ops
from .ops import Segments

try:  # same hub integration as the reference (fast3r/models/fast3r.py:45-49): from_pretrained / save_pretrained
    from huggingface_hub import PyTorchModelHubMixin as _HubMixin
except Exception:  # pragma: no cover - huggingface_hub is optional for the kernels themselves
    class _HubMixin:  # type: ignore
        def __init_subclass__(cls, **kw):
            super().__init_subclass__()

BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32


def _plain(cfg):
    """Plain python containers out of any Mapping / Sequence config (omegaconf DictConfig / ListConfig included), the
    job of OmegaConf.to_container in the reference ctor (fast3r/models/fast3r.py:59-66) without importing omegaconf."""
    from collections.abc import Mapping, Sequence
    if isinstance(cfg, Mapping):
        return {str(k): _plain(v) for k, v in cfg.items()}
    if isinstance(cfg, Sequence) and not isinstance(cfg, (str, bytes)):
        return [_plain(v) for v in cfg]
    return cfg


# --------------------------------------------------------------------------- parameter containers
class _Attention(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.qkv = nn.Linear(dim, dim * 3, bias=True)
        self.proj = nn.Linear(dim, dim)


class _Mlp(nn.Module):
    def __init__(self, dim, hidden):
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden)
        self.fc2 = nn.Linear(hidden, dim)


class _Block(nn.Module):
    """Parameter layout of fast3r/croco/models/blocks.py:197-234."""

    def __init__(self, dim, mlp_ratio, eps):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=eps)
        self.attn = _Attention(dim)
        self.norm2 = nn.LayerNorm(dim, eps=eps)
        self.mlp = _Mlp(dim, int(dim * mlp_ratio))


class _PatchEmbed(nn.Module):
    def __init__(self, patch, dim):
        super().__init__()
        self.proj = nn.Conv2d(3, dim, kernel_size=patch, stride=patch)


class CroCoEncoder(nn.Module):
    """Parameter layout of fast3r/models/fast3r.py:499-547."""

    def __init__(self, img_size=512, patch_size=16, patch_embed_cls="ManyAR_PatchEmbed", embed_dim=768,
                 num_heads=12, depth=12, mlp_ratio=4, pos_embed="RoPE100", attn_implementation="pytorch_naive",
                 **_unused):
        super().__init__()
        if not pos_embed.startswith("RoPE"):
            raise NotImplementedError("Unknown pos_embed " + pos_embed)
        self.rope_base = float(pos_embed[len("RoPE"):])
        self.patch_size, self.embed_dim, self.num_heads, self.depth = patch_size, embed_dim, num_heads, depth
        self.patch_embed_cls = patch_embed_cls
        self.patch_embed = _PatchEmbed(patch_size, embed_dim)
        self.enc_blocks = nn.ModuleList([_Block(embed_dim, mlp_ratio, 1e-6) for _ in range(depth)])
        self.enc_norm = nn.LayerNorm(embed_dim, eps=1e-6)


def _sincos_table(dim: int, n: int = 1000) -> torch.Tensor:
    """fast3r/croco/models/pos_embed.py:58-76 (float64 numpy, then .float()), used at fast3r.py:691-697."""
    omega = np.arange(dim // 2, dtype=float)
    omega /= dim / 2.0
    omega = 1.0 / 10000 ** omega
    out = np.einsum("m,d->md", np.arange(n, dtype=float), omega)
    return torch.from_numpy(np.concatenate([np.sin(out), np.cos(out)], axis=1)).float()


class Fast3RDecoder(nn.Module):
    """Parameter layout of fast3r/models/fast3r.py:654-700."""

    def __init__(self, random_image_idx_embedding: bool, enc_embed_dim: int, embed_dim: int = 768,
                 num_heads: int = 12, depth: int = 12, mlp_ratio: float = 4.0, qkv_bias: bool = True,
                 drop: float = 0.0, attn_drop: float = 0.0, attn_implementation: str = "pytorch_naive",
                 attn_bias_for_inference_enabled=True, **_unused):
        super().__init__()
        if not qkv_bias or drop or attn_drop:
            raise NotImplementedError("fast3r_b200 supports qkv_bias=True, drop=0, attn_drop=0 (the ViT-L config)")
        self.embed_dim, self.num_heads, self.depth = embed_dim, num_heads, depth
        self.random_image_idx_embedding = random_image_idx_embedding
        self.attn_bias_for_inference_enabled = attn_bias_for_inference_enabled
        self.decoder_embed = nn.Linear(enc_embed_dim, embed_dim, bias=True)
        self.dec_blocks = nn.ModuleList([_Block(embed_dim, mlp_ratio, 1e-5) for _ in range(depth)])
        self.register_buffer("image_idx_emb", _sincos_table(embed_dim), persistent=False)
        self.dec_norm = nn.LayerNorm(embed_dim, eps=1e-6)

    def draw_image_ids(self, batch_size: int, num_views: int, rank_offset: Optional[int] = None) -> torch.Tensor:
        """Exact RNG side effects of _generate_per_rank_generator / _get_random_image_pos
        (fast3r/models/fast3r.py:702-713, 738-745): one draw from the GLOBAL torch CPU RNG per forward, also in
        eval.  ``rank_offset`` None => torch.distributed rank (reference behaviour for data parallel)."""
        if not self.random_image_idx_embedding:
            return torch.arange(num_views)[None].expand(batch_size, num_views).contiguous()
        per_forward_pass_seed = torch.randint(0, 2 ** 32, (1,)).item()
        if rank_offset is None:
            rank_offset = torch.distributed.get_rank() if (torch.distributed.is_available()
                                                           and torch.distributed.is_initialized()) else 0
        g = torch.Generator()
        g.manual_seed(per_forward_pass_seed + rank_offset)
        ids = torch.zeros(batch_size, num_views, dtype=torch.long)
        max_image_idx = self.image_idx_emb.shape[0] - 1
        for b in range(batch_size):
            ids[b, 1:] = torch.randperm(max_image_idx, generator=g)[: num_views - 1] + 1
        return ids


class _RCU(nn.Module):
    def __init__(self, f):
        super().__init__()
        self.conv1 = nn.Conv2d(f, f, 3, padding=1)
        self.conv2 = nn.Conv2d(f, f, 3, padding=1)


class _Fusion(nn.Module):
    def __init__(self, f):
        super().__init__()
        self.out_conv = nn.Conv2d(f, f, 1)
        self.resConfUnit1 = _RCU(f)
        self.resConfUnit2 = _RCU(f)


class _DPT(nn.Module):
    """Parameter layout of DPTOutputAdapter_fix (fast3r/dust3r/heads/dpt_head.py:28-40,
    fast3r/croco/models/dpt_block.py:29-88, 350-382, 401-490)."""

    def __init__(self, dim_tokens, layer_dims=(96, 192, 384, 768), feature_dim=256, last_dim=128, num_channels=4):
        super().__init__()
        ld = list(layer_dims)
        self.scratch = nn.Module()
        rn = [nn.Conv2d(ld[i], feature_dim, 3, padding=1, bias=False) for i in range(4)]
        self.scratch.layer1_rn, self.scratch.layer2_rn, self.scratch.layer3_rn, self.scratch.layer4_rn = rn
        self.scratch.layer_rn = nn.ModuleList(rn)  # aliases, like the reference
        for i in range(1, 5):
            setattr(self.scratch, f"refinenet{i}", _Fusion(feature_dim))
        self.head = nn.Sequential(nn.Conv2d(feature_dim, feature_dim // 2, 3, padding=1), nn.Identity(),
                                  nn.Conv2d(feature_dim // 2, last_dim, 3, padding=1), nn.Identity(),
                                  nn.Conv2d(last_dim, num_channels, 1))
        self.act_postprocess = nn.ModuleList([
            nn.Sequential(nn.Conv2d(dim_tokens[0], ld[0], 1), nn.ConvTranspose2d(ld[0], ld[0], 4, stride=4)),
            nn.Sequential(nn.Conv2d(dim_tokens[1], ld[1], 1), nn.ConvTranspose2d(ld[1], ld[1], 2, stride=2)),
            nn.Sequential(nn.Conv2d(dim_tokens[2], ld[2], 1)),
            nn.Sequential(nn.Conv2d(dim_tokens[3], ld[3], 1), nn.Conv2d(ld[3], ld[3], 3, stride=2, padding=1)),
        ])


class PixelwiseTaskWithDPT(nn.Module):
    def __init__(self, dim_tokens, hooks_idx, depth_mode, conf_mode, num_channels=4):
        super().__init__()
        self.hooks_idx, self.depth_mode, self.conf_mode = hooks_idx, depth_mode, conf_mode
        self.dpt = _DPT(dim_tokens, num_channels=num_channels)


# --------------------------------------------------------------------------- packed (device) weights
# Every GEMM weight is packed as [N_out, taps, K] with K contiguous (include/fast3r_b200.h).
class _Packed:
    """Weights packed for one numeric path, which they carry along with the GEMM dispatch of that path.
    ``precision`` "bf16" (fast path): bf16 weights and activations.  "fp16": the same with fp16 in place of bf16.
    "fp32" (parity path): fp32 activations, which the GEMM splits on the fly into bf16 [hi | lo | hi] along K, against
    weights packed as [Whi | Whi | Wlo] (3K wide), so the same kernel accumulates hi*hi + lo*hi + hi*lo in fp32
    (fp32-level products on the bf16 tensor pipe)."""

    def __init__(self, precision: str):
        self.x3 = precision == "fp32"
        self.adt = {"bf16": BF16, "fp16": F16, "fp32": F32}[precision]  # dtype of the activations that feed a GEMM

    def _pk(self, w: torch.Tensor) -> torch.Tensor:
        w = w.detach().to(F32)
        hi = w.to(BF16 if self.x3 else self.adt)
        if not self.x3:
            return hi.contiguous()
        lo = (w - hi.float()).to(BF16)
        return torch.cat([hi, hi, lo], dim=-1).contiguous()

    def _lin(self, m) -> torch.Tensor:  # linear (out,in), 1x1 or patch conv (out,in,kh,kw) -> (out, 1, in*kh*kw)
        return self._pk(m.weight.detach().reshape(m.weight.shape[0], 1, -1))

    def _conv3(self, m) -> torch.Tensor:  # (out,in,3,3) -> (out, 9, in)
        w = m.weight.detach()
        return self._pk(w.permute(0, 2, 3, 1).reshape(w.shape[0], 9, w.shape[1]))

    def _convt(self, m) -> torch.Tensor:  # (in,out,k,k) -> ((i*k+j)*out + o, 1, in)
        w = m.weight.detach()
        k = w.shape[2]
        return self._pk(w.permute(2, 3, 1, 0).reshape(k * k * w.shape[1], 1, w.shape[0]))

    def gemm(self, a, wt, *, a_relu=False, a_relu_src=None, **kw):
        """``a``: an ``adt`` activation.  ``a_relu`` multiplies relu(a) instead: the parity path folds the ReLU into the
        operand split, the fast path reads the bf16 copy ``a_relu_src`` that the producing GEMM stored."""
        if self.x3:
            return ops.gemm_x3(a, wt, a_relu=a_relu, **kw)
        return ops.gemm(a_relu_src if a_relu else a, wt, **kw)

    def linear(self, a, wt, bias=None, **kw):
        return self.gemm(a, wt, w=a.numel() // a.shape[-1], bias=bias, **kw)


def _f32(t) -> Optional[torch.Tensor]:
    return None if t is None else t.detach().to(F32).contiguous()


class _BlockW(_Packed):
    def __init__(self, blk: _Block, precision="bf16"):
        super().__init__(precision)
        self.n1w, self.n1b = _f32(blk.norm1.weight), _f32(blk.norm1.bias)
        self.n2w, self.n2b = _f32(blk.norm2.weight), _f32(blk.norm2.bias)
        self.qkv_w, self.qkv_b = self._lin(blk.attn.qkv), _f32(blk.attn.qkv.bias)
        self.proj_w, self.proj_b = self._lin(blk.attn.proj), _f32(blk.attn.proj.bias)
        self.fc1_w, self.fc1_b = self._lin(blk.mlp.fc1), _f32(blk.mlp.fc1.bias)
        self.fc2_w, self.fc2_b = self._lin(blk.mlp.fc2), _f32(blk.mlp.fc2.bias)


class _DPTW(_Packed):
    def __init__(self, dpt: _DPT, precision="bf16"):
        super().__init__(precision)
        ap = dpt.act_postprocess
        self.ap0 = (self._lin(ap[0][0]), _f32(ap[0][0].bias), self._convt(ap[0][1]), _f32(ap[0][1].bias))
        self.ap1 = (self._lin(ap[1][0]), _f32(ap[1][0].bias), self._convt(ap[1][1]), _f32(ap[1][1].bias))
        self.ap2 = (self._lin(ap[2][0]), _f32(ap[2][0].bias))
        w31 = self._conv3(ap[3][1])  # stride-2 conv runs as im2col + linear: (out, 9, C') -> (out, 1, 9*C')
        self.ap3 = (self._lin(ap[3][0]), _f32(ap[3][0].bias), w31.reshape(w31.shape[0], 1, -1), _f32(ap[3][1].bias))
        self.rn = [self._conv3(m) for m in dpt.scratch.layer_rn]
        self.fus = {}
        for i in range(1, 5):
            f = getattr(dpt.scratch, f"refinenet{i}")
            self.fus[i] = dict(
                out_w=self._lin(f.out_conv), out_b=_f32(f.out_conv.bias),
                r1=(self._conv3(f.resConfUnit1.conv1), _f32(f.resConfUnit1.conv1.bias),
                    self._conv3(f.resConfUnit1.conv2), _f32(f.resConfUnit1.conv2.bias)),
                r2=(self._conv3(f.resConfUnit2.conv1), _f32(f.resConfUnit2.conv1.bias),
                    self._conv3(f.resConfUnit2.conv2), _f32(f.resConfUnit2.conv2.bias)))
        self.h0 = (self._conv3(dpt.head[0]), _f32(dpt.head[0].bias))
        self.h2 = (self._conv3(dpt.head[2]), _f32(dpt.head[2].bias))
        self.w4 = dpt.head[4].weight.detach().to(F32).reshape(dpt.head[4].weight.shape[0], -1).contiguous()
        self.b4 = _f32(dpt.head[4].bias)


class _ModelW(_Packed):
    def __init__(self, model: "Fast3R", precision: str, device):
        super().__init__(precision)
        enc, dec = model.encoder, model.decoder
        self.pe_w, self.pe_b = self._lin(enc.patch_embed.proj), _f32(enc.patch_embed.proj.bias)
        self.enc = [_BlockW(b, precision) for b in enc.enc_blocks]
        self.enc_nw, self.enc_nb = _f32(enc.enc_norm.weight), _f32(enc.enc_norm.bias)
        self.de_w, self.de_b = self._lin(dec.decoder_embed), _f32(dec.decoder_embed.bias)
        self.dec = [_BlockW(b, precision) for b in dec.dec_blocks]
        self.dec_nw, self.dec_nb = _f32(dec.dec_norm.weight), _f32(dec.dec_norm.bias)
        self.table = dec.image_idx_emb.detach().to(device=device, dtype=F32).contiguous()
        self.head = _DPTW(model.downstream_head.dpt, precision)
        local = model.downstream_head_local
        self.head_local = _DPTW(local.dpt, precision) if local is not None else None
        j = torch.arange(16, dtype=torch.float32)
        ang = torch.arange(256, dtype=torch.float32)[:, None] * (1.0 / (enc.rope_base ** (j / 16.0)))[None]
        self.rope_cos, self.rope_sin = ang.cos().contiguous().to(device), ang.sin().contiguous().to(device)


def _sync(device) -> None:
    """profiling=True synchronises like the reference does (fast3r.py:322-491), on the device of the views."""
    if device.type == "cuda":
        torch.cuda.synchronize(device)


def _require_cuda(device) -> None:
    """The product has exactly one compute path: the sm_90a kernels.  (tests/ replace this hook, together with
    ``fast3r_b200.model.ops``, by a CPU emulator of the C ABI to exercise the host orchestration without a GPU.)"""
    if device.type != "cuda":
        raise RuntimeError("fast3r_b200.Fast3R runs on CUDA (sm_90a) only; call model.to('cuda') first. "
                           "There is no CPU fallback.")
    L.load()


# --------------------------------------------------------------------------- the model
PRECISIONS = ("bf16", "fp32", "fp16")


class Fast3R(nn.Module, _HubMixin, repo_url="https://github.com/facebookresearch/fast3r", tags=["image-to-3d"]):
    """Drop-in replacement for fast3r.models.fast3r.Fast3R (same ctor / state_dict / forward contract, same
    huggingface_hub mixin: ``Fast3R.from_pretrained(dir_or_repo)`` / ``save_pretrained``).

    ``precision`` selects the numeric path of the kernels:
      * ``"bf16"`` (default, the benchmarked path): bf16 tensor-core operands, fp32 accumulation / residual stream /
        statistics / outputs - what the reference computes under ``torch.autocast(bfloat16)``, a little closer to fp32.
      * ``"fp32"`` (parity path): the reference's no-autocast result (``inference(..., dtype="32")``,
        fast3r/dust3r/inference_multiview.py:41-49) to ~1e-5 rel-L2: activations are stored fp32 and every tensor-core
        product is evaluated as hi*hi + lo*hi + hi*lo on bf16 pairs (3x the MMA work).
      * ``"fp16"``: the fast path with fp16 in place of every bf16 tensor (3 more mantissa bits at the same tensor-core
        rate; fp32 stays fp32) - what the reference computes under its default ``torch.autocast("cuda")`` (fp16).  A
        16-bit activation past 65504 becomes inf, as under that autocast.  Not available on a sequence-parallel
        (sharded) model."""

    def __init__(self, encoder_args: dict, decoder_args: dict, head_args: dict, freeze="none"):
        super().__init__()
        self.encoder_args = _plain(encoder_args)
        self.decoder_args = _plain(decoder_args)
        self.head_args = _plain(head_args)
        self.build_encoder(self.encoder_args)
        self.build_decoder(self.decoder_args)
        self.build_head(self.head_args)
        self.max_parallel_views_for_head = 25
        self.max_images_per_encoder_chunk = 256
        self.precision = "bf16"
        # sequence-parallel inference (set by fast3r_b200.parallel.enable_sequence_parallel)
        self.sp_group = None
        # None: per-rank seed offset like the reference (data parallel, fast3r.py:707-708); an int pins the offset
        # (sequence parallel always broadcasts the rank-0 draw so that all ranks use the single-device id stream)
        self.image_id_rank_offset = None
        self._taps = None  # set to a dict to record per-stage tensors (parity debugging / tests)
        self._host_sink = None  # set by inference(): streams finished head chunks to pinned host memory
        self._packed = {}
        self._packed_sig = {}
        self.set_freeze(freeze)

    # ---- construction (fast3r/models/fast3r.py:72-157)
    def build_encoder(self, encoder_args: dict):
        if encoder_args["encoder_type"] != "croco":
            raise ValueError(f"Unsupported encoder type for fast3r_b200: {encoder_args['encoder_type']}")
        a = deepcopy(encoder_args)
        a.pop("encoder_type")
        self.encoder = CroCoEncoder(**a)

    def build_decoder(self, decoder_args: dict):
        decoder_args["decoder_type"] = decoder_args.get("decoder_type", "fast3r")
        if decoder_args["decoder_type"] != "fast3r":
            raise ValueError(f"Unsupported decoder type for fast3r_b200: {decoder_args['decoder_type']}")
        a = deepcopy(decoder_args)
        a.pop("decoder_type")
        self.decoder = Fast3RDecoder(**a)

    def build_head(self, head_args: dict):
        self.output_mode, self.head_type = head_args["output_mode"], head_args["head_type"]
        self.depth_mode, self.conf_mode = head_args["depth_mode"], head_args["conf_mode"]
        if not (self.head_type == "dpt" and self.output_mode == "pts3d"):
            raise NotImplementedError(f"unexpected head_type={self.head_type} and output_mode={self.output_mode}")
        # the fused last-conv epilogue hard-codes postprocess.py:28-64 for depth ('exp', -inf, inf) and conf
        # ('exp', 1, inf): no clipping.  Anything else would silently differ from the reference, so refuse it.
        dm, cm = tuple(self.depth_mode), (tuple(self.conf_mode) if self.conf_mode is not None else None)
        ok = (len(dm) == 3 and dm[0] == "exp" and float(dm[1]) == float("-inf") and float(dm[2]) == float("inf")
              and cm is not None and len(cm) == 3 and cm[0] == "exp" and float(cm[1]) == 1.0
              and float(cm[2]) == float("inf"))
        if not ok:
            raise NotImplementedError("fast3r_b200 implements depth_mode=('exp',-inf,inf), conf_mode=('exp',1,inf) "
                                      f"only (got {self.depth_mode}, {self.conf_mode})")
        assert self.decoder_args["depth"] > 9
        l2 = self.decoder_args["depth"]
        ed, dd = self.encoder_args["embed_dim"], self.decoder_args["embed_dim"]
        mk = lambda: PixelwiseTaskWithDPT([ed, dd, dd, dd], [0, l2 * 2 // 4, l2 * 3 // 4, l2],  # noqa: E731
                                          self.depth_mode, self.conf_mode)
        self.downstream_head = mk()
        self.downstream_head_local = mk() if head_args.get("with_local_head", False) else None
        self.landscape_only = head_args.get("landscape_only", True)

    def set_freeze(self, freeze):
        self.freeze = freeze
        to_be_frozen = {"none": [], "encoder": [self.encoder], "sandwich": [self.encoder, self.downstream_head]}
        for m in to_be_frozen[freeze]:
            for p in m.parameters():
                p.requires_grad = False

    def set_max_parallel_views_for_head(self, max_parallel_views_for_head):
        self.max_parallel_views_for_head = max_parallel_views_for_head

    def set_precision(self, precision: str):
        if precision not in PRECISIONS:
            raise ValueError(f"precision must be one of {PRECISIONS}, got {precision!r}")
        self.precision = precision
        return self

    def load_state_dict(self, ckpt, **kw):
        r = super().load_state_dict(ckpt, **kw)
        self._packed, self._packed_sig = {}, {}
        return r

    def load_from_dust3r_checkpoint(self, dust3r_checkpoint_path: str):
        """Behaviour of fast3r/models/fast3r.py:162-239: take patch_embed / enc_blocks / enc_norm (-> encoder.*) and
        downstream_head1 (-> downstream_head.*) from a DUSt3R checkpoint; a head that does not fit leaves the current head
        untouched (and ``head_args['skip_load_pretrained_head']`` skips it).  Returns (loaded, not_loaded) key sets."""
        ckpt = torch.load(dust3r_checkpoint_path, weights_only=False)["model"]
        enc_sd, head_sd = {}, {}
        for key, value in ckpt.items():
            if key.startswith(("patch_embed", "enc_blocks", "enc_norm")):
                enc_sd["encoder." + key] = value
            elif key.startswith("downstream_head1"):
                head_sd[key.replace("downstream_head1", "downstream_head", 1)] = value
        loaded = set()
        res = self.load_state_dict(enc_sd, strict=False)
        loaded |= {k[len("encoder."):] for k in enc_sd if k not in set(res.unexpected_keys)}
        if not self.head_args.get("skip_load_pretrained_head", False):
            keep = {k: v.clone() for k, v in self.downstream_head.state_dict().items()}
            try:
                res = self.load_state_dict(head_sd, strict=False)
                loaded |= {k.replace("downstream_head", "downstream_head1", 1) for k in head_sd
                           if k not in set(res.unexpected_keys)}
            except RuntimeError:
                self.downstream_head.load_state_dict(keep)
        self._packed, self._packed_sig = {}, {}
        return loaded, set(ckpt.keys()) - loaded

    def _tap(self, name, t):
        if self._taps is not None and name not in self._taps:  # first writer wins (global head before local head)
            self._taps[name] = t.detach().float().cpu().clone()

    # ---- packed weights (one set per precision, rebuilt when a parameter changes)
    def _signature(self):
        return tuple((p.data_ptr(), p._version) for p in self.parameters())

    def _pack(self, device) -> _ModelW:
        mode = self.precision
        sig = (self._signature(), str(device))
        if mode in self._packed and self._packed_sig.get(mode) == sig:
            return self._packed[mode]
        _require_cuda(device)
        for name, prm in self.named_parameters():
            if prm.device != device:
                raise RuntimeError(f"fast3r_b200: parameter {name} lives on {prm.device} but the views are on {device}; "
                                   "call model.to(device) first (there is no CPU path)")
        enc, dec = self.encoder, self.decoder
        if enc.embed_dim // enc.num_heads != 64 or dec.embed_dim // dec.num_heads != 64:
            raise NotImplementedError("fast3r_b200 attention kernel is specialised for head_dim 64")
        P = _ModelW(self, mode, device)
        self._packed[mode], self._packed_sig[mode] = P, sig
        return P

    # ---- one transformer block (fast3r/croco/models/blocks.py:135-194, 236-239)
    @staticmethod
    def _block(x, w: _BlockW, ws, *, batch, seq, heads, eps, scale, rope=None, kv_exchange=None, segments=None):
        M, D = x.shape
        h, q, kv, att, hid = ws["h"][:M], ws["q"][:M], ws["kv"][:M], ws["att"][:M], ws["hid"][:M]
        ops.layernorm(x, w.n1w, w.n1b, eps, h)
        if rope is not None:
            w.linear(h, w.qkv_w, w.qkv_b, out0=q, ldo=D, split_col=D, out0b=kv, ldo_b=2 * D, epi=L.EPI_ROPE,
                     tok_per_img=rope["P"], grid_w=rope["gw"], rope_cols=2 * D, rope_cos=rope["cos"],
                     rope_sin=rope["sin"])
        else:
            w.linear(h, w.qkv_w, w.qkv_b, out0=q, ldo=D, split_col=D, out0b=kv, ldo_b=2 * D)
        if segments is not None:  # several samples in one sequence (forward_many): each attends to its own tokens
            if w.x3:  # parity path: one attention per segment
                for a, b in zip(segments.offsets, segments.offsets[1:]):
                    ops.attention_x3(q[a:b], kv[a:b], att[a:b], batch=1, heads=heads, sq=b - a, skv=b - a, scale=scale)
            else:
                ops.attention_segments(q, kv, att, segments, heads=heads, scale=scale)
        elif kv_exchange is None:
            (ops.attention_x3 if w.x3 else ops.attention)(q, kv, att, batch=batch, heads=heads, sq=seq, skv=seq,
                                                          scale=scale)
        else:  # sequence parallel: exchange K|V with the other ranks and attend to all keys (parallel.KVExchange)
            kv_exchange.attend(ops, q, kv, att, heads=heads, scale=scale, x3=w.x3)
        w.linear(att, w.proj_w, w.proj_b, out0=x, res0=x)
        ops.layernorm(x, w.n2w, w.n2b, eps, h)
        w.linear(h, w.fc1_w, w.fc1_b, out0=hid, act=L.ACT_GELU)
        w.linear(hid, w.fc2_w, w.fc2_b, out0=x, res0=x)

    @staticmethod
    def _workspace(M, D, hidden, device, dtype=BF16):
        e = lambda *s: torch.empty(*s, dtype=dtype, device=device)  # noqa: E731
        return dict(h=e(M, D), q=e(M, D), kv=e(M, 2 * D), att=e(M, D), hid=e(M, hidden))

    # ---- encoder (fast3r/models/fast3r.py:250-296, 549-559)
    def _encode(self, imgs: torch.Tensor, P_: _ModelW):
        enc = self.encoder
        n, _, H, W = imgs.shape
        gh, gw = H // enc.patch_size, W // enc.patch_size
        if max(gh, gw) > P_.rope_cos.shape[0]:
            raise ValueError(f"image too large for the RoPE table ({gh}x{gw} patches > {P_.rope_cos.shape[0]})")
        P, D = gh * gw, enc.embed_dim
        feats = torch.empty(n * P, D, dtype=P_.adt, device=imgs.device)
        chunk = self.max_images_per_encoder_chunk
        hidden = enc.enc_blocks[0].mlp.fc1.weight.shape[0]
        ws = self._workspace(min(n, chunk) * P, D, hidden, imgs.device, P_.adt)
        rope = dict(P=P, gw=gw, cos=P_.rope_cos, sin=P_.rope_sin)
        for s in range(0, n, chunk):
            c = min(chunk, n - s)
            M = c * P
            a0 = torch.empty(M, 3 * enc.patch_size * enc.patch_size, dtype=P_.adt, device=imgs.device)
            ops.im2col_patch(imgs[s:s + c], a0)
            x = torch.empty(M, D, dtype=F32, device=imgs.device)
            P_.linear(a0, P_.pe_w, P_.pe_b, out0=x)
            self._tap("patch_embed", x)
            for li, w in enumerate(P_.enc):
                self._block(x, w, ws, batch=c, seq=P, heads=enc.num_heads, eps=1e-6, scale=64 ** -0.5, rope=rope)
                self._tap(f"enc_block{li}", x)
            ops.layernorm(x, P_.enc_nw, P_.enc_nb, 1e-6, feats[s * P:(s + c) * P])
        return feats, P, gh, gw

    # ---- fusion decoder (fast3r/models/fast3r.py:768-808)
    def _decode(self, feats_bnp: torch.Tensor, ids: torch.Tensor, B: int, seq: int, tok_per_img: int, P_: _ModelW,
                kv_exchange=None, segments=None):
        """feats_bnp: (B*seq, D) tokens in (b, view, patch) order.  ids: image-index table rows, a (B, views) tensor
        with one row per view of tok_per_img tokens, or with tok_per_img=0 a flat (B*seq,) tensor with one row per
        token (views of different resolutions).  segments (ops.Segments, B = 1): the sequence holds several samples,
        each attending to its own tokens only."""
        dec = self.decoder
        D = dec.embed_dim
        M = feats_bnp.shape[0]
        dev = feats_bnp.device
        x = torch.empty(M, D, dtype=F32, device=dev)
        P_.linear(feats_bnp, P_.de_w, P_.de_b, out0=x, epi=L.EPI_IDXEMB, tok_per_img=tok_per_img, emb_table=P_.table,
                  emb_ids=ids.to(device=dev, dtype=torch.int32).contiguous())
        hd = D // dec.num_heads
        if (not self.training) and dec.attn_bias_for_inference_enabled:
            scale = hd ** -0.5 * (1.0 * math.log(137) / math.log(20)) ** 0.5  # blocks.py:119-124
        else:
            scale = hd ** -0.5
        hidden = dec.dec_blocks[0].mlp.fc1.weight.shape[0]
        ws = self._workspace(M, D, hidden, dev, P_.adt)
        depth = dec.depth
        hooks = {depth * 2 // 4: None, depth * 3 // 4: None}
        self._tap("dec_embed", x)
        for i, w in enumerate(P_.dec):
            if kv_exchange is not None:
                slot = kv_exchange.kv_workspace(ws["kv"].dtype, dev)
                if slot is not None:
                    ws["kv"] = slot  # the QKV GEMM writes K|V straight into this rank's exchange slot of this layer
            self._block(x, w, ws, batch=B, seq=seq, heads=dec.num_heads, eps=1e-5, scale=scale, kv_exchange=kv_exchange,
                        segments=segments)
            self._tap(f"dec_block{i}", x)
            if (i + 1) in hooks:
                if P_.x3:
                    hooks[i + 1] = x.clone()
                else:
                    t = torch.empty(M, D, dtype=P_.adt, device=dev)
                    (ops.cast_f16 if P_.adt == F16 else ops.cast_bf16)(x, t)
                    hooks[i + 1] = t
        last = torch.empty(M, D, dtype=P_.adt, device=dev)
        ops.layernorm(x, P_.dec_nw, P_.dec_nb, 1e-6, last)
        return [hooks[depth * 2 // 4], hooks[depth * 3 // 4], last]

    # ---- DPT head + postprocess (dpt_head.py:42-90, dpt_block.py, postprocess.py)
    @staticmethod
    def _rcu(hw: _DPTW, x, x_relu, w, nv, h, w_, res1=None, want_relu=False):
        """y = x + conv2(relu(conv1(relu(x)))) (+ res1); returns (y, relu(y) or None).  Fast path: relu(x) arrives as
        the 16-bit tensor x_relu and relu(y) is a second epilogue output; parity path: the ReLUs are folded into the
        operand split of the consuming conv (x_relu / the returned relu(y) are None)."""
        dev = x.device
        t = torch.empty(nv, h, w_, 256, dtype=hw.adt, device=dev)
        hw.gemm(x, w[0], a_relu=True, a_relu_src=x_relu, w=w_, h=h, nb=nv, taps=9, bias=w[1], out0=t, act=L.ACT_RELU)
        y = torch.empty(nv, h, w_, 256, dtype=hw.adt, device=dev)
        if hw.x3:
            ops.gemm_x3(t, w[2], w=w_, h=h, nb=nv, taps=9, bias=w[3], out0=y, res0=x)
            if res1 is not None:
                ops.add_f32(y, res1)
            return y, None
        yr = torch.empty(nv, h, w_, 256, dtype=hw.adt, device=dev) if want_relu else None
        ops.gemm(t, w[2], w=w_, h=h, nb=nv, taps=9, bias=w[3], out0=y, out1=yr, res0=x, res1=res1)
        return y, yr

    def _dpt(self, hooked: List[torch.Tensor], nv: int, gh: int, gw: int, H: int, W: int, hw: _DPTW,
             pts: torch.Tensor, conf: torch.Tensor):
        dev = hooked[0].device
        e = lambda *s: torch.empty(*s, dtype=hw.adt, device=dev)  # noqa: E731
        g = hw.gemm
        # act_postprocess
        a = e(nv, gh, gw, 96)
        g(hooked[0], hw.ap0[0], w=gw, h=gh, nb=nv, bias=hw.ap0[1], out0=a)
        l0 = e(nv, 4 * gh, 4 * gw, 96)
        g(a, hw.ap0[2], w=gw, h=gh, nb=nv, bias=hw.ap0[3], out0=l0, epi=L.EPI_CONVT, ct_k=4, ct_cout=96)
        a = e(nv, gh, gw, 192)
        g(hooked[1], hw.ap1[0], w=gw, h=gh, nb=nv, bias=hw.ap1[1], out0=a)
        l1 = e(nv, 2 * gh, 2 * gw, 192)
        g(a, hw.ap1[2], w=gw, h=gh, nb=nv, bias=hw.ap1[3], out0=l1, epi=L.EPI_CONVT, ct_k=2, ct_cout=192)
        l2 = e(nv, gh, gw, 384)
        g(hooked[2], hw.ap2[0], w=gw, h=gh, nb=nv, bias=hw.ap2[1], out0=l2)
        a = e(nv, gh, gw, 768)
        g(hooked[3], hw.ap3[0], w=gw, h=gh, nb=nv, bias=hw.ap3[1], out0=a)
        h3, w3 = (gh + 1) // 2, (gw + 1) // 2
        l3 = e(nv, h3, w3, 768)
        if hw.x3:  # stride-2 conv = strided im2col of the split operand (channels [hi | lo | hi]) + linear
            a3 = torch.empty(nv, gh, gw, 3 * 768, dtype=BF16, device=dev)
            ops.split3(a, a3)
            col = torch.empty(nv * h3 * w3, 27 * 768, dtype=BF16, device=dev)
            ops.im2col3x3s2(a3, col, nv, gh, gw, 3 * 768, h3, w3)
        else:
            col = e(nv * h3 * w3, 9 * 768)
            ops.im2col3x3s2(a, col, nv, gh, gw, 768, h3, w3)
        ops.gemm(col, hw.ap3[2], w=nv * h3 * w3, bias=hw.ap3[3], out0=l3)
        # layer_rn (3x3, no bias): keep x and relu(x)
        dims = [(4 * gh, 4 * gw), (2 * gh, 2 * gw), (gh, gw), (h3, w3)]
        lay, lay_r = [], []
        for i, src in enumerate([l0, l1, l2, l3]):
            hh, ww = dims[i]
            o = e(nv, hh, ww, 256)
            orl = None if hw.x3 else e(nv, hh, ww, 256)
            g(src, hw.rn[i], w=ww, h=hh, nb=nv, taps=9, out0=o, out1=orl)
            lay.append(o)
            lay_r.append(orl)
            self._tap(f"layer_rn{i}", o)

        def out_conv_up(y, f, hh, ww, ho, wo):
            # 1x1 out_conv commutes with the bilinear upsample (weights sum to 1): do it at low resolution
            z = e(nv, hh, ww, 256)
            g(y, f["out_w"], w=ww, h=hh, nb=nv, bias=f["out_b"], out0=z)
            up = e(nv, ho, wo, 256)
            ops.upsample2x(z, up, nv, hh, ww, 256, ho, wo)
            return up

        # refinenet4 (single input; output cropped to layer-3 size, dpt_head.py:69-71)
        y, _ = self._rcu(hw, lay[3], lay_r[3], hw.fus[4]["r2"], nv, h3, w3)
        path = out_conv_up(y, hw.fus[4], h3, w3, gh, gw)
        self._tap("path4", path)
        for lvl, i in ((3, 2), (2, 1), (1, 0)):
            hh, ww = dims[i]
            f = hw.fus[lvl]
            s, sr = self._rcu(hw, lay[i], lay_r[i], f["r1"], nv, hh, ww, res1=path, want_relu=True)
            y, _ = self._rcu(hw, s, sr, f["r2"], nv, hh, ww)
            path = out_conv_up(y, f, hh, ww, 2 * hh, 2 * ww)
            self._tap(f"path{lvl}", path)
        # head: conv3x3 256->128, x2 bilinear, conv3x3 128->128 + ReLU + conv1x1 128->4 + postprocess (fused)
        hh, ww = 8 * gh, 8 * gw
        t = e(nv, hh, ww, 128)
        g(path, hw.h0[0], w=ww, h=hh, nb=nv, taps=9, bias=hw.h0[1], out0=t)
        up = e(nv, H, W, 128)
        ops.upsample2x(t, up, nv, hh, ww, 128, H, W)
        g(up, hw.h2[0], w=W, h=H, nb=nv, taps=9, bias=hw.h2[1], epi=L.EPI_FINAL, w4=hw.w4, b4=hw.b4, pts=pts, conf=conf)

    def _heads(self, enc, hooked, B, P_: _ModelW, device, results):
        """The global (and local) DPT head of every shape group, in chunks of max_parallel_views_for_head views
        (fast3r.py:430-444); view i's predictions go into results[i]."""
        heads = [("pts3d_in_other_view", "conf", P_.head)]
        if P_.head_local is not None:
            heads.append(("pts3d_local", "conf_local", P_.head_local))
        step = max(1, int(self.max_parallel_views_for_head))
        if P_.x3:
            step = min(step, 8)  # fp32 feature maps + split scratch are ~5x the bf16 footprint
        for ((H, W), idxs, _, P, gh, gw), hooked_g in zip(enc, hooked):
            nvt = len(idxs) * B
            outs = {}
            for pts, conf, _hw in heads:
                outs[pts] = torch.empty(nvt, H, W, 3, dtype=F32, device=device)
                outs[conf] = torch.empty(nvt, H, W, dtype=F32, device=device)
            for s in range(0, nvt, step):
                c = min(step, nvt - s)
                hk = [t[s * P:(s + c) * P] for t in hooked_g]
                for pts, conf, hw in heads:
                    self._dpt(hk, c, gh, gw, H, W, hw, outs[pts][s:s + c], outs[conf][s:s + c])
                if self._host_sink is not None:  # D2H of this chunk overlaps the heads of the next one (SURVEY §8 f1)
                    self._host_sink.chunk_done(list(outs.values()), s, c)
            for k, i in enumerate(idxs):
                results[i].update({key: t[k * B:(k + 1) * B] for key, t in outs.items()})

    # ---- portrait views (ManyAR_PatchEmbed + landscape_only heads: fast3r/dust3r/patch_embed.py:59-105,
    #      fast3r/dust3r/utils/misc.py:74-104)
    def _portrait_flags(self, views, H, W):
        """Per view: True if it is a portrait image stored transposed in a landscape buffer (true_shape = (W, H)).  The
        reference supports that only with patch_embed_cls="ManyAR_PatchEmbed" and head landscape_only=True (training
        configuration); with PatchEmbedDust3R / landscape_only=False (what every inference caller uses) true_shape has to
        equal the stored shape (misc.py:67-72 takes the head resolution from it)."""
        flags = []
        many_ar = self.encoder.patch_embed_cls == "ManyAR_PatchEmbed" and self.landscape_only
        for v in views:
            ts = v.get("true_shape", None)
            if ts is None:
                flags.append(False)
                continue
            ts = torch.as_tensor(ts).reshape(-1, 2)
            same = bool(((ts[:, 0] == H) & (ts[:, 1] == W)).all())
            swapped = bool(((ts[:, 0] == W) & (ts[:, 1] == H)).all()) and H != W
            if same:
                flags.append(False)
            elif swapped and many_ar:
                flags.append(True)
            elif swapped:
                raise ValueError("portrait true_shape needs patch_embed_cls='ManyAR_PatchEmbed' and landscape_only=True "
                                 "(with PatchEmbedDust3R / landscape_only=False true_shape must equal the image shape)")
            else:
                raise NotImplementedError("fast3r_b200: true_shape must be the image shape or its transpose, identical for "
                                          "all batch elements of a view")
        return flags

    # ---- forward (fast3r/models/fast3r.py:302-497)
    def _check_forward(self):
        if self.training and torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError(
                "fast3r_b200.Fast3R has no backward kernels (training step, SURVEY a13 / config 5, is not built): "
                "call it under torch.no_grad() for a forward-only pass, or use model.eval()")
        if self.precision not in PRECISIONS:
            raise ValueError(f"precision must be one of {PRECISIONS}, got {self.precision!r}")

    def forward(self, views, profiling=False):
        self._check_forward()
        with torch.no_grad():
            preds, profiling_info = self._forward([views], profiling)
        return (preds[0], profiling_info) if profiling else preds[0]

    def _landscape(self, views):
        """(batch size, images in the geometry the model runs them in, portrait flag per view) of one sample's views.
        Portrait views (ManyAR_PatchEmbed + landscape_only heads) are recognised when all views share one stored shape.
        They are un-transposed (a strided view of the same pixels) and run in their true geometry - patch grid, RoPE
        positions and DPT head at (W, H); their predictions are transposed back to the landscape storage layout after
        the heads, exactly what ManyAR_PatchEmbed + transpose_to_landscape.wrapper_yes compute."""
        B, _, H, W = views[0]["img"].shape
        ps = self.encoder.patch_size
        for v in views:
            b, _, h, w = v["img"].shape
            if b != B:
                raise ValueError("all views must have the same batch size")
            if h % ps or w % ps:
                raise AssertionError(f"Input image size ({h}x{w}) is not a multiple of patch size ({ps}).")
        same_shape = all(v["img"].shape == views[0]["img"].shape for v in views)
        portrait = self._portrait_flags(views, H, W) if same_shape else [False] * len(views)
        imgs = [v["img"].swapaxes(-1, -2) if p else v["img"] for v, p in zip(views, portrait)]
        return B, imgs, portrait

    @staticmethod
    def _shape_groups(imgs) -> Dict[tuple, List[int]]:
        """Views of different resolutions (fast3r/models/fast3r.py:276-294, 364-376, 407-428): the reference encodes them
        and runs the heads view by view; here views are grouped by shape (same arithmetic per view, batched per group)."""
        groups: Dict[tuple, List[int]] = {}
        for i, im in enumerate(imgs):
            groups.setdefault(tuple(im.shape[-2:]), []).append(i)
        return groups

    def _encode_groups(self, imgs, groups, device, P_: _ModelW, keep=lambda i: True):
        """Per shape group: ((H, W), its kept views, their encoder tokens in (view, b, patch) order, P, gh, gw)."""
        enc = []
        for shape, idxs in groups.items():
            idxs = [i for i in idxs if keep(i)]
            if not idxs:  # no view of this resolution on this rank
                continue
            x = torch.cat([imgs[i].to(device, non_blocking=True) for i in idxs], dim=0).to(dtype=F32).contiguous()
            enc.append((shape, idxs) + self._encode(x, P_))
        return enc

    @staticmethod
    def _to_landscape(results, portrait):
        for r, p in zip(results, portrait):
            if p:
                for k in list(r):
                    r[k] = r[k].swapaxes(1, 2)

    def _pack_tokens(self, enc, ids, off, t0, seq, B, P_: _ModelW, device):
        """Decoder input with one image-index row per token, one index_copy / index_select per shape group instead of
        per-view slices: each of the B sequences holds its views' tokens in (view, patch) order, view i at rows
        [off[i] - t0, off[i] - t0 + P).  ids: (B, views) image ids.  Returns the (B*seq, D) tokens, their (B*seq,) ids,
        and per group the map of a decoder output back to the group's (view, b, patch) order, the head input order."""
        feats_bnp = torch.empty(B * seq, self.encoder.embed_dim, dtype=P_.adt, device=device)
        tok_ids = torch.empty(B, seq, dtype=torch.int32)
        to_heads = []
        for _, idxs, feats, P, _, _ in enc:
            base = torch.tensor([off[i] - t0 for i in idxs], dtype=torch.long)  # (n_g,)
            r = (base[:, None, None] + torch.arange(B, dtype=torch.long)[None, :, None] * seq
                 + torch.arange(P, dtype=torch.long)[None, None, :]).reshape(-1).to(device)  # (n_g, B, P) order
            feats_bnp.index_copy_(0, r, feats)
            for i in idxs:
                tok_ids[:, off[i] - t0: off[i] - t0 + P] = ids[:, i:i + 1].to(torch.int32)
            to_heads.append(lambda t, r=r: t.index_select(0, r))
        return feats_bnp, tok_ids.reshape(-1), to_heads

    def forward_many(self, samples, profiling=False):
        """Several scenes in one forward.  ``samples``: a list of view lists, each of batch size 1 (what inference()
        collates); returns one preds list per sample, each what ``forward(sample)`` returns (with ``profiling``, one
        ``profiling_info`` for the whole call).  The encoder and the DPT heads batch the views of all samples by shape;
        the decoder runs one sequence of all samples' tokens, sample after sample, whose fusion attention is block-
        diagonal (ops.attention_segments): each sample's tokens attend to that sample's tokens only.  The image ids are
        drawn per sample, in sample order, so the global torch RNG advances as for forward on each sample in turn.
        Per sample, the result equals forward(sample) up to the order of fp32 sums: GEMM plans depend on the row count,
        which packing changes.  forward_many([sample]) is bit-identical to forward(sample)."""
        self._check_forward()
        if self.sp_group is not None:
            raise NotImplementedError("forward_many does not run on a sequence-parallel (sharded) model; call forward "
                                      "per sample")
        if len(samples) == 0:
            raise ValueError("forward_many: empty sample list")
        with torch.no_grad():
            preds, profiling_info = self._forward(samples, profiling, packed=True)
        return (preds, profiling_info) if profiling else preds

    def _forward(self, samples, profiling=False, packed=False):
        """The forward of ``samples``, a list of view lists: (one preds list per sample, profiling_info or None).
        forward runs one sample, batched and, on a sequence-parallel model, sharded.  ``packed`` (forward_many) runs
        samples of batch size 1 as one decoder sequence with one attention segment per sample."""
        # (decorated with no_grad: the CUDA path has no backward kernels yet.  Training-mode FORWARD semantics - attention
        # scale 1/8, fast3r/croco/models/blocks.py:151-154 - are honoured and tested; optimisation steps are not.)
        profiling_info = {} if profiling else None
        t_start = time.time()
        imgs, portrait = [], []  # all views of all samples, sample after sample
        for s, views in enumerate(samples):  # forward_many's checks of a sample come with _landscape's, in sample order
            if packed and len(views) == 0:
                raise ValueError(f"forward_many: sample {s} has no views")
            B, sample_imgs, sample_portrait = self._landscape(views)
            if packed and B != 1:
                raise ValueError(f"forward_many packs samples of batch size 1 (sample {s} has {B}); call forward for it")
            imgs += sample_imgs
            portrait += sample_portrait
        N = len(imgs)
        first = list(accumulate([len(views) for views in samples], initial=0))  # first view of each sample
        ps = self.encoder.patch_size
        groups = self._shape_groups(imgs)
        sp = self.sp_group
        if sp is not None and self.precision == "fp16":
            raise NotImplementedError("precision='fp16' does not run on a sequence-parallel (sharded) model: its K|V "
                                      "exchange carries bf16; use precision='bf16' or 'fp32'")
        device = samples[0][0]["img"].device
        if sp is not None and device.type != "cuda":
            device = next(self.parameters()).device  # sharded forward: host views are uploaded per rank below
        P_ = self._pack(device)
        tokens = [(im.shape[-2] // ps) * (im.shape[-1] // ps) for im in imgs]
        off = list(accumulate(tokens, initial=0))  # first token of each view in the decoder sequence
        # sequence parallel: contiguous views per rank, balanced by token count (views of different resolutions)
        lo, hi = (0, N) if sp is None else sp.view_range(N, tokens)
        enc = self._encode_groups(imgs, groups, device, P_, keep=lambda i: lo <= i < hi)
        if profiling:
            _sync(device)
            profiling_info["encode_images_time"] = time.time() - t_start
        t1 = time.time()
        # image ids: same host RNG stream as the reference, one draw per sample in sample order.  Sequence parallel:
        # every rank consumes its own RNG draw (same side effect as the reference) but uses the ids rank 0 drew, so the
        # result equals the single-device forward whatever the per-rank RNG states are.
        rank_offset = 0 if sp is not None else self.image_id_rank_offset
        ids = torch.cat([self.decoder.draw_image_ids(B, len(views), rank_offset=rank_offset) for views in samples],
                        dim=1)
        if sp is not None:
            ids = sp.broadcast_ids(ids, device)
        if profiling:
            profiling_info["pos_emb_time"] = time.time() - t1
            _sync(device)
        t2 = time.time()
        segments = Segments([off[i] for i in first], device) if packed else None
        # decoder input: the tokens of each sample in (view, patch) order; to_heads[g] takes a decoder output back to
        # group g's (view, b, patch) order, the order of the head input (fast3r.py:385-398)
        if len(groups) == 1 and not packed:  # one image id per view
            (_, idxs, feats, P, _, _), = enc
            seq, tok_per_img, ids = len(idxs) * P, P, ids[:, lo:hi].contiguous()
            if B == 1:
                feats_bnp, to_heads = feats, [lambda t: t]
            else:  # (n, b, p) <-> (b, n, p)
                n = len(idxs)
                swap = lambda t, a, b: t.view(a, b, P, -1).permute(1, 0, 2, 3).contiguous().view(a * b * P, -1)  # noqa: E731
                feats_bnp, to_heads = swap(feats, n, B), [lambda t: swap(t, B, n)]
        else:
            t0 = off[lo]  # this rank's tokens are [off[lo], off[hi]) of each sample's sequence
            seq, tok_per_img = off[hi] - t0, 0
            feats_bnp, ids, to_heads = self._pack_tokens(enc, ids, off, t0, seq, B, P_, device)
        kvx = None
        if sp is not None:
            kvx = sp.make_kv_exchange(B, seq, self.decoder.embed_dim, rows=[off[b] - off[a] for a, b in sp.ranges],
                                      mixed=len(groups) > 1)
        dec_out = self._decode(feats_bnp, ids, B, seq, tok_per_img, P_, kv_exchange=kvx, segments=segments)
        if profiling:
            _sync(device)
            profiling_info["decoder_time"] = time.time() - t2
        t3 = time.time()
        hooked = [[feats] + [to_head(t) for t in dec_out] for (_, _, feats, _, _, _), to_head in zip(enc, to_heads)]
        if profiling:
            profiling_info["head_prepare_input_time"] = time.time() - t3
        t4 = time.time()
        results = [{} for _ in range(N)]
        self._heads(enc, hooked, B, P_, device, results)
        self._to_landscape(results, portrait)
        if sp is not None and sp.gather_preds:
            shapes = [v["img"].shape[-2:] for views in samples for v in views]
            results = sp.gather_results(results, N, B, *shapes[0], device, shapes=shapes)
        results = [results[a:b] for a, b in zip(first, first[1:])]
        if profiling:
            _sync(device)
            t_end = time.time()
            profiling_info["head_forward_time"] = t_end - t4
            profiling_info["total_time"] = t_end - t_start
        return results, profiling_info
