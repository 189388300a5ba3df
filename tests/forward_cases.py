"""Whole-forward cases at the view counts the project runs at (tests/test_forward_fp64_gpu.py), and the host branches each
reaches (tests/test_forward_fp64_cpu.py records them in an emulated run and fails if a branch has no case).

Weight gain: the tiny model's synthetic weights at gain 1 amplify a bf16 rounding to about 1e-2 relative error at the
output, the whole bf16 tolerance, so a per-slice bound would have no headroom left to see a host fault with.  The tiny
cases use gain 0.7, where the bf16 forward's worst slice sits near 0.7 of the bound on an H100.  ViT-L/512 at gain 1 is the
same: its bf16 worst patch reached 2.3x the bound (pts3d_local) and fp16 1.5x, with a concatenated error inside the
old tolerances; it runs at gain 0.7 too.

A case is a list of scenes, each a list of (H, W) per view, a batch size, a model, the precisions it runs in and the
entry point: ``inference`` (one scene through fast3r_b200.inference, whose host sink streams every head chunk to pinned
memory), ``forward`` (Fast3R.forward) or ``inference_many`` (several scenes in one Fast3R.forward_many).  Images are
``synth_images`` with one seed per view; weights are ``synth_state_dict``."""
from __future__ import annotations

import torch

from tests.golden.synth import synth_state_dict, synth_images

L368, L384, P512 = (368, 512), (384, 512), (512, 384)

# tiny_mixed_n34: the 6 portrait views sit between landscape ones, so a view's predictions must find their way back from
# its shape group to its place in the scene
_MIXED = [P512 if i % 6 == 3 else L368 for i in range(34)]

CASES = {
    # ViT-L/512 at the benchmark's 32 views: head chunks 25 + 7 (bf16, fp16) and 8 x 4 (parity path), host sink
    "vitl_n32": dict(model="vitl", gain=0.7, scenes=[[L368] * 32], B=1, precisions=("bf16", "fp16", "fp32"),
                     entry="inference"),
    # 320 views, 235 520 tokens: two encoder chunks of at most 256 images
    "tiny_n320": dict(model="tiny", gain=0.7, scenes=[[L368] * 320], B=1, precisions=("bf16", "fp32"), entry="forward"),
    # B=2: 32 head images in (view, b) order, so the bf16 chunk boundary at image 25 falls inside view 12
    "tiny_b2_n16": dict(model="tiny", gain=0.7, scenes=[[L368] * 16], B=2, precisions=("bf16", "fp32"), entry="forward"),
    # two shape groups through _pack_tokens; the 28-view group is split 25 + 3 into head chunks
    "tiny_mixed_n34": dict(model="tiny", gain=0.7, scenes=[_MIXED], B=1, precisions=("bf16", "fp32"), entry="forward"),
    # three scenes of different view counts and shapes in one packed forward
    "tiny_many": dict(model="tiny", gain=0.7, scenes=[[L368] * 20, [L384] * 7, [P512] * 5], B=1, precisions=("bf16",),
                      entry="inference_many"),
}

# host branches of Fast3R._forward / _encode / _heads / inference's host sink (names used by the CPU coverage test)
BRANCHES = ("encoder_chunks>1", "head_chunks>1", "head_chunk_splits_view", "batch>1", "groups>1", "packed",
            "sink_chunks>1")


def model_args(kind: str):
    from fast3r_b200 import tiny_args, vit_large_args
    return {"tiny": tiny_args, "vitl": vit_large_args}[kind]()


def state_dict(kind: str, gain: float, M=None, seed: int = 0):
    """(config, synthetic weights) of a model kind; ``M``: the fast3r_b200.model module to take the key schema from."""
    if M is None:
        import fast3r_b200.model as M
    cfg = model_args(kind)
    with torch.device("meta"):
        shapes = {k: tuple(v.shape) for k, v in M.Fast3R(*cfg).state_dict().items()}
    return cfg, synth_state_dict(shapes, seed=seed, gain=gain)


def scene_images(scenes, B: int, seed0: int = 1234, shape_map=None):
    """Per scene, the list of (B, 3, H, W) images; view k of the whole case has generator seed seed0 + k.
    ``shape_map``: replaces each (H, W) (the CPU test runs the same composition at small sizes)."""
    out, k = [], 0
    for sc in scenes:
        imgs = []
        for hw in sc:
            h, w = shape_map[hw] if shape_map else hw
            imgs.append(synth_images(1, B, h, w, seed0=seed0 + k)[0])
            k += 1
        out.append(imgs)
    return out

