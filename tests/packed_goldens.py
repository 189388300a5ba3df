"""Tiny golden scenes packed into one Fast3R.forward_many call (tests/test_packed_cpu.py, tests/test_packed_gpu.py).

All tiny fixtures share the weights (synth_state_dict, weight_seed 0).  The portrait fixture needs
patch_embed_cls="ManyAR_PatchEmbed" with landscape_only heads; the other fixtures pass no true_shape, so that
configuration runs them exactly as the default one does, and one model serves all four scenes.  Every fixture was
generated from torch.manual_seed(rng_seed) right before its forward, so each scene's image ids are drawn from that seed
(reseeded_ids)."""
import os

import torch

from tests.golden.synth import synth_state_dict, synth_images

TAGS = ["tiny_b1_n3", "tiny_single_view", "tiny_mixed_res", "tiny_portrait"]


def tiny_model(golden_dir, M=None):
    """The ManyAR / landscape_only tiny model with the fixtures' weights (M: the fast3r_b200.model module to build it
    from)."""
    if M is None:
        import fast3r_b200.model as M
    from fast3r_b200 import tiny_args
    g = torch.load(os.path.join(golden_dir, "tiny_portrait.pt"))
    enc, dec, head = tiny_args()
    enc.update(g["enc_over"])
    head.update(g["head_over"])
    model = M.Fast3R(enc, dec, head).eval()
    model.load_state_dict(synth_state_dict(g["shapes"], seed=g["weight_seed"]))
    return model


def scene(golden_dir, tag, device="cpu"):
    """(views, reference preds, rng_seed) of one fixture."""
    g = torch.load(os.path.join(golden_dir, f"{tag}.pt"))
    if tag == "tiny_mixed_res":
        imgs = [synth_images(1, g["B"], h, w, seed0=1234 + i)[0] for i, (h, w) in enumerate(g["sizes"])]
        views = [dict(img=im.to(device)) for im in imgs]
    elif tag == "tiny_portrait":
        views = [dict(img=im.to(device), true_shape=torch.tensor([g["true_shapes"][i]] * g["B"], dtype=torch.int32))
                 for i, im in enumerate(synth_images(g["N"], g["B"], g["H"], g["W"]))]
    else:
        views = [dict(img=im.to(device)) for im in synth_images(g["N"], g["B"], g["H"], g["W"])]
    return views, g["preds"], g["rng_seed"]


def reseeded_ids(model, seeds):
    """Makes the decoder draw the k-th call's image ids from torch.manual_seed(seeds[k]), as each fixture did."""
    draw, calls = model.decoder.draw_image_ids, iter(seeds)

    def reseeded(batch_size, num_views, rank_offset=None):
        torch.manual_seed(next(calls))
        return draw(batch_size, num_views, rank_offset=rank_offset)

    model.decoder.draw_image_ids = reseeded
