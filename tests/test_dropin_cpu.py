"""Drop-in boundary beyond forward(): hub mixin, config containers, DUSt3R checkpoint loading and portrait views.
CPU only: the kernels are replaced by tests/abi_emulator.py."""
import os

import pytest
import torch

from tests.conftest import rel_l2
from tests.golden.synth import synth_state_dict, synth_images


@pytest.fixture()
def emulated(monkeypatch):
    import fast3r_b200.model as M
    from tests import abi_emulator
    monkeypatch.setattr(M, "ops", abi_emulator)
    monkeypatch.setattr(M, "_require_cuda", lambda device: None)
    return M


def test_hub_mixin_roundtrip(tmp_path):
    """Fast3R.from_pretrained(local_dir) / save_pretrained like the reference (fast3r/models/fast3r.py:45-49, README.md:84)."""
    from fast3r_b200 import Fast3R, tiny_args
    m = Fast3R(*tiny_args())
    m.save_pretrained(str(tmp_path))
    assert {"config.json", "model.safetensors"} <= set(os.listdir(tmp_path))
    m2 = Fast3R.from_pretrained(str(tmp_path))
    assert m2.encoder_args == m.encoder_args and m2.decoder_args == m.decoder_args and m2.head_args == m.head_args
    for (k, a), (_, b) in zip(m.state_dict().items(), m2.state_dict().items()):
        assert torch.equal(a, b), k


def test_mapping_configs_are_accepted():
    """omegaconf DictConfig / ListConfig look like Mapping / Sequence: the ctor must turn them into plain containers
    (reference: OmegaConf.to_container, fast3r.py:59-66)."""
    from collections.abc import Mapping, Sequence
    from fast3r_b200 import Fast3R, tiny_args

    class DictCfg(Mapping):
        def __init__(self, d): self._d = {k: wrap(v) for k, v in d.items()}
        def __getitem__(self, k): return self._d[k]
        def __iter__(self): return iter(self._d)
        def __len__(self): return len(self._d)

    class ListCfg(Sequence):
        def __init__(self, v): self._v = [wrap(x) for x in v]
        def __getitem__(self, i): return self._v[i]
        def __len__(self): return len(self._v)

    def wrap(v):
        return DictCfg(v) if isinstance(v, dict) else ListCfg(v) if isinstance(v, (list, tuple)) else v

    enc, dec, head = tiny_args()
    m = Fast3R(DictCfg(enc), DictCfg(dec), DictCfg(head))
    assert type(m.head_args) is dict and type(m.head_args["depth_mode"]) is list and m.head_args == head


def test_unsupported_head_modes_are_refused():
    from fast3r_b200 import Fast3R, tiny_args
    enc, dec, head = tiny_args()
    for bad in (dict(conf_mode=["exp", 1, 100.0]), dict(depth_mode=["exp", -10.0, 10.0]), dict(depth_mode=["linear", float("-inf"), float("inf")])):
        with pytest.raises(NotImplementedError):
            Fast3R(enc, dec, dict(head, **bad))


def test_load_from_dust3r_checkpoint(tmp_path):
    """Encoder + downstream_head1 of a DUSt3R checkpoint are taken over, everything else is left (fast3r.py:162-239)."""
    from fast3r_b200 import Fast3R, tiny_args
    m = Fast3R(*tiny_args())
    sd = m.state_dict()
    g = torch.Generator().manual_seed(1)
    ck = {}
    for k, v in sd.items():
        if k.startswith("encoder."):
            ck[k[len("encoder."):]] = torch.randn(v.shape, generator=g)
        elif k.startswith("downstream_head."):
            ck[k.replace("downstream_head.", "downstream_head1.", 1)] = torch.randn(v.shape, generator=g)
    for k in list(ck):  # scratch.layer_rn.{i} aliases scratch.layer{i+1}_rn (one tensor in the module)
        if ".scratch.layer_rn." in k:
            i = int(k.split(".scratch.layer_rn.")[1].split(".")[0])
            ck[k] = ck[k.replace(f".scratch.layer_rn.{i}.", f".scratch.layer{i + 1}_rn.")]
    ck["dec_blocks.0.attn.qkv.weight"] = torch.zeros(3)   # DUSt3R decoder weights are ignored
    path = str(tmp_path / "DUSt3R_ViTLarge_BaseDecoder_512_dpt.pth")
    torch.save({"model": ck}, path)
    before = {k: v.clone() for k, v in sd.items()}
    loaded, not_loaded = m.load_from_dust3r_checkpoint(path)
    after = m.state_dict()
    assert "dec_blocks.0.attn.qkv.weight" in not_loaded
    for k in after:
        if k.startswith("encoder."):
            assert torch.equal(after[k], ck[k[len("encoder."):]]), k
        elif k.startswith("downstream_head."):
            assert torch.equal(after[k], ck[k.replace("downstream_head.", "downstream_head1.", 1)]), k
        else:
            assert torch.equal(after[k], before[k]), k


def _portrait_model_views(M, g):
    from fast3r_b200 import tiny_args
    enc, dec, head = tiny_args()
    enc.update(g["enc_over"]); head.update(g["head_over"])
    model = M.Fast3R(enc, dec, head).eval()
    model.load_state_dict(synth_state_dict(g["shapes"], seed=g["weight_seed"]))
    imgs = synth_images(g["N"], g["B"], g["H"], g["W"])
    views = [dict(img=im, true_shape=torch.tensor([g["true_shapes"][i]] * g["B"], dtype=torch.int32), idx=i,
                  instance=str(i)) for i, im in enumerate(imgs)]
    return model, views


@pytest.mark.parametrize("precision,tol", [("bf16", 2e-2), ("fp32", 1e-3)])
def test_portrait_view_against_reference_fixture(emulated, golden_dir, precision, tol):
    """ManyAR_PatchEmbed + landscape_only heads with one portrait view (stored transposed): reference outputs."""
    g = torch.load(os.path.join(golden_dir, "tiny_portrait.pt"))
    model, views = _portrait_model_views(emulated, g)
    model.set_precision(precision)
    torch.manual_seed(g["rng_seed"])
    preds = model(views)
    for p, q in zip(preds, g["preds"]):
        for k in q:
            assert p[k].shape == q[k].shape
    for k in g["preds"][0]:
        e = rel_l2(torch.cat([p[k].flatten() for p in preds]), torch.cat([q[k].flatten() for q in g["preds"]]))
        assert e < tol, (k, e)


def test_portrait_needs_manyar_configuration(emulated, golden_dir):
    from fast3r_b200 import tiny_args
    g = torch.load(os.path.join(golden_dir, "tiny_portrait.pt"))
    model = emulated.Fast3R(*tiny_args()).eval()   # PatchEmbedDust3R / landscape_only=False (inference configuration)
    imgs = synth_images(2, 1, g["H"], g["W"])
    views = [dict(img=imgs[0], true_shape=torch.tensor([[g["H"], g["W"]]])),
             dict(img=imgs[1], true_shape=torch.tensor([[g["W"], g["H"]]]))]
    with pytest.raises(ValueError):
        model(views)
