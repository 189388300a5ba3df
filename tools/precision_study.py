"""Precision study (CPU, test infrastructure): which rounding points of the CUDA path have to go beyond bf16 for
the north star's 1e-3 rel-L2?  Runs the PRODUCT host code over tests/abi_emulator.py with selectable rounding:
  gemm:  'bf16' (operands rounded to bf16) | 'fp16' (rounded to fp16) | 'x3' (a = hi+lo split, 3 products) | 'fp32'
  attn:  'bf16' (q,k,v,p,o rounded)        | 'fp16' (rounded to fp16) | 'x3'                                 | 'fp32'
(the 'fp16' rows are the rounding points of precision="fp16") and prints rel-L2 vs the reference fixture (tiny) / the fp32 oracle (ViT-L width)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import fast3r_b200.model as M  # noqa: E402
from tests import abi_emulator as E  # noqa: E402
from tests.conftest import rel_l2  # noqa: E402
from tests.golden.synth import synth_state_dict, synth_images  # noqa: E402

BF = torch.bfloat16
ROUND = {"bf16": BF, "fp16": torch.float16}  # the 16-bit storage type of the 'bf16' / 'fp16' modes


def r16(t, dt=BF):
    return t.to(dt).float()


def split(t):
    hi = r16(t)
    return hi, r16(t - hi)


def run(model, imgs, seed, gemm_mode, attn_mode):
    M.ops = E
    M._require_cuda = lambda d: None
    M.BF16 = torch.float32  # fp32 storage everywhere; rounding is injected below
    orig_gemm, orig_att = E.gemm, E.attention

    def gemm(a, wt, **kw):
        if gemm_mode in ROUND:
            return orig_gemm(r16(a, ROUND[gemm_mode]), r16(wt, ROUND[gemm_mode]), **kw)
        if gemm_mode == "x3":  # emulate hi/lo: a*w ~ ah*wh + al*wh + ah*wl: drop al*wl
            ah, al = split(a.float())
            wh, wl = split(wt.float())
            # linear in (a, w): run three times with out accumulation is awkward; emulate by operand perturbation:
            # a*w - al*wl  ==  exact product minus the dropped term; dropped term is ~2^-18 relative -> use exact
            return orig_gemm(ah + al, wh + wl, **kw)
        return orig_gemm(a, wt, **kw)

    def attention(q, kv, out, *, batch, heads, sq, skv, scale, lse=None):
        D = heads * 64
        if attn_mode in ROUND:  # q, k, v, P and O rounded to the 16-bit type, fp32 softmax statistics
            dt = ROUND[attn_mode]
            qh = r16(q.reshape(batch, sq, heads, 64).transpose(1, 2).float(), dt)
            kh = r16(kv[:, :D].reshape(batch, skv, heads, 64).transpose(1, 2).float(), dt)
            vh = r16(kv[:, D:].reshape(batch, skv, heads, 64).transpose(1, 2).float(), dt)
            s = (qh @ kh.transpose(-2, -1)) * scale
            p = torch.exp(s - s.amax(-1, keepdim=True))
            o = (r16(p, dt) @ vh) / p.sum(-1, keepdim=True)
            out.copy_(r16(o.transpose(1, 2).reshape(batch * sq, D), dt).to(out.dtype))
            return
        qh = q.reshape(batch, sq, heads, 64).transpose(1, 2).float()
        kh = kv[:, :D].reshape(batch, skv, heads, 64).transpose(1, 2).float()
        vh = kv[:, D:].reshape(batch, skv, heads, 64).transpose(1, 2).float()
        if attn_mode in ("bf16", "pv3"):
            qh, kh = r16(qh), r16(kh)
        else:
            qh, kh = sum(split(qh)), sum(split(kh))
        if attn_mode in ("bf16", "qk3"):
            vh = r16(vh)
        else:
            vh = sum(split(vh))
        s = (qh @ kh.transpose(-2, -1)) * scale
        m = s.amax(-1, keepdim=True)
        p = torch.exp(s - m)
        l = p.sum(-1, keepdim=True)
        if attn_mode in ("bf16", "qk3"):
            p = r16(p)
        elif attn_mode in ("x3", "pv3"):
            p = sum(split(p))
        o = (p @ vh) / l
        o = o.transpose(1, 2).reshape(batch * sq, D)
        if attn_mode in ("bf16", "qk3", "qk3o"):
            o = r16(o)
        out.copy_(o.to(out.dtype))

    E.gemm, E.attention = gemm, attention
    E.linear = lambda a, wt, bias=None, **kw: gemm(a, wt, w=a.numel() // a.shape[-1], bias=bias, **kw)
    try:
        torch.manual_seed(seed)
        with torch.no_grad():
            return model([dict(img=im) for im in imgs])
    finally:
        E.gemm, E.attention = orig_gemm, orig_att


def main():
    from fast3r_b200 import tiny_args, vit_large_args
    which = sys.argv[1] if len(sys.argv) > 1 else "tiny"
    if which == "tiny":
        g = torch.load(os.path.join(os.path.dirname(__file__), "..", "tests", "golden", "tiny_b1_n3.pt"))
        model = M.Fast3R(*tiny_args()).eval()
        model.load_state_dict(synth_state_dict(g["shapes"], seed=g["weight_seed"]))
        imgs = synth_images(g["N"], g["B"], g["H"], g["W"])
        ref, seed = g["preds"], g["rng_seed"]
    else:
        from oracle import fast3r_oracle as O
        enc, dec, head = vit_large_args()
        model = M.Fast3R(enc, dec, head).eval()
        shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
        sd = synth_state_dict(shapes, seed=5)
        model.load_state_dict(sd)
        imgs = synth_images(2, 1, 96, 128)
        torch.manual_seed(7)
        ref, seed = O.forward(sd, enc, dec, head, imgs), 7
    for gm, am in (("bf16", "bf16"), ("fp16", "fp16"), ("x3", "bf16"), ("x3", "qk3"), ("x3", "pv3"), ("x3", "x3"), ("fp32", "fp32")):
        preds = run(model, imgs, seed, gm, am)
        rep = {k: rel_l2(torch.cat([p[k].flatten() for p in preds]), torch.cat([p[k].float().flatten() for p in ref]))
               for k in ref[0]}
        print(f"gemm={gm:5s} attn={am:5s}", {k: f"{v:.2e}" for k, v in rep.items()}, flush=True)


if __name__ == "__main__":
    main()
