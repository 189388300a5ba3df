"""One representative launch of every kernel family at bench sizes (for `ncu --set full`): LayerNorm, patch im2col,
bilinear upsample, the four decoder linears, DPT 3x3 convolutions (plain, residual + relu copy, fused final), ConvTranspose,
attention merge, and the parity-path kernels (split3, x3 GEMM, x3 attention)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fast3r_b200 import ops, lib as L  # noqa: E402

dev, bf, f32 = "cuda", torch.bfloat16, torch.float32
r = lambda *s, dt=bf, sc=0.05: (torch.randn(*s, device=dev) * sc).to(dt)  # noqa: E731
M, D = 23552, 1024
x = r(M, D, dt=f32, sc=1.0)
w1, b1 = r(D, dt=f32, sc=1.0), r(D, dt=f32, sc=1.0)
h = torch.empty(M, D, dtype=bf, device=dev)
ops.layernorm(x, w1, b1, 1e-5, h)                                            # layernorm_kernel<8>
img = r(32, 3, 368, 512, dt=f32, sc=1.0)
ops.im2col_patch(img, torch.empty(32 * 736, 768, dtype=bf, device=dev))      # im2col_patch_kernel
nv = 8
t = r(nv, 184, 256, 128)
ops.upsample2x(t, torch.empty(nv, 368, 512, 128, dtype=bf, device=dev), nv, 184, 256, 128, 368, 512)  # upsample2x_kernel
q, kvb = torch.empty(M, D, dtype=bf, device=dev), torch.empty(M, 2 * D, dtype=bf, device=dev)
ops.linear(h, r(3 * D, 1, D), r(3 * D, dt=f32), out0=q, ldo=D, split_col=D, out0b=kvb, ldo_b=2 * D)   # qkv
ops.linear(h, r(D, 1, D), r(D, dt=f32), out0=x, res0=x)                      # proj (fp32 reduce-add epilogue)
hid = torch.empty(M, 4 * D, dtype=bf, device=dev)
ops.linear(h, r(4 * D, 1, D), r(4 * D, dt=f32), out0=hid, act=L.ACT_GELU)    # fc1 + GELU
ops.linear(hid, r(D, 1, 4 * D), r(D, dt=f32), out0=x, res0=x)                # fc2
f = r(nv, 92, 128, 256)
o, o1 = torch.empty_like(f), torch.empty_like(f)
ops.gemm(f, r(256, 9, 256), w=128, h=92, nb=nv, taps=9, bias=r(256, dt=f32), out0=o, act=L.ACT_RELU)          # conv3x3 (TMA epi)
ops.gemm(f, r(256, 9, 256), w=128, h=92, nb=nv, taps=9, bias=r(256, dt=f32), out0=o, out1=o1, res0=f, res1=f)  # RCU conv2
up = r(nv, 368, 512, 128)
ops.gemm(up, r(128, 9, 128), w=512, h=368, nb=nv, taps=9, bias=r(128, dt=f32), epi=L.EPI_FINAL, w4=r(4, 128, dt=f32),
         b4=r(4, dt=f32), pts=torch.empty(nv, 368, 512, 3, device=dev), conf=torch.empty(nv, 368, 512, device=dev))  # final fused
a96 = r(nv, 23, 32, 96)
ops.gemm(a96, r(16 * 96, 1, 96), w=32, h=23, nb=nv, bias=r(96, dt=f32), out0=torch.empty(nv, 92, 128, 96, dtype=bf, device=dev),
         epi=L.EPI_CONVT, ct_k=4, ct_cout=96)                                # ConvTranspose k4s4
sq, skv = 2944, 23552
qq, kk = r(sq, D, sc=1.0), r(skv, 2 * D, sc=1.0)
ops.attention(qq, kk, torch.empty(sq, D, dtype=bf, device=dev), batch=1, heads=16, sq=sq, skv=skv, scale=0.16)  # sliced + merge
xf = r(2944, D, dt=f32, sc=1.0)
ops.gemm_x3(xf, r(D, 1, 3 * D), w=2944, bias=r(D, dt=f32), out0=torch.empty(2944, D, dtype=f32, device=dev))   # split3 + x3 GEMM
ops.attention_x3(r(2944, D, dt=f32, sc=1.0), r(2944, 2 * D, dt=f32, sc=1.0), torch.empty(2944, D, dtype=f32, device=dev),
                 batch=1, heads=16, sq=2944, skv=2944, scale=0.16)           # attn_split_kernel + attention_x3
torch.cuda.synchronize()
