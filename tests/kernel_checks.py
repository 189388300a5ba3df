"""Per-kernel numerics checks: each CUDA op (through the C ABI) against a plain PyTorch fp32 reference of the
same op on the same bf16-rounded operands (the GEMM and attention cases: per element against float64,
tests/test_gemm_plans_gpu.py and tests/test_attention_plans_gpu.py).  Used by tests/test_kernels_gpu.py (asserting) and by
tools/gpu_check.py (report-everything mode for debugging on the GPU box)."""

import torch
import torch.nn.functional as F

from fast3r_b200 import lib as L
from fast3r_b200 import ops


def rel(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _rand(shape, seed, scale=1.0, dtype=torch.bfloat16):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype).cuda()


def check_gemm(names):
    """The GEMM cases `names` of tests/gemm_plans.CASES, each checked per element against float64 and for its launch
    plan (tests/test_gemm_plans_gpu.run_case; it raises on a failure)."""
    from tests import gemm_plans as GP
    from tests.test_gemm_plans_gpu import run_case
    for name in names:
        i, case = next((i, c) for i, c in enumerate(GP.CASES) if c["name"] == name)
        assert GP.plan_key(case) == case["key"], (name, GP.plan_key(case), case["key"])
        run_case(case, seed=1000 + i)
    return 0.0, 0.0, {}


def attention_ref(q, k, v, scale):
    a = (q.float() @ k.float().transpose(-2, -1)) * scale
    return a.softmax(-1) @ v.float()


def check_attention(names):
    """The attention cases `names` of tests/attention_plans.CASES, each checked per element against float64 in both input
    regimes (tests/test_attention_plans_gpu.run_case; it raises on a failure)."""
    from tests import attention_plans as AP
    from tests.test_attention_plans_gpu import run_case
    for name in names:
        i, case = next((i, c) for i, c in enumerate(AP.CASES) if c["name"] == name)
        assert AP.case_keys(case) == case["keys"], (name, AP.case_keys(case), case["keys"])
        for regime in ("flat", "grow"):
            run_case(case, regime, seed=2000 + 2 * i + (regime == "grow"))
    return 0.0, 0.0, {}


def check_layernorm(rows=1000, dim=1024, eps=1e-5, seed=100):
    x = _rand((rows, dim), seed, 2.0, torch.float32) + 0.5
    w, b = _rand((dim,), seed + 1, 1.0, torch.float32), _rand((dim,), seed + 2, 1.0, torch.float32)
    out = torch.zeros(rows, dim, dtype=torch.bfloat16, device="cuda")
    ops.layernorm(x, w, b, eps, out)
    ref = F.layer_norm(x, (dim,), w, b, eps)
    o32 = torch.zeros(rows, dim, dtype=torch.float32, device="cuda")
    ops.layernorm(x, w, b, eps, o32)
    return max(rel(out, ref), rel(o32, ref) * 1000), 4e-3, dict(f32=rel(o32, ref))


def check_im2col_patch(n=3, H=64, W=96, seed=110):
    img = _rand((n, 3, H, W), seed, 1.0, torch.float32)
    out = torch.zeros(n * (H // 16) * (W // 16), 768, dtype=torch.bfloat16, device="cuda")
    ops.im2col_patch(img, out)
    ref = F.unfold(img, kernel_size=16, stride=16).transpose(1, 2).reshape(-1, 768).to(torch.bfloat16)
    return float((out.float() - ref.float()).abs().max()), 1e-9, {}


def check_im2col3x3s2(n=2, H=5, W=6, C=64, seed=120):
    x = _rand((n, H, W, C), seed)
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    out = torch.zeros(n * Ho * Wo, 9 * C, dtype=torch.bfloat16, device="cuda")
    ops.im2col3x3s2(x, out, n, H, W, C, Ho, Wo)
    u = F.unfold(x.float().permute(0, 3, 1, 2), kernel_size=3, stride=2, padding=1)  # (n, C*9, L) c-major
    ref = u.reshape(n, C, 9, Ho * Wo).permute(0, 3, 2, 1).reshape(n * Ho * Wo, 9 * C)
    return float((out.float() - ref).abs().max()), 1e-9, {}


def check_upsample(n=2, H=12, W=16, C=64, crop=True, seed=130):
    x = _rand((n, H, W, C), seed)
    Ho, Wo = (2 * H - 1, 2 * W) if crop else (2 * H, 2 * W)
    out = torch.zeros(n, Ho, Wo, C, dtype=torch.bfloat16, device="cuda")
    ops.upsample2x(x, out, n, H, W, C, Ho, Wo)
    ref = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=True)
    ref = ref[:, :, :Ho, :Wo].permute(0, 2, 3, 1)
    return rel(out, ref), 4e-3, {}


def check_cast(n=4096 * 3, seed=140):
    x = _rand((n,), seed, 1.0, torch.float32)
    out = torch.zeros(n, dtype=torch.bfloat16, device="cuda")
    ops.cast_bf16(x, out)
    return float((out.float() - x.to(torch.bfloat16).float()).abs().max()), 1e-9, {}


# ---------------------------------------------------------------- parity path (hi/lo-split bf16 products, fp32 storage)
def _pack_x3(w):  # (N, taps, K) fp32 -> bf16 [Whi | Whi | Wlo]  (same packing as fast3r_b200.model._pk)
    hi = w.to(torch.bfloat16)
    lo = (w - hi.float()).to(torch.bfloat16)
    return torch.cat([hi, hi, lo], dim=-1).contiguous()


def check_split3(rows=300, k=200, seed=200):
    x = _rand((rows, k), seed, 3.0, torch.float32)
    out = torch.zeros(rows, 3 * k, dtype=torch.bfloat16, device="cuda")
    ops.split3(x, out, relu=True)
    v = F.relu(x)
    hi = v.to(torch.bfloat16)
    lo = (v - hi.float()).to(torch.bfloat16)
    ref = torch.cat([hi, lo, hi], -1)
    exact = float((out.float() - ref.float()).abs().max())
    recon = rel(out[:, :k].float() + out[:, k:2 * k].float(), v)
    return max(exact, recon / 1e-5 * 1e-9), 1e-9, dict(recon=recon)


def check_linear_x3(M=1000, K=1024, N=512, seed=210, act=L.ACT_NONE):
    a = _rand((M, K), seed, 1.0, torch.float32)
    w = _rand((N, 1, K), seed + 1, K ** -0.5, torch.float32)
    bias = _rand((N,), seed + 2, 1.0, torch.float32)
    out = torch.zeros(M, N, dtype=torch.float32, device="cuda")
    ops.gemm_x3(a, _pack_x3(w), w=M, bias=bias, out0=out, act=act)
    ref = (a.double() @ w[:, 0].double().T + bias.double())
    if act == L.ACT_GELU:
        ref = F.gelu(ref)
    return rel(out, ref), 3e-5, {}


def check_conv3x3_x3(nb=2, H=9, W=24, C=96, N=256, seed=220):
    x = _rand((nb, H, W, C), seed, 1.0, torch.float32)
    w = _rand((N, C, 3, 3), seed + 1, (9 * C) ** -0.5, torch.float32)
    bias = _rand((N,), seed + 2, 1.0, torch.float32)
    r0 = _rand((nb, H, W, N), seed + 3, 1.0, torch.float32)
    out = torch.zeros(nb, H, W, N, dtype=torch.float32, device="cuda")
    ops.gemm_x3(x, _pack_x3(w.permute(0, 2, 3, 1).reshape(N, 9, C)), a_relu=True, w=W, h=H, nb=nb, taps=9, bias=bias,
                out0=out, res0=r0)
    ref = F.conv2d(F.relu(x).double().permute(0, 3, 1, 2), w.double(), bias.double(), padding=1).permute(0, 2, 3, 1) + r0
    return rel(out, ref), 3e-5, {}


def check_upsample_f32(n=2, H=12, W=16, C=256, crop=True, seed=240):
    x = _rand((n, H, W, C), seed, 1.0, torch.float32)
    Ho, Wo = (2 * H - 1, 2 * W) if crop else (2 * H, 2 * W)
    out = torch.zeros(n, Ho, Wo, C, dtype=torch.float32, device="cuda")
    ops.upsample2x(x, out, n, H, W, C, Ho, Wo)
    ref = F.interpolate(x.permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=True)
    return rel(out, ref[:, :, :Ho, :Wo].permute(0, 2, 3, 1)), 2e-6, {}


def check_im2col_patch_f32(n=2, H=32, W=48, seed=250):
    img = _rand((n, 3, H, W), seed, 1.0, torch.float32)
    out = torch.zeros(n * (H // 16) * (W // 16), 768, dtype=torch.float32, device="cuda")
    ops.im2col_patch(img, out)
    ref = F.unfold(img, kernel_size=16, stride=16).transpose(1, 2).reshape(-1, 768)
    return float((out - ref).abs().max()), 1e-9, {}


def check_add_f32(n=4096 * 5, seed=260):
    a, b = _rand((n,), seed, 1.0, torch.float32), _rand((n,), seed + 1, 1.0, torch.float32)
    ref = a + b
    ops.add_f32(a, b)
    return float((a - ref).abs().max()), 1e-9, {}


ALL = [
    ("x3_split3", check_split3, {}),
    ("x3_linear", check_linear_x3, {}),
    ("x3_linear_gelu_tails", check_linear_x3, dict(M=333, K=256, N=96, act=L.ACT_GELU)),
    ("x3_conv3x3_c96_relu_res", check_conv3x3_x3, {}),
    ("x3_attn_tails", check_attention, dict(names=["x3_attn_tails"])),
    ("x3_attn_128", check_attention, dict(names=["x3_attn_128"])),
    ("x3_attn_peaky_long", check_attention, dict(names=["x3_attn_peaky_long"])),
    ("x3_upsample_f32", check_upsample_f32, {}),
    ("x3_im2col_patch_f32", check_im2col_patch_f32, {}),
    ("x3_add_f32", check_add_f32, {}),
    ("cast", check_cast, {}),
    ("layernorm_1024", check_layernorm, {}),
    ("layernorm_128", check_layernorm, dict(rows=77, dim=128, eps=1e-6)),
    ("im2col_patch", check_im2col_patch, {}),
    ("im2col3x3s2", check_im2col3x3s2, {}),
    ("upsample_crop", check_upsample, {}),
    ("upsample_full", check_upsample, dict(H=23, W=32, C=128, crop=False)),
    ("linear_small_tails", check_gemm, dict(names=["linear_small_tails"])),
    ("linear_qkv_shape", check_gemm, dict(names=["linear_qkv_shape"])),
    ("linear_bn256", check_gemm, dict(names=["linear_bn256"])),
    ("linear_resid_gelu", check_gemm, dict(names=["linear_resid_gelu", "linear_resid_gelu_out1"])),
    ("linear_resid_splitk", check_gemm, dict(names=["linear_resid_splitk", "linear_resid_splitk_out1"])),  # K slices
    ("linear_split", check_gemm, dict(names=["linear_split"])),
    ("rope_epilogue", check_gemm, dict(names=["rope_epilogue"])),
    ("idxemb_epilogue", check_gemm, dict(names=["idxemb_epilogue"])),
    ("conv1x1_tinymap", check_gemm, dict(names=["conv1x1_tinymap"])),
    ("conv3x3_w256", check_gemm, dict(names=["conv3x3_w256"])),
    ("conv3x3_w6_c96_res", check_gemm, dict(names=["conv3x3_w6_c96_res"])),
    ("conv3x3_w24_c192", check_gemm, dict(names=["conv3x3_w24_c192"])),
    ("conv3x3_w512", check_gemm, dict(names=["conv3x3_w512"])),
    ("convT_k4", check_gemm, dict(names=["convT_k4"])),
    ("convT_k2", check_gemm, dict(names=["convT_k2"])),
    ("final_fused", check_gemm, dict(names=["final_fused"])),
    ("attn_736_b2h2", check_attention, dict(names=["attn_736_b2h2"])),
    ("attn_128", check_attention, dict(names=["attn_128"])),
    ("attn_256x384", check_attention, dict(names=["attn_256x384"])),
    ("attn_tails_1000", check_attention, dict(names=["attn_tails_1000"])),
    ("attn_24", check_attention, dict(names=["attn_24"])),
    ("attn_long_3072", check_attention, dict(names=["attn_long_3072"])),
    ("attn_peaky", check_attention, dict(names=["attn_peaky"])),
    ("attn_q9tiles_oddpair", check_attention, dict(names=["attn_q9tiles_oddpair"])),
    ("attn_ranges_merge", check_attention, dict(names=["attn_ranges_merge"])),
    ("attn_ranges_merge_rank0", check_attention, dict(names=["attn_ranges_merge_rank0"])),
    ("attn_autosplit", check_attention, dict(names=["attn_autosplit"])),
    ("attn_skv235520_slices", check_attention, dict(names=["attn_skv235520_slices"])),
    # the bench regime: 23 552 keys (N=32 views) = 184 key blocks of lazy-rescale accumulation, flat and peaky scores
    ("attn_skv23552", check_attention, dict(names=["attn_skv23552"])),
    ("attn_skv23552_peaky", check_attention, dict(names=["attn_skv23552_peaky"])),
]
