"""Per-kernel numerics checks under their historical names: each entry runs cases of the per-element tables against
float64 (tests/test_gemm_plans_gpu.py, tests/test_attention_plans_gpu.py, tests/test_elementwise_plans_gpu.py).  Used
by tests/test_kernels_gpu.py (asserting) and by tools/gpu_check.py (report-everything mode for debugging on the GPU
box)."""


def check_gemm(names, x3=False):
    """The GEMM cases `names` of tests/gemm_plans.CASES, each checked per element against float64 and for its launch
    plan (tests/test_gemm_plans_gpu.run_case; it raises on a failure).  x3: from fp32 operands through the parity path's
    operand split."""
    from tests import gemm_plans as GP
    from tests.test_gemm_plans_gpu import run_case
    for name in names:
        i, case = next((i, c) for i, c in enumerate(GP.CASES) if c["name"] == name)
        assert GP.plan_key(case) == case["key"], (name, GP.plan_key(case), case["key"])
        run_case(case, seed=(4000 if x3 else 1000) + i, x3=x3)
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


def check_elementwise(names):
    """The element-wise cases `names` of tests/elementwise_plans.CASES, each checked per element against float64 in every
    variant (LayerNorm input regime, 16-bit type) of its key (tests/test_elementwise_plans_gpu.run_case; it raises on a
    failure)."""
    from tests import elementwise_plans as EP
    from tests.test_elementwise_plans_gpu import run_case, variants
    for name in names:
        i, case = next((i, c) for i, c in enumerate(EP.CASES) if c["name"] == name)
        assert EP.key(case) == case["key"], (name, EP.key(case), case["key"])
        for j, v in enumerate(variants(case)):
            run_case(case, v, seed=3000 + 8 * i + j)
    return 0.0, 0.0, {}


ALL = [
    ("x3_split3", check_elementwise, dict(names=["x3_split3"])),
    ("x3_linear", check_gemm, dict(names=["x3_linear"], x3=True)),
    ("x3_linear_gelu_tails", check_gemm, dict(names=["x3_linear_gelu_tails"], x3=True)),
    ("x3_conv3x3_c96_relu_res", check_gemm, dict(names=["x3_conv3x3_c96_relu_res"], x3=True)),
    ("x3_attn_tails", check_attention, dict(names=["x3_attn_tails"])),
    ("x3_attn_128", check_attention, dict(names=["x3_attn_128"])),
    ("x3_attn_peaky_long", check_attention, dict(names=["x3_attn_peaky_long"])),
    ("x3_upsample_f32", check_elementwise, dict(names=["x3_upsample_f32"])),
    ("x3_im2col_patch_f32", check_elementwise, dict(names=["x3_im2col_patch_f32"])),
    ("x3_add_f32", check_elementwise, dict(names=["x3_add_f32"])),
    ("cast", check_elementwise, dict(names=["cast"])),
    ("layernorm_1024", check_elementwise, dict(names=["layernorm_1024"])),
    ("layernorm_128", check_elementwise, dict(names=["layernorm_128"])),
    ("im2col_patch", check_elementwise, dict(names=["im2col_patch"])),
    ("im2col3x3s2", check_elementwise, dict(names=["im2col3x3s2"])),
    ("upsample_crop", check_elementwise, dict(names=["upsample_crop"])),
    ("upsample_full", check_elementwise, dict(names=["upsample_full"])),
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
