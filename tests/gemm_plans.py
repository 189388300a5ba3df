"""Launch plans of f3r_gemm, for the tests: the library's own plan rule (fast3r_b200/csrc/gemm_plan.h, compiled for the
host by g++ through tests/gemm_plan_host.cpp), the plan key of a call, and the table of GPU cases that
tests/test_gemm_plans_gpu.py runs and tests/test_gemm_plans_cpu.py checks the forward against.

A call is described by a plain dict ("descriptor"): n, k, taps, w, h, nb, epi, act, out0 (None | "bf16" | "f32"), out1
(bool), res0 (None | "bf16" | "f32" | "f32_inplace", the last aliasing out0), res1 (bool) and split_col (0: none).

The plan key names the code that runs in gemm_kernel for a call: BLOCK_N, taps, the epilogue (generic / TMA store / TMA
fp32 reduce-add), the K split, the TMA-store box width sbx, the epilogue arguments, and the tails - a partial last N
tile, K not a multiple of 64, a partial M tile (pixels outside the image), and more work items than SMs (CTAs that loop
over several tiles carry the smem-ring phase from one tile to the next)."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

from fast3r_b200 import lib as L

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "fast3r_b200", "csrc")
H100_SMS = 132  # the table's keys are those of an H100 SXM (132 SMs)

EPI_NAMES = {L.EPI_STORE: "STORE", L.EPI_ROPE: "ROPE", L.EPI_IDXEMB: "IDXEMB", L.EPI_CONVT: "CONVT",
             L.EPI_FINAL: "FINAL"}
ACT_NAMES = {L.ACT_NONE: "NONE", L.ACT_RELU: "RELU", L.ACT_GELU: "GELU"}
PLAN_FIELDS = ("bw", "bh", "bw_log2", "sbx_log2", "tiles_x", "tiles_y", "num_m_tiles", "block_n", "num_n_tiles",
          "tma_epi", "k_split")

_host = None


def host_lib():
    """gemm_plan.h compiled for the host (once per process, into a temporary directory)."""
    global _host
    if _host is None:
        if shutil.which("g++") is None:
            raise RuntimeError("g++ is needed to compile fast3r_b200/csrc/gemm_plan.h for the host")
        so = os.path.join(tempfile.mkdtemp(prefix="f3r_gemm_plan_"), "libgemm_plan_host.so")
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-I", CSRC,
          os.path.join(HERE, "gemm_plan_host.cpp"), "-o", so])
        lib = C.CDLL(so)
        lib.f3r_test_gemm_plan.argtypes = [C.POINTER(L.GemmDesc), C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]
        lib.f3r_test_gemm_plan.restype = None
        lib.f3r_test_gemm_desc_size.restype = C.c_ulong
        assert lib.f3r_test_gemm_desc_size() == C.sizeof(L.GemmDesc)
        _host = lib
    return _host


def _cdesc(d):
    """A GemmDesc with the descriptor's fields; the pointers only say which operands are present (and which alias)."""
    c = L.GemmDesc()
    c.a, c.wt = 0x1000, 0x2000
    for f in ("n", "k", "taps", "w", "h", "nb", "epi", "act", "split_col"):
        setattr(c, f, int(d.get(f, 0)))
    c.a_ld = c.k
    c.out0_f32 = int(d.get("out0") == "f32")
    res0 = d.get("res0")
    c.res0_f32 = int(res0 in ("f32", "f32_inplace"))
    c.out0 = 0x3000 if d.get("out0") else None
    c.res0 = (0x3000 if res0 == "f32_inplace" else 0x4000) if res0 else None
    c.out1 = 0x5000 if d.get("out1") else None
    c.res1 = 0x6000 if d.get("res1") else None
    return c


def plan(d, num_sms=H100_SMS, allow_tma_epi=True, allow_k_split=True):
    """The launch plan f3r_gemm chooses for descriptor d on a device with num_sms SMs, as a dict of PLAN_FIELDS."""
    out = (C.c_int * len(PLAN_FIELDS))()
    host_lib().f3r_test_gemm_plan(C.byref(_cdesc(d)), int(num_sms), int(allow_tma_epi), int(allow_k_split), out)
    return dict(zip(PLAN_FIELDS, out))


def plan_key(d, num_sms=H100_SMS):
    """Canonical string of the plan key of descriptor d."""
    p = plan(d, num_sms)
    items = p["num_m_tiles"] * p["num_n_tiles"] * p["k_split"]
    s = (f"bn{p['block_n']} taps{d['taps']} tma{p['tma_epi']} ks{p['k_split']} sbx{1 << p['sbx_log2']} "
         f"{EPI_NAMES[d['epi']]} {ACT_NAMES[d['act']]} out0:{d.get('out0') or '-'} res0:{d.get('res0') or '-'}")
    flags = [("out1", bool(d.get("out1"))), ("res1", bool(d.get("res1"))), ("split", bool(d.get("split_col"))),
          ("ntail", d["n"] % p["block_n"] != 0), ("ktail", d["k"] % 64 != 0),
          ("mtail", d["w"] % p["bw"] != 0 or d["h"] % p["bh"] != 0), ("multi", items > num_sms)]
    return s + "".join(" " + f for f, on in flags if on)


# ------------------------------------------------------------------------------------------------------ the case table
# One case per plan key of the forward (reduced to the fewest views / rows that reach the same key), then a contract
# matrix beyond the forward.  Fields besides the descriptor: ldo / ldo_b (row strides, default n / n - split_col),
# bias (default True), tok_per_img, grid_w, rope_cols (ROPE / IDXEMB), ct_k, ct_cout (CONVT), and "key": the plan
# key the case must reach on an H100 SXM.  x3 (True: the parity forward reaches the key with K = 3 k0) makes
# tests/test_gemm_plans_gpu.py also run the case from fp32 operands through ops.gemm_x3 (a_relu: with relu(A)).
S, R, I, T, F = L.EPI_STORE, L.EPI_ROPE, L.EPI_IDXEMB, L.EPI_CONVT, L.EPI_FINAL
NONE, RELU, GELU = L.ACT_NONE, L.ACT_RELU, L.ACT_GELU


def _case(name, key, **f):
    c = dict(name=name, key=key, n=None, k=None, w=None, taps=1, h=1, nb=1, epi=S, act=NONE, out0=None, out1=False, res0=None, res1=False,
          split_col=0, bias=True, ldo=None, ldo_b=0, tok_per_img=0, grid_w=0, rope_cols=0, ct_k=0, ct_cout=0, x3=False,
          a_relu=False)
    unknown = set(f) - set(c)
    assert not unknown, unknown
    c.update(f)
    return c


# ---- one case per plan key of the forward: ViT-L at 512x368 (N=32 in bf16 and fp32, N=4, one portrait view) and the
# fusion decoder of N=32 sharded over 2, 4 and 8 ranks (tests/test_gemm_plans_cpu.py records them)
FORWARD = [
    # forward bf16 N=32 368x512
    _case("fwd00", "bn256 taps1 tma1 ks1 sbx32 STORE NONE out0:f32 res0:- multi",
          n=1024, k=768, w=4352, out0="f32", x3=True),
    # forward bf16 N=32 368x512
    _case("fwd01", "bn256 taps1 tma1 ks1 sbx32 ROPE NONE out0:bf16 res0:- split multi",
          n=3072, k=1024, w=1536, epi=R, out0="bf16", split_col=1024, ldo=1024, ldo_b=2048,
          tok_per_img=736, grid_w=32, rope_cols=2048),
    # forward bf16 N=32 368x512
    _case("fwd02", "bn256 taps1 tma2 ks1 sbx32 STORE NONE out0:f32 res0:f32_inplace multi",
          n=1024, k=1024, w=4352, out0="f32", res0="f32_inplace"),
    # forward bf16 N=32 368x512
    _case("fwd03", "bn256 taps1 tma1 ks1 sbx32 STORE GELU out0:bf16 res0:- multi",
          n=4096, k=1024, w=1152, act=GELU, out0="bf16"),
    # forward bf16 N=32 368x512
    _case("fwd04", "bn256 taps1 tma1 ks1 sbx32 IDXEMB NONE out0:f32 res0:- multi",
          n=1024, k=1024, w=4352, epi=I, out0="f32", tok_per_img=736),
    # forward bf16 N=32 368x512
    _case("fwd05", "bn256 taps1 tma1 ks1 sbx32 STORE NONE out0:bf16 res0:- split multi",
          n=3072, k=1024, w=1536, out0="bf16", split_col=1024, ldo=1024, ldo_b=2048),
    # forward bf16 N=32 368x512
    _case("fwd06", "bn128 taps1 tma1 ks1 sbx32 STORE NONE out0:bf16 res0:- ntail mtail multi",
          n=96, k=1024, w=32, h=23, nb=23, out0="bf16"),
    # forward bf16 N=32 368x512
    _case("fwd07", "bn256 taps1 tma0 ks1 sbx32 CONVT NONE out0:bf16 res0:- ktail mtail multi",
          n=1536, k=96, w=32, h=23, nb=4, epi=T, out0="bf16", ct_k=4, ct_cout=96),
    # forward bf16 N=32 368x512
    _case("fwd08", "bn256 taps1 tma1 ks1 sbx32 STORE NONE out0:bf16 res0:- ntail mtail multi",
          n=192, k=1024, w=32, h=23, nb=23, out0="bf16"),
    # forward bf16 N=32 368x512
    _case("fwd09", "bn256 taps1 tma0 ks1 sbx32 CONVT NONE out0:bf16 res0:- mtail multi",
          n=768, k=192, w=32, h=23, nb=8, epi=T, out0="bf16", ct_k=2, ct_cout=192),
    # forward bf16 N=32 368x512
    _case("fwd10", "bn256 taps1 tma1 ks1 sbx32 STORE NONE out0:bf16 res0:- mtail multi",
          n=768, k=1024, w=32, h=23, nb=8, out0="bf16"),
    # forward bf16 N=32 368x512
    _case("fwd11", "bn128 taps1 tma1 ks1 sbx32 STORE NONE out0:bf16 res0:- mtail multi",
          n=768, k=6912, w=2880, out0="bf16"),
    # forward bf16 N=32 368x512
    _case("fwd12", "bn256 taps9 tma0 ks1 sbx32 STORE NONE out0:bf16 res0:- out1 ktail multi",
          n=256, k=96, taps=9, w=128, h=92, nb=2, out0="bf16", out1=True, bias=False),
    # forward bf16 N=32 368x512
    _case("fwd13", "bn256 taps9 tma0 ks1 sbx32 STORE NONE out0:bf16 res0:- out1 multi",
          n=256, k=192, taps=9, w=64, h=46, nb=6, out0="bf16", out1=True, bias=False),
    # forward bf16 N=32 368x512
    _case("fwd14", "bn256 taps9 tma0 ks1 sbx32 STORE NONE out0:bf16 res0:- out1 mtail multi",
          n=256, k=384, taps=9, w=32, h=23, nb=23, out0="bf16", out1=True, bias=False),
    # forward bf16 N=32 368x512
    _case("fwd15", "bn128 taps9 tma0 ks1 sbx16 STORE NONE out0:bf16 res0:- out1 mtail",
          n=256, k=768, taps=9, w=16, h=12, out0="bf16", out1=True, bias=False),
    # forward bf16 N=32 368x512
    _case("fwd16", "bn128 taps9 tma1 ks1 sbx16 STORE RELU out0:bf16 res0:- mtail",
          n=256, k=256, taps=9, w=16, h=12, act=RELU, out0="bf16"),
    # forward bf16 N=32 368x512
    _case("fwd17", "bn128 taps9 tma0 ks1 sbx16 STORE NONE out0:bf16 res0:bf16 mtail",
          n=256, k=256, taps=9, w=16, h=12, out0="bf16", res0="bf16"),
    # forward bf16 N=32 368x512
    _case("fwd18", "bn128 taps1 tma1 ks1 sbx16 STORE NONE out0:bf16 res0:- mtail",
          n=256, k=256, w=16, h=12, out0="bf16"),
    # forward bf16 N=32 368x512
    _case("fwd19", "bn256 taps9 tma1 ks1 sbx32 STORE RELU out0:bf16 res0:- mtail multi",
          n=256, k=256, taps=9, w=32, h=23, nb=23, act=RELU, out0="bf16"),
    # forward bf16 N=32 368x512
    _case("fwd20", "bn256 taps9 tma0 ks1 sbx32 STORE NONE out0:bf16 res0:bf16 out1 res1 mtail multi",
          n=256, k=256, taps=9, w=32, h=23, nb=23, out0="bf16", out1=True, res0="bf16", res1=True),
    # forward bf16 N=32 368x512
    _case("fwd21", "bn256 taps9 tma0 ks1 sbx32 STORE NONE out0:bf16 res0:bf16 mtail multi",
          n=256, k=256, taps=9, w=32, h=23, nb=23, out0="bf16", res0="bf16"),
    # forward bf16 N=32 368x512
    _case("fwd22", "bn256 taps9 tma1 ks1 sbx32 STORE RELU out0:bf16 res0:- multi",
          n=256, k=256, taps=9, w=64, h=46, nb=6, act=RELU, out0="bf16"),
    # forward bf16 N=32 368x512
    _case("fwd23", "bn256 taps9 tma0 ks1 sbx32 STORE NONE out0:bf16 res0:bf16 out1 res1 multi",
          n=256, k=256, taps=9, w=64, h=46, nb=6, out0="bf16", out1=True, res0="bf16", res1=True),
    # forward bf16 N=32 368x512
    _case("fwd24", "bn256 taps9 tma0 ks1 sbx32 STORE NONE out0:bf16 res0:bf16 multi",
          n=256, k=256, taps=9, w=64, h=46, nb=6, out0="bf16", res0="bf16"),
    # forward bf16 N=32 368x512
    _case("fwd25", "bn256 taps1 tma1 ks1 sbx32 STORE NONE out0:bf16 res0:- multi",
          n=256, k=256, w=64, h=46, nb=6, out0="bf16"),
    # forward bf16 N=32 368x512
    _case("fwd26", "bn128 taps9 tma1 ks1 sbx32 STORE NONE out0:bf16 res0:- multi",
          n=128, k=256, taps=9, w=256, h=184, out0="bf16"),
    # forward bf16 N=32 368x512
    _case("fwd27", "bn128 taps9 tma0 ks1 sbx32 FINAL NONE out0:- res0:- multi",
          n=128, k=128, taps=9, w=512, h=34, epi=F),
    # forward bf16 N=32 368x512
    _case("fwd28", "bn128 taps1 tma1 ks1 sbx32 STORE NONE out0:bf16 res0:- ntail mtail",
          n=96, k=1024, w=32, h=23, out0="bf16"),
    # forward bf16 N=32 368x512
    _case("fwd29", "bn128 taps1 tma0 ks1 sbx32 CONVT NONE out0:bf16 res0:- mtail multi",
          n=768, k=192, w=32, h=23, nb=4, epi=T, out0="bf16", ct_k=2, ct_cout=192),
    # forward bf16 N=32 368x512
    _case("fwd30", "bn128 taps1 tma1 ks1 sbx32 STORE NONE out0:bf16 res0:- mtail",
          n=384, k=1024, w=32, h=23, out0="bf16"),
    # forward bf16 N=32 368x512
    _case("fwd31", "bn128 taps9 tma0 ks1 sbx32 STORE NONE out0:bf16 res0:- out1 mtail",
          n=256, k=384, taps=9, w=32, h=23, out0="bf16", out1=True, bias=False),
    # forward bf16 N=32 368x512
    _case("fwd32", "bn128 taps9 tma1 ks1 sbx32 STORE RELU out0:bf16 res0:- mtail",
          n=256, k=256, taps=9, w=32, h=23, act=RELU, out0="bf16"),
    # forward bf16 N=32 368x512
    _case("fwd33", "bn128 taps9 tma0 ks1 sbx32 STORE NONE out0:bf16 res0:bf16 out1 res1 mtail",
          n=256, k=256, taps=9, w=32, h=23, out0="bf16", out1=True, res0="bf16", res1=True),
    # forward bf16 N=32 368x512
    _case("fwd34", "bn128 taps9 tma0 ks1 sbx32 STORE NONE out0:bf16 res0:bf16 mtail",
          n=256, k=256, taps=9, w=32, h=23, out0="bf16", res0="bf16"),
    # decoder bf16 N=32 rank 0/4 (8 views)
    _case("fwd35", "bn256 taps1 tma2 ks2 sbx32 STORE NONE out0:f32 res0:f32_inplace multi",
          n=1024, k=4096, w=5760, out0="f32", res0="f32_inplace"),
    # decoder bf16 N=32 rank 0/8 (4 views)
    _case("fwd36", "bn128 taps1 tma1 ks1 sbx32 IDXEMB NONE out0:f32 res0:- multi",
          n=1024, k=1024, w=2176, epi=I, out0="f32", tok_per_img=736),
    # decoder bf16 N=32 rank 0/8 (4 views)
    _case("fwd37", "bn128 taps1 tma2 ks1 sbx32 STORE NONE out0:f32 res0:f32_inplace multi",
          n=1024, k=1024, w=2176, out0="f32", res0="f32_inplace"),
    # decoder bf16 N=32 rank 0/8 (4 views)
    _case("fwd38", "bn128 taps1 tma2 ks2 sbx32 STORE NONE out0:f32 res0:f32_inplace multi",
          n=1024, k=4096, w=2944, out0="f32", res0="f32_inplace"),
    # forward fp32 N=32 368x512
    _case("fwd39", "bn256 taps1 tma1 ks1 sbx32 ROPE NONE out0:f32 res0:- split multi",
          n=3072, k=3072, w=1536, epi=R, out0="f32", split_col=1024, ldo=1024, ldo_b=2048,
          tok_per_img=736, grid_w=32, rope_cols=2048, x3=True),
    # forward fp32 N=32 368x512
    _case("fwd40", "bn256 taps1 tma1 ks1 sbx32 STORE GELU out0:f32 res0:- multi",
          n=4096, k=3072, w=1152, act=GELU, out0="f32", x3=True),
    # forward fp32 N=32 368x512
    _case("fwd41", "bn256 taps1 tma1 ks1 sbx32 STORE NONE out0:f32 res0:- split multi",
          n=3072, k=3072, w=1536, out0="f32", split_col=1024, ldo=1024, ldo_b=2048, x3=True),
    # forward fp32 N=32 368x512
    _case("fwd42", "bn128 taps1 tma1 ks1 sbx32 STORE NONE out0:f32 res0:- ntail mtail",
          n=96, k=3072, w=32, h=23, out0="f32", x3=True),
    # forward fp32 N=32 368x512
    _case("fwd43", "bn256 taps1 tma0 ks1 sbx32 CONVT NONE out0:f32 res0:- ktail mtail multi",
          n=1536, k=288, w=32, h=23, nb=4, epi=T, out0="f32", ct_k=4, ct_cout=96, x3=True),
    # forward fp32 N=32 368x512
    _case("fwd44", "bn256 taps1 tma0 ks1 sbx32 CONVT NONE out0:f32 res0:- mtail multi",
          n=768, k=576, w=32, h=23, nb=8, epi=T, out0="f32", ct_k=2, ct_cout=192, x3=True),
    # forward fp32 N=32 368x512
    _case("fwd45", "bn128 taps1 tma1 ks1 sbx32 STORE NONE out0:f32 res0:- mtail multi",
          n=384, k=3072, w=32, h=23, nb=8, out0="f32", x3=True),
    # forward fp32 N=32 368x512
    _case("fwd46", "bn256 taps1 tma1 ks1 sbx32 STORE NONE out0:f32 res0:- mtail multi",
          n=768, k=3072, w=32, h=23, nb=8, out0="f32", x3=True),
    # forward fp32 N=32 368x512
    _case("fwd47", "bn128 taps1 tma1 ks1 sbx32 STORE NONE out0:f32 res0:-",
          n=768, k=20736, w=128, out0="f32", x3=True),
    # forward fp32 N=32 368x512
    _case("fwd48", "bn256 taps9 tma1 ks1 sbx32 STORE NONE out0:f32 res0:- ktail multi",
          n=256, k=288, taps=9, w=128, h=92, nb=2, out0="f32", bias=False, x3=True),
    # forward fp32 N=32 368x512
    _case("fwd49", "bn256 taps9 tma1 ks1 sbx32 STORE NONE out0:f32 res0:- multi",
          n=256, k=576, taps=9, w=64, h=46, nb=6, out0="f32", bias=False, x3=True),
    # forward fp32 N=32 368x512
    _case("fwd50", "bn128 taps9 tma1 ks1 sbx32 STORE NONE out0:f32 res0:- mtail",
          n=256, k=1152, taps=9, w=32, h=23, out0="f32", bias=False, x3=True),
    # forward fp32 N=32 368x512
    _case("fwd51", "bn128 taps9 tma1 ks1 sbx16 STORE NONE out0:f32 res0:- mtail",
          n=256, k=2304, taps=9, w=16, h=12, out0="f32", bias=False, x3=True),
    # forward fp32 N=32 368x512
    _case("fwd52", "bn128 taps9 tma1 ks1 sbx16 STORE RELU out0:f32 res0:- mtail",
          n=256, k=768, taps=9, w=16, h=12, act=RELU, out0="f32", x3=True, a_relu=True),
    # forward fp32 N=32 368x512
    _case("fwd53", "bn128 taps9 tma0 ks1 sbx16 STORE NONE out0:f32 res0:f32 mtail",
          n=256, k=768, taps=9, w=16, h=12, out0="f32", res0="f32", x3=True),
    # forward fp32 N=32 368x512
    _case("fwd54", "bn128 taps1 tma1 ks1 sbx16 STORE NONE out0:f32 res0:- mtail",
          n=256, k=768, w=16, h=12, out0="f32", x3=True),
    # forward fp32 N=32 368x512
    _case("fwd55", "bn128 taps9 tma1 ks1 sbx32 STORE RELU out0:f32 res0:- mtail",
          n=256, k=768, taps=9, w=32, h=23, act=RELU, out0="f32", x3=True, a_relu=True),
    # forward fp32 N=32 368x512
    _case("fwd56", "bn128 taps9 tma0 ks1 sbx32 STORE NONE out0:f32 res0:f32 mtail",
          n=256, k=768, taps=9, w=32, h=23, out0="f32", res0="f32", x3=True),
    # forward fp32 N=32 368x512
    _case("fwd57", "bn128 taps1 tma1 ks1 sbx32 STORE NONE out0:f32 res0:- mtail",
          n=256, k=768, w=32, h=23, out0="f32", x3=True),
    # forward fp32 N=32 368x512
    _case("fwd58", "bn256 taps9 tma1 ks1 sbx32 STORE RELU out0:f32 res0:- multi",
          n=256, k=768, taps=9, w=64, h=46, nb=6, act=RELU, out0="f32", x3=True, a_relu=True),
    # forward fp32 N=32 368x512
    _case("fwd59", "bn256 taps9 tma0 ks1 sbx32 STORE NONE out0:f32 res0:f32 multi",
          n=256, k=768, taps=9, w=64, h=46, nb=6, out0="f32", res0="f32", x3=True),
    # forward fp32 N=32 368x512
    _case("fwd60", "bn128 taps9 tma1 ks1 sbx32 STORE NONE out0:f32 res0:- multi",
          n=128, k=768, taps=9, w=256, h=184, out0="f32", x3=True),
    # forward bf16 N=4 368x512
    _case("fwd61", "bn128 taps1 tma1 ks1 sbx32 STORE NONE out0:f32 res0:- multi",
          n=1024, k=768, w=2176, out0="f32"),
    # forward bf16 N=4 368x512
    _case("fwd62", "bn128 taps1 tma1 ks1 sbx32 STORE NONE out0:bf16 res0:-",
          n=768, k=6912, w=128, out0="bf16"),
    # forward bf16 N=4 368x512
    _case("fwd63", "bn128 taps9 tma0 ks1 sbx32 STORE NONE out0:bf16 res0:- out1 multi",
          n=256, k=192, taps=9, w=64, h=46, nb=3, out0="bf16", out1=True, bias=False),
    # forward bf16 N=4 368x512
    _case("fwd64", "bn128 taps9 tma1 ks1 sbx32 STORE RELU out0:bf16 res0:- multi",
          n=256, k=256, taps=9, w=64, h=46, nb=3, act=RELU, out0="bf16"),
    # forward bf16 N=4 368x512
    _case("fwd65", "bn128 taps9 tma0 ks1 sbx32 STORE NONE out0:bf16 res0:bf16 out1 res1 multi",
          n=256, k=256, taps=9, w=64, h=46, nb=3, out0="bf16", out1=True, res0="bf16", res1=True),
    # forward bf16 N=4 368x512
    _case("fwd66", "bn128 taps9 tma0 ks1 sbx32 STORE NONE out0:bf16 res0:bf16 multi",
          n=256, k=256, taps=9, w=64, h=46, nb=3, out0="bf16", res0="bf16"),
    # forward bf16 N=4 368x512
    _case("fwd67", "bn128 taps1 tma1 ks1 sbx32 STORE NONE out0:bf16 res0:- multi",
          n=256, k=256, w=64, h=46, nb=3, out0="bf16"),
    # forward bf16 N=1 512x368
    _case("fwd68", "bn128 taps1 tma1 ks1 sbx32 ROPE NONE out0:bf16 res0:- split mtail multi",
          n=3072, k=1024, w=736, epi=R, out0="bf16", split_col=1024, ldo=1024, ldo_b=2048,
          tok_per_img=736, grid_w=23, rope_cols=2048),
    # forward bf16 N=1 512x368
    _case("fwd69", "bn128 taps1 tma2 ks1 sbx32 STORE NONE out0:f32 res0:f32_inplace mtail",
          n=1024, k=1024, w=96, out0="f32", res0="f32_inplace"),
    # forward bf16 N=1 512x368
    _case("fwd70", "bn128 taps1 tma1 ks1 sbx32 STORE GELU out0:bf16 res0:- mtail multi",
          n=4096, k=1024, w=608, act=GELU, out0="bf16"),
    # forward bf16 N=1 512x368
    _case("fwd71", "bn128 taps1 tma2 ks2 sbx32 STORE NONE out0:f32 res0:f32_inplace mtail",
          n=1024, k=4096, w=736, out0="f32", res0="f32_inplace"),
    # forward bf16 N=1 512x368
    _case("fwd72", "bn128 taps1 tma1 ks1 sbx32 IDXEMB NONE out0:f32 res0:- mtail",
          n=1024, k=1024, w=96, epi=I, out0="f32", tok_per_img=736),
    # forward bf16 N=1 512x368
    _case("fwd73", "bn128 taps1 tma1 ks1 sbx32 STORE NONE out0:bf16 res0:- split mtail multi",
          n=3072, k=1024, w=736, out0="bf16", split_col=1024, ldo=1024, ldo_b=2048),
    # forward bf16 N=1 512x368
    _case("fwd74", "bn128 taps1 tma1 ks1 sbx8 STORE NONE out0:bf16 res0:- ntail mtail",
          n=96, k=1024, w=23, h=32, out0="bf16"),
    # forward bf16 N=1 512x368
    _case("fwd75", "bn128 taps1 tma0 ks1 sbx8 CONVT NONE out0:bf16 res0:- ktail mtail",
          n=1536, k=96, w=23, h=32, epi=T, out0="bf16", ct_k=4, ct_cout=96),
    # forward bf16 N=1 512x368
    _case("fwd76", "bn128 taps1 tma0 ks1 sbx8 CONVT NONE out0:bf16 res0:- mtail",
          n=768, k=192, w=23, h=32, epi=T, out0="bf16", ct_k=2, ct_cout=192),
    # forward bf16 N=1 512x368
    _case("fwd77", "bn128 taps1 tma1 ks1 sbx8 STORE NONE out0:bf16 res0:- mtail",
          n=384, k=1024, w=23, h=32, out0="bf16"),
    # forward bf16 N=1 512x368
    _case("fwd78", "bn128 taps9 tma0 ks1 sbx4 STORE NONE out0:bf16 res0:- out1 ktail multi",
          n=256, k=96, taps=9, w=92, h=128, out0="bf16", out1=True, bias=False),
    # forward bf16 N=1 512x368
    _case("fwd79", "bn128 taps9 tma0 ks1 sbx2 STORE NONE out0:bf16 res0:- out1",
          n=256, k=192, taps=9, w=46, h=64, out0="bf16", out1=True, bias=False),
    # forward bf16 N=1 512x368
    _case("fwd80", "bn128 taps9 tma0 ks1 sbx8 STORE NONE out0:bf16 res0:- out1 mtail",
          n=256, k=384, taps=9, w=23, h=32, out0="bf16", out1=True, bias=False),
    # forward bf16 N=1 512x368
    _case("fwd81", "bn128 taps9 tma1 ks1 sbx8 STORE RELU out0:bf16 res0:- mtail",
          n=256, k=256, taps=9, w=23, h=32, act=RELU, out0="bf16"),
    # forward bf16 N=1 512x368
    _case("fwd82", "bn128 taps9 tma0 ks1 sbx8 STORE NONE out0:bf16 res0:bf16 out1 res1 mtail",
          n=256, k=256, taps=9, w=23, h=32, out0="bf16", out1=True, res0="bf16", res1=True),
    # forward bf16 N=1 512x368
    _case("fwd83", "bn128 taps9 tma0 ks1 sbx8 STORE NONE out0:bf16 res0:bf16 mtail",
          n=256, k=256, taps=9, w=23, h=32, out0="bf16", res0="bf16"),
    # forward bf16 N=1 512x368
    _case("fwd84", "bn128 taps9 tma1 ks1 sbx2 STORE RELU out0:bf16 res0:-",
          n=256, k=256, taps=9, w=46, h=64, act=RELU, out0="bf16"),
    # forward bf16 N=1 512x368
    _case("fwd85", "bn128 taps9 tma0 ks1 sbx2 STORE NONE out0:bf16 res0:bf16 out1 res1",
          n=256, k=256, taps=9, w=46, h=64, out0="bf16", out1=True, res0="bf16", res1=True),
    # forward bf16 N=1 512x368
    _case("fwd86", "bn128 taps9 tma0 ks1 sbx2 STORE NONE out0:bf16 res0:bf16",
          n=256, k=256, taps=9, w=46, h=64, out0="bf16", res0="bf16"),
    # forward bf16 N=1 512x368
    _case("fwd87", "bn128 taps1 tma1 ks1 sbx2 STORE NONE out0:bf16 res0:-",
          n=256, k=256, w=46, h=64, out0="bf16"),
    # forward bf16 N=1 512x368
    _case("fwd88", "bn128 taps9 tma1 ks1 sbx4 STORE RELU out0:bf16 res0:- multi",
          n=256, k=256, taps=9, w=92, h=128, act=RELU, out0="bf16"),
    # forward bf16 N=1 512x368
    _case("fwd89", "bn128 taps9 tma0 ks1 sbx4 STORE NONE out0:bf16 res0:bf16 out1 res1 multi",
          n=256, k=256, taps=9, w=92, h=128, out0="bf16", out1=True, res0="bf16", res1=True),
    # forward bf16 N=1 512x368
    _case("fwd90", "bn128 taps9 tma0 ks1 sbx4 STORE NONE out0:bf16 res0:bf16 multi",
          n=256, k=256, taps=9, w=92, h=128, out0="bf16", res0="bf16"),
    # forward bf16 N=1 512x368
    _case("fwd91", "bn128 taps1 tma1 ks1 sbx4 STORE NONE out0:bf16 res0:- multi",
          n=256, k=256, w=92, h=128, out0="bf16"),
    # forward bf16 N=1 512x368
    _case("fwd92", "bn128 taps9 tma1 ks1 sbx8 STORE NONE out0:bf16 res0:- multi",
          n=128, k=256, taps=9, w=184, h=256, out0="bf16"),
    # forward bf16 N=1 512x368
    _case("fwd93", "bn128 taps9 tma0 ks1 sbx16 FINAL NONE out0:- res0:- multi",
          n=128, k=128, taps=9, w=368, h=48, epi=F),    # forward fp32 N=32 368x512 and its decoder sharded over 4 and 8 ranks: the parity path's K = 3 k of the plans above
    # whose bf16 cases have k not divisible by 3
    _case("fwd94", "bn256 taps1 tma1 ks1 sbx32 IDXEMB NONE out0:f32 res0:- multi",
          n=1024, k=3072, w=4352, epi=I, out0="f32", tok_per_img=736, x3=True),
    _case("fwd95", "bn256 taps1 tma2 ks1 sbx32 STORE NONE out0:f32 res0:f32_inplace multi",
          n=1024, k=3072, w=8192, out0="f32", res0="f32_inplace", x3=True),
    _case("fwd96", "bn256 taps1 tma2 ks2 sbx32 STORE NONE out0:f32 res0:f32_inplace multi",
          n=1024, k=3072, w=5888, out0="f32", res0="f32_inplace", x3=True),
    _case("fwd97", "bn128 taps1 tma1 ks1 sbx32 IDXEMB NONE out0:f32 res0:- multi",
          n=1024, k=3072, w=2176, epi=I, out0="f32", tok_per_img=736, x3=True),
    _case("fwd98", "bn128 taps1 tma2 ks2 sbx32 STORE NONE out0:f32 res0:f32_inplace multi",
          n=1024, k=3072, w=2944, out0="f32", res0="f32_inplace", x3=True),
    _case("fwd99", "bn128 taps9 tma0 ks1 sbx32 FINAL NONE out0:- res0:- multi",
          n=128, k=384, taps=9, w=512, h=34, epi=F, x3=True),
    # act_postprocess[3]'s stride-2 conv as the parity forward runs it (x3="stride2"): split3 of the 23x32 x 768 map,
    # im2col3x3s2 of the split operand (3 * 768 channels), then the GEMM over K = 27 * 768 against the 3x3 weight packed
    # per tap as [Whi | Whi | Wlo]
    _case("fwd_stride2_x3", "bn128 taps1 tma1 ks1 sbx32 STORE NONE out0:f32 res0:-",
          n=768, k=27 * 768, w=2 * 12 * 16, out0="f32", x3="stride2"),
]

# ---- the contract beyond the forward
_LIN = dict(out0="f32", res0="f32_inplace")
CONTRACT = [
    # act(res0 + v) with the in-place fp32 residual, with and without a K split of the same shape
    _case("inplace_none_k1", "bn128 taps1 tma2 ks1 sbx32 STORE NONE out0:f32 res0:f32_inplace mtail",
          n=256, k=1024, w=300, **_LIN),
    _case("inplace_relu_k1", "bn128 taps1 tma0 ks1 sbx32 STORE RELU out0:f32 res0:f32_inplace mtail",
          n=256, k=1024, w=300, act=RELU, **_LIN),
    _case("inplace_gelu_k1", "bn128 taps1 tma0 ks1 sbx32 STORE GELU out0:f32 res0:f32_inplace mtail",
          n=256, k=1024, w=300, act=GELU, **_LIN),
    _case("inplace_none_ksplit", "bn128 taps1 tma2 ks4 sbx32 STORE NONE out0:f32 res0:f32_inplace mtail",
          n=256, k=4096, w=300, **_LIN),
    _case("inplace_relu_ksplit", "bn128 taps1 tma0 ks1 sbx32 STORE RELU out0:f32 res0:f32_inplace mtail",
          n=256, k=4096, w=300, act=RELU, **_LIN),
    _case("inplace_gelu_ksplit", "bn128 taps1 tma0 ks1 sbx32 STORE GELU out0:f32 res0:f32_inplace mtail",
          n=256, k=4096, w=300, act=GELU, **_LIN),
    # the epilogue additions are made once, whatever the K split
    _case("inplace_idxemb_ksplit", "bn128 taps1 tma0 ks1 sbx32 IDXEMB NONE out0:f32 res0:f32_inplace mtail",
          n=256, k=4096, w=300, epi=I, tok_per_img=7, **_LIN),
    _case("inplace_rope_ksplit", "bn128 taps1 tma2 ks4 sbx32 ROPE NONE out0:f32 res0:f32_inplace mtail",
          n=256, k=4096, w=300, epi=R, tok_per_img=60, grid_w=12, rope_cols=128, **_LIN),
    _case("inplace_idxemb_per_row", "bn128 taps1 tma0 ks1 sbx32 IDXEMB NONE out0:f32 res0:f32_inplace mtail",
          n=128, k=1024, w=200, epi=I, tok_per_img=0, **_LIN),
    # bf16 residuals with the relu copy, BLOCK_N 256 with a column split and row strides wider than the columns
    _case("res_bf16_res1_out1", "bn128 taps1 tma0 ks1 sbx32 STORE NONE out0:bf16 res0:bf16 out1 res1 mtail",
          n=256, k=256, w=1000, out0="bf16", out1=True, res0="bf16", res1=True),
    _case("split_bn256_ldo", "bn256 taps1 tma1 ks1 sbx32 STORE NONE out0:bf16 res0:- split",
          n=768, k=128, w=5632, out0="bf16", split_col=256, ldo=320, ldo_b=576),
    _case("ldo_wider_f32_res", "bn128 taps1 tma0 ks1 sbx32 STORE NONE out0:f32 res0:f32 ntail mtail",
          n=96, k=192, w=300, out0="f32", res0="f32", ldo=136),
    _case("convt_bn256_k2", "bn256 taps1 tma0 ks1 sbx32 CONVT NONE out0:bf16 res0:- mtail multi",
          n=768, k=192, w=32, h=23, nb=8, epi=T, out0="bf16", ct_k=2, ct_cout=192),
    # edges: N = 32, K = 8, K = 72, a single row, one-pixel-wide maps (bw = 1) and every TMA-store box width
    _case("edge_n32", "bn128 taps1 tma1 ks1 sbx32 STORE NONE out0:bf16 res0:- ntail mtail",
          n=32, k=128, w=500, out0="bf16"),
    _case("edge_k8", "bn128 taps1 tma1 ks1 sbx32 STORE NONE out0:bf16 res0:- ktail mtail",
          n=128, k=8, w=300, out0="bf16"),
    _case("edge_k72_f32", "bn128 taps1 tma1 ks1 sbx32 STORE NONE out0:f32 res0:- ntail ktail mtail",
          n=96, k=72, w=257, out0="f32"),
    _case("edge_m1", "bn128 taps1 tma1 ks1 sbx32 STORE NONE out0:f32 res0:- ntail mtail",
          n=64, k=64, w=1, out0="f32"),
    _case("edge_m1_inplace_ksplit", "bn128 taps1 tma2 ks4 sbx32 STORE NONE out0:f32 res0:f32_inplace ntail mtail",
          n=64, k=4096, w=1, **_LIN),
    _case("edge_w1_conv3x3", "bn128 taps9 tma0 ks1 sbx1 STORE NONE out0:bf16 res0:- out1 ntail mtail",
          n=64, k=64, taps=9, w=1, h=300, nb=2, out0="bf16", out1=True),
    _case("edge_w1_store", "bn128 taps1 tma1 ks1 sbx1 STORE NONE out0:bf16 res0:- ntail mtail",
          n=64, k=64, w=1, h=257, nb=2, out0="bf16"),
    _case("edge_w2_store", "bn128 taps1 tma1 ks1 sbx2 STORE NONE out0:bf16 res0:- ntail mtail",
          n=64, k=64, w=2, h=100, nb=2, out0="bf16"),
    _case("edge_w4_store", "bn128 taps1 tma1 ks1 sbx4 STORE NONE out0:f32 res0:- ntail mtail",
          n=64, k=64, w=4, h=50, nb=2, out0="f32"),
    _case("edge_w8_store", "bn128 taps1 tma1 ks1 sbx8 STORE NONE out0:bf16 res0:- ntail mtail",
          n=64, k=64, w=8, h=20, nb=3, out0="bf16"),
    _case("edge_w16_conv3x3", "bn128 taps9 tma1 ks1 sbx16 STORE RELU out0:bf16 res0:- ntail mtail",
          n=64, k=64, taps=9, w=16, h=9, nb=3, out0="bf16", act=RELU),
    # several images whose last tile is partial in x and y
    _case("edge_nb3_partial_tiles", "bn128 taps9 tma0 ks1 sbx8 STORE NONE out0:bf16 res0:- out1 mtail",
          n=128, k=64, taps=9, w=24, h=13, nb=3, out0="bf16", out1=True),
    _case("edge_final_partial_tiles", "bn128 taps9 tma0 ks1 sbx8 FINAL NONE out0:- res0:- mtail",
          n=128, k=64, taps=9, w=40, h=13, nb=3, epi=F),
]

# ---- the hand-picked shapes of the earlier per-kernel checks (tests/kernel_checks.py runs them under these names)
KERNEL_CHECKS = [
    _case("linear_small_tails", "bn128 taps1 tma1 ks1 sbx32 STORE NONE out0:bf16 res0:- ntail mtail",
          n=96, k=192, w=300, out0="bf16"),
    _case("linear_qkv_shape", "bn256 taps1 tma1 ks1 sbx32 STORE NONE out0:bf16 res0:- multi",
          n=3072, k=1024, w=2944, out0="bf16"),
    _case("linear_bn256", "bn256 taps1 tma1 ks1 sbx32 STORE NONE out0:bf16 res0:- multi",
          n=1024, k=256, w=23552, out0="bf16"),
    _case("linear_resid_gelu", "bn128 taps1 tma2 ks1 sbx32 STORE NONE out0:f32 res0:f32_inplace mtail",
          n=512, k=1024, w=1000, **_LIN),
    _case("linear_resid_gelu_out1", "bn128 taps1 tma0 ks1 sbx32 STORE GELU out0:bf16 res0:- out1 mtail",
          n=512, k=1024, w=1000, act=GELU, out0="bf16", out1=True),
    _case("linear_resid_splitk", "bn128 taps1 tma2 ks4 sbx32 STORE NONE out0:f32 res0:f32_inplace mtail",
          n=256, k=4096, w=300, **_LIN),
    _case("linear_resid_splitk_out1", "bn128 taps1 tma0 ks1 sbx32 STORE GELU out0:bf16 res0:- out1 mtail",
          n=256, k=4096, w=300, act=GELU, out0="bf16", out1=True),
    _case("linear_split", "bn128 taps1 tma1 ks1 sbx32 STORE NONE out0:bf16 res0:- split mtail",
          n=384, k=128, w=520, out0="bf16", split_col=128, ldo=128, ldo_b=256),
    _case("rope_epilogue", "bn128 taps1 tma1 ks1 sbx32 ROPE NONE out0:bf16 res0:- mtail",
          n=384, k=128, w=120, epi=R, out0="bf16", tok_per_img=40, grid_w=8, rope_cols=256),
    _case("idxemb_epilogue", "bn128 taps1 tma1 ks1 sbx32 IDXEMB NONE out0:f32 res0:- mtail",
          n=128, k=128, w=144, epi=I, out0="f32", tok_per_img=24),
    _case("conv1x1_tinymap", "bn128 taps1 tma1 ks1 sbx32 STORE NONE out0:bf16 res0:- ntail mtail",
          n=96, k=128, w=6, h=4, nb=3, out0="bf16"),
    _case("conv3x3_w256", "bn128 taps9 tma0 ks1 sbx32 STORE NONE out0:bf16 res0:- out1",
          n=128, k=64, taps=9, w=256, h=20, nb=2, out0="bf16", out1=True),
    _case("conv3x3_w6_c96_res", "bn128 taps9 tma0 ks1 sbx32 STORE NONE out0:bf16 res0:bf16 out1 res1 ktail mtail",
          n=256, k=96, taps=9, w=6, h=4, nb=3, out0="bf16", out1=True, res0="bf16",
          res1=True),
    _case("conv3x3_w24_c192", "bn128 taps9 tma0 ks1 sbx8 STORE NONE out0:bf16 res0:- out1",
          n=256, k=192, taps=9, w=24, h=16, out0="bf16", out1=True),
    _case("conv3x3_w512", "bn128 taps9 tma0 ks1 sbx32 STORE NONE out0:bf16 res0:- out1 multi",
          n=128, k=128, taps=9, w=512, h=40, out0="bf16", out1=True),
    _case("convT_k4", "bn128 taps1 tma0 ks1 sbx32 CONVT NONE out0:bf16 res0:- ktail mtail",
          n=16 * 96, k=96, w=6, h=4, nb=2, epi=T, out0="bf16", ct_k=4, ct_cout=96),
    _case("convT_k2", "bn128 taps1 tma0 ks1 sbx32 CONVT NONE out0:bf16 res0:- mtail",
          n=4 * 192, k=192, w=6, h=4, nb=2, epi=T, out0="bf16", ct_k=2, ct_cout=192),
    _case("final_fused", "bn128 taps9 tma0 ks1 sbx32 FINAL NONE out0:- res0:-",
          n=128, k=128, taps=9, w=96, h=16, nb=2, epi=F),    # the parity path's GEMM (fp32 operands split by ops.gemm_x3)
    _case("x3_linear", "bn128 taps1 tma1 ks1 sbx32 STORE NONE out0:f32 res0:- mtail",
          n=512, k=3 * 1024, w=1000, out0="f32", x3=True),
    _case("x3_linear_gelu_tails", "bn128 taps1 tma1 ks1 sbx32 STORE GELU out0:f32 res0:- ntail mtail",
          n=96, k=3 * 256, w=333, act=GELU, out0="f32", x3=True),
    _case("x3_conv3x3_c96_relu_res", "bn128 taps9 tma0 ks1 sbx32 STORE NONE out0:f32 res0:f32 ktail mtail",
          n=256, k=3 * 96, taps=9, w=24, h=9, nb=2, out0="f32", res0="f32", x3=True, a_relu=True),
]

CASES = FORWARD + CONTRACT + KERNEL_CHECKS
