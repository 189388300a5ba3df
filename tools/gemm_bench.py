"""Times f3r_gemm on the decoder shapes (CUDA events, L2-flushed between reps).  Env knob: F3R_GEMM_DEBUG."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from fast3r_b200 import ops, lib as L
M = int(os.environ.get("M", 23552))
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
def bench(name, N, K, **kw):
    a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda") * K ** -0.5).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda")
    args = dict(kw)
    if args.pop("resid", False):
        x = torch.randn(M, N, device="cuda"); args.update(out0=x, res0=x)
    else:
        args.update(out0=torch.empty(M, N, dtype=torch.bfloat16, device="cuda"))
    ts = []
    for i in range(6):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); ops.linear(a, w, bias, **args); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    t = sorted(ts[1:])[len(ts[1:]) // 2]
    print(f"{name:8s} M={M} N={N} K={K}: {t*1e3:8.1f} us  {2*M*N*K/t/1e9:7.1f} TFLOP/s", flush=True)
bench("qkv", 3072, 1024)
bench("proj", 1024, 1024, resid=True)
bench("fc1", 4096, 1024, act=L.ACT_GELU)
bench("fc2", 1024, 4096, resid=True)
