"""Sequence-parallel parity check for views of mixed resolution (run under torchrun): the sharded forward must reproduce
the single-GPU forward of the same model on the same views when the ranks hold different token counts.

SP_ONE_GPU=1: all ranks share cuda:0 and talk over gloo (host-staged collectives); the default is one GPU per rank over
NCCL.  With the overlapped exchange disabled (all-gather, one attention call) the result must be bit-identical; the
overlapped path (key-range partials over each rank's real rows, merged by log-sum-exp) is judged like equal shards are in
tools/sp_check.py: against the fp32 oracle, next to the single-GPU forward."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from fast3r_b200 import Fast3R, tiny_args  # noqa: E402
from fast3r_b200.parallel import enable_sequence_parallel  # noqa: E402
from tests.golden.synth import synth_state_dict, synth_images  # noqa: E402

rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
one_gpu = os.environ.get("SP_ONE_GPU", "0") == "1"
torch.cuda.set_device(0 if one_gpu else lr)
if one_gpu:
    dist.init_process_group("gloo")
else:
    dist.init_process_group("nccl", device_id=torch.device("cuda", lr))

# (batch, view sizes): landscape, portrait and square views; the token counts (736 / 1024 per view) split unevenly
CASES = [(1, [(368, 512), (512, 368), (512, 512)]),
         (1, [(512, 512), (368, 512), (368, 512), (512, 368), (512, 512)]),
         (2, [(512, 512), (368, 512), (512, 368), (368, 512)])]
rl2 = lambda x, y: float((x.double() - y.double()).norm() / y.double().norm())  # noqa: E731
ok = True
for batch, sizes in CASES:
    if len(sizes) < world:
        continue
    model = Fast3R(*tiny_args()).eval()
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    model.load_state_dict(synth_state_dict(shapes, seed=0))
    model = model.cuda()
    model.image_id_rank_offset = 0           # the single-device oracle stream (rank-independent)
    imgs = [synth_images(1, batch, h, w, seed0=4321 + i)[0] for i, (h, w) in enumerate(sizes)]
    views = [dict(img=im.cuda()) for im in imgs]
    torch.manual_seed(7)
    ref = model(views)                       # single-GPU forward (every rank computes it redundantly)
    sp = enable_sequence_parallel(model, gather_preds=True)
    res = {}
    for overlap in (False, True):
        sp.overlap = overlap
        torch.manual_seed(7 + 1000 * rank)   # per-rank RNG states differ: the ids of rank 0 must be used everywhere
        out = model(views)
        kvx = next(iter(sp._kvx.values()))
        fast = kvx.fast(torch.bfloat16, views[0]["img"].device)
        same = all(a[k].shape == b[k].shape and torch.equal(a[k], b[k]) for a, b in zip(out, ref) for k in b)
        res[overlap] = (out, fast, same)
    model.sp_group = None
    rows = kvx.rows
    t = torch.tensor([0.0 if res[False][2] else 1.0], device="cpu" if one_gpu else "cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    exact = t.item() == 0.0
    ok = ok and exact and not res[False][1]
    if rank == 0:
        print(f"views={len(sizes)} batch={batch} ranges={sp.ranges} rows/rank={rows}: all-gather path "
              f"{'bit-identical' if exact else 'DIFFERS'} to single GPU", flush=True)
    out, fast, _ = res[True]
    if fast:
        from oracle import fast3r_oracle as O
        enc, dec, head = tiny_args()
        torch.manual_seed(7)
        gold = O.forward(synth_state_dict(shapes, seed=0), enc, dec, head, imgs)
        e_sp = max(rl2(torch.cat([p[k].float().cpu().flatten() for p in out]), torch.cat([p[k].flatten() for p in gold]))
                   for k in gold[0])
        e_1 = max(rl2(torch.cat([p[k].float().cpu().flatten() for p in ref]), torch.cat([p[k].flatten() for p in gold]))
                  for k in gold[0])
        t = torch.tensor([e_sp], device="cpu" if one_gpu else "cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        e_sp = t.item()
        good = e_sp < 1.3e-2 and e_sp < 1.5 * e_1 + 1e-3
        ok = ok and good and len(set(rows)) > 1
        if rank == 0:
            print(f"   path = overlapped partials (uneven rows {rows}): rel-L2 vs fp32 oracle sharded {e_sp:.3e}, "
                  f"single GPU {e_1:.3e} -> {'ok' if good else 'FAIL'}", flush=True)
    elif batch == 1:
        ok = False   # batch 1 in bf16 on CUDA must take the overlapped path
dist.barrier()
if rank == 0:
    print("SP_MIXED_OK" if ok else "SP_MIXED_FAIL")
dist.destroy_process_group()
