"""Sequence-parallel inference of the fusion decoder over the GPUs of one box (one process per GPU).

The reference has no counterpart (SURVEY.md §2a: no TP/PP/SP anywhere); the single-device result is the oracle.
Partitioning (SURVEY.md §8(e)): rank r owns a contiguous range of views, i.e. a contiguous token range of the
sequence; with views of different resolutions the ranges balance the token counts (shard_views_weighted).  Encoder
blocks, LayerNorm, all linears and the DPT heads are token/view-local and need no communication; only the global attention couples ranks: each decoder layer all-gathers K|V (bf16, S_local x 2D)
over NCCL/NVLink and every rank attends its local queries against all keys.  The image-index ids drawn by rank 0 are
broadcast to all ranks so the result equals the single-device forward whatever the per-rank RNG states are.
"""
from __future__ import annotations

import math
import os
from itertools import accumulate
from typing import List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

from .ops import attention_units


def _all_gather_into(out: torch.Tensor, inp: torch.Tensor, group=None) -> None:
    """dist.all_gather_into_tensor that also works for CUDA tensors over a gloo group (staged through the host): lets two
    ranks share ONE GPU in tests (NCCL refuses duplicate devices); NCCL groups take the direct call."""
    if inp.is_cuda and dist.get_backend(group) == "gloo":
        host_in = inp.detach().cpu().contiguous()
        host_out = torch.empty(out.shape, dtype=out.dtype)
        dist.all_gather_into_tensor(host_out, host_in, group=group)
        out.copy_(host_out)
        return
    dist.all_gather_into_tensor(out, inp, group=group)


def shard_views(num_views: int, world: int) -> List[Tuple[int, int]]:
    """Contiguous, balanced view ranges: the first (num_views % world) ranks get one extra view."""
    base, rem = divmod(num_views, world)
    out, lo = [], 0
    for r in range(world):
        n = base + (1 if r < rem else 0)
        out.append((lo, lo + n))
        lo += n
    return out


def shard_views_weighted(tokens: Sequence[int], world: int) -> List[Tuple[int, int]]:
    """Contiguous view ranges, at least one view per rank, that minimise the largest per-rank token count (the linear
    partition problem, solved exactly).  `tokens`: tokens per view.  Among the optimal partitions each rank takes the
    fewest views that reach an equal share of the tokens still unassigned, so equal token counts give exactly
    shard_views(len(tokens), world)."""
    n = len(tokens)
    if n < world:
        raise ValueError(f"sequence parallel needs at least one view per rank ({n} views, {world} ranks)")
    pre = list(accumulate(tokens, initial=0))

    def parts_needed(cap: int) -> List[int]:
        """need[i]: fewest ranges of at most `cap` tokens that cover views [i, n) (greedy from i is optimal)."""
        need, j = [0] * (n + 1), n
        for i in range(n - 1, -1, -1):
            while pre[j] - pre[i] > cap:
                j -= 1
            need[i] = 1 + need[j]
        return need

    lo_cap, hi_cap = max(tokens), pre[n]   # the optimal largest load lies in [lo_cap, hi_cap]
    while lo_cap < hi_cap:
        mid = (lo_cap + hi_cap) // 2
        if parts_needed(mid)[0] <= world:
            hi_cap = mid
        else:
            lo_cap = mid + 1
    cap, need = lo_cap, parts_needed(lo_cap)
    out, a = [], 0
    for r in range(world):
        left = world - r - 1   # ranks after this one
        if left == 0:
            out.append((a, n))
            break
        # feasible ends e: this range fits the cap, and [e, n) still splits into `left` non-empty ranges within the cap
        ends = [e for e in range(a + 1, n - left + 1) if pre[e] - pre[a] <= cap and need[e] <= left]
        share = (pre[n] - pre[a]) / (left + 1)
        e = next((e for e in ends if pre[e] - pre[a] >= share), ends[-1])
        out.append((a, e))
        a = e
    return out


def peer_key_ranges(rows: List[int], rank: int) -> List[Tuple[int, int]]:
    """Key ranges (first row, rows) that `rank` attends in the overlapped K|V exchange, in a gather buffer that holds each
    rank's rows in a slot of max(rows) rows: its own rows first, then the other ranks' rows in rank order, never a
    padding row.  Other ranks' slots that follow each other with no padding in between form one range (so with equal
    rows: the ranks before and the ranks after this one)."""
    mx = max(rows)
    peers: List[Tuple[int, int]] = []
    for p, n in enumerate(rows):
        if p == rank:
            continue
        if peers and p - 1 != rank and peers[-1][0] + peers[-1][1] == p * mx:
            peers[-1] = (peers[-1][0], peers[-1][1] + n)
        else:
            peers.append((p * mx, n))
    return [(rank * mx, rows[rank])] + peers


def assemble_kv(gathered: torch.Tensor, batch: int, rows: List[int]) -> torch.Tensor:
    """gathered: (world, batch * max_rows, C) padded per-rank K|V blocks, each laid out (b, s_local).
    Returns (batch * sum(rows), C) laid out (b, s_global) with ranks concatenated in order."""
    world, _, C = gathered.shape
    mx = max(rows)
    if batch == 1 and all(r == mx for r in rows):
        return gathered.reshape(world * mx, C)
    g = gathered.view(world, batch, mx, C)
    parts = [g[r, :, : rows[r]] for r in range(world)]  # (batch, rows_r, C)
    return torch.cat(parts, dim=1).reshape(-1, C)


class KVExchange:
    """K|V exchange + global attention of one sequence-parallel decoder forward.

    Fast path (bf16 path, batch 1, equal shards or views of mixed resolution): the QKV GEMM writes this rank's K|V
    straight into its slot of the gather buffer (`kv_workspace()`); every slot has the rows of the largest rank, so ranks
    with fewer tokens leave padding at its end.  `attend()` starts the NCCL all-gather on a side stream and meanwhile
    attends the local queries to the LOCAL keys; when the gather has landed it attends to the real rows of the other ranks
    (peer_key_ranges) and merges the partial results by their log-sum-exp (exact softmax over the union,
    f3r_attention_merge).  The exchange is hidden
    behind the local-chunk attention and every launch is key-sliced to fill the 132 SMs (ops.pick_kv_split).
    General path (batch > 1, parity precision, CPU emulator, views of one resolution in uneven shards): all-gather, then
    one attention call, bit-identical to the single-device forward.  `mixed`: the views have different resolutions, so the
    rows are almost never equal and the overlapped path takes uneven rows."""

    def __init__(self, sp, batch: int, s_local: int, dim: int, rows: List[int], mixed: bool = False):
        self.sp, self.batch, self.s_local, self.dim, self.rows = sp, batch, s_local, dim, rows
        self.mx, self.s_total = max(rows), sum(rows)
        self.even = all(r == self.mx for r in rows)
        self.mixed = mixed
        self.buf = None
        self.pad = None
        self.comm_stream = None
        self.parts = None
        self.layer = 0
        self.sym = None          # symmetric-memory transport: (2, mx, C) K|V slots of this rank, double-buffered per layer
        self.sym_state = None    # None: not tried yet, True / False

    def _setup_symmetric(self, like: torch.Tensor) -> bool:
        """Copy-engine transport: every rank exposes its K|V slot through torch symmetric memory (CUDA IPC over NVLink);
        peers PULL it with DMA copies that need no SMs.  All ranks must agree, else everybody falls back to NCCL."""
        sp = self.sp
        ok = 1
        try:
            env = os.environ.get("F3R_SP_TRANSPORT", "")
            if dist.get_backend(sp.group) != "nccl":
                raise RuntimeError("symmetric-memory transport disabled (not an NCCL group)")
            if sp.transport == "nccl" or env == "nccl":
                raise RuntimeError("symmetric-memory transport disabled")
            # measured (profiles/r02_notes.md): with 2 ranks the DMA pulls hide completely behind the local-chunk attention
            # while NCCL's kernels starve for SMs (62.9 -> 60.9 ms at N=32); with 8 ranks both take ~0.26 ms per layer
            if sp.transport == "auto" and env != "symm" and sp.world > 4:
                raise RuntimeError("NCCL all-gather preferred for more than 4 ranks")
            import torch.distributed._symmetric_memory as symm
            group = sp.group if sp.group is not None else dist.group.WORLD
            C = 2 * self.dim
            sym = symm.empty((2, self.mx, C), dtype=like.dtype, device=like.device)
            hdl = symm.rendezvous(sym, group)
            peers = [hdl.get_buffer(r, (2, self.mx, C), like.dtype) for r in range(sp.world)]
            streams = [torch.cuda.Stream(device=like.device) for _ in range(max(1, min(4, sp.world - 1)))]
        except Exception as e:  # noqa: BLE001
            ok = 0
            why = repr(e)[:200]
        on_gpu = dist.get_backend(sp.group) == "nccl"
        flag = torch.tensor([ok], device=like.device if on_gpu else "cpu", dtype=torch.int32)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=sp.group)
        if int(flag.item()) == 1:
            self.sym, self.hdl, self.peers, self.copy_streams = sym, hdl, peers, streams
            return True
        if sp.rank == 0 and ok == 0 and "preferred" not in why and "disabled" not in why:
            print(f"[fast3r_b200] symmetric-memory K|V transport unavailable ({why}); using the NCCL all-gather", flush=True)
        return False

    def _ensure(self, like: torch.Tensor):
        if self.buf is None or self.buf.dtype != like.dtype or self.buf.device != like.device:
            C = 2 * self.dim
            self.buf = torch.empty(self.sp.world, self.batch * self.mx, C, dtype=like.dtype, device=like.device)
            self.pad = None if self.even else torch.zeros(self.batch * self.mx, C, dtype=like.dtype, device=like.device)
            if like.is_cuda:
                self.comm_stream = torch.cuda.Stream(device=like.device)

    def fast(self, dtype, device) -> bool:
        return ((self.even or self.mixed) and self.batch == 1 and dtype == torch.bfloat16 and device.type == "cuda"
                and self.sp.overlap)

    def kv_workspace(self, dtype, device):
        """Where the QKV GEMM of the NEXT decoder layer should write this rank's K|V (None: any buffer; attend() copies).
        Called once per layer by Fast3R._decode."""
        if not self.fast(dtype, device):
            return None
        like = torch.empty(0, dtype=dtype, device=device)
        self._ensure(like)
        if self.sym_state is None:
            self.sym_state = self._setup_symmetric(like)
        if self.sym_state:
            return self.sym[self.layer & 1]
        return self.buf[self.sp.rank]

    def attend(self, ops, q, kv, att, *, heads: int, scale: float, x3: bool):
        sp, C = self.sp, kv.shape[-1]
        self._ensure(kv)
        if not self.fast(kv.dtype, kv.device) or x3:
            src = kv
            if not self.even:
                self.pad.view(self.batch, self.mx, C)[:, :self.s_local] = kv.view(self.batch, self.s_local, C)
                src = self.pad
            _all_gather_into(self.buf.view(-1, C), src.contiguous(), group=sp.group)
            sp.bytes_exchanged += self.buf.numel() * self.buf.element_size()
            kv_all = assemble_kv(self.buf, self.batch, self.rows)
            (ops.attention_x3 if x3 else ops.attention)(q, kv_all, att, batch=self.batch, heads=heads, sq=self.s_local,
                                                        skv=self.s_total, scale=scale)
            return
        # ---- overlapped path
        use_sym = bool(self.sym_state)
        par = self.layer & 1
        self.layer += 1
        slot = self.sym[par] if use_sym else self.buf[sp.rank]
        if kv.data_ptr() != slot.data_ptr():
            slot[:self.s_local].copy_(kv)
        compute = torch.cuda.current_stream(kv.device)
        tm = sp.timers  # optional CUDA-event trace of the phases (bench.py): list of per-call event tuples
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)] if tm is not None else None
        if ev:
            ev[0].record(compute)
        self.comm_stream.wait_stream(compute)  # K|V of this layer is complete; previous layer's readers are done
        if use_sym:
            # every rank's K|V of this layer sits in its symmetric slot `par`: barrier on the side stream, then pull the
            # peers' slots with copy-engine DMA (no SMs, unlike NCCL's kernels) on a few streams in parallel.  The slot is
            # reused two layers later; by then every peer has passed the next layer's barrier, i.e. finished these pulls.
            with torch.cuda.stream(self.comm_stream):
                if ev:
                    ev[4].record(self.comm_stream)
                self.hdl.barrier(channel=par)
            ready = torch.cuda.Event()
            ready.record(self.comm_stream)
            for i in range(1, sp.world):
                p_ = (sp.rank + i) % sp.world   # staggered so that not all ranks hit the same peer first
                st = self.copy_streams[(i - 1) % len(self.copy_streams)]
                st.wait_event(ready)
                with torch.cuda.stream(st):
                    n = self.rows[p_]
                    self.buf[p_][:n].copy_(self.peers[p_][par][:n], non_blocking=True)
            for st in self.copy_streams:
                self.comm_stream.wait_stream(st)
            if ev:
                ev[5].record(self.comm_stream)
            # the real rows of every rank (the whole buffer when the rows are equal); padding is not pulled
            sp.bytes_exchanged += self.s_total * C * self.buf.element_size()
        else:
            with torch.cuda.stream(self.comm_stream):
                if ev:
                    ev[4].record(self.comm_stream)
                _all_gather_into(self.buf.view(-1, C), slot, group=sp.group)
                if ev:
                    ev[5].record(self.comm_stream)
            sp.bytes_exchanged += self.buf.numel() * self.buf.element_size()   # the all-gather moves the padding too

        def peers_landed():
            if ev:
                ev[1].record(compute)
            compute.wait_stream(self.comm_stream)  # the other ranks' keys have landed

        # with symmetric memory the local keys are read where the QKV GEMM wrote them
        slots = self.partials(ops, q, slot[:self.s_local] if use_sym else None, heads=heads, scale=scale,
                              peers_landed=peers_landed)
        if ev:
            ev[2].record(compute)
        ops.attention_merge(self.parts[0], self.parts[1], slots, att, batch=1, heads=heads, sq=self.s_local)
        if ev:
            ev[3].record(compute)
            tm.append(ev)

    def partials(self, ops, q, local, *, heads: int, scale: float, peers_landed) -> int:
        """Overlapped path after the exchange has started: attends the local queries to this rank's keys (`local`, or its
        slot of the gather buffer when None), calls `peers_landed()`, then attends to the other ranks' real rows of the
        gather buffer (peer_key_ranges), each range key-sliced (ops.pick_kv_split) into the partial buffers `self.parts`.
        Returns the number of partials to merge."""
        sl = self.s_local
        rows_total = self.sp.world * self.mx
        units = attention_units(1, heads, sl)
        ranges = peer_key_ranges(self.rows, self.sp.rank)
        splits = [ops.pick_kv_split(units, (n + 127) // 128) for _, n in ranges]
        slots = sum(splits)
        if self.parts is None or self.parts[0].shape[0] < slots:
            self.parts = (torch.empty(slots, sl, heads * 64, dtype=torch.float32, device=q.device),
                          torch.empty(slots, 1, heads, sl, dtype=torch.float32, device=q.device))
        part_o, part_lse = self.parts
        kv_all = self.buf.view(-1, self.buf.shape[-1])
        base = 0
        for i, ((row0, n), ns) in enumerate(zip(ranges, splits)):
            if i == 1:
                peers_landed()
            if i == 0 and local is not None:
                ops.attention_partial(q, local, part_o, part_lse, part_base=base, n_split=ns, batch=1, heads=heads, sq=sl,
                                      kv_rows_total=sl, kv_row0=0, skv=n, scale=scale)
            else:
                ops.attention_partial(q, kv_all, part_o, part_lse, part_base=base, n_split=ns, batch=1, heads=heads,
                                      sq=sl, kv_rows_total=rows_total, kv_row0=row0, skv=n, scale=scale)
            base += ns
        if len(ranges) == 1:
            peers_landed()
        return slots


class SequenceParallel:
    def __init__(self, group=None, gather_preds: bool = True):
        if not dist.is_initialized():
            raise RuntimeError("torch.distributed must be initialised (torchrun) before enabling sequence parallel")
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.gather_preds = gather_preds
        self.overlap = True   # False: always all-gather first, then one attention call (A/B measurements)
        self.timers = None    # set to a list to collect CUDA-event traces of KVExchange.attend (bench.py)
        self.transport = "auto"   # "auto": copy-engine pulls from symmetric peer memory for <= 4 ranks (if available),
        #                           NCCL all-gather otherwise; "symm" / "nccl" force one (also F3R_SP_TRANSPORT)
        self._kvx = {}
        self._ranges = None
        self.bytes_exchanged = 0

    def view_range(self, num_views: int, tokens: Optional[Sequence[int]] = None) -> Tuple[int, int]:
        """This rank's views [lo, hi).  `tokens`: tokens per view (views of different resolutions); the ranges minimise
        the largest per-rank token count (shard_views_weighted).  Every rank sees the same view shapes, so all ranks
        agree on the ranges without communicating."""
        self._ranges = shard_views_weighted(tokens if tokens is not None else [1] * num_views, self.world)
        return self._ranges[self.rank]

    @property
    def ranges(self) -> List[Tuple[int, int]]:
        """The view range of every rank, as set by the last view_range call."""
        return self._ranges

    def broadcast_ids(self, ids: torch.Tensor, device) -> torch.Tensor:
        """Every rank uses the image ids drawn by rank 0 of the group (the single-device stream), whatever its own CPU
        RNG state is; each rank has still consumed its own draw, like the reference does per forward."""
        if self.world == 1:
            return ids
        src = dist.get_global_rank(self.group, 0) if self.group is not None else 0
        on_gpu = dist.get_backend(self.group) == "nccl"
        t = ids.to(device) if on_gpu else ids.clone()
        dist.broadcast(t, src=src, group=self.group)
        return t.cpu()

    def make_kv_exchange(self, batch: int, s_local: int, dim: int, rows: Optional[List[int]] = None,
                         mixed: bool = False):
        """Per-forward exchange object for the fusion decoder (one per `_decode` call).  `rows`: tokens per sample of every
        rank (default: all views have the token count of this rank's views); `mixed`: views of different resolutions."""
        if rows is None:
            tok_per_view = s_local // (self._ranges[self.rank][1] - self._ranges[self.rank][0])
            rows = [(hi - lo) * tok_per_view for lo, hi in self._ranges]
        key = (batch, s_local, dim, tuple(rows), mixed)
        if key not in self._kvx:   # buffers (and the symmetric-memory rendezvous) are reused across forwards
            self._kvx = {key: KVExchange(self, batch, s_local, dim, list(rows), mixed)}
        self._kvx[key].layer = 0
        return self._kvx[key]

    def gather_results(self, final_results, num_views, batch, H, W, device, shapes=None):
        """All ranks end up with the preds of every view (API parity with the single-device forward).  `shapes`: the
        (H, W) of every view's predictions (default: (H, W) for all).  Each rank sends its views' predictions flattened
        into one buffer padded to the largest rank's and splits what it receives by these shapes, which every rank knows."""
        shapes = [tuple(s) for s in shapes] if shapes is not None else [(H, W)] * num_views
        lo, hi = self._ranges[self.rank]
        keys = [k for k in ("pts3d_in_other_view", "conf", "pts3d_local", "conf_local") if k in final_results[lo]]
        out = [dict() for _ in range(num_views)]
        for k in keys:
            chan = tuple(final_results[lo][k].shape[3:])   # (3,) for point maps, () for confidences
            numel = [batch * h * w * math.prod(chan) for h, w in shapes]
            sizes = [sum(numel[a:b]) for a, b in self._ranges]
            loc = torch.cat([final_results[i][k].reshape(-1) for i in range(lo, hi)])
            send = torch.zeros(max(sizes), dtype=loc.dtype, device=device)
            send[: loc.numel()] = loc
            recv = torch.empty(self.world, max(sizes), dtype=loc.dtype, device=device)
            _all_gather_into(recv.view(-1), send, group=self.group)
            for r, (a, b) in enumerate(self._ranges):
                o = 0
                for i in range(a, b):
                    out[i][k] = recv[r, o:o + numel[i]].view((batch,) + shapes[i] + chan)
                    o += numel[i]
        return out


def enable_sequence_parallel(model, group=None, gather_preds: bool = True) -> SequenceParallel:
    sp = SequenceParallel(group, gather_preds)
    model.sp_group = sp
    return sp
