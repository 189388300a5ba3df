"""Sequence-parallel inference of the fusion decoder over the GPUs of one box (one process per GPU).

The reference has no counterpart (SURVEY.md §2a: no TP/PP/SP anywhere); the single-device result is the oracle.
Partitioning (SURVEY.md §8(e)): rank r owns a contiguous range of views, i.e. a contiguous token range of the
N*P-token sequence.  Encoder blocks, LayerNorm, all linears and the DPT heads are token/view-local and need no
communication; only the global attention couples ranks: each decoder layer all-gathers K|V (bf16, S_local x 2D)
over NCCL/NVLink and every rank attends its local queries against all keys.  The image-index ids drawn by rank 0 are
broadcast to all ranks so the result equals the single-device forward whatever the per-rank RNG states are.
"""
from __future__ import annotations

import os
from typing import List, Tuple

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

    Fast path (bf16 path, batch 1, equal shards): the QKV GEMM writes this rank's K|V straight into its slot of the
    gather buffer (`kv_workspace()`); `attend()` starts the NCCL all-gather on a side stream and meanwhile attends the
    local queries to the LOCAL keys; when the gather has landed it attends to the key ranges of the other ranks and merges
    the partial results by their log-sum-exp (exact softmax over the union, f3r_attention_merge).  The exchange is hidden
    behind the local-chunk attention and every launch is key-sliced to fill the 132 SMs (ops.pick_kv_split).
    General path (batch > 1, uneven shards, parity precision, CPU emulator): all-gather, then one attention call."""

    def __init__(self, sp, batch: int, s_local: int, dim: int, rows: List[int]):
        self.sp, self.batch, self.s_local, self.dim, self.rows = sp, batch, s_local, dim, rows
        self.mx, self.s_total = max(rows), sum(rows)
        self.even = all(r == self.mx for r in rows)
        self.buf = None
        self.pad = None
        self.comm_stream = None
        self.parts = None
        self.layer = 0
        self.sym = None          # symmetric-memory transport: (2, s_local, C) K|V slots of this rank, double-buffered per layer
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
            sym = symm.empty((2, self.s_local, C), dtype=like.dtype, device=like.device)
            hdl = symm.rendezvous(sym, group)
            peers = [hdl.get_buffer(r, (2, self.s_local, C), like.dtype) for r in range(sp.world)]
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
        return self.even and self.batch == 1 and dtype == torch.bfloat16 and device.type == "cuda" and self.sp.overlap

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
            slot.copy_(kv)
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
                    self.buf[p_].copy_(self.peers[p_][par], non_blocking=True)
            for st in self.copy_streams:
                self.comm_stream.wait_stream(st)
            if ev:
                ev[5].record(self.comm_stream)
        else:
            with torch.cuda.stream(self.comm_stream):
                if ev:
                    ev[4].record(self.comm_stream)
                _all_gather_into(self.buf.view(-1, C), slot, group=sp.group)
                if ev:
                    ev[5].record(self.comm_stream)
        sp.bytes_exchanged += self.buf.numel() * self.buf.element_size()
        S, sl = self.s_total, self.s_local
        lo, hi = sp.rank * sl, (sp.rank + 1) * sl
        units = attention_units(1, heads, sl)
        # local keys first (straight from this rank's slot), then the other ranks' ranges of the gather buffer
        ranges = [(lo, sl)] + [r for r in ((0, lo), (hi, S - hi)) if r[1] > 0]
        splits = [ops.pick_kv_split(units, (n + 127) // 128) for _, n in ranges]
        slots = sum(splits)
        if self.parts is None or self.parts[0].shape[0] < slots:
            self.parts = (torch.empty(slots, sl, heads * 64, dtype=torch.float32, device=kv.device),
                          torch.empty(slots, 1, heads, sl, dtype=torch.float32, device=kv.device))
        part_o, part_lse = self.parts
        kv_all = self.buf.view(-1, C)
        base = 0
        for i, ((row0, n), ns) in enumerate(zip(ranges, splits)):
            if i == 1:
                if ev:
                    ev[1].record(compute)
                compute.wait_stream(self.comm_stream)  # the other ranks' keys have landed
            if i == 0 and use_sym:   # the local keys are read where the QKV GEMM wrote them
                ops.attention_partial(q, slot, part_o, part_lse, part_base=base, n_split=ns, batch=1, heads=heads, sq=sl,
                                      kv_rows_total=sl, kv_row0=0, skv=n, scale=scale)
            else:
                ops.attention_partial(q, kv_all, part_o, part_lse, part_base=base, n_split=ns, batch=1, heads=heads,
                                      sq=sl, kv_rows_total=S, kv_row0=row0, skv=n, scale=scale)
            base += ns
        if len(ranges) == 1:
            compute.wait_stream(self.comm_stream)
        if ev:
            ev[2].record(compute)
        ops.attention_merge(part_o, part_lse, slots, att, batch=1, heads=heads, sq=sl)
        if ev:
            ev[3].record(compute)
            tm.append(ev)


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

    def view_range(self, num_views: int) -> Tuple[int, int]:
        self._ranges = shard_views(num_views, self.world)
        if any(hi - lo == 0 for lo, hi in self._ranges):
            raise ValueError(f"sequence parallel needs at least one view per rank ({num_views} views, {self.world} ranks)")
        return self._ranges[self.rank]

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

    def make_kv_exchange(self, batch: int, s_local: int, dim: int):
        """Per-forward exchange object for the fusion decoder (one per `_decode` call)."""
        tok_per_view = s_local // (self._ranges[self.rank][1] - self._ranges[self.rank][0])
        rows = [(hi - lo) * tok_per_view for lo, hi in self._ranges]
        key = (batch, s_local, dim, tuple(rows))
        if key not in self._kvx:   # buffers (and the symmetric-memory rendezvous) are reused across forwards
            self._kvx = {key: KVExchange(self, batch, s_local, dim, rows)}
        self._kvx[key].layer = 0
        return self._kvx[key]

    def gather_results(self, final_results, num_views, batch, H, W, device):
        """All ranks end up with the preds of every view (API parity with the single-device forward)."""
        keys = [k for k in ("pts3d_in_other_view", "conf", "pts3d_local", "conf_local")
                if k in final_results[self._ranges[self.rank][0]]]
        mxv = max(hi - lo for lo, hi in self._ranges)
        lo, hi = self._ranges[self.rank]
        out = [dict() for _ in range(num_views)]
        for k in keys:
            loc = torch.cat([final_results[i][k] for i in range(lo, hi)], dim=0)  # (n_loc*B, ...)
            tail = loc.shape[1:]
            send = torch.zeros((mxv * batch,) + tuple(tail), dtype=loc.dtype, device=device)
            send[: loc.shape[0]] = loc
            recv = torch.empty((self.world, mxv * batch) + tuple(tail), dtype=loc.dtype, device=device)
            _all_gather_into(recv.view((-1,) + tuple(tail)), send, group=self.group)
            for r, (a, b) in enumerate(self._ranges):
                for i in range(a, b):
                    out[i][k] = recv[r, (i - a) * batch:(i - a + 1) * batch]
        return out


def enable_sequence_parallel(model, group=None, gather_preds: bool = True) -> SequenceParallel:
    sp = SequenceParallel(group, gather_preds)
    model.sp_group = sp
    return sp
