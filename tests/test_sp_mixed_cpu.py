"""Sequence parallelism over views of mixed resolution, on the CPU: token-balanced sharding, the sharded forward of the
product host code over the C-ABI emulator on a 2-rank gloo group, and the key ranges of the overlapped K|V exchange
when ranks hold different token counts."""
import itertools
import os
import socket
from types import SimpleNamespace

import pytest
import torch
from torch.overrides import TorchFunctionMode

from tests.conftest import rel_l2
from tests.golden.synth import synth_state_dict, synth_images


# ------------------------------------------------------------------ token-balanced sharding
def _best_max_load(tokens, world):
    """Brute force over every split into `world` non-empty contiguous ranges."""
    n, best = len(tokens), None
    for cuts in itertools.combinations(range(1, n), world - 1):
        b = (0,) + cuts + (n,)
        load = max(sum(tokens[b[i]:b[i + 1]]) for i in range(world))
        best = load if best is None else min(best, load)
    return best


def _check_partition(ranges, n, world):
    assert len(ranges) == world and ranges[0][0] == 0 and ranges[-1][1] == n
    assert all(a < b for a, b in ranges)
    assert all(ranges[i][1] == ranges[i + 1][0] for i in range(world - 1))


def test_equal_tokens_reproduce_shard_views():
    from fast3r_b200.parallel import shard_views, shard_views_weighted
    for world in range(1, 9):
        for n in range(world, 40):
            for tok in (1, 736):
                assert shard_views_weighted([tok] * n, world) == shard_views(n, world), (n, world, tok)
    assert shard_views_weighted([1024] * 1000, 8) == shard_views(1000, 8)
    assert shard_views_weighted([3] * 5, 2) == [(0, 3), (3, 5)]


@pytest.mark.parametrize("tokens,world,ranges,load", [
    ([24, 12, 24, 6], 2, [(0, 2), (2, 4)], 36),              # the four resolutions of tiny_mixed_res
    ([736, 736, 1024, 1024, 736, 736], 2, [(0, 3), (3, 6)], 2496),
    ([1024, 736, 736, 736, 736], 2, [(0, 2), (2, 5)], 2208),  # shard_views' (0, 3) | (3, 5) would load 2496
    ([100, 1, 1, 1, 1, 1], 3, [(0, 1), (1, 4), (4, 6)], 100),
    ([1, 1, 1, 1, 1, 100], 3, [(0, 4), (4, 5), (5, 6)], 100),
    ([5, 5, 5, 5, 20], 2, [(0, 4), (4, 5)], 20),
])
def test_weighted_sharding_hand_checked(tokens, world, ranges, load):
    from fast3r_b200.parallel import shard_views_weighted
    got = shard_views_weighted(tokens, world)
    assert got == ranges
    assert max(sum(tokens[a:b]) for a, b in got) == load == _best_max_load(tokens, world)


def test_weighted_sharding_is_optimal_on_random_sets():
    from fast3r_b200.parallel import shard_views_weighted
    g = torch.Generator().manual_seed(0)
    for _ in range(300):
        world = int(torch.randint(1, 5, (1,), generator=g))
        n = int(torch.randint(world, 10, (1,), generator=g))
        choices = torch.tensor([384, 576, 736, 1024, 1472])
        tokens = choices[torch.randint(0, 5, (n,), generator=g)].tolist()
        got = shard_views_weighted(tokens, world)
        _check_partition(got, n, world)
        assert max(sum(tokens[a:b]) for a, b in got) == _best_max_load(tokens, world), (tokens, world, got)


def test_fewer_views_than_ranks_raises():
    from fast3r_b200.parallel import shard_views_weighted, SequenceParallel
    with pytest.raises(ValueError, match="at least one view per rank"):
        shard_views_weighted([736, 1024, 736], 4)
    sp = SequenceParallel.__new__(SequenceParallel)   # the range logic only; no process group needed
    sp.world, sp.rank = 4, 0
    with pytest.raises(ValueError, match="at least one view per rank"):
        sp.view_range(3, [736, 1024, 736])


# ------------------------------------------------------------------ sharded forward over gloo (2 ranks, emulator)
class _RowwiseProducts(TorchFunctionMode):
    """Runs every matmul of the emulator one row at a time and every convolution one image at a time.  The CPU BLAS picks
    its blocking by the row count, so the same row can round differently when a rank holds fewer views than the single
    device; in this mode a row's result depends on its own data only, as it does in the sm_90a kernels (the same
    condition under which the GPU forward is bit-identical, tools/sp_check.py), and the sharded forward can be compared
    bit for bit."""

    def __torch_function__(self, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        name = getattr(func, "__name__", "")   # `a @ b` arrives as Tensor.matmul
        if name in ("matmul", "__matmul__") and args[0].dim() >= 2 and args[0].shape[-2] > 1:
            a, b = args
            return torch.cat([a[..., i:i + 1, :] @ b for i in range(a.shape[-2])], dim=-2)
        if name == "conv2d" and args[0].shape[0] > 1:
            x, rest = args[0], args[1:]
            return torch.cat([func(x[i:i + 1], *rest, **kwargs) for i in range(x.shape[0])])
        return func(*args, **kwargs)


def _model(M, g):
    from fast3r_b200 import tiny_args
    model = M.Fast3R(*tiny_args()).eval()
    model.load_state_dict(synth_state_dict(g["shapes"], seed=g["weight_seed"]))
    return model


def _sp_worker(rank, world, port, golden_dir, batch, seed_skew, ret):
    import torch.distributed as dist
    import fast3r_b200.model as M
    from tests import abi_emulator
    from fast3r_b200.parallel import enable_sequence_parallel
    M.ops = abi_emulator
    M._require_cuda = lambda device: None
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    g = torch.load(os.path.join(golden_dir, "tiny_mixed_res.pt"))
    model = _model(M, g)
    model.image_id_rank_offset = 0
    imgs = [synth_images(1, batch, h, w, seed0=1234 + i)[0] for i, (h, w) in enumerate(g["sizes"])]
    views = [dict(img=im) for im in imgs]
    with _RowwiseProducts():
        torch.manual_seed(g["rng_seed"])
        ref = model(views)                                   # un-sharded forward in this process
        sp = enable_sequence_parallel(model, gather_preds=True)
        torch.manual_seed(g["rng_seed"] + seed_skew * rank)  # ranks > 0 may hold a different CPU RNG state
        out = model(views)
        sp.gather_preds = False                              # each rank keeps its own views only
        torch.manual_seed(g["rng_seed"])
        own = model(views)
    res = dict(ranges=sp.ranges, rows=next(iter(sp._kvx.values())).rows)
    res["bitwise"] = all(torch.equal(p[k], q[k]) and p[k].shape == q[k].shape for p, q in zip(out, ref) for k in q)
    res["fix"] = max(rel_l2(p[k], q[k]) for p, q in zip(out, g["preds"]) for k in q) if batch == g["B"] else None
    lo, hi = sp.ranges[rank]
    res["own"] = all((lo <= i < hi) == bool(p) for i, p in enumerate(own)) and all(
        torch.equal(own[i][k], ref[i][k]) for i in range(lo, hi) for k in ref[i])
    ret[rank] = res
    dist.destroy_process_group()


@pytest.mark.parametrize("batch,seed_skew", [(1, 0), (1, 1000), (2, 0)])
def test_mixed_resolution_forward_over_gloo(golden_dir, batch, seed_skew):
    """Views at four resolutions split 36 | 30 tokens over 2 ranks: the sharded forward (general path: all-gather, one
    attention call) equals the un-sharded forward of the same process bit for bit, and the reference fixture within the
    single-device tolerance (the fixture has batch 1)."""
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    procs = [ctx.Process(target=_sp_worker, args=(r, 2, port, golden_dir, batch, seed_skew, ret)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
    assert set(ret.keys()) == {0, 1}, dict(ret)
    for r in (0, 1):
        res = ret[r]
        assert res["ranges"] == [(0, 2), (2, 4)] and res["rows"] == [36, 30], res
        assert res["bitwise"], (r, res)
        assert res["own"], (r, res)
        if batch == 1:
            assert res["fix"] < 3e-2, (r, res["fix"])


# ------------------------------------------------------------------ overlapped exchange: key ranges with uneven rows
class _RecordingOps:
    """Stands in for fast3r_b200.ops: records the key ranges the overlapped path hands to attention_partial."""

    def __init__(self):
        self.calls = []

    @staticmethod
    def pick_kv_split(units, key_blocks):
        from fast3r_b200.ops import pick_kv_split
        return pick_kv_split(units, key_blocks)

    def attention_partial(self, q, kv, part_o, part_lse, *, part_base, n_split, batch, heads, sq, kv_rows_total,
                          kv_row0, skv, scale):
        assert kv.shape[0] == batch * kv_rows_total and kv_row0 + skv <= kv_rows_total
        self.calls.append((kv, kv_row0, skv, part_base, n_split))


def _exchange(rows, rank, heads=2):
    from fast3r_b200.parallel import KVExchange
    sp = SimpleNamespace(rank=rank, world=len(rows))
    kvx = KVExchange(sp, 1, rows[rank], heads * 64, rows)
    kvx.buf = torch.zeros(len(rows), max(rows), 2 * heads * 64, dtype=torch.bfloat16)
    return kvx


def _partials(kvx, ops, q, local):
    landed = []
    n = kvx.partials(ops, q, local, heads=2, scale=0.2, peers_landed=lambda: landed.append(len(getattr(ops, "calls", []))))
    return n, landed


@pytest.mark.parametrize("rows", [[36, 30], [30, 36], [736, 1024, 736], [1024, 736, 1024, 1024], [5000, 4100, 300]])
@pytest.mark.parametrize("use_local", [False, True])
def test_overlapped_ranges_cover_real_rows_once(rows, use_local):
    mx = max(rows)
    for rank in range(len(rows)):
        kvx = _exchange(rows, rank)
        ops = _RecordingOps()
        local = torch.zeros(rows[rank], 4 * 64, dtype=torch.bfloat16) if use_local else None
        q = torch.zeros(rows[rank], 2 * 64, dtype=torch.bfloat16)
        n_parts, landed = _partials(kvx, ops, q, local)
        assert landed == [1]                         # the peers' keys are waited for after the local partial only
        covered = []
        for i, (kv, row0, skv, base, ns) in enumerate(ops.calls):
            if i == 0 and use_local:
                assert kv is local and row0 == 0
                row0 = rank * mx
            else:
                assert kv.data_ptr() == kvx.buf.data_ptr()
            covered += list(range(row0, row0 + skv))
        real = [p * mx + j for p in range(len(rows)) for j in range(rows[p])]
        assert sorted(covered) == real               # every real row exactly once, no padding row
        assert covered[:rows[rank]] == list(range(rank * mx, rank * mx + rows[rank]))   # local rows first
        assert n_parts == sum(c[4] for c in ops.calls) and [c[3] for c in ops.calls] == list(
            itertools.accumulate([0] + [c[4] for c in ops.calls[:-1]]))


@pytest.mark.parametrize("world,sl", [(2, 36), (3, 736), (4, 1024), (8, 4600)])
def test_overlapped_ranges_equal_rows_unchanged(world, sl):
    """Equal rows: the local range, then the ranks before and the ranks after it as one range each (the launches of
    single-resolution runs)."""
    from fast3r_b200.parallel import peer_key_ranges
    S = world * sl
    for rank in range(world):
        lo, hi = rank * sl, (rank + 1) * sl
        today = [(lo, sl)] + [r for r in ((0, lo), (hi, S - hi)) if r[1] > 0]
        assert peer_key_ranges([sl] * world, rank) == today
        ops = _RecordingOps()
        _partials(_exchange([sl] * world, rank), ops, torch.zeros(sl, 128, dtype=torch.bfloat16), None)
        assert [(row0, skv) for _, row0, skv, _, _ in ops.calls] == today


@pytest.mark.parametrize("rows", [[36, 30], [130, 70, 200]])
def test_overlapped_partials_equal_attention_over_all_keys(rows):
    """The emulated partials over the padded gather buffer merged by log-sum-exp equal one attention over the
    concatenated real keys (padding filled with garbage that must not be read)."""
    from tests import abi_emulator as E
    from fast3r_b200.parallel import assemble_kv
    heads, mx = 2, max(rows)
    D = heads * 64
    g = torch.Generator().manual_seed(5)
    for rank in range(len(rows)):
        kvx = _exchange(rows, rank)
        kvx.buf = torch.full((len(rows), mx, 2 * D), 1e4).bfloat16()
        for p, n in enumerate(rows):
            kvx.buf[p, :n] = torch.randn(n, 2 * D, generator=g).bfloat16()
        q = torch.randn(rows[rank], D, generator=g).bfloat16()
        n_parts, _ = _partials(kvx, E, q, None)
        out, ref = torch.zeros(rows[rank], D).bfloat16(), torch.zeros(rows[rank], D).bfloat16()
        E.attention_merge(kvx.parts[0], kvx.parts[1], n_parts, out, batch=1, heads=heads, sq=rows[rank])
        E.attention(q, assemble_kv(kvx.buf, 1, rows), ref, batch=1, heads=heads, sq=rows[rank], skv=sum(rows), scale=0.2)
        assert rel_l2(out.float(), ref.float()) < 6e-3


def test_overlapped_path_selection():
    """Batch 1 in bf16 takes the overlapped path with equal rows, and with uneven rows when the views have mixed
    resolutions; views of one resolution in uneven shards keep the all-gather path (bit-identical to one device)."""
    from fast3r_b200.parallel import KVExchange
    sp, cuda = SimpleNamespace(rank=0, world=2, overlap=True), torch.device("cuda")
    assert KVExchange(sp, 1, 72, 128, [72, 72]).fast(torch.bfloat16, cuda)
    assert not KVExchange(sp, 1, 72, 128, [72, 48]).fast(torch.bfloat16, cuda)
    assert KVExchange(sp, 1, 72, 128, [72, 48], mixed=True).fast(torch.bfloat16, cuda)
    assert not KVExchange(sp, 2, 72, 128, [72, 48], mixed=True).fast(torch.bfloat16, cuda)
    assert not KVExchange(sp, 1, 72, 128, [72, 48], mixed=True).fast(torch.float32, cuda)
