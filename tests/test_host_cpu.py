"""CPU-side checks: key schema, RNG stream, loud failure without CUDA, collation helpers and the sequence-parallel host
logic over a 2-rank gloo group."""
import os
import socket

import numpy as np
import pytest
import torch


def test_state_dict_schema_matches_reference(golden_dir):
    from fast3r_b200 import Fast3R, tiny_args
    g = torch.load(os.path.join(golden_dir, "tiny_b1_n3.pt"))
    m = Fast3R(*tiny_args())
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == g["shapes"]


def test_vitl_param_count():
    from fast3r_b200 import Fast3R, vit_large_args
    with torch.device("meta"):
        m = Fast3R(*vit_large_args())
    n = sum(p.numel() for p in m.parameters())
    assert abs(n / 1e6 - 647.55) < 0.01, n  # SURVEY.md §6: 647.55 M params
    assert len(m.state_dict()) == 720  # SURVEY.md §8(b)


def test_image_id_rng_stream_matches_reference(golden_dir):
    from fast3r_b200 import Fast3R, tiny_args
    g = torch.load(os.path.join(golden_dir, "tiny_b1_n3.pt"))
    m = Fast3R(*tiny_args())
    torch.manual_seed(g["rng_seed"])
    assert torch.equal(m.decoder.draw_image_ids(g["B"], g["N"]), g["image_ids"])
    from oracle.fast3r_oracle import image_idx_table
    assert torch.equal(m.decoder.image_idx_emb, image_idx_table(128))


def test_image_ids_at_the_1000_view_limit():
    """N = 1000 is the model's maximum (image-index table has 1000 rows, fast3r/models/fast3r.py:694,742)."""
    from fast3r_b200 import Fast3R, tiny_args
    from oracle.fast3r_oracle import draw_image_ids
    m = Fast3R(*tiny_args())
    torch.manual_seed(3)
    a = m.decoder.draw_image_ids(2, 1000)
    torch.manual_seed(3)
    b = draw_image_ids(2, 1000)
    assert torch.equal(a, b) and a.shape == (2, 1000)
    assert sorted(a[0].tolist()) == list(range(1000))  # a permutation: every table row used exactly once
    with pytest.raises(RuntimeError):
        m.decoder.draw_image_ids(1, 1001)              # like the reference: randperm(999) cannot fill 1000 slots


def test_no_cpu_fallback():
    from fast3r_b200 import Fast3R, tiny_args
    m = Fast3R(*tiny_args()).eval()
    views = [dict(img=torch.zeros(1, 3, 32, 32)) for _ in range(2)]
    with pytest.raises(RuntimeError, match="CUDA"):
        m(views)
    from fast3r_b200 import ops
    with pytest.raises(RuntimeError):
        ops.cast_bf16(torch.zeros(8), torch.zeros(8, dtype=torch.bfloat16))


def test_training_step_fails_loudly():
    from fast3r_b200 import Fast3R, tiny_args
    m = Fast3R(*tiny_args()).train()
    with pytest.raises(NotImplementedError, match="backward"):
        m([dict(img=torch.zeros(1, 3, 32, 32))])


def test_collate_like_reference():
    from fast3r_b200.inference import collate_with_cat, to_cpu, check_if_same_size
    views = [dict(img=torch.zeros(1, 3, 16, 32), true_shape=np.int32([[16, 32]]), idx=i, instance=str(i))
             for i in range(3)]
    assert check_if_same_size(views)
    batch = collate_with_cat([tuple(views)])
    assert isinstance(batch, list) and len(batch) == 3
    assert torch.is_tensor(batch[0]["true_shape"]) and batch[0]["true_shape"].shape == (1, 2)
    assert batch[1]["idx"] == [1] and batch[2]["instance"] == ["2"]
    res = collate_with_cat([to_cpu(dict(views=list(batch), preds=[dict(conf=torch.ones(1, 16, 32))] * 3, loss=None))])
    assert res["loss"] is None and len(res["preds"]) == 3


def test_shard_views_and_assemble():
    from fast3r_b200.parallel import shard_views, assemble_kv
    assert shard_views(1000, 8) == [(i * 125, (i + 1) * 125) for i in range(8)]
    assert shard_views(5, 2) == [(0, 3), (3, 5)]
    B, C = 2, 4
    rows = [3, 2]
    full = torch.arange(B * 5 * C, dtype=torch.float32).view(B, 5, C)
    g = torch.zeros(2, B * 3, C)
    g[0].view(B, 3, C)[:, :3] = full[:, :3]
    g[1].view(B, 3, C)[:, :2] = full[:, 3:]
    assert torch.equal(assemble_kv(g, B, rows), full.reshape(-1, C))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _sp_worker(rank, world, port, n_views, batch, tok, C, ret):
    import torch.distributed as dist
    from fast3r_b200.parallel import SequenceParallel
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    sp = SequenceParallel(gather_preds=True)
    lo, hi = sp.view_range(n_views)
    full = torch.arange(batch * n_views * tok * C, dtype=torch.float32).view(batch, n_views * tok, C)
    local = full[:, lo * tok:hi * tok].contiguous().view(-1, C)
    kvx = sp.make_kv_exchange(batch, (hi - lo) * tok, C // 2)
    seen = {}

    class FakeOps:  # the general path hands the assembled K|V of ALL ranks to one attention call
        @staticmethod
        def attention(q, kv_all, att, *, batch, heads, sq, skv, scale):
            seen.update(kv=kv_all, skv=skv, sq=sq, batch=batch)

    kvx.attend(FakeOps, None, local, None, heads=1, scale=1.0, x3=False)
    ok = seen["skv"] == n_views * tok and seen["sq"] == (hi - lo) * tok and torch.equal(seen["kv"], full.reshape(-1, C))
    # result gathering
    fr = [dict() for _ in range(n_views)]
    for i in range(lo, hi):
        fr[i]["conf"] = torch.full((batch, 2, 3), float(i))
    out = sp.gather_results(fr, n_views, batch, 2, 3, torch.device("cpu"))
    ok = ok and all(float(out[i]["conf"].mean()) == float(i) for i in range(n_views))
    ret[rank] = bool(ok)
    dist.destroy_process_group()


@pytest.mark.parametrize("n_views,batch", [(4, 1), (5, 2)])
def test_sequence_parallel_host_logic_gloo(n_views, batch):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    port = _free_port()
    procs = [ctx.Process(target=_sp_worker, args=(r, 2, port, n_views, batch, 3, 4, ret)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
    assert dict(ret) == {0: True, 1: True}


def test_pick_kv_split_invariants():
    """ops.pick_kv_split: key slicing only when it fills more of the 132 SMs, every slice keeps >= 16 key blocks, and the
    decoder shapes of the sequence-parallel runs (16 heads, 192-row query tiles) map to fixed choices."""
    from fast3r_b200.ops import pick_kv_split, NUM_SMS
    for units in (1, 16, 64, 132, 192, 368, 395, 396, 736, 1472, 23552):
        for blocks in (1, 6, 15, 16, 23, 32, 92, 184, 1840):
            s = pick_kv_split(units, blocks)
            assert 1 <= s <= 8
            assert s == 1 or blocks // s >= 16
            if units >= 3 * NUM_SMS:
                assert s == 1
            waves = lambda k: -(-units * k // NUM_SMS) / k  # noqa: E731
            assert waves(s) <= waves(1) + 1e-9            # never worse than one slice
    assert pick_kv_split(192, 184) == 2      # 2 waves at 73 % -> 3 waves of halves at 97 %
    assert pick_kv_split(368, 184) == 5      # 3 waves at 93 % -> 14 waves of fifths at 99.6 %
    assert pick_kv_split(1472, 184) == 1     # 12 waves: never sliced (>= 3 waves)
    assert pick_kv_split(192, 23) == 1       # N=4: slices would be too short
