"""Launch plans of the attention kernels, for the tests: the plan key of a call, computed with the library's own host
rules, and the table of GPU cases that tests/test_attention_plans_gpu.py runs and tests/test_attention_plans_cpu.py checks
the forward against.

A call is described by a plain dict ("descriptor") with the arguments of one C-ABI entry point:
  entry "attention"  f3r_attention: batch, heads, sq, skv, ldo, lse (bool)
  entry "partial"    f3r_attention_partial: batch, heads, sq, skv, kv_rows_total, kv_row0, n_split, part_base
  entry "segments"   f3r_attention_segments: offsets (host list), heads, n_split, ldo, part (bool: key-slice partials)
  entry "x3"         f3r_attention_x3: batch, heads, sq, skv, ldo, lse (bool)
  entry "merge"      f3r_attention_merge: n_parts, batch, heads, sq, ldo

The plan key names the code path a call takes in attention_kernel<kSeg>, attention_x3_kernel and
attention_merge_kernel: the entry point; the last query tile (how many of the 64-row consumer warpgroups hold rows of
it, and whether it is full); the key blocks of the smallest and the largest key slice, as classes of the shared-memory
ring (bf16: 3 stages, x3: 2 stages); the last key block of the range (full, one valid key, or another partial count); the
key range (kv_row0 > 0, rows of the buffer after the range, batch > 1); the key split (one slice, an even or an uneven
partition); for segments, a segment with fewer key blocks than the split (neutral partials), one shorter than a key
block, and one whose start is not a multiple of the query tile; and a row stride of the output wider than heads * 64.
A segments call has one key per segment; the other calls have one key."""
from fast3r_b200 import ops

KB = 128                     # keys per key block (both kernels)
BF16_TILE = ops.ATT_Q_TILE   # 192 query rows = 3 consumer warpgroups
X3_TILE = 128                # 128 query rows = 2 consumer warpgroups


def _cdiv(a, b):
    return -(-a // b)


def _kb_class(n, x3):
    """Key blocks of one slice as a class of the smem ring: bf16 (3 stages) 1, 2, 3, 4-6, 7+; x3 (2 stages) 1, 2, 3-4, 5+."""
    if x3:
        return str(n) if n <= 2 else "3-4" if n <= 4 else "5+"
    return str(n) if n <= 3 else "4-6" if n <= 6 else "7+"


def _tile(sq, tile):
    r = sq - (_cdiv(sq, tile) - 1) * tile
    return f"tile{_cdiv(r, 64)}/{tile // 64}" + ("" if r == tile else "p")


def _last_block(skv):
    v = skv - (_cdiv(skv, KB) - 1) * KB
    return "full" if v == KB else "one" if v == 1 else "part"


def slices(nkv, n_split):
    """(first key block, key blocks) of each slice: the kernel's partition j0 = s * nkv / n_split."""
    return [(s * nkv // n_split, (s + 1) * nkv // n_split - s * nkv // n_split) for s in range(n_split)]


def _blocks(skv, n_split, x3=False):
    nkv = _cdiv(skv, KB)
    sizes = [n for _, n in slices(nkv, n_split)]
    lo, hi = _kb_class(min(sizes), x3), _kb_class(max(sizes), x3)
    split = "1" if n_split == 1 else "even" if nkv % n_split == 0 else "uneven"
    return f"kb:{lo}" + ("" if lo == hi else f"..{hi}") + f" last:{_last_block(skv)} split:{split}"


def _flags(*pairs):
    return "".join(" " + f for f, on in pairs if on)


def plan_keys(d):
    """Sorted list of the plan keys of descriptor d (one per segment for a segments call, else one)."""
    e = d["entry"]
    heads = d["heads"]
    wide = d.get("ldo", heads * 64) > heads * 64
    if e == "merge":
        return [f"merge parts:{d['n_parts']}" + _flags(("batch", d["batch"] > 1), ("ldo", wide))]
    if e == "x3":
        return [("x3+lse" if d["lse"] else "x3") + f" {_tile(d['sq'], X3_TILE)} "
                + _blocks(d["skv"], 1, x3=True) + _flags(("batch", d["batch"] > 1), ("ldo", wide))]
    if e == "segments":
        keys = set()
        off = d["offsets"]
        for a, b in zip(off, off[1:]):
            n = b - a
            if n == 0:
                continue  # no query tile, no work item
            ns = min(d["n_split"], _cdiv(n, KB))
            keys.add(("seg+part" if d["part"] else "seg") + f" {_tile(n, BF16_TILE)} " + _blocks(n, ns)
                     + _flags(("neutral", ns < d["n_split"]), ("short", n < KB), ("unaligned", a % BF16_TILE != 0),
                              ("ldo", wide and not d["part"])))
        return sorted(keys)
    if e == "attention":
        head, row0, total, ns = "attn+lse" if d["lse"] else "attn", 0, d["skv"], 1
    else:
        head, row0, total, ns = "partial", d["kv_row0"], d["kv_rows_total"], d["n_split"]
    return [f"{head} {_tile(d['sq'], BF16_TILE)} " + _blocks(d["skv"], ns)
            + _flags(("row0", row0 > 0), ("tail", total > row0 + d["skv"]), ("batch", d["batch"] > 1),
                     ("ldo", e == "attention" and wide))]


# ------------------------------------------------------------------------------------------------------ the case table
# A case is a dict: name, kind, keys (the plan keys its calls reach, sorted), and the fields of its kind:
#   "attention"  batch, heads, sq, skv, ldo, lse, scale                         one f3r_attention
#   "split"      batch, heads, sq, kv_rows_total, ranges [(kv_row0, skv, n_split)], base (slots before the first),
#                ldo, scale, direct (also one f3r_attention over the whole buffer)
#                f3r_attention_partial per range into consecutive slots from `base`, then f3r_attention_merge of them
#   "segments"   offsets, heads, n_split, ldo, scale                           f3r_attention_segments (n_split > 1:
#                partials into one slot per slice, then f3r_attention_merge, as ops.attention_segments)
#   "x3"         batch, heads, sq, skv, ldo, lse, scale                         one f3r_attention_x3
#   "merge"      n_parts, batch, heads, sq, ldo, neutral (slots that hold neutral partials, LSE = -inf), holes (slots
#                that are neutral in every other row)                           f3r_attention_merge of given partials
DEFAULT_SCALE = 0.125


def case_calls(c):
    """Descriptors of the calls that case c makes, in order."""
    k = c["kind"]
    if k == "attention":
        return [dict(entry="attention", batch=c["batch"], heads=c["heads"], sq=c["sq"], skv=c["skv"], ldo=c["ldo"],
                     lse=c["lse"])]
    if k == "x3":
        return [dict(entry="x3", batch=c["batch"], heads=c["heads"], sq=c["sq"], skv=c["skv"], ldo=c["ldo"], lse=c["lse"])]
    if k == "merge":
        return [dict(entry="merge", n_parts=c["n_parts"], batch=c["batch"], heads=c["heads"], sq=c["sq"], ldo=c["ldo"])]
    if k == "segments":
        part = c["n_split"] > 1
        out = [dict(entry="segments", offsets=c["offsets"], heads=c["heads"], n_split=c["n_split"], ldo=c["ldo"],
                    part=part)]
        if part:
            out.append(dict(entry="merge", n_parts=c["n_split"], batch=1, heads=c["heads"], sq=c["offsets"][-1],
                            ldo=c["ldo"]))
        return out
    out, base = [], c["base"]
    for row0, skv, ns in c["ranges"]:
        out.append(dict(entry="partial", batch=c["batch"], heads=c["heads"], sq=c["sq"], skv=skv,
                        kv_rows_total=c["kv_rows_total"], kv_row0=row0, n_split=ns, part_base=base))
        base += ns
    out.append(dict(entry="merge", n_parts=base - c["base"], batch=c["batch"], heads=c["heads"], sq=c["sq"],
                    ldo=c["ldo"]))
    if c["direct"]:
        out.append(dict(entry="attention", batch=c["batch"], heads=c["heads"], sq=c["sq"], skv=c["kv_rows_total"],
                        ldo=c["ldo"], lse=True))
    return out


def case_keys(c):
    return sorted({k for d in case_calls(c) for k in plan_keys(d)})


def _case(name, kind, keys, **f):
    c = dict(name=name, kind=kind, keys=sorted(keys), batch=1, heads=2, ldo=None, lse=False, scale=DEFAULT_SCALE,
             base=0, direct=False, neutral=(), holes=())
    unknown = set(f) - set(c) - {"sq", "skv", "kv_rows_total", "ranges", "offsets", "n_split", "n_parts", "qscale"}
    assert not unknown, unknown
    c.update(f)
    if c["ldo"] is None:
        c["ldo"] = c["heads"] * 64
    return c


def attn(name, keys, **f):
    return _case(name, "attention", keys, **f)


def split(name, keys, **f):
    return _case(name, "split", keys, **f)


def seg(name, keys, **f):
    return _case(name, "segments", keys, **f)


def x3(name, keys, **f):
    return _case(name, "x3", keys, **f)


def merge(name, keys, **f):
    return _case(name, "merge", keys, **f)


# ---- one reduced case per plan key of the forward (tests/test_attention_plans_cpu.py records them): ViT-L at 368x512
# (N=32, N=4, N=320) and 512x368 in bf16 and fp32, forward_many, and the sequence-parallel attention of N=32 on 2, 4 and
# 8 ranks, of N=320 and N=1000 on 8 ranks and of mixed resolutions on 3 ranks (KVExchange.partials and the merge; the
# parity path's all-gather attention_x3)
T1, T2, T3 = 193, 320, 384          # last query tile: 1, 2 or 3 (full) warpgroups with rows
K7, K7P = 7 * 128, 7 * 128 + 40     # key blocks 7+: last block full / partial
FORWARD = [
    attn("fwd_attn_t1_k7", ["attn tile1/3p kb:7+ last:full split:1"], sq=T1, skv=K7),
    attn("fwd_attn_t2_k7", ["attn tile2/3p kb:7+ last:full split:1"], sq=T2, skv=K7),
    attn("fwd_attn_t3_k4", ["attn tile3/3 kb:4-6 last:full split:1"], sq=T3, skv=512),
    attn("fwd_attn_t3_k6_batch", ["attn tile3/3 kb:4-6 last:full split:1 batch"], batch=2, sq=192, skv=768),
    attn("fwd_attn_t3p_k5", ["attn tile3/3p kb:4-6 last:part split:1"], sq=330, skv=600),
    attn("fwd_attn_736_batch", ["attn tile3/3p kb:4-6 last:part split:1 batch"], batch=2, sq=736, skv=736),
    # KVExchange: the local range (whole buffer, or the rank's slot: tail), the ranks after (row0), and a middle rank's
    # three ranges, merged
    split("fwd_sp_t1_local", ["merge parts:1", "partial tile1/3p kb:7+ last:full split:1"],
          sq=T1, kv_rows_total=K7, ranges=[(0, K7, 1)]),
    split("fwd_sp_t1_rank0", ["merge parts:2", "partial tile1/3p kb:7+ last:full split:1 row0",
                              "partial tile1/3p kb:7+ last:full split:1 tail"],
          sq=T1, kv_rows_total=2 * K7, ranges=[(0, K7, 1), (K7, K7, 1)]),
    split("fwd_sp_t1_rank1", ["merge parts:3", "partial tile1/3p kb:7+ last:full split:1 row0",
                              "partial tile1/3p kb:7+ last:full split:1 row0 tail",
                              "partial tile1/3p kb:7+ last:full split:1 tail"],
          sq=T1, kv_rows_total=4 * K7, ranges=[(K7, K7, 1), (0, K7, 1), (2 * K7, 2 * K7, 1)]),
    split("fwd_sp_t2_local", ["merge parts:1", "partial tile2/3p kb:7+ last:full split:1"],
          sq=T2, kv_rows_total=K7, ranges=[(0, K7, 1)]),
    split("fwd_sp_t2_rank1", ["merge parts:3", "partial tile2/3p kb:7+ last:full split:1 row0",
                              "partial tile2/3p kb:7+ last:full split:1 row0 tail",
                              "partial tile2/3p kb:7+ last:full split:1 tail"],
          sq=T2, kv_rows_total=4 * K7, ranges=[(K7, K7, 1), (0, K7, 1), (2 * K7, 2 * K7, 1)]),
    split("fwd_sp_t1p_local", ["merge parts:1", "partial tile1/3p kb:7+ last:part split:1"],
          sq=T1, kv_rows_total=K7P, ranges=[(0, K7P, 1)]),
    split("fwd_sp_t1p_rank1", ["merge parts:3", "partial tile1/3p kb:7+ last:part split:1 row0",
                               "partial tile1/3p kb:7+ last:part split:1 row0 tail",
                               "partial tile1/3p kb:7+ last:part split:1 tail"],
          sq=T1, kv_rows_total=4 * K7P, ranges=[(K7P, K7P, 1), (0, K7P, 1), (2 * K7P, 2 * K7P, 1)]),
    # mixed resolutions: slots of max(rows) rows, the last rank's slot padded (NaN rows that must not be read)
    split("fwd_sp_mixed_rank0", ["merge parts:3", "partial tile3/3 kb:7+ last:full split:1 row0 tail",
                                 "partial tile3/3 kb:7+ last:part split:1 row0 tail",
                                 "partial tile3/3 kb:7+ last:part split:1 tail"],
          sq=T3, kv_rows_total=3 * K7P, ranges=[(0, K7P, 1), (K7P, K7P, 1), (2 * K7P, K7, 1)]),
    split("fwd_sp_mixed_local", ["merge parts:1", "partial tile3/3 kb:7+ last:part split:1"],
          sq=T3, kv_rows_total=K7P, ranges=[(0, K7P, 1)]),
    split("fwd_sp_mixed_rank2", ["merge parts:3", "partial tile1/3p kb:7+ last:full split:1 row0 tail", "partial tile1/3p kb:7+ last:full split:uneven tail"],
          sq=T1, kv_rows_total=3 * 1920, ranges=[(3840, K7, 1), (0, 15 * 128, 2)]),
    # forward_many: one aligned segment, then segments that start 64 rows into a query tile
    seg("fwd_seg_scenes", ["seg tile1/3p kb:7+ last:full split:1", "seg tile3/3 kb:4-6 last:full split:1 unaligned",
                           "seg tile3/3 kb:7+ last:full split:1 unaligned"],
        offsets=[0, 1024, 1792, 2944], n_split=1),
    x3("fwd_x3_t1_k5", ["x3 tile1/2p kb:5+ last:full split:1"], sq=129, skv=640),
    x3("fwd_x3_t2_k5", ["x3 tile2/2 kb:5+ last:full split:1"], sq=256, skv=640),
    x3("fwd_x3_t2_k5_batch", ["x3 tile2/2 kb:5+ last:full split:1 batch"], batch=2, sq=128, skv=768),
    x3("fwd_x3_t2p_k6", ["x3 tile2/2p kb:5+ last:part split:1"], sq=200, skv=700),
    x3("fwd_x3_736_batch", ["x3 tile2/2p kb:5+ last:part split:1 batch"], batch=2, sq=736, skv=736),
]

# ---- the contract beyond the forward: every ring class, one valid key, lse, key slices even and uneven with and
# without part_base, segments with neutral partials, short and unaligned segments, wider ldo, merges of 1 to 8 parts
CONTRACT = [
    attn("lse_k1_one", ["attn+lse tile1/3p kb:1 last:one split:1"], sq=64, skv=1, lse=True),
    attn("lse_k2_part", ["attn+lse tile2/3p kb:2 last:part split:1"], sq=100, skv=200, lse=True),
    attn("lse_k3_full_ldo", ["attn+lse tile3/3 kb:3 last:full split:1 ldo"], sq=192, skv=384, lse=True, ldo=192),
    attn("lse_k4_one", ["attn+lse tile1/3p kb:4-6 last:one split:1 batch"], batch=2, sq=193, skv=385, lse=True),
    attn("lse_k7_one_ldo", ["attn+lse tile3/3p kb:7+ last:one split:1 ldo"], sq=150, skv=769, lse=True, ldo=136),
    attn("attn_k2_one", ["attn tile1/3p kb:2 last:one split:1"], sq=10, skv=129),
    split("slices_even_base", ["merge parts:3", "partial tile3/3 kb:3 last:full split:even"],
          sq=192, kv_rows_total=9 * 128, ranges=[(0, 9 * 128, 3)], base=2),
    split("slices_uneven_lse_base", ["merge parts:3 batch ldo", "partial tile2/3p kb:2..3 last:one split:uneven batch"],
          batch=2, sq=100, kv_rows_total=6 * 128 + 1, ranges=[(0, 6 * 128 + 1, 3)], base=1, ldo=192),
    split("slices_k1", ["merge parts:4", "partial tile1/3p kb:1 last:part split:even row0 tail"],
          sq=30, kv_rows_total=700, ranges=[(100, 500, 4)]),
    split("slices_k1_k4", ["merge parts:5", "partial tile2/3p kb:1..2 last:part split:uneven row0", "partial tile2/3p kb:4-6 last:full split:1 tail"],
          sq=128, kv_rows_total=1140, ranges=[(0, 512, 1), (512, 628, 4)]),
    split("slices_k7_uneven_8", ["merge parts:8", "partial tile1/3p kb:7+ last:part split:uneven row0 tail"],
          sq=250, kv_rows_total=8000, ranges=[(77, 7500, 8)]),
    seg("seg_neutral_short", ["merge parts:3", "seg+part tile1/3p kb:1..2 last:part split:uneven unaligned", "seg+part tile2/3p kb:1 last:part split:1 neutral short", "seg+part tile3/3p kb:3..4-6 last:part split:uneven unaligned"],
        offsets=[0, 100, 700, 700, 2000], n_split=3),
    seg("seg_neutral_one", ["merge parts:2", "seg+part tile1/3p kb:1 last:one split:1 neutral short unaligned", "seg+part tile2/3p kb:1..2 last:part split:uneven unaligned", "seg+part tile3/3p kb:1 last:one split:even"],
        offsets=[0, 129, 130, 430], n_split=2),
    seg("seg_ldo_short", ["seg tile1/3p kb:1 last:one split:1 short ldo", "seg tile1/3p kb:1 last:part split:1 short unaligned ldo", "seg tile3/3 kb:3 last:full split:1 unaligned ldo"],
        offsets=[0, 1, 65, 449], n_split=1, ldo=192),
    x3("x3_lse_k1_one", ["x3+lse tile1/2p kb:1 last:one split:1"], sq=1, skv=1, lse=True),
    x3("x3_lse_k2_ldo", ["x3+lse tile2/2p kb:2 last:part split:1 ldo"], sq=100, skv=250, lse=True, ldo=136),
    x3("x3_k3_one_batch", ["x3 tile1/2p kb:3-4 last:one split:1 batch"], batch=2, sq=129, skv=257),
    x3("x3_lse_k4_full", ["x3+lse tile2/2 kb:3-4 last:full split:1"], sq=128, skv=512, lse=True),
] + [
    merge(f"merge_{n}", [f"merge parts:{n}" + (" batch" if n % 2 else "") + (" ldo" if n > 4 else "")],
          n_parts=n, batch=1 + n % 2, sq=150 + n, ldo=128 + 64 * (n > 4), neutral=(n - 1,) if n > 1 else (),
          holes=(0,) if n > 2 else ())
    for n in range(1, 9)
]

# ---- the earlier relative-L2 attention checks (tests/kernel_checks.py runs them under these names)
S2 = 0.16019
KERNEL_CHECKS = [
    attn("attn_736_b2h2", ["attn+lse tile3/3p kb:4-6 last:part split:1 batch"], batch=2, sq=736, skv=736, lse=True),
    attn("attn_128", ["attn+lse tile2/3p kb:1 last:full split:1"], heads=1, sq=128, skv=128, lse=True),
    attn("attn_256x384", ["attn+lse tile1/3p kb:3 last:full split:1"], sq=256, skv=384, lse=True),
    attn("attn_tails_1000", ["attn+lse tile1/3p kb:7+ last:part split:1"], heads=3, sq=1000, skv=1000, lse=True,
         scale=S2),
    attn("attn_24", ["attn+lse tile1/3p kb:1 last:part split:1 batch"], batch=3, sq=24, skv=24, lse=True),
    attn("attn_long_3072", ["attn+lse tile2/3p kb:7+ last:full split:1"], sq=512, skv=3072, lse=True, scale=S2),
    attn("attn_peaky", ["attn+lse tile2/3p kb:7+ last:full split:1"], sq=512, skv=2048, lse=True, scale=0.5,
         qscale=3.0),
    attn("attn_q9tiles_oddpair", ["attn+lse tile3/3p kb:7+ last:part split:1"], sq=2300, skv=1000, lse=True, scale=S2),
    split("attn_ranges_merge", ["merge parts:6", "partial tile2/3p kb:3 last:part split:even tail", "partial tile2/3p kb:4-6 last:part split:1 row0 tail", "partial tile2/3p kb:4-6 last:part split:even row0"],
          sq=700, kv_rows_total=2944, ranges=[(736, 736, 1), (0, 736, 2), (1472, 1472, 3)], scale=S2),
    split("attn_ranges_merge_rank0", ["merge parts:3", "partial tile2/3p kb:4-6 last:part split:1 tail", "partial tile2/3p kb:4-6 last:part split:even row0"],
          sq=300, kv_rows_total=1500, ranges=[(0, 500, 1), (500, 1000, 2)], scale=S2),
    split("attn_autosplit", ["attn+lse tile1/3p kb:7+ last:part split:1", "merge parts:2", "partial tile1/3p kb:7+ last:part split:even"],
          heads=4, sq=600, kv_rows_total=4000, ranges=[(0, 4000, 2)], scale=S2, direct=True),
    split("attn_skv235520_slices", ["attn+lse tile3/3 kb:7+ last:full split:1", "merge parts:4",
                                    "partial tile3/3 kb:7+ last:full split:even"],
          heads=1, sq=192, kv_rows_total=235520, ranges=[(0, 235520, 4)], scale=S2, direct=True),
    attn("attn_skv23552", ["attn+lse tile2/3p kb:7+ last:full split:1"], sq=512, skv=23552, lse=True, scale=S2),
    attn("attn_skv23552_peaky", ["attn+lse tile1/3p kb:7+ last:full split:1"], heads=1, sq=256, skv=23552, lse=True,
         scale=0.5, qscale=3.0),
    x3("x3_attn_tails", ["x3+lse tile1/2p kb:5+ last:part split:1 batch"], batch=2, sq=300, skv=736, lse=True, scale=S2),
    x3("x3_attn_128", ["x3+lse tile2/2 kb:1 last:full split:1"], heads=1, sq=128, skv=128, lse=True),
    x3("x3_attn_peaky_long", ["x3+lse tile2/2 kb:5+ last:full split:1"], sq=256, skv=4096, lse=True, scale=0.5,
       qscale=3.0),
    # pipeline edges: the prologue, the steady-state trip and the PV-only last block with short key ranges
    attn("attn_skv200", ["attn+lse tile2/3p kb:2 last:part split:1"], sq=300, skv=200, lse=True, scale=S2),
    attn("attn_skv129", ["attn+lse tile3/3p kb:2 last:one split:1 batch"], batch=2, heads=1, sq=130, skv=129, lse=True,
         scale=S2),
    attn("attn_skv256", ["attn+lse tile1/3p kb:2 last:full split:1"], sq=256, skv=256, lse=True),
    attn("attn_skv385_peaky", ["attn+lse tile1/3p kb:4-6 last:one split:1"], sq=200, skv=385, lse=True, scale=0.5,
         qscale=3.0),
    split("attn_ranges_skv200", ["merge parts:3", "partial tile2/3p kb:1 last:part split:even row0",
                                 "partial tile2/3p kb:2 last:part split:1 tail"],
          sq=300, kv_rows_total=400, ranges=[(0, 200, 1), (200, 200, 2)], scale=S2),
    split("attn_ranges_skv330", ["merge parts:6", "partial tile2/3p kb:1 last:part split:even row0",
                                 "partial tile2/3p kb:1..2 last:part split:uneven tail",
                                 "partial tile2/3p kb:3 last:part split:1 row0 tail"],
          sq=300, kv_rows_total=990, ranges=[(330, 330, 1), (0, 330, 2), (660, 330, 3)], scale=S2),
    # query tiles: one row in the last tile's first warpgroup, one row in its third, whole tiles
    split("attn_sq193_ranges", ["merge parts:3", "partial tile1/3p kb:1 last:part split:even tail",
                                "partial tile1/3p kb:2 last:part split:1 row0"],
          sq=193, kv_rows_total=400, ranges=[(200, 200, 1), (0, 200, 2)], scale=S2),
    attn("attn_sq321", ["attn+lse tile3/3p kb:3 last:part split:1 batch"], batch=2, sq=321, skv=300, lse=True, scale=S2),
    attn("attn_sq384", ["attn+lse tile3/3 kb:3 last:full split:1"], sq=384, skv=384, lse=True),
]

CASES = FORWARD + CONTRACT + KERNEL_CHECKS
