"""Segments whose filter survivors are designed slice by slice, for the survivor paths of the scan kernel
(pinot_b200/csrc/pb200_scan.cuh): the GROUP BY survivor queue and its pipelined last batch, the aggregation-only deferred
gathers, per-row probing of later filter leaves, bitmap-skipped slices and the flushes at segment changes and at exit.

Geometry.  A slice is 1024 segment rows, 1024-aligned whatever the warps per CTA (W) and the grid; lane l of the warp that
handles slice i owns rows i * 1024 + 32 l .. + 31.  CTA tile T holds slices T * W .. T * W + W - 1 (warp w: slice
T * W + w), so under `grid` 1 warp w sees slices w, W + w, 2 W + w, ... in consecutive tiles.

Columns (every segment):
  p1     INT, values 0..3: 1 on the designed rows and on the decoys, else 0, 2 or 3;
  p2     INT, values 0..1: 1 on the designed rows, 0 on the decoys, else random.  `p1 = 1 AND p2 = 1` matches exactly the
         designed rows; the planner runs the p1 leaf first (1 of 4 dictIds against 1 of 2), so a slice's decoys set the
         warp's per-lane maximum that the p2 leaf sees (per-row probing when it is <= sparse_max);
  inv    INT with an inverted index: 1 on every row of the skipped slices (and on one row that survives nothing), else 0;
         `inv = 0` leaves the skipped slices without a doc, so the bitmap skips them;
  k24, kb, k70  group keys over 24, 10 000 and 70 000 values (every segment with enough rows holds all of them, so
         segments merge by dictId);
  rid, blk = rid // 16, bit = 1 << (rid % 16): SUM(bit) GROUP BY blk is each 16-row block's exact match mask;
  v      INT with INT_MIN and INT_MAX, r the same kind of values kept raw, f FLOAT (quarters: exact in double),
  l      LONG (positive, sums above 2^53)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Sequence

import numpy as np

SLICE = 1024
LANES = 32
INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
S_EDGES = [0, 1, 2, 3, 4, 5, 31, 32, 33, 127, 128, 129, 255, 256, 257, 383, 384, 385, 511, 512, 513, 1023, 1024]
NONZERO = [s for s in S_EDGES if s]
KEY_SPACES = {"k24": 24, "kb": 10_000, "k70": 70_000}
# per-lane maxima after the first leaf that the decoys produce: on both sides of sparse_max (4) and sparse_max_agg
# (4; 2 for GROUP BY), and none
DECOY_PRE = [0, 4, 5, 2, 3, 32, 1]


@dataclass(frozen=True)
class Slice:
    s: int                  # designed survivors
    layout: str = "packed"  # packed | spread | one_lane
    pre: int = 0            # per-lane count after the first leaf: decoys fill every lane below it up to it
    skipped: bool = False   # inv = 1 on every row: `inv = 0` skips the slice
    lane: int = 7           # one_lane: the lane holding the rows


def layouts_for(s: int) -> List[str]:
    return ["packed", "spread", "one_lane"] if s <= LANES else ["packed", "spread"]


def all_items() -> List[Slice]:
    """Every S edge in every layout it has (one-lane: S <= 32)."""
    return [Slice(s, lay) for s in S_EDGES for lay in layouts_for(s)]


def designed_offsets(sl: Slice, rows: int) -> np.ndarray:
    """Offsets inside the slice of its designed survivors."""
    j = np.arange(sl.s)
    if sl.layout == "packed":
        off = j
    elif sl.layout == "spread":   # round robin over lanes: each lane holds floor(S/32) or ceil(S/32)
        off = LANES * (j % LANES) + j // LANES
    else:
        assert sl.s <= LANES, sl
        off = LANES * sl.lane + j
    assert np.all(off < rows), (sl, rows)
    return off.astype(np.int64)


def decoy_offsets(sl: Slice, designed: np.ndarray, rows: int) -> np.ndarray:
    """Rows that pass the first leaf only: every lane with fewer than `pre` designed rows is topped up to `pre`."""
    taken = np.zeros(SLICE, dtype=bool)
    taken[designed] = True
    out = []
    for lane in range(LANES):
        lo, hi = LANES * lane, min(LANES * lane + LANES, rows)
        free = [o for o in range(lo, hi) if not taken[o]]
        need = max(0, min(sl.pre, hi - lo) - int(taken[lo:hi].sum()))
        out += free[:need]
    return np.array(out, dtype=np.int64)


def per_lane(mask_slice: np.ndarray) -> np.ndarray:
    """Counts per lane of a slice's bool mask (padded to 1024 rows)."""
    m = np.zeros(SLICE, dtype=bool)
    m[:len(mask_slice)] = mask_slice
    return m.reshape(LANES, LANES).sum(axis=1)


@dataclass
class SegmentPlan:
    name: str
    num_docs: int
    slices: List[Slice]
    keys: Dict[str, int]

    @property
    def num_slices(self) -> int:
        return -(-self.num_docs // SLICE)


@dataclass
class Planned:
    """A built segment's columns and what was designed: `designed` (p1 = 1 AND p2 = 1), `decoy` (p1 = 1 only) and
    `skipped` (rows of the slices `inv = 0` skips)."""
    plan: SegmentPlan
    columns: Dict[str, np.ndarray]
    designed: np.ndarray
    decoy: np.ndarray
    skipped: np.ndarray


def build_columns(plan: SegmentPlan, seed: int) -> Planned:
    n = plan.num_docs
    assert len(plan.slices) == plan.num_slices, (plan.name, len(plan.slices), plan.num_slices)
    rng = np.random.default_rng(seed)
    designed, decoy, skipped = (np.zeros(n, dtype=bool) for _ in range(3))
    for i, sl in enumerate(plan.slices):
        base, rows = i * SLICE, min(SLICE, n - i * SLICE)
        d = designed_offsets(sl, rows)
        designed[base + d] = True
        decoy[base + decoy_offsets(sl, d, rows)] = True
        if sl.skipped:
            skipped[base:base + rows] = True
    rid = np.arange(n, dtype=np.int64)
    p1 = rng.choice(np.array([0, 2, 3]), size=n)
    p1[designed | decoy] = 1
    p2 = rng.integers(0, 2, size=n)
    p2[designed] = 1
    p2[decoy] = 0
    inv = np.zeros(n, dtype=np.int64)
    inv[skipped] = 1
    spare = np.nonzero(~designed & ~skipped)[0]
    inv[spare[0]] = 1   # the dictionary is {0, 1} in every segment
    cols = {"p1": p1, "p2": p2, "inv": inv, "rid": rid, "blk": rid // 16, "bit": 1 << (rid % 16)}
    for name, size in plan.keys.items():
        assert n >= size, (plan.name, name)
        cols[name] = rng.permutation(n) % size
    v = rng.integers(-5000, 5000, size=n)
    v[rng.random(n) < 0.02] = INT_MAX
    v[rng.random(n) < 0.02] = INT_MIN
    cols["v"] = v
    r = rng.integers(INT_MIN, INT_MAX + 1, size=n)
    r[rng.random(n) < 0.02] = INT_MAX
    r[rng.random(n) < 0.02] = INT_MIN
    cols["r"] = r
    cols["f"] = rng.integers(-40, 40, size=n) / 4.0
    cols["l"] = (1 << 40) + rng.integers(0, 1 << 30, size=n)
    out = {k: x.astype(np.int32) for k, x in cols.items() if k not in ("f", "l")}
    out["f"] = cols["f"].astype(np.float32)
    out["l"] = cols["l"].astype(np.int64)
    for c, card in (("p1", 4), ("p2", 2), ("inv", 2)):
        assert len(np.unique(out[c])) == card, (plan.name, c)
    return Planned(plan, out, designed, decoy, skipped)


# ------------------------------------------------------------------------------------------------------------------
# the slice sequences
# ------------------------------------------------------------------------------------------------------------------
RAGGED_ROWS = [1, 1023, 513, 31, 33, 129, 640, 1000, 2, 1022, 257, 100]


def _layout(s: int, k: int) -> str:
    lays = layouts_for(s)
    return lays[k % len(lays)]


def hand_over_plans(warps: int, keys=("k24", "kb")) -> List[SegmentPlan]:
    """Two-tile segments laid out per warp for `warps` W, such that under `grid` 1 every non-zero S edge is followed,
    in the same warp's next tile, by a non-zero S, by S = 0, by a bitmap-skipped slice, by the segment's ragged last
    slice and by the segment's end.  Segment i (S edge s = NONZERO[i]) puts, in warp column [tile 0, tile 1]:
      warp 0:      [s, S = 0]          warp 1: [s, skipped]       warp 2: [s, next edge]  (the next edge then ends)
      warp W - 1:  [s, ragged last slice]
      the others:  pairs of every (S, layout) item in turn.
    Two more segments without a ragged slice are exactly 12 and 16 slices long (multiples of 6 x 1024 and 8 x 1024)."""
    items = all_items()
    cursor = 0
    plans = []

    def filler():
        nonlocal cursor
        it = items[cursor % len(items)]
        cursor += 1
        return Slice(it.s, it.layout, DECOY_PRE[cursor % len(DECOY_PRE)])

    for i, s in enumerate(NONZERO):
        nxt = NONZERO[(i + 1) % len(NONZERO)]
        r = RAGGED_ROWS[i % len(RAGGED_ROWS)]
        pre = DECOY_PRE[i % len(DECOY_PRE)]
        cols = [[Slice(s, _layout(s, i), pre), Slice(0, "packed", DECOY_PRE[(i + 1) % len(DECOY_PRE)])],
                [Slice(s, _layout(s, i + 1), pre), Slice(64, "spread", 0, skipped=True)],
                [Slice(s, _layout(s, i + 2), pre), Slice(nxt, _layout(nxt, i), pre)]]
        while len(cols) < warps - 1:
            cols.append([filler(), filler()])
        ragged_s = [r, 0, min(r, 130), 1][i % 4]
        cols.append([Slice(s, _layout(s, i), pre), Slice(ragged_s, "packed", DECOY_PRE[i % len(DECOY_PRE)])])
        slices = [cols[w][t] for t in range(2) for w in range(warps)]
        plans.append(SegmentPlan(f"ho{warps}_{i}", (2 * warps - 1) * SLICE + r, slices, {k: KEY_SPACES[k] for k in keys}))
    for n in (12 * SLICE, 16 * SLICE):
        slices = [filler() for _ in range(n // SLICE)]
        plans.append(SegmentPlan(f"ho{warps}_full{n}", n, slices, {k: KEY_SPACES[k] for k in keys}))
    return plans


def long_plan(name: str, num_slices: int, ragged: int, keys=("k24", "kb", "k70"), start: int = 0) -> SegmentPlan:
    """Every (S, layout) item in turn, a skipped slice every seventh; a ragged last slice of `ragged` rows (0: none)."""
    items = all_items()
    slices = []
    for i in range(num_slices):
        it = items[(start + i) % len(items)]
        sl = Slice(it.s, it.layout, DECOY_PRE[i % len(DECOY_PRE)], skipped=i % 7 == 3)
        slices.append(sl)
    if ragged:
        slices[-1] = Slice(min(slices[-1].s, ragged), "packed", 0)
    n = (num_slices - (1 if ragged else 0)) * SLICE + ragged
    return SegmentPlan(name, n, slices, {k: KEY_SPACES[k] for k in keys})


def successors(plan: SegmentPlan, warps: int) -> List[tuple]:
    """(slice, what follows it in the same warp's next tile under grid 1): a Slice, "ragged" (the segment's ragged last
    slice), "empty" (a slot past the segment's last row) or "end"."""
    tiles = -(-plan.num_slices // warps)
    ragged = plan.num_docs % SLICE != 0
    out = []
    for i, sl in enumerate(plan.slices):
        j = i + warps
        if j // warps >= tiles:
            nxt = "end"
        elif j >= plan.num_slices:
            nxt = "empty"
        elif ragged and j == plan.num_slices - 1:
            nxt = "ragged"
        else:
            nxt = plan.slices[j]
        out.append((sl, nxt))
    return out


# ------------------------------------------------------------------------------------------------------------------
# the device hash table (pb200_scan.cuh hash_slot, pb200_plan.cpp lay_out_table)
# ------------------------------------------------------------------------------------------------------------------
M64 = (1 << 64) - 1


def mix64_32(z: int) -> int:
    """pb200_scan.cuh mix64_32: the SplitMix64 finaliser, low 32 bits."""
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return (z ^ (z >> 31)) & 0xFFFFFFFF


def mix64_32_np(z: np.ndarray) -> np.ndarray:
    z = z.astype(np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return ((z ^ (z >> np.uint64(31))) & np.uint64(0xFFFFFFFF)).astype(np.int64)


def hash_capacity(limit: int) -> int:
    """lay_out_table: cap = max(2^16, the least power of two >= 2 (numGroupsLimit + 1))."""
    cap = 1 << 16
    while cap < 2 * (max(limit, 1) + 1):
        cap <<= 1
    return cap


def raw_key(ids: Sequence[int], cards: Sequence[int]) -> int:
    """sum of dictId_g * mult_g, column 0 least significant."""
    key, mult = 0, 1
    for i, c in zip(ids, cards):
        key += i * mult
        mult *= c
    return key


def keys_at_table_end(card_a: int, card_b: int, limit: int, count: int, last: int = 16) -> List[tuple]:
    """`count` dictId pairs (a, b) whose home slot is among the table's `last` slots: their probe chains run past
    h_mask and wrap to slot 0."""
    cap = hash_capacity(limit)
    a, b = np.meshgrid(np.arange(card_a, dtype=np.int64), np.arange(card_b, dtype=np.int64), indexing="ij")
    key = (a + b * card_a).reshape(-1)
    slot = mix64_32_np(key) & (cap - 1)
    pick = np.nonzero(slot >= cap - last)[0][:count]
    assert len(pick) == count, (len(pick), count)
    return [(int(k % card_a), int(k // card_a)) for k in key[pick]]


def hash_segment_columns(pairs: Sequence[tuple], card: int, seed: int, slices_before: int = 6) -> Planned:
    """A segment whose designed rows carry group keys (ha, hb) = pairs[k] in row order: `slices_before` slices of 100
    spread survivors, then a last slice of 130 packed survivors -- its pipelined last batch holds the final two pairs
    (queue entries 128 and 129).  Every other row takes ha / hb values so that both dictionaries are 0 .. card - 1."""
    plan = SegmentPlan(f"hash{seed}", slices_before * SLICE + 200,
                       [Slice(100, "spread", 5) for _ in range(slices_before)] + [Slice(130, "packed", 0)], {})
    p = build_columns(plan, seed)
    rows = np.nonzero(p.designed)[0]
    assert len(rows) == 100 * slices_before + 130 and 2 < len(pairs) <= len(rows)
    body = [tuple(x) for x in list(pairs)[:-2]]
    fill = [body[k % len(body)] for k in range(len(rows) - 2)]
    fill += [tuple(pairs[-2]), tuple(pairs[-1])]
    rng = np.random.default_rng(seed + 1)
    ha = rng.permutation(plan.num_docs) % card
    hb = rng.permutation(plan.num_docs) % card
    free = np.nonzero(~p.designed)[0]
    assert len(free) >= card
    ha[free[:card]] = np.arange(card)
    hb[free[:card]] = np.arange(card)
    ha[rows] = [x for x, _ in fill]
    hb[rows] = [y for _, y in fill]
    p.columns["ha"] = ha.astype(np.int32)
    p.columns["hb"] = hb.astype(np.int32)
    return p


def distinct_pairs(base: Sequence[tuple], card: int, total: int) -> List[tuple]:
    """`base`, then more distinct pairs until there are `total`."""
    out, seen = list(base), set(base)
    k = 0
    while len(out) < total:
        pr = (k % card, (k // card + 1) % card)
        if pr not in seen:
            out.append(pr)
            seen.add(pr)
        k += 1
    return out


# ------------------------------------------------------------------------------------------------------------------
# the routes the GPU tests take, and the plan each query shape gets on them (tests/test_survivor_plan_cpu.py pins it)
# ------------------------------------------------------------------------------------------------------------------
F = "p1 = 1 AND p2 = 1"
FI = "inv = 0 AND p1 = 1 AND p2 = 1"   # a doc-mask leaf as well: bitmap-skipped slices
GB_SPEC = f"SELECT SUM(v), COUNT(*) FROM t WHERE {F} GROUP BY k24"
GB_BLK = f"SELECT SUM(bit) FROM t WHERE {F} GROUP BY blk"
GB_INV = f"SELECT SUM(v), COUNT(*) FROM t WHERE {FI} GROUP BY k24"
GB_KB = f"SELECT SUM(v), COUNT(*) FROM t WHERE {F} GROUP BY kb"
GB_KB_INV = f"SELECT SUM(v), COUNT(*) FROM t WHERE {FI} GROUP BY kb"
GB_K70 = f"SELECT SUM(v), COUNT(*) FROM t WHERE {FI} GROUP BY k70"
MIX1 = f"SELECT SUM(f), COUNT(*) FROM t WHERE {F} GROUP BY k24"                   # one pipelined aggregation
MIX2 = f"SELECT SUM(v), MAX(f) FROM t WHERE {FI} GROUP BY k24"                    # exactly two
MIX4 = f"SELECT SUM(v), SUM(f), MIN(v), MAX(f), AVG(l), COUNT(*) FROM t WHERE {F} GROUP BY k24"   # two + four at once
MIX3 = f"SELECT MIN(v), MAX(f), SUM(v) FROM t WHERE {FI} GROUP BY kb"             # two pipelined, a sum at once
MIX_K70 = f"SELECT SUM(v), MAX(f), MIN(v) FROM t WHERE {F} GROUP BY k70"
GB_RAW = f"SELECT SUM(r), MIN(r), COUNT(*) FROM t WHERE {F} GROUP BY k24"
AGG_SUM = f"SELECT SUM(v), COUNT(*), AVG(v) FROM t WHERE {F}"
AGG_MIX = f"SELECT SUM(v), MIN(v), MAX(f), SUM(l), SUM(f), MAX(rid) FROM t WHERE {FI}"   # MIN / MAX: MinMaxLeft
AGG_RAW = f"SELECT SUM(r), MIN(r), MAX(r), COUNT(*) FROM t WHERE {F}"

# (id, knobs, segment set, queries).  Segment sets: "w6" / "w8" (hand_over_plans(6 / 8): the warp width the route runs
# at), "big" (long_plan segments holding the 70 000-value key).
ROUTES = [
    ("spec", {}, "w6", [GB_SPEC, GB_BLK]),
    ("spec_8_warp_table", {}, "w8", [GB_KB]),
    ("generic", {"spec": 0}, "w6", [GB_SPEC, GB_INV, GB_BLK]),
    ("generic_8_warp_table", {"spec": 0}, "w8", [GB_KB, GB_KB_INV]),
    ("global_stride1", {"smem_groups": 0, "table_stride": 1}, "w6", [GB_SPEC, GB_INV]),
    ("global_stride16", {"smem_groups": 0, "table_stride": 16}, "w6", [GB_INV, MIX2]),
    ("global_70000_keys", {}, "big", [GB_K70, MIX_K70]),
    ("hash", {"dense_max": 1}, "w6", [GB_SPEC, GB_INV, MIX4]),
    ("no_carrier", {"pack_count": 0}, "w6", [GB_SPEC, GB_INV]),
    ("no_carrier_8_warp_table", {"pack_count": 0}, "w8", [GB_KB_INV]),
    ("no_gb_defer", {"gb_defer": 0}, "w6", [GB_SPEC, GB_INV, MIX4]),
    ("mixes", {}, "w6", [MIX1, MIX2, MIX4, MIX3, GB_RAW]),
    ("agg_defer", {}, "w6", [AGG_SUM, AGG_MIX, AGG_RAW]),
    ("agg_no_defer", {"defer": 0}, "w6", [AGG_SUM, AGG_MIX, AGG_RAW]),
    ("agg_sparse0", {"sparse_max_agg": 0}, "w6", [AGG_SUM, AGG_MIX]),
    ("agg_sparse2", {"sparse_max_agg": 2}, "w6", [AGG_SUM, AGG_MIX]),
    ("agg_sparse4", {"sparse_max_agg": 4}, "w6", [AGG_SUM, AGG_RAW]),
    ("agg_sparse32", {"sparse_max_agg": 32}, "w6", [AGG_SUM, AGG_MIX]),
    ("agg_w8", {"warps": 8}, "w8", [AGG_SUM, AGG_MIX]),
    ("agg_w8_no_defer", {"warps": 8, "defer": 0}, "w8", [AGG_SUM, AGG_MIX]),
    # geometry, crossed with the routes where it matters
    ("grid1", {"grid": 1}, "w6", [GB_SPEC, GB_INV, MIX4, AGG_SUM, AGG_MIX]),
    ("grid1_w8", {"grid": 1, "warps": 8}, "w8", [GB_SPEC, GB_INV, MIX4, AGG_SUM, AGG_MIX]),
    ("grid1_8_warp_table", {"grid": 1}, "w8", [GB_KB, GB_KB_INV]),
    ("grid1_generic", {"grid": 1, "spec": 0}, "w6", [GB_SPEC, GB_BLK]),
    ("grid1_global", {"grid": 1, "smem_groups": 0}, "w6", [GB_SPEC, MIX2]),
    ("grid1_hash", {"grid": 1, "dense_max": 1}, "w6", [GB_INV, MIX2]),
    ("grid1_no_gb_defer", {"grid": 1, "gb_defer": 0}, "w6", [MIX4]),
    ("grid1_stages2", {"grid": 1, "stages": 2}, "w6", [GB_INV, MIX4, AGG_MIX]),
    ("grid1_no_skip", {"grid": 1, "skip": 0}, "w6", [GB_INV, AGG_MIX]),
    ("grid1_sparse0", {"grid": 1, "sparse_max": 0}, "w6", [GB_SPEC, GB_INV, AGG_SUM]),
    ("grid1_sparse32", {"grid": 1, "sparse_max": 32}, "w6", [GB_SPEC, GB_INV, AGG_SUM]),
    ("grid1_agg_sparse0", {"grid": 1, "sparse_max_agg": 0}, "w6", [AGG_SUM, AGG_RAW]),
    ("grid1_agg_no_defer", {"grid": 1, "defer": 0}, "w6", [AGG_SUM]),
    ("grid7", {"grid": 7}, "w6", [GB_SPEC, GB_INV, MIX4, AGG_MIX]),
    ("grid7_w8", {"grid": 7, "warps": 8}, "w8", [GB_INV, AGG_SUM]),
    ("stages2", {"stages": 2}, "w6", [GB_SPEC, AGG_SUM]),
    ("no_skip", {"skip": 0}, "w6", [GB_INV, AGG_MIX]),
    ("sparse0", {"sparse_max": 0}, "w6", [GB_SPEC, MIX2]),
    ("sparse32", {"sparse_max": 32}, "w6", [GB_INV, MIX2, AGG_MIX]),
]

# (W, SPEC, DEFER, smem_groups, smem_copies, hashed, num_defer_codes, defer_agg, sparse_max, sparse_max_agg, carrier_agg)
# of every (route, query) above, pinned by tests/test_survivor_plan_cpu.py.  GROUP BY blk: smem_groups is the segment's
# block count (None here), its copies follow from it.
EXPECTED_PLAN = {
    ("spec", GB_SPEC): (6, 1, 0, 24, 32, 0, 1, -1, 4, 2, 0),
    ("spec", GB_BLK): (6, 1, 0, None, None, 0, 1, -1, 4, 2, 0),
    ("spec_8_warp_table", GB_KB): (8, 1, 0, 10000, 1, 0, 1, -1, 4, 2, 0),
    ("generic", GB_SPEC): (6, 0, 0, 24, 32, 0, 1, -1, 4, 2, 0),
    ("generic", GB_INV): (6, 0, 0, 24, 32, 0, 1, -1, 4, 2, 0),
    ("generic", GB_BLK): (6, 0, 0, None, None, 0, 1, -1, 4, 2, 0),
    ("generic_8_warp_table", GB_KB): (8, 0, 0, 10000, 1, 0, 1, -1, 4, 2, 0),
    ("generic_8_warp_table", GB_KB_INV): (8, 0, 0, 10000, 1, 0, 1, -1, 4, 2, 0),
    ("global_stride1", GB_SPEC): (6, 0, 0, 0, 0, 0, 1, -1, 4, 2, 0),
    ("global_stride1", GB_INV): (6, 0, 0, 0, 0, 0, 1, -1, 4, 2, 0),
    ("global_stride16", GB_INV): (6, 0, 0, 0, 0, 0, 1, -1, 4, 2, 0),
    ("global_stride16", MIX2): (6, 0, 0, 0, 0, 0, 2, -1, 4, 2, -1),
    ("global_70000_keys", GB_K70): (6, 0, 0, 0, 0, 0, 1, -1, 4, 2, 0),
    ("global_70000_keys", MIX_K70): (6, 0, 0, 0, 0, 0, 2, -1, 4, 2, -1),
    ("hash", GB_SPEC): (6, 0, 0, 0, 0, 1, 1, -1, 4, 2, 0),
    ("hash", GB_INV): (6, 0, 0, 0, 0, 1, 1, -1, 4, 2, 0),
    ("hash", MIX4): (6, 0, 0, 0, 0, 1, 2, -1, 4, 2, 0),
    ("no_carrier", GB_SPEC): (6, 1, 0, 24, 32, 0, 1, -1, 4, 2, -1),
    ("no_carrier", GB_INV): (6, 0, 0, 24, 32, 0, 1, -1, 4, 2, -1),
    ("no_carrier_8_warp_table", GB_KB_INV): (8, 0, 0, 10000, 1, 0, 1, -1, 4, 2, -1),
    ("no_gb_defer", GB_SPEC): (6, 0, 0, 24, 32, 0, 0, -1, 4, 2, 0),
    ("no_gb_defer", GB_INV): (6, 0, 0, 24, 32, 0, 0, -1, 4, 2, 0),
    ("no_gb_defer", MIX4): (6, 0, 0, 0, 0, 0, 0, -1, 4, 2, 0),
    ("mixes", MIX1): (6, 0, 0, 0, 0, 0, 1, -1, 4, 2, -1),
    ("mixes", MIX2): (6, 0, 0, 0, 0, 0, 2, -1, 4, 2, -1),
    ("mixes", MIX4): (6, 0, 0, 0, 0, 0, 2, -1, 4, 2, 0),
    ("mixes", MIX3): (6, 0, 0, 0, 0, 0, 2, -1, 4, 2, -1),
    ("mixes", GB_RAW): (6, 0, 0, 0, 0, 0, 1, -1, 4, 2, -1),
    ("agg_defer", AGG_SUM): (6, 0, 1, 0, 0, 0, 0, 0, 4, 4, 0),
    ("agg_defer", AGG_MIX): (6, 0, 1, 0, 0, 0, 0, 0, 4, 4, 0),
    ("agg_defer", AGG_RAW): (6, 0, 1, 0, 0, 0, 0, -1, 4, 4, 0),
    ("agg_no_defer", AGG_SUM): (6, 0, 1, 0, 0, 0, 0, -1, 4, 4, 0),
    ("agg_no_defer", AGG_MIX): (6, 0, 1, 0, 0, 0, 0, -1, 4, 4, 0),
    ("agg_no_defer", AGG_RAW): (6, 0, 1, 0, 0, 0, 0, -1, 4, 4, 0),
    ("agg_sparse0", AGG_SUM): (6, 0, 1, 0, 0, 0, 0, 0, 4, 0, 0),
    ("agg_sparse0", AGG_MIX): (6, 0, 1, 0, 0, 0, 0, 0, 4, 0, 0),
    ("agg_sparse2", AGG_SUM): (6, 0, 1, 0, 0, 0, 0, 0, 4, 2, 0),
    ("agg_sparse2", AGG_MIX): (6, 0, 1, 0, 0, 0, 0, 0, 4, 2, 0),
    ("agg_sparse4", AGG_SUM): (6, 0, 1, 0, 0, 0, 0, 0, 4, 4, 0),
    ("agg_sparse4", AGG_RAW): (6, 0, 1, 0, 0, 0, 0, -1, 4, 4, 0),
    ("agg_sparse32", AGG_SUM): (6, 0, 1, 0, 0, 0, 0, 0, 4, 32, 0),
    ("agg_sparse32", AGG_MIX): (6, 0, 1, 0, 0, 0, 0, 0, 4, 32, 0),
    ("agg_w8", AGG_SUM): (8, 0, 1, 0, 0, 0, 0, 0, 4, 4, 0),
    ("agg_w8", AGG_MIX): (8, 0, 1, 0, 0, 0, 0, 0, 4, 4, 0),
    ("agg_w8_no_defer", AGG_SUM): (8, 0, 0, 0, 0, 0, 0, -1, 4, 4, 0),
    ("agg_w8_no_defer", AGG_MIX): (8, 0, 0, 0, 0, 0, 0, -1, 4, 4, 0),
    ("grid1", GB_SPEC): (6, 1, 0, 24, 32, 0, 1, -1, 4, 2, 0),
    ("grid1", GB_INV): (6, 0, 0, 24, 32, 0, 1, -1, 4, 2, 0),
    ("grid1", MIX4): (6, 0, 0, 0, 0, 0, 2, -1, 4, 2, 0),
    ("grid1", AGG_SUM): (6, 0, 1, 0, 0, 0, 0, 0, 4, 4, 0),
    ("grid1", AGG_MIX): (6, 0, 1, 0, 0, 0, 0, 0, 4, 4, 0),
    ("grid1_w8", GB_SPEC): (8, 0, 0, 24, 32, 0, 1, -1, 4, 2, 0),
    ("grid1_w8", GB_INV): (8, 0, 0, 24, 32, 0, 1, -1, 4, 2, 0),
    ("grid1_w8", MIX4): (8, 0, 0, 0, 0, 0, 2, -1, 4, 2, 0),
    ("grid1_w8", AGG_SUM): (8, 0, 1, 0, 0, 0, 0, 0, 4, 4, 0),
    ("grid1_w8", AGG_MIX): (8, 0, 1, 0, 0, 0, 0, 0, 4, 4, 0),
    ("grid1_8_warp_table", GB_KB): (8, 1, 0, 10000, 1, 0, 1, -1, 4, 2, 0),
    ("grid1_8_warp_table", GB_KB_INV): (8, 0, 0, 10000, 1, 0, 1, -1, 4, 2, 0),
    ("grid1_generic", GB_SPEC): (6, 0, 0, 24, 32, 0, 1, -1, 4, 2, 0),
    ("grid1_generic", GB_BLK): (6, 0, 0, None, None, 0, 1, -1, 4, 2, 0),
    ("grid1_global", GB_SPEC): (6, 0, 0, 0, 0, 0, 1, -1, 4, 2, 0),
    ("grid1_global", MIX2): (6, 0, 0, 0, 0, 0, 2, -1, 4, 2, -1),
    ("grid1_hash", GB_INV): (6, 0, 0, 0, 0, 1, 1, -1, 4, 2, 0),
    ("grid1_hash", MIX2): (6, 0, 0, 0, 0, 1, 2, -1, 4, 2, -1),
    ("grid1_no_gb_defer", MIX4): (6, 0, 0, 0, 0, 0, 0, -1, 4, 2, 0),
    ("grid1_stages2", GB_INV): (6, 0, 0, 24, 32, 0, 1, -1, 4, 2, 0),
    ("grid1_stages2", MIX4): (6, 0, 0, 0, 0, 0, 2, -1, 4, 2, 0),
    ("grid1_stages2", AGG_MIX): (6, 0, 1, 0, 0, 0, 0, 0, 4, 4, 0),
    ("grid1_no_skip", GB_INV): (6, 0, 0, 24, 32, 0, 1, -1, 4, 2, 0),
    ("grid1_no_skip", AGG_MIX): (6, 0, 1, 0, 0, 0, 0, 0, 4, 4, 0),
    ("grid1_sparse0", GB_SPEC): (6, 1, 0, 24, 32, 0, 1, -1, 0, 0, 0),
    ("grid1_sparse0", GB_INV): (6, 0, 0, 24, 32, 0, 1, -1, 0, 0, 0),
    ("grid1_sparse0", AGG_SUM): (6, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0),
    ("grid1_sparse32", GB_SPEC): (6, 1, 0, 24, 32, 0, 1, -1, 32, 2, 0),
    ("grid1_sparse32", GB_INV): (6, 0, 0, 24, 32, 0, 1, -1, 32, 2, 0),
    ("grid1_sparse32", AGG_SUM): (6, 0, 1, 0, 0, 0, 0, 0, 32, 32, 0),
    ("grid1_agg_sparse0", AGG_SUM): (6, 0, 1, 0, 0, 0, 0, 0, 4, 0, 0),
    ("grid1_agg_sparse0", AGG_RAW): (6, 0, 1, 0, 0, 0, 0, -1, 4, 0, 0),
    ("grid1_agg_no_defer", AGG_SUM): (6, 0, 1, 0, 0, 0, 0, -1, 4, 4, 0),
    ("grid7", GB_SPEC): (6, 1, 0, 24, 32, 0, 1, -1, 4, 2, 0),
    ("grid7", GB_INV): (6, 0, 0, 24, 32, 0, 1, -1, 4, 2, 0),
    ("grid7", MIX4): (6, 0, 0, 0, 0, 0, 2, -1, 4, 2, 0),
    ("grid7", AGG_MIX): (6, 0, 1, 0, 0, 0, 0, 0, 4, 4, 0),
    ("grid7_w8", GB_INV): (8, 0, 0, 24, 32, 0, 1, -1, 4, 2, 0),
    ("grid7_w8", AGG_SUM): (8, 0, 1, 0, 0, 0, 0, 0, 4, 4, 0),
    ("stages2", GB_SPEC): (6, 1, 0, 24, 32, 0, 1, -1, 4, 2, 0),
    ("stages2", AGG_SUM): (6, 0, 1, 0, 0, 0, 0, 0, 4, 4, 0),
    ("no_skip", GB_INV): (6, 0, 0, 24, 32, 0, 1, -1, 4, 2, 0),
    ("no_skip", AGG_MIX): (6, 0, 1, 0, 0, 0, 0, 0, 4, 4, 0),
    ("sparse0", GB_SPEC): (6, 1, 0, 24, 32, 0, 1, -1, 0, 0, 0),
    ("sparse0", MIX2): (6, 0, 0, 0, 0, 0, 2, -1, 0, 0, -1),
    ("sparse32", GB_INV): (6, 0, 0, 24, 32, 0, 1, -1, 32, 2, 0),
    ("sparse32", MIX2): (6, 0, 0, 0, 0, 0, 2, -1, 32, 2, -1),
    ("sparse32", AGG_MIX): (6, 0, 1, 0, 0, 0, 0, 0, 32, 32, 0),
}
