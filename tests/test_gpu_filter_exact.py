"""-m gpu: every filter route of the scan kernel against the value-space reference (tests/filter_ref.py).

The matched doc set is read back exactly from each kernel through `rid` (an INT column holding the doc index, stored
sorted, dictId == doc):

* aggregation only: COUNT(*), SUM(rid), MIN(rid), MAX(rid), DISTINCTCOUNT(rid) -- the DISTINCTCOUNT set is the doc set;
* COUNT(*) alone (no projected column: with only doc-mask / doc-range leaves the kernel runs without its TMA pipe);
* GROUP BY rid with COUNT(*) (global dense table): the keys are the doc set;
* GROUP BY blk with SUM(bit), blk = rid // 16, bit = 1 << (rid % 16) (shared-memory table): each group's exact sum is its
  block's 16-row match mask.

num_docs_scanned must equal the reference's count everywhere.  Segments: dictionary INT columns whose dictionaries span
the one-sided range shortcuts (cardinality 2^b and 2^(b-1) + 1 for b up to 17, where the segment has the rows), a raw
INT column at INT_MIN / INT_MAX, LONG at the int64 ends, FLOAT, DOUBLE, STRING, sorted columns (DOC_RANGES) and two
inverted columns: one random, one clustered in runs (non-monotone) whose postings mix run, bitmap and array containers
and leave whole 1024-row slices without a match.  Sizes 1 .. 196 609 give 1 to 4 roaring containers and ragged tails.
Trees: flat ANDs of 1-8 leaves (the conjunction route) and nested AND / OR / NOT (the postfix program), each run under
the kernel's tuning knobs."""
import time

import numpy as np
import pytest

from filter_ref import matching_docs_many
from gpu_util import to_device, tuned
from pinot_b200.plan_maker import B200Context, B200PlanMaker, UnsupportedQueryError
from pinot_b200.query import Aggregation, Filter, Predicate, QueryContext
from test_filter_ref_cpu import literal_pool, random_leaf, random_tree

pytestmark = pytest.mark.gpu

INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
SIZES = [1, 31, 33, 1_025, 8_193, 65_537, 131_073, 196_609]
WIDTHS = [1, 2, 7, 8, 15, 16, 17]
KNOBS = [{}, {"sparse_max": 0}, {"sparse_max": 32}, {"skip": 0}, {"warps": 8}, {"grid": 1}, {"grid": 7}, {"stages": 2},
         {"sparse_max_agg": 32}]
LIMIT = 1 << 20


def _segment(oracle, n, seed):
    rng = np.random.default_rng(seed)
    rid = np.arange(n, dtype=np.int32)
    cols = {"rid": rid, "blk": rid // 16, "bit": (1 << (rid % 16)).astype(np.int32), "srt": rid // 37}
    for b in WIDTHS:
        for card in sorted({1 << b, (1 << (b - 1)) + 1}):
            if card <= n:
                ids = np.concatenate([rng.permutation(card), rng.integers(0, card, size=n - card)])
                cols[f"c{b}_{card}"] = (ids * 3 - 7).astype(np.int32)
    r = rng.integers(-1000, 1000, size=n).astype(np.int32)
    r[rng.integers(0, n, size=max(1, n // 50))] = INT_MAX
    r[rng.integers(0, n, size=max(1, n // 50))] = INT_MIN
    cols["r"] = r
    cols["l"] = np.array([INT64_MIN, INT64_MAX, -1, 0, 5, 1 << 53], dtype=np.int64)[rng.integers(0, 6, size=n)]
    cols["f"] = (rng.integers(-20, 20, size=n) / 4.0).astype(np.float32)
    cols["d"] = rng.integers(-20, 20, size=n) / 3.0
    cols["s"] = np.array([b"a", b"ab", b"b", b"ba", b"zz"])[rng.integers(0, 5, size=n)]
    cols["inv"] = rng.integers(0, 40, size=n).astype(np.int32)
    # clustered in runs of 2000 rows cycling 3, 1, 4, 0, 2 (run containers, slices without value 3); in the second 64K
    # chunk every other row is 5 (bitmap container) and every 97th 6 (array container)
    ic = np.array([3, 1, 4, 0, 2], dtype=np.int32)[(rid // 2000) % 5]
    ic[(rid >= 65_536) & (rid < 98_304) & (rid % 2 == 0)] = 5
    ic[(rid >= 65_536) & (rid % 97 == 0)] = 6
    if n > 1 and np.all(np.diff(ic) >= 0):
        ic[0] = 7   # never stored as sorted
    cols["ic"] = ic
    return oracle.build_segment(f"fx{n}_{seed}", cols, inverted=["inv", "ic"], raw=["r"])


@pytest.fixture(scope="module")
def ctx():
    c = B200Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pm(ctx):
    return B200PlanMaker(ctx)


@pytest.fixture(scope="module")
def segs(oracle, ctx):
    out = []
    with tuned(ctx, raw_dict_max=0):   # "r" stays a raw 32-bit column (RAW_RANGE leaves)
        for n in SIZES:
            seg = _segment(oracle, n, n)
            out.append((seg, to_device(ctx, seg)))
    yield out
    for _, dev in out:
        dev.destroy()


def _leaves(seg, rng, k):
    """k seeded leaves over the segment's filter columns: pools of stored values, neighbours, fractions and literals
    beyond int32 / int64, plus IN / NOT IN over dictIds 31 / 32 / 63 / 64 / card - 1 and raw bounds at INT_MIN / INT_MAX."""
    names = [c.name for c in seg.columns if c.name not in ("bit",)]
    pools = {c.name: literal_pool(np.asarray(c.raw_values if c.raw_values is not None else c.dict_values),
                                  c.data_type in (0, 1)) for c in seg.columns if c.name in names}
    out = []
    for _ in range(k):
        c = names[int(rng.integers(0, len(names)))]
        out.append(random_leaf(rng, c, pools[c]))
    for c in seg.columns:
        if c.name.startswith("c") and c.name[1].isdigit():
            v = [int(x) for x in np.asarray(c.dict_values)[[i for i in (31, 32, 63, 64, c.cardinality - 1) if i < c.cardinality]]]
            out += [Predicate("IN", c.name, v), Predicate("NOT_IN", c.name, v), Predicate("IN", c.name, v + [-8, 10 ** 12]),
                    Predicate("RANGE", c.name, [], v[0], None, True, True), Predicate("RANGE", c.name, [], None, v[-1], True, False)]
    for lo, hi, li, ui in [(INT_MIN, INT_MAX, True, True), (INT_MIN, INT_MAX, False, False), (INT_MAX, None, True, True),
                           (INT_MAX, None, False, True), (None, INT_MIN, True, True), (None, INT_MIN, True, False),
                           (INT_MIN - 1, INT_MAX + 1, True, True), (-0.5, 0.5, True, True), (2.5, 2.5, True, True),
                           (None, INT_MIN + 0.5, True, True), (INT_MAX - 0.5, None, False, True)]:
        out.append(Predicate("RANGE", "r", [], lo, hi, li, ui))
    out += [Predicate("EQ", "r", [INT_MAX]), Predicate("EQ", "r", [INT_MIN]), Predicate("EQ", "r", [0.5]),
            Predicate("EQ", "r", [INT_MAX + 1])]
    n = seg.num_docs
    for a, b in [(0, 31), (32, 1023), (1024, 2047), (31, 32), (n - 1, n - 1), (n // 2, n)]:
        out.append(Predicate("RANGE", "rid", [], a, b, True, True))
    out += [Predicate("IN", "ic", [3]), Predicate("IN", "ic", [5, 6]), Predicate("NOT_IN", "ic", [3, 5]),
            Predicate("EQ", "ic", [6]), Predicate("RANGE", "srt", [], 3, 5, True, False)]
    return [p for p in out if p.type != "NEQ" or p.column != "r"]   # NEQ / IN on a raw column is not accelerated


def _accelerated(p):
    return not (p.column == "r" and p.type in ("IN", "NOT_IN", "NEQ"))


def _trees(seg, seed):
    rng = np.random.default_rng(seed)
    leaves = [p for p in _leaves(seg, rng, 40) if _accelerated(p)]
    pick = lambda: leaves[int(rng.integers(0, len(leaves)))]   # noqa: E731
    trees = list(leaves)
    for k in range(1, 9):   # flat conjunctions, doc-mask leaves among them
        trees.append(Filter("AND", [pick() for _ in range(k)]) if k > 1 else pick())
        trees.append(Filter("AND", [Predicate("IN", "ic", [3, 5])] + [pick() for _ in range(k - 1)]))
    for _ in range(30):
        t = random_tree(rng, pick)
        if _shape(t)[0] <= 8 and _shape(t)[1] <= 16:
            trees.append(t)
    same = pick()
    trees.append(Filter("OR", [same, Filter("NOT", [same])]))
    trees.append(Filter("AND", [same, Filter("NOT", [Filter("NOT", [same])])]))
    trees.append(_deep(pick, 8))                                    # 8 leaves, stack depth 8
    trees.append(_not_chain(pick, 8, 7))                            # 8 leaves, 16 nodes
    return trees


def _shape(t):
    """(leaves, nodes) of a tree."""
    if isinstance(t, Predicate):
        return 1, 1
    s = [_shape(c) for c in t.children]
    return sum(x for x, _ in s), 1 + sum(y for _, y in s)


def _deep(pick, k):
    """AND(l, OR(l, AND(l, ...))): every operand stays on the stack until the last leaf."""
    t = pick()
    for j in range(k - 1):
        t = Filter("AND" if j % 2 else "OR", [pick(), t])
    return t


def _not_chain(pick, leaves, nots):
    t = Filter("AND", [pick() for _ in range(leaves)])
    for _ in range(nots):
        t = Filter("NOT", [t])
    return t


def _q(aggs, flt=None, group_by=()):
    return QueryContext(aggregations=aggs, filter=flt, group_by=list(group_by), num_groups_limit=LIMIT,
                        max_initial_result_holder_capacity=LIMIT)


AGG = [Aggregation("COUNT"), Aggregation("SUM", "rid"), Aggregation("MIN", "rid"), Aggregation("MAX", "rid"),
       Aggregation("DISTINCTCOUNT", "rid")]


def _check_agg(b, ref, what):
    want = np.nonzero(ref)[0]
    k = len(want)
    assert b.stats.num_docs_scanned == k, what
    assert int(b.longs[0][0]) == k, what
    assert b.doubles[1][0] == float(want.sum()), what
    assert b.doubles[2][0] == (float(want[0]) if k else float("inf")), what
    assert b.doubles[3][0] == (float(want[-1]) if k else float("-inf")), what
    got = np.sort(np.asarray(b.distinct.get((4, 0), np.zeros(0)), dtype=np.int64))
    assert np.array_equal(got, want), what


def _check_count(b, ref, what):
    assert b.stats.num_docs_scanned == int(ref.sum()), what
    assert int(b.longs[0][0]) == int(ref.sum()), what


def _check_gb_rid(b, ref, what):
    want = np.nonzero(ref)[0]
    assert b.stats.num_docs_scanned == len(want), what
    keys = np.sort(b.keys[:, 0].astype(np.int64)) if b.num_groups > 0 else np.zeros(0, dtype=np.int64)
    assert np.array_equal(keys, want), what
    assert b.num_groups <= 0 or np.all(b.longs[0][:b.num_groups] == 1), what


def _check_gb_blk(b, ref, what):
    assert b.stats.num_docs_scanned == int(ref.sum()), what
    got = np.zeros(len(ref), dtype=bool)
    for g in range(max(b.num_groups, 0)):
        blk, mask = int(b.keys[g, 0]), int(b.doubles[0][g])
        for j in range(16):
            if mask >> j & 1:
                got[blk * 16 + j] = True
    assert np.array_equal(got, ref), what


def _run_all(oracle, pm, segs, seed, group_by, what):
    ran = refused = 0
    for seg, dev in segs:
        trees = _trees(seg, seed + seg.num_docs)
        refs = matching_docs_many(oracle, seg, trees)
        for t, ref in zip(trees, refs):
            tag = f"{what} n={seg.num_docs}: {t}"
            try:
                b = pm.execute_segments([dev], _q(AGG, t))[0]
            except UnsupportedQueryError as e:   # 8 warps: a ring too small for this many touched bits per row
                assert "too wide" in str(e), tag
                refused += 1
                continue
            ran += 1
            _check_agg(b, ref, "agg " + tag)
            _check_count(pm.execute_segments([dev], _q([Aggregation("COUNT")], t))[0], ref, "count " + tag)
            if group_by:
                _check_gb_rid(pm.execute_segments([dev], _q([Aggregation("COUNT")], t, ["rid"]))[0], ref, "gb rid " + tag)
                _check_gb_blk(pm.execute_segments([dev], _q([Aggregation("SUM", "bit")], t, ["blk"]))[0], ref, "gb blk " + tag)
    assert refused <= ran // 10, (what, ran, refused)


@pytest.mark.parametrize("knobs", KNOBS, ids=[",".join(f"{k}={v}" for k, v in kn.items()) or "defaults" for kn in KNOBS])
def test_every_tree_on_every_segment(oracle, ctx, pm, segs, knobs):
    """Aggregation-only and COUNT(*) observables under each knob; the group-by observables at the defaults and with
    per-row probing forced on (sparse_max 32) or off (sparse_max 0)."""
    t0 = time.perf_counter()
    with tuned(ctx, **knobs):
        _run_all(oracle, pm, segs, 100, knobs in ({}, {"sparse_max": 0}, {"sparse_max": 32}), str(knobs))
    print(f"{knobs}: {time.perf_counter() - t0:.1f} s")


def test_limits_of_the_filter_program(oracle, pm, segs):
    """8 leaves, 16 nodes and stack depth 8 run; one past each is refused with UnsupportedQueryError, never rows."""
    seg, dev = segs[-3]
    rng = np.random.default_rng(3)
    # leaves no segment can prove constant: the plan maker would answer a constant tree without the kernel
    leaves = [Predicate("IN", "inv", [j, j + 7]) for j in range(12)] + \
             [Predicate("RANGE", "c7_128", [], 3 * j - 7, 3 * j + 200, True, j % 2 == 0) for j in range(12)]
    pick = lambda: leaves[int(rng.integers(0, len(leaves)))]   # noqa: E731
    ok = [_deep(pick, 8), _not_chain(pick, 8, 7), Filter("AND", [pick() for _ in range(8)])]
    for t, ref in zip(ok, matching_docs_many(oracle, seg, ok)):
        _check_agg(pm.execute_segments([dev], _q(AGG, t))[0], ref, f"limit {t}")
    for t in [_deep(pick, 9), _not_chain(pick, 8, 8), Filter("AND", [pick() for _ in range(9)])]:
        with pytest.raises(UnsupportedQueryError):
            pm.execute_segments([dev], _q(AGG, t))


def test_per_segment_submission_of_17_segments(oracle, ctx, pm):
    """17 segments with different dictionaries in one submission (two launch chunks): each segment's doc set."""
    hs, devs = [], []
    try:
        with tuned(ctx, raw_dict_max=0):
            for j in range(17):
                hs.append(_segment(oracle, 700 + 431 * j, 5_000 + j))
                devs.append(to_device(ctx, hs[-1]))
        rng = np.random.default_rng(17)
        cols = ["c1_2", "c2_4", "c7_128", "c7_65", "inv", "ic", "f", "s", "srt", "rid"]
        pools = {c: literal_pool(np.asarray(hs[0].column(c).dict_values), c not in ("f", "s")) for c in cols}

        def leaf():
            c = cols[int(rng.integers(0, len(cols)))]
            return random_leaf(rng, c, pools[c])
        for _ in range(12):
            t = random_tree(rng, leaf)
            if _shape(t)[0] > 8 or _shape(t)[1] > 16:
                continue
            blocks = pm.execute_segments(devs, _q(AGG, t))
            for s, b in zip(hs, blocks):
                _check_agg(b, matching_docs_many(oracle, s, [t])[0], f"17 segs n={s.num_docs}: {t}")
    finally:
        for d in devs:
            d.destroy()


def test_filter_clauses(oracle, pm, segs):
    """COUNT(*) FILTER (WHERE tree) next to a plain COUNT(*): the clause's count is the reference's."""
    for seg, dev in segs[3:6]:
        trees = _trees(seg, 7)[-12:]
        for t, ref in zip(trees, matching_docs_many(oracle, seg, trees)):
            b = pm.execute_segments([dev], _q([Aggregation("COUNT", None, t), Aggregation("COUNT")]))[0]
            assert int(b.longs[0][0]) == int(ref.sum()), (seg.num_docs, t)
            assert int(b.longs[1][0]) == seg.num_docs, (seg.num_docs, t)
