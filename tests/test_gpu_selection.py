"""-m gpu: selection queries (SELECT columns WHERE ... LIMIT n) against the value-space reference (tests/selection_ref.py):
doc ids, segments and every value equal, in order.

Segments of 1 .. 196 609 rows hold dictionary INT / LONG (at the int64 ends) / FLOAT / DOUBLE / STRING columns, a sorted
column (doc-range leaves), an inverted one, and a raw INT column at INT_MIN / INT_MAX -- streamed raw, and with the
dictionary synthesised at load.  Filters cover no filter, a filter folded to EMPTY, ranges, IN / NOT IN, inverted EQ, doc
ranges and AND / OR / NOT trees; limits 0, 1, matches - 1, matches, matches + 1 and one whose output exceeds the 512 KB
mapped-write bound.  LIMIT >= matches returns the whole match mask of the segment, so those cases check the kernel's
mask output bit for bit against filter_ref.  Then the scan kernel's knobs, a 17-segment submission (two launch chunks)
merged and per segment, the prefix pass with and without its rescan, and four threads on one context.
ORDER BY: 1-3 mixed ASC / DESC items over every stored type (raw INT at INT_MIN / INT_MAX, LONG at the int64 ends), a
low-cardinality first key whose threshold bucket holds far more than LIMIT rows, order columns that are not selected,
and merged submissions whose segments have different dictionaries (tops merged by value)."""
import threading

import numpy as np
import pytest

from gpu_util import to_device, tuned
from pinot_b200.plan_maker import B200Context, B200PlanMaker, UnsupportedQueryError
from pinot_b200.query import Filter, Predicate
from pinot_b200.sql import SelectionQuery, parse_selection
from selection_ref import assert_rows_equal, expected

pytestmark = pytest.mark.gpu

INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
SIZES = [1, 31, 32, 1_025, 49_157, 196_609]
COLUMNS = ["rid", "i", "l", "f", "d", "s", "r"]
KNOBS = [{"sparse_max": 0}, {"sparse_max": 32}, {"skip": 0}, {"warps": 8}, {"grid": 1}, {"grid": 7}, {"stages": 2}]


def _segment(oracle, n, seed, name=None):
    rng = np.random.default_rng(seed)
    rid = np.arange(n, dtype=np.int32)
    r = rng.integers(-1000, 1000, size=n).astype(np.int32)
    r[rng.integers(0, n, size=max(1, n // 40))] = INT_MAX
    r[rng.integers(0, n, size=max(1, n // 40))] = INT_MIN
    cols = {"rid": rid,
            "i": (rng.integers(0, 300, size=n) * 7 - 1000).astype(np.int32),
            "l": np.array([INT64_MIN, INT64_MAX, -1, 0, 5, 1 << 53], dtype=np.int64)[rng.integers(0, 6, size=n)],
            "f": (rng.integers(-20, 20, size=n) / 4.0).astype(np.float32),
            "d": rng.integers(-20, 20, size=n) / 3.0,
            "s": np.array([b"a", b"ab", b"b", b"ba", b"zz"])[rng.integers(0, 5, size=n)],
            "r": r,
            "inv": rng.integers(0, 40, size=n).astype(np.int32)}
    return oracle.build_segment(name or f"sel{n}_{seed}", cols, inverted=["inv"], raw=["r"])


def _filters(n):
    return [None,
            Predicate("RANGE", "i", [], 10 ** 9, None, True, True),                     # folds to EMPTY on the host
            Predicate("RANGE", "i", [], -500, 400, True, False),
            Predicate("IN", "s", ["ab", "zz"]),
            Predicate("NOT_IN", "i", [-1000, -993, 1093]),
            Predicate("EQ", "inv", [7]),
            Predicate("RANGE", "rid", [], n // 3, n - 2, True, True),                   # sorted column: doc ranges
            Predicate("RANGE", "r", [], INT_MAX, None, True, True),
            Predicate("RANGE", "r", [], None, INT_MIN, True, True),
            Filter("AND", [Predicate("RANGE", "f", [], -2.0, 3.0, True, True), Predicate("RANGE", "l", [], 0, None, True, True)]),
            Filter("OR", [Predicate("EQ", "inv", [3]), Filter("NOT", [Predicate("RANGE", "d", [], -5.0, None, True, True)]),
                          Filter("AND", [Predicate("IN", "s", ["b"]), Predicate("RANGE", "rid", [], 0, n // 2, True, True)])])]


@pytest.fixture(scope="module")
def ctx():
    c = B200Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pm(ctx):
    return B200PlanMaker(ctx)


@pytest.fixture(scope="module", params=["raw", "synthesised"])
def segs(request, oracle, ctx):
    out = []
    with tuned(ctx, raw_dict_max=0 if request.param == "raw" else 1 << 20):
        for n in SIZES:
            seg = _segment(oracle, n, n)
            out.append((seg, to_device(ctx, seg)))
    yield out
    for _, dev in out:
        dev.destroy()


def _check(oracle, pm, pairs, flt, columns, limit, merge=False, what="", order_by=()):
    q = SelectionQuery(columns=columns, filter=flt, limit=limit, order_by=list(order_by))
    got = pm.execute_selection([d for _, d in pairs], q, merge=merge)
    want = expected(oracle, [s for s, _ in pairs], flt, columns if columns is not None else sorted(pairs[0][1].column_names), limit, merge,
                    order_by)
    blocks = [got] if merge else got
    assert len(blocks) == len(want)
    for b, w in zip(blocks, want):
        assert_rows_equal(b, w, what)
        assert b.stats.num_docs_scanned == w["matched"], what   # whole segments are scanned below the prefix length
        assert b.stats.num_entries_scanned_post_filter == b.num_rows * len(b.names), what
    return want


def test_limits_and_filters(oracle, pm, segs):
    for seg, dev in segs:
        n = seg.num_docs
        for fi, flt in enumerate(_filters(n)):
            m = expected(oracle, [seg], flt, [], n, False)[0]["matched"]
            for limit in sorted({0, 1, max(m - 1, 0), m, m + 1}):
                _check(oracle, pm, [(seg, dev)], flt, COLUMNS, limit, what=f"n={n} filter={fi} limit={limit}")


def test_large_output_and_star(oracle, pm, segs):
    seg, dev = segs[-1]
    # 100 000 rows x (8 + 7 x 8) bytes: beyond the mapped-write bound, staged and copied with one DMA
    _check(oracle, pm, [(seg, dev)], None, COLUMNS, 100_000, what="large")
    _check(oracle, pm, [(seg, dev)], Predicate("RANGE", "i", [], 0, None, True, True), None, 20, what="select *")
    _check(oracle, pm, [(seg, dev)], None, ["s", "s", "rid"], 5, what="repeated column")


def test_knobs(oracle, ctx, pm, segs):
    for knobs in KNOBS:
        with tuned(ctx, **knobs):
            for seg, dev in segs[3:]:
                for flt in _filters(seg.num_docs)[2:]:
                    _check(oracle, pm, [(seg, dev)], flt, ["rid", "i", "s"], seg.num_docs, what=f"{knobs}")


def test_many_segments(oracle, ctx, pm):
    pairs = []
    try:
        for k in range(17):
            seg = _segment(oracle, 3_000 + 977 * k, 100 + k)
            pairs.append((seg, to_device(ctx, seg)))
        for flt in (None, Predicate("RANGE", "i", [], 1000, None, True, True), Predicate("EQ", "inv", [11])):
            for limit in (0, 7, 5_000, 100_000):
                _check(oracle, pm, pairs, flt, ["rid", "l", "s"], limit, merge=True, what=f"merged {limit}")
                _check(oracle, pm, pairs, flt, ["rid", "l", "s"], limit, merge=False, what=f"per segment {limit}")
    finally:
        for _, d in pairs:
            d.destroy()


def test_prefix_rescan(oracle, ctx, pm):
    n = 1_500_000
    seg = _segment(oracle, n, 7, name="prefix")
    dev = to_device(ctx, seg)
    try:
        # matches everywhere: the prefix holds the first 10, nothing is rescanned and the statistics count the prefix
        got = pm.execute_selection([dev], SelectionQuery(columns=["rid"], filter=Predicate("RANGE", "i", [], 0, None, True, True), limit=10))[0]
        want = expected(oracle, [seg], Predicate("RANGE", "i", [], 0, None, True, True), ["rid"], 10, False)[0]
        assert_rows_equal(got, want, "prefix")
        assert 0 < got.stats.num_docs_scanned < want["matched"]
        # matches only beyond the prefix: rescanned over the whole segment
        flt = Predicate("RANGE", "rid", [], 1_400_000, None, True, True)
        _check(oracle, pm, [(seg, dev)], flt, ["rid", "i", "r"], 10, what="rescan")
        flt = Filter("AND", [Predicate("RANGE", "i", [], 0, None, True, True), Predicate("RANGE", "rid", [], 1_048_000, None, True, True)])
        _check(oracle, pm, [(seg, dev)], flt, ["rid", "i"], 3_000, what="rescan across the prefix end")
    finally:
        dev.destroy()


def test_refusals(pm, segs):
    _, dev = segs[0]
    with pytest.raises(UnsupportedQueryError):
        pm.execute_selection([dev], SelectionQuery(columns=["rid"], limit=1_000_001))
    with pytest.raises(ValueError):
        pm.execute_selection([dev], parse_selection("SELECT rid FROM t ORDER BY i, l, f, d, s, r, inv, rid, i LIMIT 3"))


def test_threads(oracle, ctx, segs):
    pairs = segs[3:]
    errors = []

    def work(t):
        try:
            pm = B200PlanMaker(ctx)
            for k in range(6):
                flt = _filters(pairs[k % len(pairs)][0].num_docs)[(t + k) % 11]
                seg, dev = pairs[(t + k) % len(pairs)]
                _check(oracle, pm, [(seg, dev)], flt, ["rid", "f", "s"], 50 + t, what=f"thread {t}")
        except Exception as e:  # noqa: BLE001
            errors.append(e)
    threads = [threading.Thread(target=work, args=(t,)) for t in range(4)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors


ORDERS = [[("i", True)], [("i", False)], [("s", True), ("rid", False)], [("l", False), ("f", True)],
          [("r", True)], [("r", False), ("d", True)], [("inv", True), ("s", False), ("l", True)], [("f", False)]]


def test_order_by(oracle, pm, segs):
    for seg, dev in segs:
        n = seg.num_docs
        for fi, flt in enumerate(_filters(n)[:1] + _filters(n)[2:]):
            m = expected(oracle, [seg], flt, [], n, False)[0]["matched"]
            for oi, order in enumerate(ORDERS):
                for limit in sorted({0, 1, 10, max(m - 1, 0), m + 1}):
                    _check(oracle, pm, [(seg, dev)], flt, ["rid", "s", "d"], limit, what=f"n={n} f={fi} o={oi} l={limit}",
                           order_by=order)


def test_order_by_low_cardinality_and_unselected(oracle, ctx, pm):
    # first key of 3 values over 200 000 rows: the threshold bucket holds ~66 000 rows for LIMIT 5 / 1000
    rng = np.random.default_rng(11)
    n = 200_000
    seg = oracle.build_segment("lowcard", {"k": rng.integers(0, 3, size=n).astype(np.int32),
                                           "v": rng.integers(-50, 50, size=n).astype(np.int32),
                                           "s": np.array([b"p", b"q"])[rng.integers(0, 2, size=n)]})
    dev = to_device(ctx, seg)
    try:
        for order in ([("k", True)], [("k", False), ("v", True)], [("s", True), ("k", False), ("v", False)]):
            for limit in (5, 1000, 150_000):
                _check(oracle, pm, [(seg, dev)], None, ["v"], limit, what=f"{order} {limit}", order_by=order)
                _check(oracle, pm, [(seg, dev)], Predicate("RANGE", "v", [], 0, None, True, True), ["s"], limit,
                       what=f"{order} {limit} filtered", order_by=order)
    finally:
        dev.destroy()


def test_order_by_many_segments(oracle, ctx, pm):
    # 17 segments (two launch chunks) with different dictionaries: merged tops by value, ties by (segment, doc id)
    pairs = []
    try:
        for k in range(17):
            seg = _segment(oracle, 2_000 + 613 * k, 300 + k)
            pairs.append((seg, to_device(ctx, seg)))
        for order in ([("i", False)], [("s", True), ("l", False)], [("f", True), ("r", True), ("rid", False)]):
            for limit in (0, 1, 25, 40_000):
                for merge in (True, False):
                    _check(oracle, pm, pairs, Predicate("RANGE", "d", [], -3.0, None, True, True), ["rid", "i", "s"], limit,
                           merge=merge, what=f"{order} {limit} {merge}", order_by=order)
    finally:
        for _, d in pairs:
            d.destroy()


def test_order_by_knobs(oracle, ctx, pm, segs):
    for knobs in KNOBS:
        with tuned(ctx, **knobs):
            seg, dev = segs[-1]
            _check(oracle, pm, [(seg, dev)], _filters(seg.num_docs)[2], ["rid"], 100, what=f"{knobs}", order_by=[("s", False), ("i", True)])
