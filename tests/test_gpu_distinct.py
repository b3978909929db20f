"""-m gpu: DISTINCT queries (SELECT DISTINCT columns WHERE ... [ORDER BY columns] LIMIT n) against the value-space
reference (tests/distinct_ref.py): every tuple, its first-occurrence doc id and segment index, in order, and the statistics.

Segments of 1 .. 196 609 rows hold dictionary INT (at INT_MIN / INT_MAX), LONG (at the int64 ends), FLOAT, DOUBLE and
STRING columns and a raw INT column whose dictionary is synthesised at load; DISTINCT over 1-4 of them.  Filters are
selection's shapes; limits 0, 1, distinct - 1, distinct, distinct + 1 and an output above the 512 KB mapped-write bound.
ORDER BY with 1-3 mixed ASC / DESC items, including items that leave ties (broken by first occurrence).  Key spaces of
one value, of exactly 2^24 (accepted) and just above (refused).  The prefix route final and with a rescan (LIMIT at the
prefix's distinct count and one above it), merged and per segment.  17 domain-bound segments (two launch chunks) merged
and per segment, the merge refusal without a domain and the by-value merge of per-segment results.  The scan knobs, and
four threads on one context."""
import threading

import numpy as np
import pytest

from distinct_ref import expected
from gpu_util import to_device, tuned
from pinot_b200._lib import E_INVALID, Pb200Error
from pinot_b200.plan_maker import B200Context, B200PlanMaker, DictionaryDomain, UnsupportedQueryError, merge_distinct_blocks
from pinot_b200.query import Filter, Predicate
from pinot_b200.sql import DistinctQuery
from selection_ref import assert_rows_equal

pytestmark = pytest.mark.gpu

INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
SIZES = [1, 31, 32, 1_025, 49_157, 196_609]
COLSETS = [["i"], ["s", "l"], ["f", "d", "r"], ["i", "s", "f", "l"]]
KNOBS = [{"sparse_max": 0}, {"sparse_max": 32}, {"skip": 0}, {"warps": 8}, {"grid": 1}, {"grid": 7}, {"stages": 2}]


def _segment(oracle, n, seed, name=None):
    rng = np.random.default_rng(seed)
    i = (rng.integers(0, 60, size=n) * 7 - 200).astype(np.int32)
    i[rng.integers(0, n, size=max(1, n // 50))] = INT_MAX
    i[rng.integers(0, n, size=max(1, n // 50))] = INT_MIN
    cols = {"rid": np.arange(n, dtype=np.int32),
            "i": i,
            "l": np.array([INT64_MIN, INT64_MAX, -1, 0, 5, 1 << 53], dtype=np.int64)[rng.integers(0, 6, size=n)],
            "f": (rng.integers(-20, 20, size=n) / 4.0).astype(np.float32),
            "d": rng.integers(-6, 6, size=n) / 3.0,
            "s": np.array([b"a", b"ab", b"b", b"ba", b"zz"])[rng.integers(0, 5, size=n)],
            "r": rng.integers(-1000, 1000, size=n).astype(np.int32) * 1000,
            "inv": rng.integers(0, 40, size=n).astype(np.int32)}
    return oracle.build_segment(name or f"dst{n}_{seed}", cols, inverted=["inv"], raw=["r"])


def _filters(n):
    return [None,
            Predicate("RANGE", "i", [], 10 ** 9, None, True, True),                     # folds to EMPTY on the host
            Predicate("RANGE", "i", [], -100, 200, True, False),
            Predicate("IN", "s", ["ab", "zz"]),
            Predicate("NOT_IN", "i", [-200, -193, 213]),
            Predicate("EQ", "inv", [7]),
            Predicate("RANGE", "rid", [], n // 3, n - 2, True, True),                   # sorted column: doc ranges
            Predicate("RANGE", "r", [], 0, None, True, True),
            Filter("AND", [Predicate("RANGE", "f", [], -2.0, 3.0, True, True), Predicate("RANGE", "l", [], 0, None, True, True)]),
            Filter("OR", [Predicate("EQ", "inv", [3]), Filter("NOT", [Predicate("RANGE", "d", [], -1.0, None, True, True)]),
                          Filter("AND", [Predicate("IN", "s", ["b"]), Predicate("RANGE", "rid", [], 0, n // 2, True, True)])])]


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
    for n in SIZES:   # the raw INT column "r" gets a dictionary synthesised at load (the default raw_dict_max)
        seg = _segment(oracle, n, n)
        out.append((seg, to_device(ctx, seg)))
    yield out
    for _, dev in out:
        dev.destroy()


def _cut(w, limit):
    return dict(w, doc_ids=w["doc_ids"][:limit], segment_index=w["segment_index"][:limit], columns=[c[:limit] for c in w["columns"]])


def _check_block(b, w, ncols, what, full_scan=True):
    assert_rows_equal(b, w, what)
    if full_scan:
        assert b.stats.num_docs_scanned == w["matched"], what
        assert b.stats.num_entries_scanned_post_filter == w["matched"] * ncols, what


def _check(oracle, pm, pairs, flt, columns, limit, merge=False, what="", order_by=(), want=None):
    q = DistinctQuery(columns=columns, filter=flt, limit=limit, order_by=list(order_by))
    got = pm.execute_distinct([d for _, d in pairs], q, merge=merge)
    if want is None:
        want = expected(oracle, [s for s, _ in pairs], flt, columns, limit, merge, order_by)
    blocks = [got] if merge else got
    assert len(blocks) == len(want)
    for b, w in zip(blocks, want):
        _check_block(b, _cut(w, limit), len(columns), what)
    return got


def test_limits_and_filters(oracle, pm, segs):
    for seg, dev in segs:
        n = seg.num_docs
        for fi, flt in enumerate(_filters(n)):
            for cols in COLSETS:
                full = expected(oracle, [seg], flt, cols, None, False)
                d = len(full[0]["doc_ids"])
                for limit in sorted({0, 1, max(d - 1, 0), d, d + 1}):
                    _check(oracle, pm, [(seg, dev)], flt, cols, limit, what=f"n={n} f={fi} {cols} l={limit}", want=full)


ORDERS = [([("i", True)], ["i"]), ([("i", False)], ["i", "s"]), ([("s", False)], ["s", "i", "l"]),
          ([("l", False), ("f", True)], ["f", "l", "s"]), ([("r", True), ("d", False)], ["d", "r"]),
          ([("s", True), ("f", False), ("i", True)], ["i", "s", "f", "d"]), ([("d", False)], ["d", "s"])]


def test_order_by(oracle, pm, segs):
    for seg, dev in segs:
        n = seg.num_docs
        for fi, flt in enumerate(_filters(n)[:1] + _filters(n)[2:]):
            for oi, (order, cols) in enumerate(ORDERS):
                full = expected(oracle, [seg], flt, cols, None, False, order)
                d = len(full[0]["doc_ids"])
                for limit in sorted({0, 1, 10, max(d - 1, 0), d + 1}):
                    _check(oracle, pm, [(seg, dev)], flt, cols, limit, what=f"n={n} f={fi} o={oi} l={limit}", order_by=order, want=full)


def test_large_output_and_key_spaces(oracle, ctx, pm, segs):
    seg, dev = segs[-1]
    # most of the 196 609 rows hold distinct (i, r, s) tuples, 32 bytes each: beyond the mapped-write bound (staged, one DMA)
    _check(oracle, pm, [(seg, dev)], None, ["i", "r", "s"], 1_000_000, what="large")
    _check(oracle, pm, [(seg, dev)], None, ["i", "r", "s"], 1_000_000, what="large ordered", order_by=[("r", False), ("s", True)])
    n = 2 * 4096
    rng = np.random.default_rng(9)
    a = np.arange(n, dtype=np.int32) % 4096
    rng.shuffle(a)
    kseg = oracle.build_segment("keyspace", {"one": np.full(n, 5, dtype=np.int32), "a": a, "b": (a * 7 + 3) % 4096,
                                             "c": np.arange(n, dtype=np.int32) % 4097})
    kdev = to_device(ctx, kseg)
    try:
        _check(oracle, pm, [(kseg, kdev)], None, ["one"], 10, what="one value")
        _check(oracle, pm, [(kseg, kdev)], None, ["a", "one", "b"], 100, what="2^24 keys")        # 4096 x 1 x 4096
        _check(oracle, pm, [(kseg, kdev)], None, ["b", "a"], 5000, what="2^24 keys ordered", order_by=[("a", False)])
        with pytest.raises(UnsupportedQueryError):
            pm.execute_distinct([kdev], DistinctQuery(columns=["a", "c"], limit=10))              # 4096 x 4097
    finally:
        kdev.destroy()


def test_refusals(pm, segs):
    _, dev = segs[0]
    with pytest.raises(UnsupportedQueryError):
        pm.execute_distinct([dev], DistinctQuery(columns=["i"], limit=1_000_001))
    with pytest.raises(Pb200Error) as e:
        pm.execute_distinct([dev], DistinctQuery(columns=["i"], order_by=[("s", True)], limit=3))   # not a DISTINCT column
    assert e.value.code == E_INVALID
    with pytest.raises(UnsupportedQueryError):
        pm.execute_distinct([dev], DistinctQuery(columns=["i", "s", "l", "f", "d", "r", "inv", "rid", "i"], limit=3))


def test_prefix_route(oracle, ctx, pm):
    """The prefix covers docs [0, P), P >= 2^20 whole tiles (< 1 100 000 at 6 or 8 warps); `late` = doc // 100 000 holds 11
    distinct values there.  LIMIT 11 is final after the prefix, LIMIT 12 needs the rescan; num_docs_scanned tells which."""
    n = 1_500_000
    pairs = []
    try:
        for k in range(2):
            rng = np.random.default_rng(70 + k)
            seg = oracle.build_segment(f"dprefix{k}", {"late": (np.arange(n) // 100_000).astype(np.int32),
                                                        "v": rng.integers(0, 50, size=n).astype(np.int32)})
            pairs.append((seg, to_device(ctx, seg)))
        for merge in (False, True):
            use = pairs if merge else pairs[:1]
            for limit, final in ((5, True), (11, True), (12, False), (15, False)):
                what = f"late limit={limit} merge={merge}"
                got = pm.execute_distinct([d for _, d in use], DistinctQuery(columns=["late"], limit=limit), merge=merge)
                want = expected(oracle, [s for s, _ in use], None, ["late"], limit, merge)
                b = got if merge else got[0]
                _check_block(b, want[0], 1, what, full_scan=False)
                if final:
                    assert b.stats.num_docs_scanned < n * len(use), what
                else:   # merged: segment 0 was truncated first, both truncated segments are scanned again in full
                    assert b.stats.num_docs_scanned == n * len(use), what
            # v >= 10: the prefix holds all 40 values, LIMIT 40 is final, LIMIT 41 rescans (and still finds 40)
            for limit, final in ((40, True), (41, False)):
                flt = Predicate("RANGE", "v", [], 10, None, True, True)
                got = pm.execute_distinct([d for _, d in use], DistinctQuery(columns=["v"], filter=flt, limit=limit), merge=merge)
                want = expected(oracle, [s for s, _ in use], flt, ["v"], limit, merge)
                for b, w in zip([got] if merge else got, want):
                    _check_block(b, w, 1, f"v limit={limit} merge={merge}", full_scan=not final)
                    if final:
                        assert b.stats.num_docs_scanned < w["matched"]
        # ORDER BY scans every doc
        _check(oracle, pm, pairs, None, ["late"], 3, merge=False, what="ordered", order_by=[("late", False)])
    finally:
        for _, d in pairs:
            d.destroy()


def test_many_segments_domain(oracle, ctx, pm):
    pairs = []
    domain = None
    try:
        for k in range(17):
            seg = _segment(oracle, 3_000 + 977 * k, 200 + k)
            pairs.append((seg, to_device(ctx, seg)))
        devs = [d for _, d in pairs]
        flt = Predicate("RANGE", "r", [], -500_000, None, True, True)
        # "r" (2 000 values, a few thousand rows per segment) has a different dictionary in every segment: bind a domain
        with pytest.raises(UnsupportedQueryError):
            pm.execute_distinct(devs, DistinctQuery(columns=["s", "r"], filter=flt, limit=10), merge=True)
        for order in ([], [("s", False), ("r", True)]):
            # per segment, unbound: the by-value merge equals the merged reference
            per = pm.execute_distinct(devs, DistinctQuery(columns=["s", "r"], filter=flt, limit=40, order_by=order))
            merged = merge_distinct_blocks(per, order, 40)
            assert_rows_equal(merged, expected(oracle, [s for s, _ in pairs], flt, ["s", "r"], 40, True, order)[0], f"by value {order}")
        domain = DictionaryDomain.build(ctx, devs, ["i", "s", "l"])
        for d in devs:
            d.bind_domain(domain)
        for cols, order in ((["i", "s"], []), (["i", "s"], [("s", False), ("i", True)]), (["l"], [("l", True)])):
            for limit in (0, 7, 5_000):
                for merge in (True, False):
                    _check(oracle, pm, pairs, flt, cols, limit, merge=merge, what=f"bound {cols} {order} {limit} {merge}", order_by=order)
    finally:
        for _, d in pairs:
            d.destroy()
        if domain is not None:
            domain.release()


def test_knobs(oracle, ctx, pm, segs):
    for knobs in KNOBS:
        with tuned(ctx, **knobs):
            for seg, dev in segs[3:]:
                for flt in _filters(seg.num_docs)[2:]:
                    _check(oracle, pm, [(seg, dev)], flt, ["s", "i"], 1000, what=f"{knobs}")
                    _check(oracle, pm, [(seg, dev)], flt, ["s", "i"], 10, what=f"{knobs} ordered", order_by=[("i", False)])


def test_threads(oracle, ctx, segs):
    pairs = segs[3:]
    errors = []

    def work(t):
        try:
            pm = B200PlanMaker(ctx)
            for k in range(6):
                seg, dev = pairs[(t + k) % len(pairs)]
                flt = _filters(seg.num_docs)[(t + k) % 10]
                _check(oracle, pm, [(seg, dev)], flt, COLSETS[(t + k) % 4], 20 + t, what=f"thread {t}",
                       order_by=[(COLSETS[(t + k) % 4][0], t % 2 == 0)] if k % 2 else [])
        except Exception as e:  # noqa: BLE001
            errors.append(e)
    threads = [threading.Thread(target=work, args=(t,)) for t in range(4)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
