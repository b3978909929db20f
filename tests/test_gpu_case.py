"""-m gpu: SUM / AVG / MIN / MAX over CASE WHEN (DESIGN.md section 3.19) against the per-row reference tests/case_ref.py:
sums within gamma_n * sum|x| of the exact sum (NaN / +-inf / +0.0 by rule), MIN / MAX bit for bit in Double.compare
order, AVG counts exact.

Segments of 1 .. 100 003 rows hold INT, LONG (at the int64 ends and 2^53 + 1), FLOAT, DOUBLE and STRING condition
columns, branch values with NaN, +-inf and -0.0, and raw INT / DOUBLE columns (dictionaries synthesised at load).
Aggregation only and GROUP BY on the shared-memory, dense and hash tables, the count carrier on and off, with and without
WHERE, next to column and arithmetic expression aggregations; 17 merged segments whose STRING dictionaries differ;
ORDER BY ... LIMIT, HAVING, post-aggregation ORDER BY, a FILTER clause, the CLI, the statistics, the DataTable refusal
and the library's refusals."""
import json

import numpy as np
import pytest

from case_ref import row_values
from expr_ref import check_value
from filter_ref import matching_docs
from gpu_util import to_device, tuned
from pinot_b200 import cli, sql
from pinot_b200._lib import Pb200Error, UnsupportedQueryError
from pinot_b200.plan_maker import B200Context, B200PlanMaker, DictionaryDomain
from pinot_b200.query import Aggregation, Predicate, QueryContext

pytestmark = pytest.mark.gpu

INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
SIZES = [1, 31, 33, 4096, 100_003]
FNS = ["SUM", "AVG", "MIN", "MAX"]
STATUS = np.array([b"ok", b"error", b"warn", b"retry", b"fatal error"])
CASES = [
    "CASE WHEN s = 'error' THEN i ELSE 0 END",
    "CASE WHEN s IN ('warn', 'retry', 'nope') THEN d ELSE -d END",
    "CASE WHEN i > 1000 AND NOT l BETWEEN -5 AND 5 THEN l WHEN f <= 2.5 THEN f * 2 ELSE 0.5 END",
    "CASE WHEN s LIKE '%error' OR e > 10.5 THEN e / j WHEN s NOT IN ('ok') THEN i - l ELSE d END",
    "CASE WHEN l = 9007199254740993 THEN 1 WHEN l > 4611686018427387904 THEN 2 WHEN l < -9007199254740992 THEN 3 ELSE 0 END",
    "CASE WHEN REGEXP_LIKE(s, '^w') THEN ri WHEN ri < 0 THEN rd ELSE i * j END",
    "CASE WHEN i <> 5 AND i != 7.5 THEN 1 ELSE 0 END",
    "CASE WHEN i >= 2.5 THEN i ELSE 0 END",
]


def _segment(oracle, n, seed, name=None, statuses=STATUS, raw_double=True):
    rng = np.random.default_rng(seed)
    i = (rng.integers(-300, 300, size=n) * 7).astype(np.int32)
    i[rng.integers(0, n, size=max(1, n // 50))] = INT_MAX
    i[rng.integers(0, n, size=max(1, n // 50))] = INT_MIN
    longs = np.array([INT64_MIN, INT64_MAX, (1 << 53) + 1, -(1 << 53) - 1, (1 << 62) + 3, 0, 5, -5], dtype=np.int64)
    lv = rng.integers(-10_000, 10_000, size=n).astype(np.int64)
    lv[rng.integers(0, n, size=max(1, n // 20))] = longs[rng.integers(0, len(longs), size=max(1, n // 20))]
    d = rng.integers(-600, 600, size=n) / 3.0
    d[rng.integers(0, n, size=max(1, n // 90))] = -0.0
    if n > 1000:
        d[rng.integers(0, n, size=2)] = np.nan
        d[rng.integers(0, n, size=1)] = np.inf
    cols = {"rid": np.arange(n, dtype=np.int32), "i": i, "j": rng.integers(-3, 4, size=n).astype(np.int32), "l": lv,
            "f": (rng.integers(-40, 40, size=n) / 8.0 + 0.0625).astype(np.float32),   # no -0.0 or NaN: a condition column
            "e": rng.integers(-100, 100, size=n) / 4.0 + 0.125,                        # likewise
            "d": d, "s": statuses[rng.integers(0, len(statuses), size=n)],
            "ri": rng.integers(-1_000_000, 1_000_000, size=n).astype(np.int32), "rd": rng.integers(-50, 50, size=n) / 4.0 if raw_double else rng.integers(-50, 50, size=n).astype(np.int32),
            "g": rng.integers(0, 10, size=n).astype(np.int32), "h": rng.integers(0, 3000, size=n).astype(np.int32)}
    return oracle.build_segment(name or f"case{n}_{seed}", cols, raw=["ri", "rd"])


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
    for n in SIZES:
        seg = _segment(oracle, n, n)
        out.append((seg, to_device(ctx, seg)))
    yield out
    for _, dev in out:
        dev.destroy()


def _arg(text):
    return sql.parse(f"SELECT SUM({text}) FROM t").aggregations[0].column


def _query(aggs, flt=None, group_by=()):
    return QueryContext(aggregations=list(aggs), filter=flt, group_by=list(group_by), limit=100_000)


def _py(v):
    return v.decode("utf-8") if isinstance(v, bytes) else (v.item() if hasattr(v, "item") else v)


def _check(oracle, data, dev, q, b, what):
    rows = 1 if b.num_groups < 0 else b.num_groups
    got = {tuple(_py(dev.dictionary_value(c, int(b.keys[r, k]))) for k, c in enumerate(q.group_by)): r for r in range(rows)}
    checked = 0
    for a, agg in enumerate(q.aggregations):
        if agg.function not in FNS or not (agg.column or "").startswith("case("):
            continue
        ref = row_values(oracle, data, q.filter, q.group_by, agg.column)
        if q.group_by:
            assert set(got) == set(ref), f"{what} {agg}: groups differ"
        for key, r in got.items():
            xs = ref.get(key, [])
            d, l = float(b.doubles[a][r]), int(b.longs[a][r])
            assert check_value(agg.function, d, l, xs), f"{what} {agg.function}({agg.column}) {key}: {d!r} ({l}) over {len(xs)} rows"
        checked += 1
    assert checked


FILTERS = [None, Predicate("RANGE", "i", [], -1500, 1800, True, False)]


def _aggs(k):
    return [Aggregation(fn, _arg(CASES[(k + m) % len(CASES)])) for m, fn in enumerate(FNS)]


def test_aggregation_only(oracle, pm, segs):
    for seg, dev in segs:
        for flt in FILTERS:
            for k in range(len(CASES)):
                q = _query(_aggs(k) + [Aggregation("COUNT")], flt)
                _check(oracle, [seg], dev, q, pm.execute_segments([dev], q)[0], f"n={seg.num_docs} k={k}")


@pytest.mark.parametrize("knobs", [dict(), dict(dense_max=1), dict(smem_groups=0), dict(pack_count=0), dict(pack_count=1)],
                         ids=["default", "hash", "no_smem", "no_carrier", "carrier"])
def test_group_by(oracle, ctx, pm, segs, knobs):
    """Shared-memory (g), dense (h, smem_groups=0) and hash (dense_max=1) tables; the count carrier on and off; next to a
    column aggregation and an arithmetic expression."""
    with tuned(ctx, **knobs):
        for seg, dev in segs[2:]:
            for gb in (["g"], ["h"]):
                for flt in FILTERS:
                    q = _query([Aggregation("SUM", _arg(CASES[0])), Aggregation("COUNT"), Aggregation("MIN", _arg(CASES[2])),
                                Aggregation("AVG", _arg(CASES[3])), Aggregation("MAX", _arg(CASES[5])), Aggregation("SUM", "times(i,j)")],
                               flt, group_by=gb)
                    b = pm.execute_segments([dev], q)[0]
                    _check(oracle, [seg], dev, q, b, f"{knobs} n={seg.num_docs} {gb}")


def test_next_to_column_aggregations(oracle, pm, segs):
    """Column aggregations in a query with CASE keep the values they have alone."""
    seg, dev = segs[4]
    for gb in ([], ["g"]):
        base = _query([Aggregation("COUNT"), Aggregation("SUM", "i"), Aggregation("MAX", "l")], FILTERS[1], group_by=gb)
        withc = _query([Aggregation("SUM", _arg(CASES[1]))] + base.aggregations, FILTERS[1], group_by=gb)
        a, b = pm.execute_segments([dev], base)[0], pm.execute_segments([dev], withc)[0]
        assert a.num_groups == b.num_groups
        for r in range(1 if a.num_groups < 0 else a.num_groups):
            for x in range(3):
                assert int(a.longs[x][r]) == int(b.longs[x + 1][r]) and float(a.doubles[x][r]) == float(b.doubles[x + 1][r])
        _check(oracle, [seg], dev, withc, b, f"with columns {gb}")


def test_statistics(oracle, pm, segs):
    seg, dev = segs[4]
    matched = int(np.count_nonzero(matching_docs(oracle, seg, FILTERS[1])))
    q = _query([Aggregation("SUM", _arg("CASE WHEN s = 'error' AND g > 3 THEN i WHEN s = 'ok' THEN i * j ELSE 0 END"))],
               FILTERS[1], group_by=["g"])
    b = pm.execute_segments([dev], q)[0]
    assert b.stats.num_docs_scanned == matched
    assert b.stats.num_entries_scanned_post_filter == matched * 4   # g, s, i, j: each column once


def test_synthesised_raw_condition_and_streamed_refusal(oracle, ctx, pm):
    seg = _segment(oracle, 8193, 5)
    dev = to_device(ctx, seg)
    try:
        q = _query([Aggregation("SUM", _arg("CASE WHEN ri > 0 THEN rd ELSE ri END")), Aggregation("MAX", _arg(CASES[5]))], group_by=["g"])
        _check(oracle, [seg], dev, q, pm.execute_segments([dev], q)[0], "synthesised")
    finally:
        dev.destroy()
    with tuned(ctx, raw_dict_max=0):   # ri streamed as 32-bit values: a value leaf yes, a condition column no
        dev = to_device(ctx, _segment(oracle, 8193, 6, raw_double=False))   # a raw DOUBLE column is only loaded with a dictionary
        try:
            q = _query([Aggregation("SUM", _arg("CASE WHEN i > 0 THEN ri ELSE 0 END"))])
            pm.execute_segments([dev], q)
            with pytest.raises(UnsupportedQueryError):
                pm.execute_segments([dev], _query([Aggregation("SUM", _arg("CASE WHEN ri > 0 THEN i ELSE 0 END"))]))
        finally:
            dev.destroy()


def test_seventeen_segments_merged(oracle, ctx, pm):
    """Merged on the device over a domain for the key; each segment's STRING dictionary its own, 'error' present in some."""
    data = []
    for k in range(17):
        statuses = STATUS if k % 3 == 0 else np.array([b"ok", b"warn", b"x%d" % k])
        data.append(_segment(oracle, 3000 + 41 * k, 700 + k, name=f"case17_{k}", statuses=statuses))
    devs = [to_device(ctx, s) for s in data]
    domain = DictionaryDomain.build(ctx, devs, ["g", "h"])
    try:
        for d in devs:
            d.bind_domain(domain)
        for gb in ([], ["g"], ["g", "h"]):
            q = _query([Aggregation("SUM", _arg(CASES[0])), Aggregation("AVG", _arg(CASES[1])), Aggregation("MIN", _arg(CASES[3])),
                        Aggregation("MAX", _arg("CASE WHEN s LIKE 'x%' THEN i ELSE l END")), Aggregation("COUNT")], FILTERS[1], group_by=gb)
            _check(oracle, data, devs[0], q, pm.execute_segments(devs, q, merge=True)[0], f"merged {gb}")
            # per segment too
            for s, b in zip(data, pm.execute_segments(devs, q)):
                _check(oracle, [s], devs[0], q, b, f"per segment {gb}")
    finally:
        for d in devs:
            d.destroy()
        domain.release()


def test_order_by_having_post_and_filter_clause(oracle, pm, segs):
    seg, dev = segs[4]
    case = "CASE WHEN s = 'error' THEN 1 ELSE 0 END"
    ref = row_values(oracle, [seg], None, ["h"], _arg(case))
    q = sql.parse(f"SELECT h, SUM({case}) FROM t GROUP BY h ORDER BY SUM({case}) DESC, h LIMIT 5")
    b = pm.execute_segments([dev], q, merge=True)[0]
    want = sorted(ref, key=lambda k: (-sum(ref[k]), k[0]))[:5]
    assert [(_py(dev.dictionary_value("h", int(b.keys[r, 0]))),) for r in range(5)] == want
    q = sql.parse(f"SELECT h, SUM({case}) FROM t GROUP BY h HAVING SUM({case}) > 3")
    b = pm.execute_segments([dev], q, merge=True)[0]
    assert b.num_groups == sum(1 for xs in ref.values() if sum(xs) > 3)
    q = sql.parse(f"SELECT h, SUM({case}) / COUNT(*) FROM t GROUP BY h ORDER BY SUM({case}) / COUNT(*) DESC, h LIMIT 5")
    b = pm.execute_segments([dev], q, merge=True)[0]
    want = sorted(ref, key=lambda k: (-(sum(ref[k]) / len(ref[k])), k[0]))[:5]
    assert [(_py(dev.dictionary_value("h", int(b.keys[r, 0]))),) for r in range(5)] == want
    q = sql.parse(f"SELECT g, SUM({case}) FILTER (WHERE j > 0), COUNT(*) FROM t GROUP BY g")
    b = pm.execute_segments([dev], q)[0]
    fref = row_values(oracle, [seg], Predicate("RANGE", "j", [], 0, None, False, True), ["g"], _arg(case))
    for r in range(b.num_groups):
        key = (_py(dev.dictionary_value("g", int(b.keys[r, 0]))),)
        assert check_value("SUM", float(b.doubles[0][r]), 0, fref.get(key, [])), key


def test_cli_and_datatable_refusal(oracle, ctx, pm, segs, tmp_path, capsys):
    from segment_dir_util import write_segment_dir
    seg, dev = segs[3]
    q = sql.parse(f"SELECT g, SUM({CASES[0]}) FROM t GROUP BY g")
    b = pm.execute_segments([dev], q, keep_handle=True, defer=False)[0]
    try:
        with pytest.raises((UnsupportedQueryError, Pb200Error)):
            pm.to_datatable(dev, q, b)
    finally:
        b.release(ctx)
    data = [_segment(oracle, 3000 + k, 950 + k, name=f"casecli{k}") for k in range(2)]
    dirs = [str(write_segment_dir(tmp_path / f"s{k}", s)) for k, s in enumerate(data)]
    ref = row_values(oracle, data, None, ["g"], _arg(CASES[0]))
    for extra in ([], ["--merge-on-device"]):
        argv = [f"SELECT g, SUM({CASES[0]}) FROM t GROUP BY g ORDER BY g LIMIT 100", "--json"]
        for d in dirs:
            argv += ["--segment-dir", d]
        capsys.readouterr()
        assert cli.main(argv + extra) == 0
        out = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
        assert len(out["rows"]) == len(ref), extra
        for g, total in out["rows"]:
            assert check_value("SUM", float(total), 0, ref[(int(g),)]), (extra, g)


def test_refusals(oracle, ctx, pm, segs):
    seg, dev = segs[3]
    for text in ("CASE WHEN d > 1 THEN i ELSE 0 END",            # DOUBLE condition column with NaN / -0.0
                 "CASE WHEN s > 'ok' THEN i ELSE 0 END",          # STRING range
                 "CASE WHEN l > 9007199254740993.5 THEN 1 ELSE 0 END",   # LONG against a non-integral literal beyond 2^53
                 "CASE WHEN i > 0 THEN f ELSE i END",             # FLOAT branch next to an INT branch
                 "CASE WHEN i > 0 THEN f ELSE 16777217 END",      # ... or an integer beyond 2^24
                 "CASE WHEN s = 'ok' THEN year(l) ELSE 0 END",    # time function
                 "CASE WHEN i LIKE 'a%' THEN 1 ELSE 0 END"):      # pattern on INT
        with pytest.raises(UnsupportedQueryError):
            pm.execute_segments([dev], _query([Aggregation("SUM", _arg(text))]))
    for ok in ("CASE WHEN i > 0 THEN f ELSE d END", "CASE WHEN i > 0 THEN f ELSE 16777216 END", "CASE WHEN i > 0 THEN f ELSE i + 0 END"):
        q = _query([Aggregation("SUM", _arg(ok))])
        _check(oracle, [seg], dev, q, pm.execute_segments([dev], q)[0], ok)
    with pytest.raises(Pb200Error):
        pm.execute_segments([dev], _query([Aggregation("SUM", _arg("CASE WHEN nosuch = 1 THEN i ELSE 0 END"))]))
    with pytest.raises(UnsupportedQueryError):   # GROUP BY deferred to a later finalize, as for arithmetic expressions
        pm.execute_segments([dev], _query([Aggregation("SUM", _arg(CASES[0]))], group_by=["g"]), merge=True, keep_handle=True)
