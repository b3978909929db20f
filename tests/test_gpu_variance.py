"""-m gpu: VAR_POP / VAR_SAMP / STDDEV_POP / STDDEV_SAMP against the exact reference (tests/variance_ref.py): every value
within 1 ulp of the exact rational (in practice equal to it rounded once), and bit-identical across routes and knobs.

Columns: INT at INT_MIN and INT_MAX (k up to 2^32 - 1 in one group), LONG near +2^62 and -2^62, dyadic FLOAT and DOUBLE, a
raw INT column whose dictionary is synthesised at load and a DATETRUNC derived column.  Routes: aggregation only, the
dense global table, the shared-memory table, the hash table, 17 segments merged over a domain and per segment, ORDER BY
ASC / DESC with LIMIT and ties.  Four threads race on the first limb build of one dictionary.  Every refusal."""
import ctypes as C
import threading

import numpy as np
import pytest

import variance_ref as vr
from gpu_util import to_device, tuned
from percentile_ref import group_values
from pinot_b200 import cli, sql
from pinot_b200._lib import E_UNSUPPORTED, UnsupportedQueryError
from pinot_b200.plan_maker import B200Context, B200PlanMaker, DictionaryDomain
from pinot_b200.query import Aggregation, Filter, Predicate, QueryContext

pytestmark = pytest.mark.gpu

INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
SIZES = [1, 1_025, 49_157]
COLUMNS = ["i", "lp", "ln", "f", "d", "r"]
FNS = list(vr.FUNCTIONS)
HOUR = 3_600_000


def _segment(oracle, n, seed, name=None):
    rng = np.random.default_rng(seed)
    i = (rng.integers(0, 3000, size=n) * 7 - 9000).astype(np.int32)
    i[rng.integers(0, n, size=max(1, n // 50))] = INT_MAX
    i[rng.integers(0, n, size=max(1, n // 50))] = INT_MIN
    cols = {"rid": np.arange(n, dtype=np.int32),
            "i": i,
            "lp": ((1 << 62) + rng.integers(0, 1 << 32, size=n)).astype(np.int64),
            "ln": (-(1 << 62) + rng.integers(0, 1 << 32, size=n)).astype(np.int64),
            "lw": rng.integers(0, 1 << 40, size=n).astype(np.int64),              # range >= 2^32: refused
            "f": (rng.integers(-400, 400, size=n) / 8.0).astype(np.float32),
            "d": rng.integers(-60000, 60000, size=n) / 8.0,
            "d3": rng.integers(-600, 600, size=n) / 10.0,                          # 0.1-steps: refused
            "r": rng.integers(-1000, 1000, size=n).astype(np.int32) * 1000,
            "ts": (1_700_000_000_000 + rng.integers(0, 10 * 24 * HOUR, size=n)).astype(np.int64),
            "g": rng.integers(0, 10, size=n).astype(np.int32),
            "h": rng.integers(0, 300, size=n).astype(np.int32),
            "s": np.array([b"a", b"ab", b"b"])[rng.integers(0, 3, size=n)]}
    return oracle.build_segment(name or f"var{n}_{seed}", cols, raw=["r"])


def _filters(n):
    return [None,
            Predicate("RANGE", "i", [], 10 ** 10, None, True, True),   # folds to EMPTY on the host
            Predicate("RANGE", "i", [], -5000, 9000, True, False),
            Predicate("IN", "g", [1, 4, 7]),
            Filter("AND", [Predicate("RANGE", "f", [], -20.0, 30.0, True, True), Predicate("RANGE", "rid", [], 0, n // 2, True, True)])]


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


def _query(aggs, flt=None, group_by=(), order_by=(), limit=100_000, **kw):
    return QueryContext(aggregations=list(aggs), filter=flt, group_by=list(group_by), order_by=list(order_by), limit=limit,
                        num_groups_limit=100_000, **kw)


def _key_of(seg, group_by, keys_row):
    out = []
    for j, c in enumerate(group_by):
        v = seg.value_of(c, int(keys_row[j]))
        out.append(v.decode() if isinstance(v, bytes) else (v.item() if hasattr(v, "item") else v))
    return tuple(out)


def _check(oracle, data, q, b, what, values=None):
    """Every VAR / STDDEV of block b against the reference over the segments `data`; returns {(a, key): value}."""
    got = {}
    refs = {}
    rows = 1 if b.num_groups < 0 else b.num_groups
    for a, agg in enumerate(q.aggregations):
        if agg.function not in vr.FUNCTIONS:
            continue
        if agg.column not in refs:
            refs[agg.column] = values if values is not None else group_values(oracle, data, q.filter, q.group_by, agg.column)
        ref = refs[agg.column]
        if q.group_by:
            assert b.num_groups == len(ref) or q.order_by, what
        for g in range(rows):
            key = () if b.num_groups < 0 else _key_of(data[0], q.group_by, b.keys[g])
            sums = vr.exact_sums(ref[key])
            v = float(b.doubles[a][g])
            assert vr.within_one_ulp(v, agg.function, sums), f"{what} a={a} key={key}: {v!r} vs {vr.final(agg.function, sums)!r}"
            assert int(b.longs[a][g]) == sums[0], what
            got[(a, key)] = np.float64(v).tobytes()
    return got


def _sets(col, extra=()):
    """All four functions of one column, in two queries: the column's three internal sums and at most three of the
    caller's aggregations fit the six a query has"""
    return [[Aggregation(fn, col) for fn in FNS[:3]], [Aggregation(FNS[3], col)] + list(extra)]


def test_aggregation_only(oracle, pm, segs):
    for seg, dev in segs:
        for fi, flt in enumerate(_filters(seg.num_docs)):
            for col in COLUMNS:
                for aggs in _sets(col, [Aggregation("COUNT")]):
                    q = _query(aggs, flt)
                    _check(oracle, [seg], q, pm.execute_segments([dev], q)[0], f"n={seg.num_docs} f={fi} {col}")


def test_extremes_in_one_group(oracle, ctx, pm):
    """k = 0 and k = 2^32 - 1 in one group at the largest n the test affords: the 128-bit bounds on the device."""
    n = 100_003
    cols = {"i": np.where(np.arange(n) % 2 == 0, INT_MIN, INT_MAX).astype(np.int32), "g": np.zeros(n, dtype=np.int32)}
    cols["i"][0] = 5
    seg = oracle.build_segment("var_ext", cols)
    dev = to_device(ctx, seg)
    try:
        for gb in ([], ["g"]):
            for aggs in _sets("i"):
                q = _query(aggs, group_by=gb)
                _check(oracle, [seg], q, pm.execute_segments([dev], q)[0], f"extremes {gb}")
    finally:
        dev.destroy()


ROUTES = [("smem", {}), ("global", {"smem_groups": 0}), ("hash", {"dense_max": 1}), ("no_carrier", {"pack_count": 0}),
          ("warps8", {"warps": 8}), ("no_defer", {"defer": 0, "gb_defer": 0}), ("grid1", {"grid": 1})]


def test_routes_bit_identical(oracle, ctx, pm, segs):
    seg, dev = segs[-1]
    shapes = [([Aggregation("VARPOP", "i"), Aggregation("STDDEVSAMP", "i"), Aggregation("SUM", "i")], []),
              ([Aggregation("STDDEVSAMP", "d"), Aggregation("VARPOP", "d"), Aggregation("SUM", "i")], ["g"]),   # count carrier
              ([Aggregation("VARSAMP", "lp"), Aggregation("STDDEVPOP", "lp"), Aggregation("COUNT")], ["g"]),
              ([Aggregation("VARSAMP", "r"), Aggregation("STDDEVPOP", "r")], ["h"]),
              ([Aggregation("STDDEVPOP", "f"), Aggregation("COUNT")], ["h", "g"]),
              ([Aggregation("VARPOP", "ln"), Aggregation("AVG", "ln")], ["g", "s"])]
    for si, (aggs, gb) in enumerate(shapes):
        for fi, flt in enumerate(_filters(seg.num_docs)[2:4]):
            q = _query(aggs, flt, group_by=gb)
            first = None
            for name, knobs in ROUTES:
                with tuned(ctx, **knobs):
                    got = _check(oracle, [seg], q, pm.execute_segments([dev], q)[0], f"shape {si} f={fi} {name}")
                if first is None:
                    first = got
                assert got == first, f"shape {si} f={fi}: {name} differs from the shared-memory route"


def test_order_by_with_ties(oracle, pm, segs):
    seg, dev = segs[-1]
    for asc in (True, False):
        for limit in (1, 3, 10):
            q = _query([Aggregation("COUNT"), Aggregation("STDDEVPOP", "i")], None, group_by=["h"],
                       order_by=[("stddevpop(i)", asc)], limit=limit, min_segment_group_trim_size=1)
            b = pm.execute_segments([dev], q)[0]
            ref = group_values(oracle, [seg], None, ["h"], "i")
            val = {k: vr.final("STDDEVPOP", vr.exact_sums(v)) for k, v in ref.items()}
            want = sorted(ref, key=lambda k: (val[k] if asc else -val[k], k))
            got = [_key_of(seg, ["h"], b.keys[g]) for g in range(b.num_groups)]
            assert got == want[:len(got)] and len(got) >= limit, (asc, limit)
            # ties: a constant column gives 0 in every group (and -inf for VARSAMP of one-row groups), keys break them
            q = _query([Aggregation("VARSAMP", "g")], Predicate("EQ", "g", [3]), group_by=["h"],
                       order_by=[("var_samp(g)", asc)], limit=limit, min_segment_group_trim_size=1)
            b = pm.execute_segments([dev], q)[0]
            ref = group_values(oracle, [seg], q.filter, ["h"], "g")
            val = {k: vr.final("VARSAMP", vr.exact_sums(v)) for k, v in ref.items()}
            want = sorted(ref, key=lambda k: (val[k] if asc else -val[k], k))
            assert [_key_of(seg, ["h"], b.keys[g]) for g in range(b.num_groups)] == want[:b.num_groups]


def test_seventeen_segments_merged_on_device(oracle, ctx, pm):
    data = [_segment(oracle, 20_000 + 37 * k, 1000 + k, name=f"var17_{k}") for k in range(17)]
    devs = [to_device(ctx, s) for s in data]
    domain = None
    flt = Predicate("RANGE", "i", [], -5000, 9000, True, False)
    try:
        for gb in ([], ["g"]):
            for aggs in ([Aggregation("STDDEVSAMP", "i"), Aggregation("VARPOP", "i"), Aggregation("COUNT")],
                         [Aggregation("VARSAMP", "d"), Aggregation("STDDEVPOP", "d")]):
                q = _query(aggs, flt, group_by=gb)
                per_seg = cli.final_rows(q, cli.merge_blocks(q, devs, pm.execute_segments(devs, q)))
                refs = {a.column: group_values(oracle, data, flt, gb, a.column) for a in aggs if a.column}
                assert len(per_seg) == len(refs[aggs[0].column])
                for row in per_seg:
                    key = tuple(row[:len(gb)])
                    for a, agg in enumerate(aggs):
                        if agg.function in FNS:
                            assert row[len(gb) + a] == vr.final(agg.function, vr.exact_sums(refs[agg.column][key])), (gb, agg, key)
                if domain is None:
                    with pytest.raises(UnsupportedQueryError):   # no shared dictionary: refused, never merged by dictId
                        pm.execute_segments(devs, q, merge=True)
                    domain = DictionaryDomain.build(ctx, devs, ["i", "d", "g"])
                    for d in devs:
                        d.bind_domain(domain)
                merged = pm.execute_segments(devs, q, merge=True)[0]
                _check(oracle, data, q, merged, f"merged {gb}")
                assert cli.final_rows(q, cli.merge_blocks(q, devs[:1], [merged])) == per_seg
    finally:
        for d in devs:
            d.destroy()
        if domain is not None:
            domain.release()


def test_derived_column(oracle, ctx, pm, segs):
    seg, dev = segs[-1]
    q = sql.parse("SELECT g, VAR_POP(DATETRUNC('HOUR', ts)), STDDEV_SAMP(DATETRUNC('HOUR', ts)) FROM t GROUP BY g LIMIT 100")
    col = q.aggregations[0].column
    assert q.aggregations[1].column == col
    b = pm.execute_segments([dev], q)[0]
    ts = group_values(oracle, [seg], None, ["g"], "ts")
    buckets = {k: (v // HOUR) * HOUR for k, v in ts.items()}
    _check(oracle, [seg], q, b, "datetrunc", values=buckets)


def test_racing_first_build(oracle, ctx, pm):
    seg = _segment(oracle, 30_011, 77, name="var_race")
    dev = to_device(ctx, seg)
    try:
        q = _query(_sets("d")[0], group_by=["g"])
        out, errors = [None] * 4, []
        start = threading.Barrier(4)

        def run(t):
            try:
                start.wait()
                b = pm.execute_segments([dev], q)[0]
                out[t] = [(tuple(b.keys[g]), np.asarray([b.doubles[a][g] for a in range(3)]).tobytes()) for g in range(b.num_groups)]
            except Exception as e:   # noqa: BLE001 -- reported below
                errors.append(e)
        threads = [threading.Thread(target=run, args=(t,)) for t in range(4)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        assert not errors, errors
        assert out[0] == out[1] == out[2] == out[3]
        _check(oracle, [seg], q, pm.execute_segments([dev], q)[0], "after the race")
    finally:
        dev.destroy()


def test_empty_and_single_row(oracle, pm, segs):
    seg, dev = segs[0]   # one row: *POP 0, *SAMP -inf
    for gb in ([], ["g"]):
        got = []
        for aggs in _sets("i"):
            q = _query(aggs, group_by=gb)
            b = pm.execute_segments([dev], q)[0]
            _check(oracle, [seg], q, b, f"one row {gb}")
            got += [float(b.doubles[a][0]) for a in range(len(aggs))]
        assert got == [0.0, float("-inf"), 0.0, float("-inf")]
    seg, dev = segs[-1]
    flt = Filter("AND", [Predicate("RANGE", "rid", [], 0, 5, True, True), Predicate("RANGE", "rid", [], 10, 20, True, True)])
    for aggs in _sets("d", [Aggregation("COUNT")]):
        b = pm.execute_segments([dev], _query(aggs, flt))[0]
        assert all(float(b.doubles[a][0]) == float("-inf") for a, x in enumerate(aggs) if x.function in FNS)
        assert all(int(b.longs[a][0]) == 0 for a in range(len(aggs)))


def test_refusals(oracle, ctx, pm, segs):
    seg, dev = segs[-1]
    for col in ("s", "lw", "d3"):   # STRING, LONG range >= 2^32, 0.1-steps
        with pytest.raises(UnsupportedQueryError):
            pm.execute_segments([dev], _query([Aggregation("VARPOP", col)]))
    with pytest.raises(UnsupportedQueryError):   # more than 6 aggregations with the 3 internal sums of each column
        pm.execute_segments([dev], _query([Aggregation("VARPOP", "i"), Aggregation("VARPOP", "d"), Aggregation("COUNT")]))
    pm.execute_segments([dev], _query([Aggregation("VARPOP", "i"), Aggregation("STDDEVSAMP", "i"), Aggregation("SUM", "i")]))
    with pytest.raises(UnsupportedQueryError):   # FILTER (WHERE ...) clause
        pm.execute_segments([dev], _query([Aggregation("VARPOP", "i", filter=Predicate("EQ", "g", [1]))]))
    with pytest.raises(UnsupportedQueryError):   # a clause on another function
        pm.execute_segments([dev], _query([Aggregation("COUNT", filter=Predicate("EQ", "g", [1])), Aggregation("VARPOP", "i")]))
    q = _query([Aggregation("VARPOP", "i")], group_by=["g"])
    with pytest.raises(UnsupportedQueryError):   # deferred finalize (cross-GPU reduce)
        pm.execute_segments([dev], q, merge=True, keep_handle=True)
    for gb in ([], ["g"]):
        q = _query([Aggregation("VARPOP", "i"), Aggregation("SUM", "i")], group_by=gb)
        b = pm.execute_segments([dev], q, merge=True, keep_handle=True, defer=False)[0]
        try:
            p, n = C.c_void_p(), C.c_int64()
            for kind in range(4):
                assert ctx.lib.pb200_result_device_buffers(b.handle, kind, C.byref(p), C.byref(n)) == E_UNSUPPORTED
        finally:
            b.release(ctx)
    q = _query([Aggregation("STDDEVPOP", "i")])
    b = pm.execute_segments([dev], q, keep_handle=True, defer=False)[0]
    try:
        with pytest.raises(UnsupportedQueryError):   # DataTable bytes of the reference's VarianceTuple
            pm.to_datatable(dev, q, b)
    finally:
        b.release(ctx)
    with tuned(ctx, raw_dict_max=0):   # raw INT streamed as 32-bit values: no dictIds
        raw = to_device(ctx, _segment(oracle, 5_000, 5, name="var_raw"))
    try:
        with pytest.raises(UnsupportedQueryError):
            pm.execute_segments([raw], _query([Aggregation("VARPOP", "r")]))
    finally:
        raw.destroy()


def test_cli_over_segment_directories(oracle, tmp_path, capsys):
    """SELECT g, STDDEV_SAMP(m), VAR_POP(m) ... ORDER BY STDDEV_SAMP(m) DESC LIMIT 10 over segment directories: the same
    rows from per-segment moments merged by value and from one submission merged on the device."""
    import json
    from segment_dir_util import write_segment_dir
    rng = np.random.default_rng(31)
    data, dirs = [], []
    for i, version in enumerate(["v1", "v3", "v3"]):
        n = 9_000 + 13 * i
        seg = oracle.build_segment(f"varcli{i}", {"g": rng.integers(0, 20 + i, size=n).astype(np.int32),
                                                  "m": (rng.integers(-3000, 3000, size=n) * (i + 1)).astype(np.int32)})
        data.append(seg)
        dirs.append(write_segment_dir(str(tmp_path / f"seg{i}"), seg, version))
    text = "SELECT g, STDDEV_SAMP(m), VAR_POP(m) FROM t GROUP BY g ORDER BY STDDEV_SAMP(m) DESC LIMIT 10"
    q = sql.parse(text)
    ref = group_values(oracle, data, None, ["g"], "m")
    want = sorted(([k[0], vr.final("STDDEVSAMP", vr.exact_sums(v)), vr.final("VARPOP", vr.exact_sums(v))] for k, v in ref.items()),
                  key=lambda r: (-r[1], r[0]))[:q.limit]
    rows = []
    for on_device in (False, True):
        argv = [text, "--json"] + [x for d in dirs for x in ("--segment-dir", d)] + (["--merge-on-device"] if on_device else [])
        assert cli.main(argv) == 0
        rows.append(json.loads(capsys.readouterr().out.strip().splitlines()[-1])["rows"])
    assert rows[0] == rows[1] == want
