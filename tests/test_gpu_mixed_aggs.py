"""-m gpu: queries that mix aggregation functions, every aggregation held to the one reference of tests/mixed_ref.py on
every route.

An aggregation's state is found by its position: DISTINCTSUM / DISTINCTAVG / DISTINCTCOUNTHLL read the bitset of the
first DISTINCTCOUNT or reader of their column, DISTINCTCOUNTHLLs of one column and log2m share one estimate, PERCENTILEs
of one column one histogram, VAR / STDDEV of one column one set of internal sums appended behind the caller's
aggregations.  The shapes here put owners and non-owners side by side: pinned ones, and a seeded draw of up to six
aggregations biased towards repeated columns.  A drawn query over the VAR / STDDEV cap (the caller's aggregations plus 3
internal sums per VAR / STDDEV column at most 6) must be refused, never answered.

Routes: aggregation only; GROUP BY on the shared-memory, dense and hash tables and on two columns; the scan knobs; several
segments in one per-segment submission; 17 segments bound to a domain and merged on the device, and the same merged by
value; a filter that matches every doc and an empty one; FILTER clauses.  ORDER BY (with and without a LIMIT trim) and
HAVING on non-owners.  Each aggregation of a mixed query equals the same aggregation run alone and in a permuted query.
The loopback combine over two ranks."""
import math
import random

import numpy as np
import pytest

import exact_ref
import mixed_ref
from filter_ref import matching_docs
from gpu_util import to_device, tuned
from pinot_b200 import cli, sql
from pinot_b200._lib import UnsupportedQueryError
from pinot_b200.plan_maker import B200Context, B200PlanMaker, DictionaryDomain
from pinot_b200.query import MOMENT_FUNCTIONS

pytestmark = pytest.mark.gpu

INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
SIZES = [1, 33, 8_193, 100_003]
MAX_AGGS = 6


def _segment(oracle, n, seed, name=None):
    """x: INT on a grid of 7 with INT_MIN / INT_MAX; y: INT 0..399; l: LONG near 2^62 on a grid of 2^28; f / d: FLOAT /
    DOUBLE eighths (no NaN or infinity: VAR / STDDEV refuse them); t: INT time with ties, ts: LONG time; r: raw INT; keys g
    (10 values), h (3 000) and s (STRING).  Value columns keep at most a few thousand distinct values, so that two
    PERCENTILE histograms per group stay within the device budget on the hash table (parse's num_groups_limit)."""
    rng = np.random.default_rng(seed)
    x = (rng.integers(-300, 300, size=n) * 7).astype(np.int32)
    x[rng.integers(0, n, size=max(1, n // 80))] = INT_MAX
    x[rng.integers(0, n, size=max(1, n // 80))] = INT_MIN
    cols = {"rid": np.arange(n, dtype=np.int32),
            "x": x,
            "y": rng.integers(0, 400, size=n).astype(np.int32),
            "l": ((1 << 62) + (rng.integers(0, 600, size=n) << 28) + 7).astype(np.int64),
            "f": (rng.integers(-400, 400, size=n) / 8.0).astype(np.float32),
            "d": rng.integers(-600, 600, size=n) / 8.0,
            "t": rng.integers(0, max(2, n // 4), size=n).astype(np.int32),
            "ts": (1_700_000_000_000 + rng.integers(0, 1 << 30, size=n)).astype(np.int64),
            "r": rng.integers(-1000, 1000, size=n).astype(np.int32) * 1000,
            "g": rng.integers(0, 10, size=n).astype(np.int32),
            "h": rng.integers(0, 3000, size=n).astype(np.int32),
            "s": np.array([b"a", b"bc", b"d", b"ef"])[rng.integers(0, 4, size=n)]}
    return oracle.build_segment(name or f"mix{n}_{seed}", cols, raw=["r"])


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
    out = {}
    for n in SIZES:
        seg = _segment(oracle, n, 7 + n)
        out[n] = (seg, to_device(ctx, seg))
    yield out
    for _, dev in out.values():
        dev.destroy()


# ------------------------------------------------------------------------------------------------------------ shapes
PINNED = [
    "PERCENTILE(x, 10), PERCENTILE(x, 90), PERCENTILE(y, 50)",
    "DISTINCTSUM(x), DISTINCTCOUNT(x), DISTINCTAVG(x), DISTINCTCOUNTHLL(x)",
    "DISTINCTCOUNT(x), DISTINCTSUM(x), DISTINCTAVG(x), DISTINCTCOUNTHLL(x)",
    "DISTINCTCOUNTHLL(x), DISTINCTCOUNTHLL(x, 8), DISTINCTCOUNTHLL(x, 12)",
    "STDDEV_POP(x), VAR_SAMP(x), PERCENTILE(x, 50)",
    "STDDEV_POP(x), VAR_SAMP(x), LASTWITHTIME(x, t, 'INT')",
    "VAR_POP(x), STDDEV_SAMP(x), SUM(y)",     # at the cap: 3 + 3; SUM(y) may carry the counts, a limb sum never
    "VAR_POP(d), AVG(y), SUM(y)",
    "SUM(x), VAR_POP(x), DISTINCTCOUNTHLL(x)",   # an INT SUM over the column of the limb sums, and an HLL beside them
    "SUM(x * d), STDDEV_POP(y), MIN(y - x)",     # expressions beside VAR / STDDEV: the limb sums follow them
    "SUM(x * d), MIN(x - y), PERCENTILE(d, 25), DISTINCTAVG(d), DISTINCTCOUNTHLL(d, 12), FIRSTWITHTIME(d, ts, 'DOUBLE')",
    "MAX(f * y), AVG(l - x), STDDEV_SAMP(d)",
    "MIN(y + r), DISTINCTCOUNT(l), DISTINCTSUM(l), LASTWITHTIME(l, ts, 'LONG'), PERCENTILE(l, 100), SUM(f)",
    "SUM(f), AVG(d), MIN(l), MAX(r), DISTINCTCOUNT(s), DISTINCTCOUNTHLL(s)",
    "PERCENTILE(r, 50), DISTINCTSUM(r), VAR_SAMP(r)",
    "LASTWITHTIME(y, ts, 'INT'), FIRSTWITHTIME(y, ts, 'INT'), PERCENTILE(y, 75), PERCENTILE(y, 0), DISTINCTAVG(y), MAX(y)",
]
OVER_CAP = ["VAR_POP(x), STDDEV_SAMP(x), SUM(y), COUNT(*)", "VAR_POP(x), VAR_POP(y)",
            "PERCENTILE(x, 50), DISTINCTSUM(y), SUM(y), STDDEV_POP(d), MAX(f)"]

# the random draw: each function with the columns it takes (VAR / STDDEV not over l: the values of an integer column must
# span less than 2^32 for them)
DRAW = {"COUNT(*)": None, "SUM": "xylfdr", "AVG": "xyfd", "MIN": "xylfds", "MAX": "xylfdr", "DISTINCTCOUNT": "xylfs",
        "DISTINCTSUM": "xyld", "DISTINCTAVG": "xyfr", "DISTINCTCOUNTHLL": "xylds", "PERCENTILE": "xyldr",
        "VAR_POP": "xyd", "VAR_SAMP": "xyf", "STDDEV_POP": "xyr", "STDDEV_SAMP": "yd", "LASTWITHTIME": "xyl",
        "FIRSTWITHTIME": "yd", "EXPR": "xyd"}
TYPES = {"x": "INT", "y": "INT", "l": "LONG", "f": "FLOAT", "d": "DOUBLE", "r": "INT", "s": "STRING"}


def _draw(rng):
    """Up to six aggregations over two columns, so that most share a column with another."""
    pool = rng.sample("xyd", 1) + rng.sample("xylfdr", 1)
    out = []
    for _ in range(rng.randint(2, MAX_AGGS)):
        fn = rng.choice(list(DRAW))
        cols = [c for c in pool if DRAW[fn] is None or c in DRAW[fn]] or list(DRAW[fn] or "x")
        c = rng.choice(cols)
        if fn == "COUNT(*)":
            out.append(fn)
        elif fn == "PERCENTILE":
            out.append(f"PERCENTILE({c}, {rng.choice([0, 10, 50, 90, 100])})")
        elif fn == "DISTINCTCOUNTHLL":
            out.append(f"DISTINCTCOUNTHLL({c}, {rng.choice([8, 8, 12, 4])})")
        elif fn.endswith("WITHTIME"):
            out.append(f"{fn}({c}, {rng.choice(['t', 'ts'])}, '{TYPES[c]}')")
        elif fn == "EXPR":
            out.append(f"{rng.choice(['SUM', 'MIN', 'MAX', 'AVG'])}({c} {rng.choice('*-+')} {rng.choice('xyd')})")
        else:
            out.append(f"{fn}({c})")
    return ", ".join(out)


DRAWN = [_draw(random.Random(1000 + i)) for i in range(10)]


def over_cap(select):
    """The VAR / STDDEV rule: the caller's aggregations plus 3 internal sums per VAR / STDDEV column at most 6."""
    aggs = parse(select).aggregations
    return len(aggs) + 3 * len({a.column for a in aggs if a.function in MOMENT_FUNCTIONS}) > MAX_AGGS


def parse(select, group_by=(), where=None, tail=""):
    text = f"SELECT {', '.join(list(group_by) + [select])} FROM t" + (f" WHERE {where}" if where else "") + \
        (f" GROUP BY {', '.join(group_by)}" if group_by else "") + (tail or " LIMIT 1000000")
    return sql.parse(text, num_groups_limit=20_000)


class Decoder:
    """dictId -> stored value from the test's own data: a segment's dictionary or, for segments bound to a domain, the sorted
    union of their dictionaries (DictionaryDomain's id space).  Only a raw column, whose dictionary is synthesised at load,
    is read through the product (IndexSegment.dictionary_value)."""

    def __init__(self, data, dev, domain=False):
        self.data, self.dev, self.domain, self.unions = data, dev, domain, {}

    def __call__(self, column, i):
        c = self.data[0].column(column)
        if not c.has_dictionary:
            return self.dev.dictionary_value(column, i)
        if not self.domain:
            return self.data[0].value_of(column, i)
        if column not in self.unions:
            self.unions[column] = np.unique(np.concatenate([exact_ref._dictionary(s.column(column)) for s in self.data]))
        return self.unions[column][i]


class Refs:
    """The reference of each (segments, query) once: the routes of one query share it."""

    def __init__(self, oracle):
        self.oracle, self.cache = oracle, {}

    def __call__(self, data, q):
        key = (tuple(s.name for s in data), repr(q.aggregations), repr(q.filter), tuple(q.group_by))
        if key not in self.cache:
            self.cache[key] = mixed_ref.reference(self.oracle, data, q)
        return self.cache[key]


@pytest.fixture(scope="module")
def refs(oracle):
    return Refs(oracle)


def run_checked(pm, refs, data, devs, q, what, merge=False, all_groups=True):
    """Runs q; a query over the cap must be refused naming VAR/STDDEV.  Returns the per-aggregation values of each block
    (mixed_ref.check_block), or None when refused."""
    if len(q.aggregations) + 3 * len({a.column for a in q.aggregations if a.function in MOMENT_FUNCTIONS}) > MAX_AGGS:
        try:
            blocks = pm.execute_segments(devs, q, merge=merge)
        except UnsupportedQueryError as e:
            assert "VAR/STDDEV" in str(e), (what, str(e))
            return None
        # a filter the host folds to EMPTY is answered without a device plan, so without its limits
        assert not any(matching_docs(refs.oracle, s, q.filter).any() for s in data), f"{what}: over the cap, not refused"
    else:
        blocks = pm.execute_segments(devs, q, merge=merge)
    if merge:
        return [mixed_ref.check_block(q, blocks[0], refs(data, q), Decoder(data, devs[0], domain=True), what, all_groups)]
    return [mixed_ref.check_block(q, b, refs([s], q), Decoder([s], dev), f"{what} seg {i}", all_groups)
            for i, (b, s, dev) in enumerate(zip(blocks, data, devs))]


# ------------------------------------------------------------------------------------------------------------ routes
def test_refusals_over_the_cap(pm, refs, segs):
    data, dev = segs[8_193]
    assert not any(over_cap(s) for s in PINNED), [s for s in PINNED if over_cap(s)]
    for select in OVER_CAP:
        assert over_cap(select)
        for gb in ((), ("g",)):
            with pytest.raises(UnsupportedQueryError, match="VAR/STDDEV"):
                pm.execute_segments([dev], parse(select, gb))
    assert sum(over_cap(s) for s in DRAWN) >= 1 and sum(not over_cap(s) for s in DRAWN) >= 5, DRAWN


@pytest.mark.parametrize("n", SIZES)
def test_aggregation_only(pm, refs, segs, n):
    data, dev = segs[n]
    for select in PINNED + DRAWN:
        for where in (None, "x > -9000 AND g <> 3", "rid >= 0", "rid < 0"):
            run_checked(pm, refs, [data], [dev], parse(select, where=where), f"n={n} {select} WHERE {where}")


@pytest.mark.parametrize("n", SIZES)
def test_group_by_tables(ctx, pm, refs, segs, n):
    """g: 10 groups (the shared-memory table where every function may use it), h: 3 000 (dense), (g, s) two columns,
    h with dense_max=1: the hash table."""
    data, dev = segs[n]
    routes = [(("g",), {})] + ([(("g", "s"), {}), (("h",), {}), (("h",), {"dense_max": 1})] if 1 < n < 100_000 else [])
    for select in PINNED + DRAWN:
        for gb, knobs in routes:
            with tuned(ctx, **knobs):
                run_checked(pm, refs, [data], [dev], parse(select, gb, where="y < 390"), f"n={n} {select} BY {gb} {knobs}")


KNOBS = [{"pack_count": 0}, {"pack_count": 1}, {"pack_shift": 2}, {"warps": 8}, {"spec": 0}, {"defer": 0, "gb_defer": 0},
         {"grid": 1}]


def test_scan_knobs(ctx, pm, refs, segs):
    data, dev = segs[8_193]
    for select in PINNED:
        for gb in ((), ("g",)):
            q = parse(select, gb)
            first = None
            for knobs in KNOBS:
                with tuned(ctx, **knobs):
                    got = run_checked(pm, refs, [data], [dev], q, f"{select} BY {gb} {knobs}")
                assert got is not None, f"{select} BY {gb} {knobs}: refused"
                first = got if first is None else first
                assert got == first, f"{select} BY {gb}: {knobs} differs from {KNOBS[0]}"


def test_per_segment_submission(pm, refs, segs):
    """Several segments, different data, one submission with one result each: a per-result stride error reads another
    segment's record."""
    pairs = [segs[n] for n in (33, 8_193, 1, 100_003)]
    data, devs = [p[0] for p in pairs], [p[1] for p in pairs]
    for select in PINNED + DRAWN[:4]:
        for gb in ((), ("g",)):
            run_checked(pm, refs, data, devs, parse(select, gb, where="x <> 0"), f"per segment {select} BY {gb}")


def _exact_rows(q, rows, data):
    """final_rows without the floating and expression sums (they add in any order), floats by their bits."""
    loose = {len(q.group_by) + a for a, agg in enumerate(q.aggregations) if mixed_ref.summed_in_any_order(data, agg)}
    return [[np.float64(v).tobytes() if isinstance(v, float) else v for i, v in enumerate(r) if i not in loose]
            for r in rows]


def _check_merged_sums(q, table, ref, what):
    """The floating and expression SUM / AVG of a by-value merge (cli.merge_blocks) within their bound of the reference."""
    for key, vals in table.items():
        want = ref[tuple(float(k) if isinstance(k, float) else mixed_ref._plain(k) for k in key)]
        for a, agg in enumerate(q.aggregations):
            if agg.function == "SUM" and (mixed_ref.is_expression(agg) or want[a].kind == "exact" and want[a].value.kind != "int"):
                mixed_ref.check_one(agg, want[a], float(vals[a]), 0, None, None, None, f"{what} key={key} a={a}")
            elif agg.function == "AVG" and (mixed_ref.is_expression(agg) or want[a].value.kind != "int"):
                mixed_ref.check_one(agg, want[a], float(vals[a][0]), int(vals[a][1]), None, None, None, f"{what} key={key} a={a}")


def test_seventeen_segments_merged(oracle, ctx, pm, refs):
    """17 segments bound to one domain, merged on the device (past one 16-segment launch chunk), against the reference
    over all their rows; the same segments merged by value (cli.merge_blocks / final_rows) give the same rows."""
    data = [_segment(oracle, 3_000 + 37 * k, 500 + k, name=f"mix17_{k}") for k in range(17)]
    devs = [to_device(ctx, s) for s in data]
    domain = DictionaryDomain.build(ctx, devs, ["x", "y", "l", "f", "d", "t", "ts", "g", "h", "s"])
    try:
        for d in devs:
            d.bind_domain(domain)
        for select in PINNED + DRAWN[:4]:
            for gb in ((), ("g",)):
                q = parse(select, gb, where="y <> 5")
                if any(a.column == "r" for a in q.aggregations):   # stored raw: a dictionary per segment, none shared
                    with pytest.raises(UnsupportedQueryError, match="different dictionary"):
                        pm.execute_segments(devs, q, merge=True)
                    continue
                merged = run_checked(pm, refs, data, devs, q, f"17 merged {select} BY {gb}", merge=True)
                if merged is None:
                    continue
                by_value = cli.merge_blocks(q, devs, pm.execute_segments(devs, q))
                _check_merged_sums(q, by_value, refs(data, q), f"by value: {select} BY {gb}")
                per_seg = cli.final_rows(q, by_value)
                on_device = cli.final_rows(q, cli.merge_blocks(q, devs[:1], pm.execute_segments(devs, q, merge=True)))
                assert _exact_rows(q, per_seg, data) == _exact_rows(q, on_device, data), f"by value: {select} BY {gb}"
    finally:
        for d in devs:
            d.destroy()
        domain.release()


# --------------------------------------------------------------------------------------------------- FILTER clauses
CLAUSED = ["COUNT(*) FILTER (WHERE g = 1), SUM(x) FILTER (WHERE y > 100), SUM(x), MIN(f) FILTER (WHERE g = 1), "
           "DISTINCTCOUNT(y) FILTER (WHERE y > 100), MAX(l) FILTER (WHERE s = 'a')",
           "DISTINCTCOUNT(x), DISTINCTCOUNT(x) FILTER (WHERE g < 5), AVG(d) FILTER (WHERE g < 5), AVG(d), "
           "MIN(y) FILTER (WHERE x > 0), MAX(y) FILTER (WHERE x > 0)"]


@pytest.mark.parametrize("gb", [(), ("g",), ("h",)], ids=["agg", "g", "h"])
def test_filter_clauses(pm, refs, segs, gb):
    data, dev = segs[8_193]
    for select in CLAUSED:
        run_checked(pm, refs, [data], [dev], parse(select, gb, where="rid > 10"), f"clauses {select} BY {gb}")
    for extra, name in (("PERCENTILE(x, 50)", "PERCENTILE"), ("DISTINCTSUM(y)", "DISTINCTSUM"), ("VAR_POP(x)", "VAR/STDDEV"),
                        ("DISTINCTCOUNTHLL(y)", "DISTINCTCOUNTHLL"), ("LASTWITHTIME(x, t, 'INT')", "WITHTIME")):
        with pytest.raises(UnsupportedQueryError, match=name):
            pm.execute_segments([dev], parse(f"SUM(x) FILTER (WHERE g = 1), COUNT(*), {extra}", gb))


# ---------------------------------------------------------------------------------------- ORDER BY / HAVING non-owners
ORDERED = [  # (select, the non-owner ORDER BY / HAVING names)
    ("PERCENTILE(x, 10), PERCENTILE(x, 90), COUNT(*)", "PERCENTILE(x, 90)"),
    ("DISTINCTCOUNT(y), DISTINCTAVG(y), PERCENTILE(y, 50)", "DISTINCTAVG(y)"),
    ("STDDEV_POP(y), VAR_SAMP(y), MAX(x)", "VAR_SAMP(y)"),
    # ORDER BY names the first aggregation that matches, which for HLLs of one column and log2m is the estimate's owner:
    # here the ordered HLL reads a DISTINCTCOUNT's set, and the second HLL shares its estimate
    ("DISTINCTCOUNT(y), DISTINCTCOUNTHLL(y, 4), DISTINCTCOUNTHLL(y, 4)", "DISTINCTCOUNTHLL(y, 4)"),
]


@pytest.mark.parametrize("select,item", ORDERED, ids=["percentile", "distinctavg", "varsamp", "hll"])
def test_order_by_and_having_on_non_owners(pm, refs, segs, select, item):
    data, dev = segs[8_193]
    base = parse(select, ("h",))
    ref = refs([data], base)
    a = _index_of(base, item)
    val = {k: mixed_ref.final(base.aggregations[a], w[a]) for k, w in ref.items()}
    for desc in (False, True):
        for limit in (5, 1_000_000):
            q = parse(select, ("h",), tail=f" ORDER BY {item}{' DESC' if desc else ''} LIMIT {limit}")
            b = pm.execute_segments([dev], q)[0]
            want = sorted(ref, key=lambda k: ((-val[k] if desc else val[k]), k))
            got = mixed_ref.block_rows(q, b, Decoder([data], dev))
            assert got == want[:len(got)] and len(got) >= min(limit, len(want)), f"{select} ORDER BY {item} LIMIT {limit}"
            mixed_ref.check_block(q, b, ref, Decoder([data], dev), f"ordered {select}", all_groups=limit > len(want))
    # the cut lies halfway between two neighbouring reference values far apart in ulps, so that a value within its
    # contract (VAR / STDDEV: one ulp) falls on the same side of it
    finite = sorted({v for v in val.values() if np.isfinite(v)})
    lo, hi = next((u, w) for u, w in zip(finite[len(finite) // 2:], finite[len(finite) // 2 + 1:]) if w - u > 8 * math.ulp(w))
    cut = (lo + hi) / 2
    q = parse(select, ("h",), tail=f" HAVING {item} > {cut!r} LIMIT 1000000")
    b = pm.execute_segments([dev], q)[0]
    got = mixed_ref.block_rows(q, b, Decoder([data], dev))
    assert set(got) == {k for k, v in val.items() if v > cut}, f"HAVING {item} > {cut}"
    mixed_ref.check_block(q, b, ref, Decoder([data], dev), f"having {select}", all_groups=False)


def _index_of(q, item):
    order = sql.parse(f"SELECT {item} FROM t GROUP BY h ORDER BY {item}")
    fn, col, arg = order.aggregations[0].function, order.aggregations[0].column, order.aggregations[0].arg
    return next(i for i, a in enumerate(q.aggregations) if (a.function, a.column, a.arg) == (fn, col, arg))


# ------------------------------------------------------------------------------------------- position does not matter
def test_position_does_not_matter(pm, refs, segs):
    """Each aggregation of a mixed query equals the same aggregation alone and in the query's aggregations reversed and
    rotated, bit for bit (floating and expression sums: each held to its bound by check_block)."""
    data, dev = segs[8_193]
    for select in [s for s in PINNED + DRAWN if not over_cap(s)]:
        items = [str(a) for a in parse(select).aggregations]
        texts = _split(select)
        for gb in ((), ("g",)):
            mixed = run_checked(pm, refs, [data], [dev], parse(select, gb), f"{select} BY {gb}")[0]
            for perm in (texts[::-1], texts[1:] + texts[:1]):
                got = run_checked(pm, refs, [data], [dev], parse(", ".join(perm), gb), f"{perm} BY {gb}")[0]
                for key, row in mixed.items():
                    for a, v in enumerate(row):
                        if v is not None:
                            assert got[key][perm.index(texts[a])] == v, f"{items[a]} moved in {perm} BY {gb} key {key}"
            for a, text in enumerate(texts):
                alone = run_checked(pm, refs, [data], [dev], parse(text, gb), f"{text} alone BY {gb}")[0]
                for key, row in mixed.items():
                    if row[a] is not None:
                        assert alone[key][0] == row[a], f"{items[a]} alone differs from in {select} BY {gb} key {key}"


def _split(select):
    """The aggregation texts of a SELECT list (commas inside parentheses kept)."""
    out, depth, cur = [], 0, ""
    for ch in select:
        depth += ch == "("
        depth -= ch == ")"
        if ch == "," and depth == 0:
            out.append(cur.strip())
            cur = ""
        else:
            cur += ch
    return out + [cur.strip()]


# ------------------------------------------------------------------------------------------------------ across GPUs
def test_loopback_combine(oracle):
    """execute_and_combine over two ranks on one GPU (tests/loopback_dist.py)."""
    from loopback_dist import run_ranks, values
    from pinot_b200.distributed import execute_and_combine, global_domain
    world = 2
    hosts = [[_segment(oracle, 2_000 + 301 * r + 7 * i, 900 + 10 * r + i, name=f"mixl{r}_{i}") for i in range(1 + r)]
             for r in range(world)]
    ctxs = [B200Context(0) for _ in range(world)]
    devs = [[to_device(c, h) for h in hs] for c, hs in zip(ctxs, hosts)]
    doms = []
    try:
        doms = values(run_ranks(world, lambda dist: global_domain(ctxs[dist.get_rank()], devs[dist.get_rank()],
                                                                  ["x", "y", "l", "d", "g", "h", "s"], dist)))
        everything = [h for hs in hosts for h in hs]

        def combine(text):
            return run_ranks(world, lambda dist: execute_and_combine(
                B200PlanMaker(ctxs[dist.get_rank()]), devs[dist.get_rank()], sql.parse(text, num_groups_limit=1_000_000), dist))

        for text in ("SELECT g, COUNT(*), SUM(x), MIN(d), MAX(l), AVG(y), DISTINCTCOUNT(y) FROM t WHERE y < 390 GROUP BY g",
                     "SELECT DISTINCTSUM(x), DISTINCTCOUNTHLL(y), SUM(x * d), COUNT(*), SUM(y), SUM(d) FROM t",
                     "SELECT DISTINCTCOUNT(x), DISTINCTAVG(x), DISTINCTCOUNTHLL(x), MIN(y - d), MAX(y) FROM t WHERE g <> 2"):
            q = sql.parse(text, num_groups_limit=1_000_000)
            got = values(combine(text))
            assert all(g is None for g in got[1:]), text
            mixed_ref.check_block(q, got[0], mixed_ref.reference(oracle, everything, q), Decoder(everything, devs[0][0], domain=True),
                                  f"world {world}: {text}")
        for last in ("PERCENTILE(x, 50)", "VAR_POP(y)", "LASTWITHTIME(x, t, 'INT')"):
            text = f"SELECT COUNT(*), SUM(x), MIN(d), DISTINCTCOUNT(y), MAX(l), {last} FROM t"
            outcomes = combine(text)
            for r, o in enumerate(outcomes):
                assert isinstance(o.error, UnsupportedQueryError), (text, r, repr(o.error))
                assert o.calls == [], (text, r, o.calls)
    finally:
        for ds in devs:
            for d in ds:
                d.destroy()
        for dom in doms:
            dom.release()
        for c in ctxs:
            c.close()
