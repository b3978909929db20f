"""-m gpu: segments bound to a dictionary domain against the exact references of their UNBOUND selves.

Binding a segment (pb200_segment_bind_domain) rewrites its forward index in place -- unpacked at the segment's width sb,
remapped, repacked at the domain's width db -- re-indexes its inverted-index offsets (ids absent from the segment get
empty posting lists), and from then on every filter leaf and the non-scan shortcut speak domain ids.  None of that may
change an answer in value space, so every reference here comes from the oracle-built host segments, never bound:

* the re-encoded stream byte for byte (pack_fixed_bits of the remapped dictIds at db bits, zero padding included), the
  remap, the widths, and the values read back through the selection kernel and a GROUP BY -- for db == sb (remapped), db
  == sb + 1, db far above sb (20, 24 and 25 bits, over fabricated domain dictionaries), the identity at the minimal width
  and the identity of a column registered wider than it needs, sb from 1 to 17, sorted columns included; sizes cover
  ragged 32-row groups and both CTA tile widths;
* domain dictionaries at the type edges: INT and LONG extremes, FLOAT / DOUBLE -0.0, 0.0, +-inf, +-max, subnormals and
  NaNs of both signs (union built in both part orders), STRING prefixes, multi-byte UTF-8 and differing padded widths;
* every filter route (scan range, scan IN / NOT IN, inverted IN / NOT IN, doc ranges, AND / OR / NOT programs) over
  segments whose values interleave (segment i holds the values = i mod 3), read back exactly through `rid`;
* COUNT / SUM / AVG / MIN / MAX / DISTINCTCOUNT per segment and merged on every GROUP BY route, over key spaces only the
  domain makes large (an almost empty 2^20 + 1 dense table, LONG_MAP, and an ARRAY_MAP key space that must be refused),
  and the non-scan shortcut, whose ids must be domain ids.

Widths above 25 bits need domain dictionaries of more than 2^25 entries and are not covered."""
import contextlib
import math
import time

import numpy as np
import pytest

import float_edges_ref as fe
from exact_ref import assert_exact, reference as exact_reference
from filter_ref import matching_docs, matching_docs_many
from gpu_util import to_device, tuned
from oracle import segment_builder as sb
from pinot_b200 import sql
from pinot_b200.plan_maker import B200Context, B200PlanMaker, DictionaryDomain, UnsupportedQueryError
from pinot_b200.query import Aggregation, Filter, Predicate
from pinot_b200.sql import SelectionQuery
from selection_ref import assert_rows_equal, expected as expected_rows
from test_filter_ref_cpu import literal_pool, random_leaf, random_tree
from test_gpu_filter_exact import AGG, _check_agg, _check_count, _check_gb_blk, _check_gb_rid, _q, _shape

pytestmark = pytest.mark.gpu

INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
SIZES = [1, 31, 33, 6_143, 6_145, 8_191, 8_193, 65_537, 196_609]
LIMIT = 1 << 20


@pytest.fixture(scope="module")
def ctx():
    c = B200Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pm(ctx):
    return B200PlanMaker(ctx)


def _bits(card):
    """bits_for_cardinality: PinotDataBitSet.getNumBitsPerValue(card - 1)."""
    return max(1, (card - 1).bit_length())


def _be(values, data_type=sb.INT):
    return np.frombuffer(np.asarray(values).astype(sb._NP_BE[data_type]).tobytes(), dtype=np.uint8).copy()


def _rows(rng, card, n):
    """n dictIds over 0 .. card - 1, each at least once (card <= n)."""
    return np.concatenate([rng.permutation(card), rng.integers(0, card, size=n - card)]).astype(np.int32)


def _spread(rng, card):
    """`card` sorted distinct INT values from just above INT_MIN, gaps of 1 .. 2^13."""
    return (INT_MIN + np.cumsum(rng.integers(1, 1 << 13, size=card))).astype(np.int32)


def _column(name, dict_values, ids, bits=None):
    """Dictionary INT column with the rows dict_values[ids]; `bits` registers the stream wider than the minimal width."""
    if bits is None:
        return sb.build_column(name, dict_values[ids])
    return sb.ColumnData(name, sb.INT, True, bits, len(dict_values), False, 4, sb.pack_fixed_bits(ids, bits),
                         _be(dict_values), None, dict_values, ids)


def _domain_values(dom, column):
    """The domain dictionary decoded: a numpy array (numeric) or a list of str."""
    info, raw = dom.info(column), dom.dictionary_bytes(column).tobytes()
    if info["stored_type"] == sb.STRING:
        w = info["entry_bytes"]
        return [raw[i * w:(i + 1) * w].rstrip(b"\0").decode("utf-8") for i in range(info["cardinality"])]
    be = sb._NP_BE[info["stored_type"]]
    return np.frombuffer(raw, dtype=be).astype(be[1:])


def _py(v):
    return v.item() if hasattr(v, "item") else v


def _table(q, block, values):
    """Value-space table of a block whose ids are domain ids, decoded through the domain dictionaries `values`."""
    rows = 1 if block.num_groups < 0 else block.num_groups
    out = {}
    for g in range(rows):
        key = () if block.num_groups < 0 else tuple(_py(values[c][int(block.keys[g, j])]) for j, c in enumerate(q.group_by))
        vals = []
        for a, agg in enumerate(q.aggregations):
            if agg.function == "COUNT":
                vals.append(int(block.longs[a][g]))
            elif agg.function == "AVG":
                vals.append((float(block.doubles[a][g]), int(block.longs[a][g])))
            elif agg.function == "DISTINCTCOUNT":
                vals.append(frozenset(_py(values[agg.column][int(d)]) for d in block.distinct.get((a, g), ())))
            else:
                vals.append(float(block.doubles[a][g]))
        out[key] = vals
    return out


# ------------------------------------------------------------------------------------------- 1. re-encoded streams
def _width_cases(n):
    """(column, segment cardinality, registered bits or None = minimal, domain cardinality) of every width pair a segment
    of n rows holds with real rows; sb = b."""
    out = []
    for b in range(1, 18):
        cs = 1 if b == 1 else (1 << (b - 1)) + 1
        if cs > n:
            break
        out += [(f"eq{b}", cs, None, max(2, 1 << b)),   # db == sb, not the identity
                (f"up{b}", cs, None, (1 << b) + 1),     # db == sb + 1
                (f"id{b}", cs, None, cs),               # identity at the minimal width
                (f"iw{b}", cs, b + 4, cs)]              # identity of a stream registered 4 bits wider than it needs
    return out


def _check_reencoded(oracle, pm, seg, dev, dom, cases, what):
    """cases: {column: (domain values, the segment's dictionary)}, the segment's dictIds in seg.column(c).dict_ids."""
    n = seg.num_docs
    for name, (dvals, sdict) in cases.items():
        c = seg.column(name)
        db = _bits(len(dvals))
        tag = f"{what} {name}: sb={c.bits} db={db} card {c.cardinality} -> {len(dvals)}"
        assert dom.info(name)["bits"] == db and dom.info(name)["cardinality"] == len(dvals), tag
        assert np.array_equal(_domain_values(dom, name), dvals), tag
        assert (dev.column_info(name)["bits"], dev.column_info(name)["cardinality"]) == (db, len(dvals)), tag
        remap = np.searchsorted(dvals, sdict)
        assert np.array_equal(dev.local_ids(name), remap), tag
        assert np.array_equal(dev.read_index(name, "fwd"), sb.pack_fixed_bits(remap[c.dict_ids], db)), tag
    names = list(cases)
    for k in range(0, len(names), 7):   # the whole segment through the selection kernel
        cols = ["rid"] + names[k:k + 7]
        got = pm.execute_selection([dev], SelectionQuery(columns=cols, limit=n))[0]
        assert_rows_equal(got, expected_rows(oracle, [seg], None, cols, n, False)[0], f"{what} select {cols}")
    for name, (dvals, sdict) in cases.items():
        b = pm.execute_segments([dev], _q([Aggregation("COUNT")], None, [name]))[0]
        keys = b.keys[:b.num_groups, 0].astype(np.int64)
        order = np.argsort(keys)
        want, counts = np.unique(sdict[seg.column(name).dict_ids], return_counts=True)
        assert np.array_equal(dvals[keys[order]], want), f"{what} GROUP BY {name}"
        assert np.array_equal(b.longs[0][:b.num_groups][order], counts), f"{what} GROUP BY {name}"
        assert b.stats.num_docs_scanned == n, f"{what} GROUP BY {name}"


@pytest.mark.parametrize("n", SIZES)
def test_reencoded_stream_at_every_width_pair(oracle, ctx, pm, n):
    t0 = time.perf_counter()
    rng = np.random.default_rng(n)
    cols, cases = [sb.build_column("rid", np.arange(n, dtype=np.int32))], {}
    for name, cs, bits, dcard in _width_cases(n):
        dvals = _spread(rng, dcard)
        sdict = dvals if dcard == cs else dvals[np.sort(rng.choice(dcard, size=cs, replace=False))]
        cols.append(_column(name, sdict, _rows(rng, cs, n), bits))
        cases[name] = (dvals, sdict)
    # a sorted column: its sorted index was expanded into a fixed-bit stream at load, which the bind re-encodes
    dvals = _spread(rng, 8192)
    sdict = dvals[np.sort(rng.choice(8192, size=min(4097, n), replace=False))]
    cols.append(_column("srt", sdict, np.sort(_rows(rng, len(sdict), n))))
    assert cols[-1].is_sorted
    cases["srt"] = (dvals, sdict)
    seg = sb.SegmentData(f"widths{n}", n, cols)
    dev, dom = to_device(ctx, seg), None
    try:
        names = list(cases)
        dom = DictionaryDomain.from_dictionaries(ctx, names, [dev.column_index(c) for c in names], [sb.INT] * len(names),
                                                 [[_be(sd), _be(dv)] for dv, sd in cases.values()])
        dev.bind_domain(dom)
        _check_reencoded(oracle, pm, seg, dev, dom, cases, f"n={n}")
    finally:
        dev.destroy()
        if dom is not None:
            dom.release()
    print(f"n={n}: {len(cases)} columns, {time.perf_counter() - t0:.1f} s")


# (column, domain cardinality -> db 20 / 24 / 25, the segment's cardinality at most)
WIDE = [("w20", (1 << 19) + 1, 2), ("w24", (1 << 23) + 1, 4097), ("w25", (1 << 24) + 1, (1 << 17) + 1)]


def test_reencoded_stream_into_wide_domains(oracle, ctx, pm):
    """db of 20, 24 and 25 bits: domain dictionaries fabricated as sorted INT sequences (only a few of their values occur
    in any segment), one domain shared by segments of several sizes; sb from 1 to 18."""
    t0 = time.perf_counter()
    rng = np.random.default_rng(2025)
    dvals = {c: (INT_MIN + 1 + np.arange(card, dtype=np.int64) * ((1 << 32) // card - 1)).astype(np.int32)
             for c, card, _ in WIDE}
    names = [c for c, _, _ in WIDE]
    dom = DictionaryDomain.from_dictionaries(ctx, names, [1, 2, 3], [sb.INT] * 3, [[_be(dvals[c][::3]), _be(dvals[c])] for c in names])
    devs = []
    try:
        for n in (1, 33, 8_193, 196_609):
            cols, cases = [sb.build_column("rid", np.arange(n, dtype=np.int32))], {}
            for c, card, most in WIDE:
                cs = min(most, n)
                sdict = dvals[c][np.sort(rng.choice(card, size=cs, replace=False))]
                cols.append(_column(c, sdict, _rows(rng, cs, n)))
                cases[c] = (dvals[c], sdict)
            seg = sb.SegmentData(f"wide{n}", n, cols)
            devs.append(to_device(ctx, seg))
            devs[-1].bind_domain(dom)
            _check_reencoded(oracle, pm, seg, devs[-1], dom, cases, f"wide n={n}")
    finally:
        for d in devs:
            d.destroy()
        dom.release()
    print(f"wide domains: {time.perf_counter() - t0:.1f} s")


# ------------------------------------------------------------------------------------------------ 2. type edges
F_MAX, D_MAX = float(np.finfo(np.float32).max), float(np.finfo(np.float64).max)
F_SUB, D_SUB = fe.float_of(1), fe.double_of(1)   # smallest subnormals


def _edge_segments(oracle):
    """Four segments, each holding some of the type edges (every pool value occurs; v is an unbound filter column)."""
    f = lambda *xs: np.array([fe.float_of(x) if isinstance(x, int) else x for x in xs], dtype=np.float32)   # noqa: E731
    d = lambda *xs: np.array([fe.double_of(x) if isinstance(x, int) and x > 1 << 60 else x for x in xs], dtype=np.float64)   # noqa: E731
    pools = [
        dict(i=[INT_MIN, 5, 7], l=[INT64_MIN, (1 << 53) - 1, 3],
             f=f(-0.0, math.inf, F_MAX, fe.F_NAN, 1.5), d=d(-0.0, math.inf, D_MAX, fe.D_NAN, 1.5),
             s=[b"a", b"ab", b"zzzz"]),
        dict(i=[-1, 0, 5], l=[(1 << 53) + 1, 3, -7],
             f=f(0.0, -math.inf, -F_MAX, fe.F_NEG_NAN), d=d(0.0, -math.inf, -D_MAX, fe.D_NEG_NAN),
             s=["é".encode(), b"ab", b"b"]),
        dict(i=[INT_MAX, 9, -1], l=[INT64_MAX, INT64_MIN, 0],
             f=np.array([F_SUB, -F_SUB, -0.0, 2.5], dtype=np.float32), d=np.array([D_SUB, -D_SUB, -0.0, 2.5]),
             s=["日本".encode(), "".encode(), b"a"]),
        dict(i=[INT_MIN, INT_MAX, 0], l=[INT64_MAX, (1 << 53) + 1, (1 << 53) - 1],
             f=f(0.0, 1.5, fe.F_PAYLOAD_NAN), d=d(0.0, 1.5, fe.D_PAYLOAD_NAN),
             s=["\U0001F600".encode(), b"abc", b"a" * 7]),
    ]
    rng = np.random.default_rng(77)
    segs = []
    for j, p in enumerate(pools):
        n = 600 + 317 * j
        cols = []
        for c in ("i", "l", "f", "d", "s"):
            pool = p[c] if isinstance(p[c], np.ndarray) else np.array(p[c], dtype={"i": np.int32, "l": np.int64, "s": None}[c])
            rows = pool[np.concatenate([np.arange(len(pool)), rng.integers(0, len(pool), size=n - len(pool))])]
            cols.append(fe.build_dict_column(c, rows) if c in ("f", "d") else sb.build_column(c, rows))
        cols.append(sb.build_column("v", rng.integers(-1000, 1000, size=n).astype(np.int32)))
        segs.append(sb.SegmentData(f"edges{j}", n, cols))
    return segs


def _float_dictionary(parts, data_type):
    """The domain's FLOAT / DOUBLE dictionary: Pinot's unique values over the parts in part order (the first NaN's bits)."""
    values = np.concatenate([np.asarray(p) for p in parts])
    return np.array(fe.unique_values(values, data_type), dtype=values.dtype)


@pytest.mark.parametrize("reverse", [False, True], ids=["parts", "parts_reversed"])
def test_domain_dictionary_at_the_type_edges(oracle, ctx, pm, reverse):
    t0 = time.perf_counter()
    segs = _edge_segments(oracle)
    if reverse:
        segs = segs[::-1]
    devs = [to_device(ctx, s) for s in segs]
    dom = None
    try:
        dom = DictionaryDomain.build(ctx, devs, ["i", "l", "f", "d", "s"])
        for c, be in (("i", ">i4"), ("l", ">i8")):
            want = np.unique(np.concatenate([s.column(c).dict_values for s in segs]))
            assert dom.dictionary_bytes(c).tobytes() == want.astype(be).tobytes(), c
        for c, dt in (("f", sb.FLOAT), ("d", sb.DOUBLE)):
            want = _float_dictionary([s.column(c).dict_values for s in segs], dt)
            assert dom.dictionary_bytes(c).tobytes() == want.astype(sb._NP_BE[dt]).tobytes(), (c, reverse)
        strings = sorted({bytes(v) for s in segs for v in s.column("s").dict_values})   # UTF-8 byte order
        assert dom.info("s")["entry_bytes"] == max(len(v) for v in strings)
        assert _domain_values(dom, "s") == [v.decode("utf-8") for v in strings]
        assert len({s.column("s").dict_entry_bytes for s in segs}) == len(segs)   # every segment pads differently
        values = {c: _domain_values(dom, c) for c in ("i", "l", "f", "d", "s")}
        for d in devs:
            d.bind_domain(dom)
        for s, d in zip(segs, devs):   # every bound row decodes to its original value (floats: bits; NaN: a NaN)
            for c in ("i", "l", "f", "d", "s"):
                col = s.column(c)
                ids = sb.unpack_fixed_bits(d.read_index(c, "fwd"), s.num_docs, d.column_info(c)["bits"])
                decoded = {int(i): d.dictionary_value(c, int(i)) for i in np.unique(ids)}
                orig = np.asarray(col.dict_values)[col.dict_ids]
                for i, v in zip(ids.tolist(), orig):
                    got = decoded[i]
                    if c == "s":
                        assert got == v.decode("utf-8"), (s.name, c, got, v)
                    elif c in ("f", "d"):
                        assert math.isnan(got) if math.isnan(v) else fe.bits_of(got) == fe.bits_of(float(v)), (s.name, c, got, v)
                    else:
                        assert got == int(v), (s.name, c, got, v)
        for text in ("SELECT MIN(i), MAX(i), DISTINCTCOUNT(i), MIN(l), MAX(l), DISTINCTCOUNT(l) FROM t WHERE v >= -600",
                     "SELECT DISTINCTCOUNT(s), MIN(i), MAX(l) FROM t WHERE v < 600",
                     "SELECT MIN(f), MAX(f), DISTINCTCOUNT(f), MIN(d), MAX(d), DISTINCTCOUNT(d) FROM t WHERE v >= -600",
                     "SELECT MIN(i), MAX(i), MIN(l), MAX(l), DISTINCTCOUNT(s) FROM t",   # non-scan per segment
                     "SELECT MIN(f), MAX(f), DISTINCTCOUNT(f), MIN(d), MAX(d), DISTINCTCOUNT(d) FROM t"):
            q = sql.parse(text)
            groups = [([s], pm.execute_segments([d], q)[0], s.name) for s, d in zip(segs, devs)]
            groups.append((segs, pm.execute_segments(devs, q, merge=True)[0], "merged"))
            for part, block, what in groups:
                what = f"{what} {q.aggregations}"
                if q.aggregations[0].column in ("f", "d"):
                    ref = fe.reference(oracle, part, q)[()]
                    for a, agg in enumerate(q.aggregations):
                        dt = part[0].column(agg.column).data_type
                        if agg.function == "DISTINCTCOUNT":
                            got = frozenset(fe.identity(values[agg.column][int(i)], dt) for i in block.distinct.get((a, 0), ()))
                            assert got == ref[a], (what, agg)
                        else:
                            assert fe.check_value(float(block.doubles[a][0]), ref[a]), (what, agg, block.doubles[a][0], ref[a])
                            i = int(block.dict_ids[a][0])
                            assert fe.identity(values[agg.column][i], dt) == fe.identity(ref[a], dt), (what, agg, i, ref[a])
                else:
                    ref = exact_reference(oracle, part, q)
                    assert_exact(q, _table(q, block, values), ref, what)
                    for a, agg in enumerate(q.aggregations):
                        if agg.function in ("MIN", "MAX"):
                            assert values[agg.column][int(block.dict_ids[a][0])] == ref[()][a], (what, agg)
    finally:
        for d in devs:
            d.destroy()
        if dom is not None:
            dom.release()
    print(f"type edges (reverse={reverse}): {time.perf_counter() - t0:.1f} s")


# --------------------------------------------------------------------------------- 3. filter routes over domain ids
FILTER_GROUPS = [[1, 33, 8_193], [6_145, 65_537, 196_609]]
WIDTHS3 = [1, 2, 7, 8, 15, 16, 17]
STRINGS = [b"a", b"aa", b"ab", b"b", b"ba", b"bb", b"c", b"ca", b"cb"]
BOUND3 = [f"c{b}" for b in WIDTHS3] + ["inv", "ic", "srt", "l", "d", "s"]


def _interleaved_segment(oracle, n, i):
    """Segment i of a triple whose bound columns hold only values = i (mod 3): every remap skips ids, and two thirds
    of the domain's ids are absent from the segment.  rid / blk / bit read the doc set back (test_gpu_filter_exact)."""
    rng = np.random.default_rng(1000 * n + i)
    rid = np.arange(n, dtype=np.int32)
    cols = {"rid": rid, "blk": rid // 16, "bit": (1 << (rid % 16)).astype(np.int32), "srt": (rid // 37) * 3 + i - 30}
    for b in WIDTHS3:
        cols[f"c{b}"] = ((_rows(rng, min(1 << b, n), n) - 5) * 3 + i).astype(np.int32)
    cols["inv"] = (rng.integers(0, 40, size=n) * 3 + i).astype(np.int32)
    ic = np.array([3, 1, 4, 0, 2], dtype=np.int32)[(rid // 2000) % 5]   # runs of 2000 rows: run containers
    ic[(rid >= 65_536) & (rid < 98_304) & (rid % 2 == 0)] = 5           # bitmap container
    ic[(rid >= 65_536) & (rid % 97 == 0)] = 6                           # array container
    if n > 1 and np.all(np.diff(ic) >= 0):
        ic[0] = 7   # never stored as sorted
    cols["ic"] = ic * 3 + i
    cols["l"] = np.array([-(1 << 61), -1, 0, 5, 1 << 53, 1 << 61], dtype=np.int64)[rng.integers(0, 6, size=n)] * 3 + i
    cols["d"] = (rng.integers(-20, 20, size=n) * 3 + i) / 4.0
    cols["s"] = np.array(STRINGS[i::3])[rng.integers(0, 3, size=n)]
    return oracle.build_segment(f"il{n}_{i}", cols, inverted=["inv", "ic"])


@pytest.fixture(scope="module")
def interleaved(oracle, ctx):
    """[(host segments, bound device segments, domain)] per size group."""
    out = []
    try:
        for sizes in FILTER_GROUPS:
            segs = [_interleaved_segment(oracle, n, i) for i, n in enumerate(sizes)]
            devs = [to_device(ctx, s) for s in segs]
            out.append((segs, devs, None))
            dom = DictionaryDomain.build(ctx, devs, BOUND3)
            out[-1] = (segs, devs, dom)
            for d in devs:
                d.bind_domain(dom)
        yield out
    finally:
        for _, devs, dom in out:
            for d in devs:
                d.destroy()
            if dom is not None:
                dom.release()


def _union(segs, column):
    return np.unique(np.concatenate([np.asarray(s.column(column).dict_values) for s in segs]))


def _domain_leaves(segs, rng, k):
    """Leaves over the union of the triple's values: seeded random ones, then per bound INT column the domain's first
    and last id, ranges whose ends sit on values of one other segment only, ranges covering two or three ids of other
    segments only (EMPTY for the third), IN / NOT IN over absent values."""
    pools = {c: literal_pool(_union(segs, c), c not in ("d", "s")) for c in BOUND3}
    out = []
    for _ in range(k):
        c = BOUND3[int(rng.integers(0, len(BOUND3)))]
        out.append(random_leaf(rng, c, pools[c]))
    for c in [f"c{b}" for b in WIDTHS3] + ["inv", "ic", "srt"]:
        u = [int(x) for x in _union(segs, c)]
        m = len(u) // 2
        out += [Predicate("IN", c, [u[0]]), Predicate("IN", c, [u[-1]]), Predicate("NOT_IN", c, [u[0], u[-1]]),
                Predicate("IN", c, u[m:m + 3] + [u[0] - 1]), Predicate("NOT_IN", c, u[1:4]), Predicate("EQ", c, [u[m]]),
                Predicate("NEQ", c, [u[-1]]),
                Predicate("RANGE", c, [], u[min(1, len(u) - 1)], u[max(-2, -len(u))], True, True),
                Predicate("RANGE", c, [], u[m], u[min(m + 1, len(u) - 1)], True, True),
                Predicate("RANGE", c, [], u[m], u[min(m + 2, len(u) - 1)], False, False),
                Predicate("RANGE", c, [], u[m], None, False, True), Predicate("RANGE", c, [], None, u[m], True, False)]
    return out


def _domain_trees(segs, seed):
    rng = np.random.default_rng(seed)
    leaves = _domain_leaves(segs, rng, 24)
    pick = lambda: leaves[int(rng.integers(0, len(leaves)))]   # noqa: E731
    trees = list(leaves)
    for k in range(2, 9):   # flat conjunctions
        trees.append(Filter("AND", [pick() for _ in range(k)]))
    for _ in range(30):
        t = random_tree(rng, pick)
        if _shape(t)[0] <= 8 and _shape(t)[1] <= 16:
            trees.append(t)
    same = pick()
    trees += [Filter("OR", [same, Filter("NOT", [same])]), Filter("AND", [same, Filter("NOT", [Filter("NOT", [same])])])]
    return trees


FILTER_KNOBS = [{}, {"sparse_max": 0}, {"sparse_max": 32}]


@pytest.mark.parametrize("knobs", FILTER_KNOBS, ids=[",".join(f"{k}={v}" for k, v in kn.items()) or "defaults" for kn in FILTER_KNOBS])
def test_every_filter_route_over_domain_ids(oracle, ctx, pm, interleaved, knobs):
    """Each tree in one submission over the bound triple; per segment the doc set through every observable of
    test_gpu_filter_exact, against the tree evaluated on the unbound segment's values."""
    t0 = time.perf_counter()
    ran = 0
    with tuned(ctx, **knobs):
        for segs, devs, _ in interleaved:
            trees = _domain_trees(segs, 31 + segs[0].num_docs)
            refs = [matching_docs_many(oracle, s, trees) for s in segs]
            for j, t in enumerate(trees):
                observables = [(AGG, (), _check_agg), ([Aggregation("COUNT")], (), _check_count),
                               ([Aggregation("COUNT")], ["rid"], _check_gb_rid), ([Aggregation("SUM", "bit")], ["blk"], _check_gb_blk)]
                for aggs, gb, check in observables:
                    for s, b, ref in zip(segs, pm.execute_segments(devs, _q(aggs, t, gb)), refs):
                        check(b, ref[j], f"{knobs} {check.__name__} n={s.num_docs}: {t}")
                ran += 1
    print(f"{knobs}: {ran} trees, {time.perf_counter() - t0:.1f} s")


# ----------------------------------------------------------------------- 4. aggregation and GROUP BY over domain ids
AGG_SIZES = [33, 8_193, 40_001]
BIG, HUGE, WIDE3 = (1 << 20) + 1, (1 << 16) + 1, 1 << 21   # domain cardinalities of big, h1 / h2, a1 / a2 / a3
BOUND4 = ["g", "k", "l", "s", "f", "big", "h1", "h2", "a1", "a2", "a3"]
ROUTES = {"default": {}, "global": {"smem_groups": 0}, "spec_off": {"spec": 0}, "hash": {"dense_max": 1},
          "sparse_0": {"sparse_max": 0}, "sparse_32": {"sparse_max": 32}, "carrier_off": {"pack_count": 0},
          "stride_16": {"table_stride": 16}}
AGG_QUERIES = [
    "SELECT COUNT(*), SUM(v), AVG(v), MIN(k), MAX(k), DISTINCTCOUNT(k) FROM t WHERE v > -500000000 GROUP BY g",
    "SELECT COUNT(*), SUM(f), AVG(v), MIN(l), MAX(l), DISTINCTCOUNT(s) FROM t WHERE g != 7 GROUP BY big",   # 2^20 + 1 keys
    "SELECT COUNT(*), SUM(v), MIN(f), MAX(f), DISTINCTCOUNT(g) FROM t GROUP BY h1, h2",                    # LONG_MAP
    "SELECT COUNT(*), SUM(v), MIN(k), MAX(k), DISTINCTCOUNT(l) FROM t WHERE s != 'b' GROUP BY g, s",
    "SELECT COUNT(*), SUM(v), AVG(f), MIN(k), MAX(l), DISTINCTCOUNT(big) FROM t WHERE k < 0 OR v > 100",
    "SELECT COUNT(*), MIN(k), MAX(k), MIN(l), MAX(l), DISTINCTCOUNT(s) FROM t",   # non-scan per segment
    "SELECT MIN(f), MAX(f), DISTINCTCOUNT(k), DISTINCTCOUNT(big) FROM t",
]


def _agg_segment(oracle, n, i, rng):
    """Segment i: bound keys and arguments = i (mod 3) where they are INT, so no two segments share a value; big, h1, h2
    and a1..a3 hold a few ids of domains far larger than any segment."""
    def ids_mod(card, count):
        return np.sort(rng.choice(np.arange(i, card, 3), size=count, replace=False))
    cols = {"g": (_rows(rng, min(100, n), n) * 3 + i).astype(np.int32)}
    kpool = np.array([INT_MIN + i, INT_MAX - 2 + i] + list(rng.integers(-10_000, 10_000, size=40) * 3 + i), dtype=np.int64)
    cols["k"] = kpool[rng.integers(0, len(kpool), size=n)].astype(np.int32)
    lpool = np.array([INT64_MIN + 2 + i, INT64_MAX - 2 + i, (1 << 53) + i, (1 << 53) + 3 + i, -7 * 3 + i], dtype=np.int64)
    cols["l"] = lpool[rng.integers(0, len(lpool), size=n)]
    cols["s"] = np.array(STRINGS[i::3])[rng.integers(0, 3, size=n)]
    cols["f"] = (rng.integers(-500, 500, size=n) * 3 + i) / 8.0
    cols["big"] = ids_mod(BIG, 100)[rng.integers(0, 100, size=n)].astype(np.int32) * 2 - 1_000_000
    for c in ("h1", "h2"):
        cols[c] = ids_mod(HUGE, 300)[rng.integers(0, 300, size=n)].astype(np.int32) * 5
    for c in ("a1", "a2", "a3"):
        cols[c] = ids_mod(WIDE3, 50)[rng.integers(0, 50, size=n)].astype(np.int32) - 7
    v = rng.integers(-1_000_000, 1_000_000, size=n).astype(np.int32)
    v[rng.integers(0, n, size=max(1, n // 20))] = INT_MAX
    v[rng.integers(0, n, size=max(1, n // 20))] = INT_MIN
    cols["v"] = v
    return oracle.build_segment(f"agg{n}_{i}", cols)


FABRICATED = {"big": np.arange(BIG, dtype=np.int32) * 2 - 1_000_000, "h1": np.arange(HUGE, dtype=np.int32) * 5,
              "h2": np.arange(HUGE, dtype=np.int32) * 5, "a1": np.arange(WIDE3, dtype=np.int32) - 7,
              "a2": np.arange(WIDE3, dtype=np.int32) - 7, "a3": np.arange(WIDE3, dtype=np.int32) - 7}


@pytest.fixture(scope="module")
def agg_bound(oracle, ctx):
    """(host segments, bound device segments, domain, decoded domain dictionaries)."""
    rng = np.random.default_rng(404)
    segs = [_agg_segment(oracle, n, i, rng) for i, n in enumerate(AGG_SIZES)]
    devs = [to_device(ctx, s) for s in segs]
    dom = None
    try:
        types = [segs[0].column(c).data_type for c in BOUND4]
        parts = [[s.column(c).dict for s in segs] + ([_be(FABRICATED[c])] if c in FABRICATED else []) for c in BOUND4]
        widths = [[s.column(c).dict_entry_bytes for s in segs] if c == "s" else None for c in BOUND4]
        dom = DictionaryDomain.from_dictionaries(ctx, BOUND4, [devs[0].column_index(c) for c in BOUND4], types, parts, widths)
        for c, card in (("big", BIG), ("h1", HUGE), ("a1", WIDE3)):
            assert dom.info(c)["cardinality"] == card
        for d in devs:
            d.bind_domain(dom)
        yield segs, devs, dom, {c: _domain_values(dom, c) for c in BOUND4}
    finally:
        for d in devs:
            d.destroy()
        if dom is not None:
            dom.release()


@contextlib.contextmanager
def _route(ctx, knobs):
    """tuned() for the knobs it knows; "spec" (not among its defaults) is restored to 1 here."""
    knobs = dict(knobs)
    spec = knobs.pop("spec", None)
    try:
        if spec is not None:
            ctx.set_tuning("spec", spec)
        with tuned(ctx, **knobs):
            yield
    finally:
        if spec is not None:
            ctx.set_tuning("spec", 1)


def _check_block(q, block, values, ref, docs, what):
    """assert_exact of the decoded table, num_docs_scanned, and every MIN / MAX dictId the domain id of its value."""
    got = _table(q, block, values)
    assert_exact(q, got, ref, what)
    assert block.stats.num_docs_scanned == docs, (what, block.stats.num_docs_scanned, docs)
    for g, key in enumerate(got):
        for a, agg in enumerate(q.aggregations):
            if agg.function in ("MIN", "MAX"):
                assert _py(values[agg.column][int(block.dict_ids[a][g])]) == ref[key][a], (what, key, agg.function, agg.column)


@pytest.mark.parametrize("route", list(ROUTES))
def test_every_aggregation_route_over_domain_ids(oracle, ctx, pm, agg_bound, route):
    """Per segment and merged, against exact_ref over the unbound segments; GROUP BY a1, a2, a3 (2^63 raw keys) is
    refused with UnsupportedQueryError, never answered."""
    t0 = time.perf_counter()
    segs, devs, _, values = agg_bound
    with _route(ctx, ROUTES[route]):
        for text in AGG_QUERIES:
            q = sql.parse(text, num_groups_limit=LIMIT)
            docs = [int(matching_docs(oracle, s, q.filter).sum()) for s in segs]
            for s, b, n in zip(segs, pm.execute_segments(devs, q), docs):
                _check_block(q, b, values, exact_reference(oracle, [s], q), n, f"{route} n={s.num_docs}: {text}")
                if q.group_by == ["h1", "h2"]:
                    assert b.regime == "LONG_MAP", (route, b.regime)
            merged = pm.execute_segments(devs, q, merge=True)[0]
            _check_block(q, merged, values, exact_reference(oracle, segs, q), sum(docs), f"{route} merged: {text}")
        q = sql.parse("SELECT COUNT(*), SUM(v) FROM t GROUP BY a1, a2, a3", num_groups_limit=LIMIT)
        for d in devs:
            with pytest.raises(UnsupportedQueryError):
                pm.execute_segments([d], q)
        with pytest.raises(UnsupportedQueryError):
            pm.execute_segments(devs, q, merge=True)
    print(f"{route}: {time.perf_counter() - t0:.1f} s")
