"""CPU: the value-space filter reference (tests/filter_ref.py) on known answers, the oracle's filter and the product's
predicate resolution (pb200h::matching_dict_ids / leaf_to_device, through the tests/host_probe shim) against it.

Literals are compared with stored values by their exact numeric value.  On an INT / LONG column `x = 2.5` matches
nothing, `x >= 2.5` is `x >= 3`, `x < -2.5` is `x <= -3`, and a literal beyond the column's range makes the predicate
constant (2^63 on a LONG column is above every value, not INT64_MAX or a wrapped negative)."""
import ctypes as C

import numpy as np
import pytest

from filter_ref import matching_docs, matching_docs_many
from oracle import segment_builder as sb
from pinot_b200 import _lib, sql
from pinot_b200.plan_maker import _marshal_query
from pinot_b200.query import Aggregation, Filter, Predicate, QueryContext
from test_host_logic_cpu import _leaf_docs, probe  # noqa: F401  (probe: the g++ shim fixture)

INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
F32_MAX = float(np.finfo(np.float32).max)
F64_MAX = float(np.finfo(np.float64).max)

# {column: values in doc order}; the same values as a dictionary column and, suffix "r", as a raw one
X = [2, -3, 3, 1, -2]
N_KNOWN = 8   # every column repeats its values up to 8 docs
KNOWN_COLUMNS = {c: np.resize(np.asarray(v, dtype=t), N_KNOWN) for c, v, t in [
    ("x", X, np.int32),
    ("xl", X, np.int64),
    ("i", [0, INT_MAX, -1, INT_MIN, 1], np.int32),
    ("l", [0, INT64_MAX, -1, INT64_MIN, 1], np.int64),
    ("f", [1.5, -np.inf, F32_MAX, np.float32(0.1), -F32_MAX, np.inf, -1.5], np.float32),
    ("d", [0.1, -np.inf, F64_MAX, 5e-324, -F64_MAX, np.inf, -5e-324, 0.0], np.float64),
    ("s", [b"b", b"ab", "é".encode(), b"a", b"abc", b"ba", b"zz"], None)]}
KNOWN_COLUMNS["xs"] = np.sort(KNOWN_COLUMNS["x"])   # ascending: stored as a sorted column
ALL = object()


def _p(sql_cond):
    return sql.parse(f"SELECT COUNT(*) FROM t WHERE {sql_cond}").filter


# (column, predicate as SQL or Predicate, matching values or ALL)
KNOWN = [
    # fractional literals on INT / LONG (dictionary, sorted and raw)
    *[(c, f"{c} {cond}", want) for c in ("x", "xl", "xs") for cond, want in [
        (">= 2.5", {3}), ("> 2.5", {3}), ("< 2.5", {-3, -2, 1, 2}), ("<= 2.5", {-3, -2, 1, 2}), ("= 2.5", set()),
        ("!= 2.5", ALL), ("BETWEEN 1.5 AND 2.5", {2}), (">= -2.5", {-2, 1, 2, 3}), ("< -2.5", {-3}), ("> -2.5", {-2, 1, 2, 3}),
        ("<= -2.5", {-3}), ("IN (2.5, 3)", {3}), ("NOT IN (2.5, -3)", {-2, 1, 2, 3}), ("> -3.5", ALL), ("<= 3.0", ALL),
        ("< 3.0", {-3, -2, 1, 2}), ("BETWEEN 2.25 AND 2.75", set()), ("BETWEEN -2.5 AND -1.5", {-2})]],
    # INT at its ends, and literals beyond int32 / int64 (a 32-bit or 64-bit wrap would find -1)
    ("i", "i >= 2147483647", {INT_MAX}), ("i", "i > 2147483647", set()), ("i", "i >= 2147483647.5", set()),
    ("i", "i > 2147483646.5", {INT_MAX}), ("i", "i <= -2147483648", {INT_MIN}), ("i", "i < -2147483648", set()),
    ("i", "i < -2147483647.5", {INT_MIN}), ("i", "i >= 2147483648", set()), ("i", "i < 2147483648", ALL),
    ("i", "i > -2147483649", ALL), ("i", "i = 4294967295", set()), ("i", "i = -4294967297", set()),
    ("i", "i IN (4294967295, 0)", {0}), ("i", "i != 4294967295", ALL), ("i", "i = 18446744073709551615", set()),
    ("i", "i < 9223372036854775808", ALL), ("i", "i > -9223372036854775809", ALL), ("i", "i BETWEEN -1.5 AND 0.5", {-1, 0}),
    # LONG at its ends and beyond int64 (a ctypes int64 wraps 2^63 to INT64_MIN and 2^64 - 1 to -1)
    ("l", "l >= 9223372036854775807", {INT64_MAX}), ("l", "l > 9223372036854775806", {INT64_MAX}),
    ("l", "l > 9223372036854775807", set()), ("l", "l >= 9223372036854775808", set()),
    ("l", "l < 9223372036854775808", ALL), ("l", "l = 9223372036854775808", set()),
    ("l", "l != 9223372036854775808", ALL), ("l", "l = 18446744073709551615", set()),
    ("l", "l < -9223372036854775809", set()), ("l", "l <= -9223372036854775808", {INT64_MIN}),
    ("l", "l < -9223372036854775807", {INT64_MIN}), ("l", "l BETWEEN -1.5 AND 0.5", {-1, 0}),
    ("l", "l >= 9200000000000000000.0", {INT64_MAX}), ("l", "l < 10000000000000000000.0", ALL),
    ("l", "l NOT IN (9223372036854775807, 9223372036854775808)", {INT64_MIN, -1, 0, 1}),
    # FLOAT: the literal as (float)literal
    ("f", "f = 0.1", {float(np.float32(0.1))}), ("f", "f BETWEEN -1.5 AND 1.5", {-1.5, float(np.float32(0.1)), 1.5}),
    ("f", Predicate("RANGE", "f", [], F32_MAX, None, False, True), {np.inf}),
    ("f", Predicate("RANGE", "f", [], None, -F32_MAX, True, False), {-np.inf}),
    ("f", Predicate("RANGE", "f", [], 1e39, None, True, True), {np.inf}),       # (float)1e39 = inf
    ("f", Predicate("RANGE", "f", [], 1e39, None, False, True), set()),
    ("f", Predicate("NEQ", "f", [-np.inf]), {1.5, F32_MAX, float(np.float32(0.1)), -F32_MAX, np.inf, -1.5}),
    # DOUBLE: subnormals, +-max, +-inf
    ("d", "d > 0", {5e-324, 0.1, F64_MAX, np.inf}), ("d", "d < 4.9e-324", {-np.inf, -F64_MAX, -5e-324, 0.0}),
    ("d", "d = 0.1", {0.1}), ("d", Predicate("RANGE", "d", [], F64_MAX, None, False, True), {np.inf}),
    ("d", Predicate("RANGE", "d", [], -F64_MAX, 5e-324, True, False), {-F64_MAX, -5e-324, 0.0}),
    ("d", Predicate("IN", "d", [np.inf, -np.inf, 1.0]), {np.inf, -np.inf}),
    # STRING: bytewise order of the unpadded UTF-8 bytes
    ("s", "s >= 'ab' AND s < 'b'", {b"ab", b"abc"}), ("s", "s > 'a'", {b"ab", b"abc", b"b", b"ba", b"zz", "é".encode()}),
    ("s", "s < 'ab'", {b"a"}), ("s", "s BETWEEN 'abc' AND 'b'", {b"abc", b"b"}), ("s", "s > 'zz'", {"é".encode()}),
    ("s", "s = 'ab'", {b"ab"}), ("s", "s NOT IN ('a', 'zzz', 'b')", {b"ab", b"abc", b"ba", b"zz", "é".encode()}),
    ("s", "s < 'a'", set()), ("s", "s > 'ab' AND s < 'abc'", set()),
]
RAW = ["x", "xl", "i", "l", "f", "d"]


@pytest.fixture(scope="module")
def known_seg(oracle):
    cols = dict(KNOWN_COLUMNS)
    cols.update({c + "r": KNOWN_COLUMNS[c] for c in RAW})
    return oracle.build_segment("known", cols, raw=[c + "r" for c in RAW])


def _cases():
    """Every known case on the dictionary column and, where there is one, the raw twin."""
    for col, pred, want in KNOWN:
        node = _p(pred) if isinstance(pred, str) else pred
        yield col, node, want
        if col in RAW:
            yield col + "r", _rename(node, col, col + "r"), want


def _rename(node, old, new):
    if isinstance(node, Predicate):
        return Predicate(node.type, new if node.column == old else node.column, list(node.values), node.lower, node.upper,
                         node.lower_inclusive, node.upper_inclusive)
    return Filter(node.type, [_rename(c, old, new) for c in node.children])


def _values_of(seg, col, mask):
    vals = KNOWN_COLUMNS[col[:-1] if col.endswith("r") and col[:-1] in RAW else col]
    return {v.item() if hasattr(v, "item") else v for v in vals[mask]}


def _want_mask(seg, col, want):
    vals = KNOWN_COLUMNS[col[:-1] if col.endswith("r") and col[:-1] in RAW else col]
    if want is ALL:
        return np.ones(seg.num_docs, dtype=bool)
    return np.array([v.item() in want if hasattr(v, "item") else v in want for v in vals])


def test_known_answers_of_the_reference(oracle, known_seg):
    n = 0
    for col, node, want in _cases():
        got = matching_docs(oracle, known_seg, node)
        assert np.array_equal(got, _want_mask(known_seg, col, want)), (col, node, _values_of(known_seg, col, got))
        n += 1
    assert n > 100


def test_oracle_filter_on_known_answers(oracle, known_seg):
    """The oracle's filter resolves fractional and out-of-range literals by exact value too (dictionary, sorted and raw)."""
    for col, node, want in _cases():
        docs, _ = oracle.filter_doc_ids(known_seg, QueryContext([Aggregation("COUNT", None)], filter=node))
        got = np.zeros(known_seg.num_docs, dtype=bool)
        got[docs] = True
        assert np.array_equal(got, _want_mask(known_seg, col, want)), (col, node, _values_of(known_seg, col, got))


# ------------------------------------------------------------------------------------------------ seeded random trees
def _random_segment(oracle, n=3000, seed=11):
    rng = np.random.default_rng(seed)
    i = rng.integers(-40, 40, size=n).astype(np.int32) * 3
    i[:2] = [INT_MIN, INT_MAX]
    l = rng.integers(-30, 30, size=n).astype(np.int64) * 1_000_000_007
    l[:2] = [INT64_MIN, INT64_MAX]
    cols = {
        "i": i, "ir": rng.permutation(i),
        "l": l, "lr": rng.permutation(l),
        "f": (rng.integers(-50, 50, size=n) / 4.0).astype(np.float32),
        "d": rng.integers(-50, 50, size=n) / 3.0,
        "s": np.array([b"a", b"ab", b"b", b"ba", b"c", b"cz"])[rng.integers(0, 6, size=n)],
        "srt": np.sort(rng.integers(0, 60, size=n)).astype(np.int32),
        "inv": rng.integers(0, 50, size=n).astype(np.int32),
    }
    return oracle.build_segment("rand", cols, inverted=["inv", "s"], raw=["ir", "lr"])


def literal_pool(values: np.ndarray, integral: bool):
    """Literals for one column: stored values (first, last, inner), absent neighbours, and for INT / LONG fractions next to
    stored values and literals beyond int32 / int64."""
    u = np.unique(values)
    present = [u[0], u[-1], u[len(u) // 2], u[min(1, len(u) - 1)], u[max(-2, -len(u))]]
    if values.dtype.kind == "S":
        return [v.decode() for v in present] + ["", "aa", "bb", "zzz"]
    present = [v.item() for v in present]
    if not integral:
        return present + [present[0] - 0.5, present[1] + 0.5, present[2] + 1e-3]
    mid = present[2]
    return present + [mid + 1, mid - 1, mid + 0.5, mid - 0.5, present[0] - 0.5, present[1] + 0.5, float(mid),
                      INT_MAX + 1, INT_MIN - 1, INT_MAX + 0.5, INT64_MAX + 1, INT64_MIN - 1, 1e19, -1e19, (1 << 64) - 1]


def random_leaf(rng, col, pool):
    k = rng.integers(0, 6)
    v = lambda: pool[int(rng.integers(0, len(pool)))]   # noqa: E731
    if k == 0:
        return Predicate("EQ", col, [v()])
    if k == 1:
        return Predicate("NEQ", col, [v()])
    if k == 2:
        return Predicate("IN", col, [v() for _ in range(int(rng.integers(1, 5)))])
    if k == 3:
        return Predicate("NOT_IN", col, [v() for _ in range(int(rng.integers(1, 5)))])
    lo, hi = (v() if rng.random() < 0.8 else None), (v() if rng.random() < 0.8 else None)
    return Predicate("RANGE", col, [], lo, hi, bool(rng.random() < 0.5), bool(rng.random() < 0.5))


def random_tree(rng, leaf, depth=3, nots=True):
    """AND / OR of 2-3 children and (nots) NOT, down to `depth`."""
    if depth == 0 or rng.random() < 0.35:
        return leaf()
    t = ("AND", "OR", "NOT")[int(rng.integers(0, 3 if nots else 2))]
    if t == "NOT":
        return Filter("NOT", [random_tree(rng, leaf, depth - 1, nots)])
    return Filter(t, [random_tree(rng, leaf, depth - 1, nots) for _ in range(int(rng.integers(2, 4)))])


def test_random_trees_match_the_oracle(oracle):
    """300 seeded trees over every column type and index kind, literals from literal_pool: the oracle's doc set must equal
    the reference's (with integral in-range literals this is parity, with the others the shared literal semantics).
    NOT nodes are left out here (NEQ / NOT_IN leaves stay): an AND whose operands include a NOT over a scan or OR
    iterator comes back from the oracle's iterator chain (AndDocIdIterator -> NotDocIdIterator.advance) with a few extra
    docs at the segment's tail on this segment.  That is a defect of the oracle's iterator model, not of literal
    resolution, and is not fixed here; the device tests hold the product's NOT trees to the reference instead."""
    seg = _random_segment(oracle)
    pools = {c.name: literal_pool(np.asarray(c.raw_values if c.raw_values is not None else c.dict_values),
                                  c.data_type in (sb.INT, sb.LONG)) for c in seg.columns}
    names = list(pools)
    rng = np.random.default_rng(2024)

    def leaf():
        c = names[int(rng.integers(0, len(names)))]
        return random_leaf(rng, c, pools[c])
    trees = [random_tree(rng, leaf, nots=False) for _ in range(300)]
    refs = matching_docs_many(oracle, seg, trees)
    for t, ref in zip(trees, refs):
        docs, _ = oracle.filter_doc_ids(seg, QueryContext([Aggregation("COUNT", None)], filter=t))
        assert np.array_equal(docs, np.nonzero(ref)[0]), t


# ------------------------------------------------------------------------------------------------ the product's resolution
def _column_struct(col):
    nm = col.name.encode()
    has_inv = col.inv is not None and not col.is_sorted
    return _lib.HColumn(nm, col.data_type, 1, col.bits, col.cardinality, int(col.is_sorted), col.dict_entry_bytes,
                        col.fwd.ctypes.data, len(col.fwd), col.dict.ctypes.data, len(col.dict),
                        col.inv.ctypes.data if has_inv else None, len(col.inv) if has_inv else 0), nm


def _leaves_for(col, pool):
    preds = []
    for v in pool:
        preds += [Predicate(t, col, [v]) for t in ("EQ", "NEQ")]
        preds += [Predicate("IN", col, [v, pool[0]]), Predicate("NOT_IN", col, [v, pool[1]])]
        for li in (True, False):
            preds += [Predicate("RANGE", col, [], v, None, li, True), Predicate("RANGE", col, [], None, v, True, li),
                      Predicate("RANGE", col, [], v, pool[1], li, not li)]
    return preds


def _dict_columns(oracle):
    seg = _random_segment(oracle)
    known = oracle.build_segment("known", KNOWN_COLUMNS, inverted=["x"])
    out = []
    for s in (seg, known):
        for c in s.columns:
            if c.has_dictionary:
                out.append((s, c, literal_pool(np.asarray(c.dict_values), c.data_type in (sb.INT, sb.LONG))))
    return out


def test_product_matching_dict_ids_against_the_reference(oracle, probe):  # noqa: F811
    """pb200h::matching_dict_ids (what a star-tree predicate and every dictionary leaf resolve to): the docs whose dictId it
    returns are exactly the reference's docs."""
    checked = 0
    for seg, col, pool in _dict_columns(oracle):
        cstruct, _keep = _column_struct(col)
        ids_of_doc = np.asarray(col.dict_ids)
        for p in _leaves_for(col.name, pool):
            hq, keep = _marshal_query(QueryContext([Aggregation("COUNT", None)], filter=p), False)
            out = np.zeros(col.cardinality + 1, dtype=np.int32)
            m = probe.probe_matching_dict_ids(C.byref(cstruct), hq.filter, hq.literals, out.ctypes.data, len(out))
            assert 0 <= m <= col.cardinality, (col.name, p, m)
            got = np.isin(ids_of_doc, out[:m])
            assert np.array_equal(got, matching_docs(oracle, seg, p)), (col.name, p)
            checked += 1
    assert checked > 2000


def test_product_leaf_to_device_against_the_reference(oracle, probe):  # noqa: F811
    """pb200h::leaf_to_device on dictionary, sorted and inverted columns: the device leaf it builds matches the reference's
    docs (evaluated on the dictIds as the kernel would)."""
    probe.probe_leaf_to_device.restype = C.c_int64
    probe.probe_leaf_to_device.argtypes = [C.POINTER(_lib.HColumn), C.c_int32, C.POINTER(_lib.HFilterNode),
                                           C.POINTER(_lib.HLiteral), C.c_void_p, C.c_void_p, C.c_int64]
    checked = 0
    for seg, col, pool in _dict_columns(oracle):
        cstruct, _keep = _column_struct(col)
        for p in _leaves_for(col.name, pool):
            hq, keep = _marshal_query(QueryContext([Aggregation("COUNT", None)], filter=p), False)
            out4 = np.zeros(4, dtype=np.int32)
            ids = np.zeros(2 * col.cardinality + 8, dtype=np.int32)
            m = probe.probe_leaf_to_device(C.byref(cstruct), seg.num_docs, hq.filter, hq.literals, out4.ctypes.data,
                                           ids.ctypes.data, len(ids))
            assert m >= 0, (col.name, p, m)
            got = np.zeros(seg.num_docs, dtype=bool)
            got[_leaf_docs(int(out4[0]), int(out4[2]), int(out4[3]), ids[:m], col.dict_ids, seg.num_docs)] = True
            assert np.array_equal(got, matching_docs(oracle, seg, p)), (col.name, p, int(out4[0]))
            checked += 1
    assert checked > 2000
