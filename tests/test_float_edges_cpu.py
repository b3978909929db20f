"""CPU: FLOAT / DOUBLE at NaN, -0.0 and +-inf in the product's host logic, against tests/float_edges_ref.py.

* Dictionaries synthesised from raw values (raw_forward.cpp): every NaN bit pattern is one entry, the last one.
* The ORDER BY key (pb200_order.h): every NaN is one value after +inf, -0.0 before 0.0.
* Predicate resolution: on stored and sorted dictionaries the oracle's doc set (the reference's binary search of the
  dictionary); on a synthesised dictionary the doc set of the raw value comparisons (NaN matches only NEQ / NOT_IN, 0 both
  zeros).
* The CLI's by-value merge: float keys by identity, MIN / MAX and ORDER BY in Double.compare order."""
import ctypes as C
import math
import os
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest

import float_edges_ref as fr
from oracle import segment_builder as sb
from pinot_b200 import _lib, cli, sql
from pinot_b200.plan_maker import _marshal_query
from pinot_b200.query import Aggregation, Predicate, QueryContext
from test_host_logic_cpu import _leaf_docs, probe  # noqa: F401  (probe: the host_probe g++ shim fixture)
from test_order_by_cpu import ALL, DOUBLE, keyfn  # noqa: F401  (keyfn: pb200_order.h compiled with g++)

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

DMAX, FMAX = 1.7976931348623157e308, 3.4028234663852886e38
D_NANS = [fr.D_NAN, fr.D_NEG_NAN, fr.D_PAYLOAD_NAN, fr.D_SIGNALLING_NAN]
F_NANS = [fr.F_NAN, fr.F_NEG_NAN, fr.F_PAYLOAD_NAN, fr.F_SIGNALLING_NAN]


def edge_values(data_type):
    """Every NaN pattern, both zeros, both infinities, the extremes, both smallest subnormals and a few plain values."""
    if data_type == sb.DOUBLE:
        nans = [fr.double_of(b) for b in D_NANS]
        plain = [-math.inf, -DMAX, -1.5, -5e-324, -0.0, 0.0, 5e-324, 1.5, 2.0, DMAX, math.inf]
        return np.array(nans + plain, dtype=np.float64)
    nans = [fr.float_of(b) for b in F_NANS]
    plain = np.array([-math.inf, -FMAX, -1.5, -1e-45, -0.0, 0.0, 1e-45, 1.5, 2.0, FMAX, math.inf], dtype=np.float32)
    return np.concatenate([np.array(nans, dtype=np.float32), plain])


def edge_column(data_type, n, seed):
    rng = np.random.default_rng(seed)
    pool = edge_values(data_type)
    v = pool[rng.integers(0, len(pool), size=n)]
    v[: len(pool)] = pool
    return v


def synthesize(probe, values, data_type):  # noqa: F811
    be = np.ascontiguousarray(values.astype(sb._NP_BE[data_type])).view(np.uint8)
    n = len(values)
    dict_out = np.zeros(n * 8 + 8, dtype=np.uint8)
    fwd_out = np.zeros(n * 4 + 8, dtype=np.uint8)
    card, bits = C.c_int32(), C.c_int32()
    assert probe.probe_synthesize_dictionary(be.ctypes.data, data_type, n, 1 << 20, dict_out.ctypes.data, len(dict_out),
                                             fwd_out.ctypes.data, len(fwd_out), C.byref(card), C.byref(bits)) == 1
    width = 4 if data_type == sb.FLOAT else 8
    dict_be = dict_out[: card.value * width].copy()
    entries = np.frombuffer(dict_be.tobytes(), dtype=sb._NP_BE[data_type])
    ids = sb.unpack_fixed_bits(fwd_out, n, bits.value).astype(np.int64)
    return dict_be, entries, ids


@pytest.mark.parametrize("data_type", [sb.FLOAT, sb.DOUBLE])
def test_synthesised_dictionary_has_one_nan_last(probe, data_type):  # noqa: F811
    values = edge_column(data_type, 5000, 1)
    _, entries, ids = synthesize(probe, values, data_type)
    want = fr.unique_values(values, data_type)
    assert [fr.identity(x, data_type) for x in entries] == [fr.identity(x, data_type) for x in want]
    assert sum(math.isnan(x) for x in entries) == 1 and math.isnan(entries[-1])
    assert [fr.bits_of(x, data_type) for x in entries[:-1]] == [fr.bits_of(x, data_type) for x in want[:-1]]
    # every row's id decodes to its own value (one id for all NaNs, two for the zeros)
    assert all(fr.identity(entries[i], data_type) == fr.identity(v, data_type) for i, v in zip(ids, values))


def test_order_key_puts_every_nan_after_inf(keyfn):  # noqa: F811
    nans = [fr.double_of(b) for b in D_NANS] + [float(fr.float_of(b)) for b in F_NANS]
    keys = {keyfn.probe_order_key(DOUBLE, 0, ALL, x, 0) for x in nans}
    assert len(keys) == 1
    inf = keyfn.probe_order_key(DOUBLE, 0, ALL, math.inf, 0)
    assert keys.pop() > inf
    for x in nans:   # DESC: NaN first
        assert keyfn.probe_order_key(DOUBLE, 1, ALL, x, 0) < keyfn.probe_order_key(DOUBLE, 1, ALL, math.inf, 0)
    assert keyfn.probe_order_key(DOUBLE, 0, ALL, -0.0, 0) < keyfn.probe_order_key(DOUBLE, 0, ALL, 0.0, 0)
    vals = list(edge_values(sb.DOUBLE).tolist())
    got = sorted(vals, key=lambda x: keyfn.probe_order_key(DOUBLE, 0, ALL, x, 0))
    assert [fr.identity(x) for x in got] == [fr.identity(x) for x in sorted(vals, key=fr.ORDER)]


@pytest.fixture(scope="module")
def float_probe(probe):  # noqa: F811  (probe builds the library first)
    src = os.path.join(HERE, "float_probe", "float_probe.cpp")
    out = os.path.join(HERE, "float_probe", "libfloat_probe.so")
    libdir = os.path.join(ROOT, "pinot_b200")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(_lib.LIB_PATH)):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", f"-I{cuda_inc}", "-o", out, src, f"-L{libdir}",
                        "-lpinot_b200", f"-Wl,-rpath,{libdir}"], check=True)
    lib = C.CDLL(out)
    lib.probe_synthesized_leaf.restype = C.c_int64
    lib.probe_synthesized_leaf.argtypes = [C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(_lib.HFilterNode),
                                           C.POINTER(_lib.HLiteral), C.c_void_p, C.c_void_p, C.c_int64]
    probe.probe_leaf_to_device.restype = C.c_int64
    probe.probe_leaf_to_device.argtypes = [C.POINTER(_lib.HColumn), C.c_int32, C.POINTER(_lib.HFilterNode),
                                           C.POINTER(_lib.HLiteral), C.c_void_p, C.c_void_p, C.c_int64]
    return lib


def predicates(column, data_type):
    big = DMAX if data_type == sb.DOUBLE else FMAX
    lits = [0, -0.0, 1.5, big, -big, 2.0, 0.75]
    out = []
    for v in lits:
        out += [Predicate("EQ", column, [v]), Predicate("NEQ", column, [v])]
    for vs in ([0], [-0.0, 1.5], [big, 0.75], [2.0, -big, 0]):
        out += [Predicate("IN", column, vs), Predicate("NOT_IN", column, vs)]
    for lo, hi in ((-1.0, 1.0), (-0.0, 0.0), (0, None), (None, -0.0), (-5e-324, 5e-324), (-big, big), (1.5, big), (None, 0)):
        for li in (True, False):
            for ui in (True, False):
                out.append(Predicate("RANGE", column, [], lo, hi, li, ui))
    return out


@pytest.mark.parametrize("data_type", [sb.FLOAT, sb.DOUBLE])
def test_raw_predicates_follow_the_value_comparisons(probe, float_probe, data_type):  # noqa: F811
    """A synthesised dictionary: the device leaf (and matching_dict_ids) select exactly the rows Java's <, > and == select.
    NaN rows match only NEQ / NOT_IN; `x = 0` and `x = -0.0` match both zeros."""
    n = 3000
    values = edge_column(data_type, n, 2)
    dict_be, entries, ids = synthesize(probe, values, data_type)
    seg = sb.SegmentData("raw", n, [sb.ColumnData("x", data_type, False, 0, 0, False, 0, None, None, None, raw_values=values)])
    for p in predicates("x", data_type):
        want = fr.raw_doc_ids(seg, p)
        hq, _keep = _marshal_query(QueryContext([Aggregation("COUNT", None)], filter=p), False)
        out4 = np.zeros(4, dtype=np.int32)
        buf = np.zeros(2 * len(entries) + 8, dtype=np.int32)
        m = float_probe.probe_synthesized_leaf(data_type, dict_be.ctypes.data, len(entries), n, 1, hq.filter, hq.literals,
                                               out4.ctypes.data, buf.ctypes.data, len(buf))
        assert m >= 0, (p, m)
        got = _leaf_docs(int(out4[0]), int(out4[2]), int(out4[3]), buf[:m], ids, n)
        assert np.array_equal(got, want), (p, len(got), len(want))
        m = float_probe.probe_synthesized_leaf(data_type, dict_be.ctypes.data, len(entries), n, 0, hq.filter, hq.literals,
                                               out4.ctypes.data, buf.ctypes.data, len(buf))
        assert np.array_equal(np.nonzero(np.isin(ids, buf[:m]))[0], want), p


@pytest.mark.parametrize("data_type", [sb.FLOAT, sb.DOUBLE])
@pytest.mark.parametrize("layout", ["scan", "inverted", "sorted"])
def test_stored_dictionary_predicates_match_the_oracle(oracle, probe, float_probe, data_type, layout):  # noqa: F811
    """A dictionary the segment stores (with a NaN entry and both zeros): the reference searches it with the binary search
    of BaseImmutableDictionary.insertionIndexOf, whose `<` / `>` call a NaN entry equal to any literal it lands on and
    -0.0 equal to 0.0.  So `x = 0` matches whichever zero the search meets, and a search that meets NaN matches its rows.
    The product keeps that parity: its doc set is the oracle's, consequences included."""
    n = 2500
    values = edge_column(data_type, n, {"scan": 3, "inverted": 4, "sorted": 5}[layout])
    neg = layout == "scan"   # the NaN entry Java keeps is the first NaN's bits: here with and without the sign bit
    values[np.isnan(values)] = fr.double_of(fr.D_NEG_NAN if neg else fr.D_NAN) if data_type == sb.DOUBLE else \
        fr.float_of(fr.F_NEG_NAN if neg else fr.F_NAN)
    if layout == "sorted":
        values = fr.sorted_rows(values)
    col = fr.build_dict_column("x", values, inverted=layout == "inverted", lib=oracle)
    assert col.is_sorted == (layout == "sorted")
    seg = sb.SegmentData("stored", n, [col])
    has_inv = col.inv is not None
    cstruct = _lib.HColumn(b"x", data_type, 1, col.bits, col.cardinality, int(col.is_sorted), col.dict_entry_bytes,
                           col.fwd.ctypes.data, len(col.fwd), col.dict.ctypes.data, len(col.dict),
                           col.inv.ctypes.data if has_inv else None, len(col.inv) if has_inv else 0)
    for p in predicates("x", data_type):
        q = QueryContext([Aggregation("COUNT", None)], filter=p)
        want = fr.doc_ids(oracle, seg, q)
        hq, _keep = _marshal_query(q, False)
        out4 = np.zeros(4, dtype=np.int32)
        buf = np.zeros(2 * col.cardinality + 8, dtype=np.int32)
        m = probe.probe_leaf_to_device(C.byref(cstruct), n, hq.filter, hq.literals, out4.ctypes.data, buf.ctypes.data, len(buf))
        assert m >= 0, (p, m)
        got = _leaf_docs(int(out4[0]), int(out4[2]), int(out4[3]), buf[:m], col.dict_ids, n)
        assert np.array_equal(got, want), (layout, p, len(got), len(want))


# ------------------------------------------------------------------------------------------------ cli by-value merge
class _Seg:
    def __init__(self, dictionary):
        self.dictionary = dictionary

    def dictionary_value(self, column, dict_id):
        return self.dictionary[dict_id]


def _block(keys, doubles, longs, distinct=None):
    g = len(keys)
    return SimpleNamespace(num_groups=g, keys=np.array(keys, dtype=np.int32).reshape(g, 1),
                           doubles=[np.array(d, dtype=np.float64) for d in doubles],
                           longs=[np.array(v, dtype=np.int64) for v in longs], distinct=distinct or {}, histograms={}, moments={})


def test_cli_merges_float_keys_by_identity_and_orders_them_totally():
    nan_a, nan_b = fr.double_of(fr.D_NAN), fr.double_of(fr.D_NEG_NAN)
    s0 = _Seg([-0.0, 0.0, 1.0, nan_a])
    s1 = _Seg([0.0, 1.0, nan_b])
    q = sql.parse("SELECT COUNT(*), MIN(m), MAX(m), DISTINCTCOUNT(x) FROM t GROUP BY x ORDER BY x DESC LIMIT 10")
    b0 = _block([0, 1, 2, 3], [[0, 0, 0, 0], [5.0, -0.0, 1.0, 2.0], [5.0, 0.0, 1.0, 2.0], [0, 0, 0, 0]], [[1, 2, 3, 4], [0] * 4, [0] * 4, [1] * 4],
                {(3, 0): [0], (3, 1): [1], (3, 2): [2], (3, 3): [3]})
    b1 = _block([0, 1, 2], [[0, 0, 0], [0.0, nan_b, 7.0], [-0.0, nan_b, 7.0], [0, 0, 0]], [[10, 20, 30], [0] * 3, [0] * 3, [1] * 3],
                {(3, 0): [0], (3, 1): [1], (3, 2): [2]})
    table = cli.merge_blocks(q, [s0, s1], [b0, b1])
    assert len(table) == 4   # -0.0, 0.0, 1.0, NaN: the two NaN keys meet, the zeros stay apart
    rows = cli.final_rows(q, table)
    assert [fr.identity(r[0]) for r in rows] == [fr.D_NAN, fr.identity(1.0), fr.identity(0.0), fr.identity(-0.0)]
    assert [r[1] for r in rows] == [34, 23, 12, 1]
    nan_row, one_row, zero_row = rows[0], rows[1], rows[2]
    assert fr.same_double(one_row[2], 1.0) and math.isnan(one_row[3])   # NaN sorts last: MAX is NaN, MIN is not ...
    assert fr.same_double(zero_row[2], -0.0) and fr.same_double(zero_row[3], 0.0)   # ... and MIN(-0.0, 0.0) is -0.0
    assert fr.check_value(nan_row[2], 2.0) and fr.check_value(nan_row[3], 7.0)
    assert [r[4] for r in rows] == [1, 1, 1, 1]   # DISTINCTCOUNT(x) of each key: one value, NaN bits or not


def _distinct_block(values, seg):
    from pinot_b200.plan_maker import ExecutionStatistics, SelectionResultsBlock
    n = len(values)
    return SelectionResultsBlock(["x"], [np.array(values, dtype=np.float64)], np.arange(n, dtype=np.int32),
                                 np.full(n, seg, dtype=np.int32), ExecutionStatistics(n, 0, 0, n))


@pytest.mark.parametrize("asc", [True, False])
def test_distinct_merge_by_identity_in_double_compare_order(asc):
    """The by-value DISTINCT merge of per-segment blocks: two NaN bit patterns are one row, -0.0 and 0.0 are two, and the
    order is Double.compare (NaN after +inf)."""
    from pinot_b200.plan_maker import merge_distinct_blocks
    b0 = _distinct_block([-0.0, fr.double_of(fr.D_NAN), 1.0, math.inf], 0)
    b1 = _distinct_block([0.0, fr.double_of(fr.D_NEG_NAN), 2.0, -math.inf], 1)
    got = merge_distinct_blocks([b0, b1], [("x", asc)], 10)
    want = [-math.inf, -0.0, 0.0, 1.0, 2.0, math.inf, math.nan]
    want = want if asc else want[::-1]
    assert [fr.identity(float(v)) for v in got.columns[0]] == [fr.identity(v) for v in want]
    top = merge_distinct_blocks([b0, b1], [("x", asc)], 2)   # a LIMIT that ends inside the zeros / at NaN
    assert [fr.identity(float(v)) for v in top.columns[0]] == [fr.identity(v) for v in want[:2]]
