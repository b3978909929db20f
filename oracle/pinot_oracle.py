"""ctypes binding of the CPU parity oracle -- TEST INFRASTRUCTURE ONLY (see oracle/pinot_oracle.h).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / ``--impl reference`` legs may import this module.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np

from pinot_b200.query import Filter, QueryContext, postfix

from . import segment_builder as sb

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libpinot_oracle.so")

_TYPE_CODES = {"AND": 0, "OR": 1, "NOT": 2, "EQ": 3, "NEQ": 4, "IN": 5, "NOT_IN": 6, "RANGE": 7}
_FN_CODES = {"COUNT": 0, "SUM": 1, "MIN": 2, "MAX": 3, "AVG": 4, "DISTINCTCOUNT": 5}
REGIMES = {0: "NONE", 1: "ARRAY", 2: "INT_MAP", 3: "LONG_MAP", 4: "ARRAY_MAP", 5: "NO_DICTIONARY"}


class _Column(C.Structure):
    _fields_ = [("data_type", C.c_int32), ("has_dictionary", C.c_int32), ("bits_per_value", C.c_int32),
                ("cardinality", C.c_int32), ("is_sorted", C.c_int32), ("dict_entry_bytes", C.c_int32),
                ("fwd", C.c_void_p), ("fwd_len", C.c_int64), ("dict", C.c_void_p), ("dict_len", C.c_int64),
                ("inv", C.c_void_p), ("inv_len", C.c_int64)]


class _Segment(C.Structure):
    _fields_ = [("num_docs", C.c_int32), ("num_columns", C.c_int32), ("columns", C.POINTER(_Column))]


class _Literal(C.Structure):
    _fields_ = [("i", C.c_int64), ("d", C.c_double), ("s", C.c_char_p)]


class _FilterNode(C.Structure):
    _fields_ = [("type", C.c_int32), ("column", C.c_int32), ("num_children", C.c_int32),
                ("lower_inclusive", C.c_int32), ("upper_inclusive", C.c_int32), ("lower_unbounded", C.c_int32),
                ("upper_unbounded", C.c_int32), ("num_values", C.c_int32), ("values_offset", C.c_int32)]


class _Agg(C.Structure):
    _fields_ = [("function", C.c_int32), ("column", C.c_int32)]


class _Query(C.Structure):
    _fields_ = [("num_filter_nodes", C.c_int32), ("filter", C.POINTER(_FilterNode)), ("literals", C.POINTER(_Literal)),
                ("num_group_by", C.c_int32), ("group_by_columns", C.POINTER(C.c_int32)), ("num_aggs", C.c_int32),
                ("aggs", C.POINTER(_Agg)), ("num_groups_limit", C.c_int32),
                ("max_initial_result_holder_capacity", C.c_int32), ("and_scan_reordering", C.c_int32),
                ("num_doc_ids", C.c_int64), ("doc_ids", C.c_void_p),
                ("agg_filter_nodes", C.POINTER(_FilterNode)), ("agg_filter_start", C.POINTER(C.c_int32)),
                ("agg_filter_count", C.POINTER(C.c_int32))]


class _StarPredicate(C.Structure):
    _fields_ = [("dimension", C.c_int32), ("num_ids", C.c_int32), ("ids", C.c_void_p)]


def build(force: bool = False) -> str:
    """Compiles oracle/_build/libpinot_oracle.so with the committed Makefile (g++)."""
    src = os.path.join(_HERE, "pinot_oracle.cpp")
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < max(
            os.path.getmtime(src), os.path.getmtime(os.path.join(_HERE, "pinot_oracle.h"))):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _LIB_PATH


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


@dataclass
class OracleResult:
    """One segment's results block (AggregationResultsBlock / GroupByResultsBlock + ExecutionStatistics)."""
    num_groups: int  # -1 = aggregation only
    regime: str
    groups_limit_reached: bool
    stats: Tuple[int, int, int, int]  # docsScanned, entriesInFilter, entriesPostFilter, totalDocs
    keys: np.ndarray  # [G, k] dictIds
    doubles: List[np.ndarray]  # per aggregation [G or 1]
    longs: List[np.ndarray]
    distinct: Dict[Tuple[int, int], np.ndarray] = field(default_factory=dict)  # (agg, group) -> sorted dictIds
    # group-by position j of a RAW column -> its on-the-fly dictionary (id -> value): keys[:, j] are ids into it
    raw_key_values: Dict[int, np.ndarray] = field(default_factory=dict)
    # aggregation index of a DISTINCTCOUNT over a RAW column -> value numbering (number -> value): distinct[(a, g)] holds numbers
    raw_distinct_values: Dict[int, np.ndarray] = field(default_factory=dict)


class Oracle:
    def __init__(self):
        self.lib = C.CDLL(build())
        L = self.lib
        L.po_execute.restype = C.c_void_p
        L.po_execute.argtypes = [C.POINTER(_Segment), C.POINTER(_Query)]
        L.po_result_error.restype = C.c_char_p
        L.po_result_error.argtypes = [C.c_void_p]
        for f in ("po_result_num_groups", "po_result_regime", "po_result_groups_limit_reached"):
            getattr(L, f).restype = C.c_int32
            getattr(L, f).argtypes = [C.c_void_p]
        L.po_result_stats.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
        L.po_result_group_keys.argtypes = [C.c_void_p, C.c_void_p]
        L.po_result_agg_double.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
        L.po_result_agg_long.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
        L.po_result_distinct.restype = C.c_int64
        L.po_result_distinct.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int64]
        L.po_result_raw_key_values.restype = C.c_int64
        L.po_result_raw_key_values.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64]
        L.po_result_raw_distinct_values.restype = C.c_int64
        L.po_result_raw_distinct_values.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64]
        L.po_result_free.argtypes = [C.c_void_p]
        L.po_filter_doc_ids.restype = C.c_int64
        L.po_filter_doc_ids.argtypes = [C.POINTER(_Segment), C.POINTER(_Query), C.c_void_p, C.c_int64,
                                        C.POINTER(C.c_int64)]
        L.po_num_bits_per_value.restype = C.c_int32
        L.po_bitset_write.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_void_p]
        L.po_bitset_read.restype = C.c_int32
        L.po_bitset_read.argtypes = [C.c_void_p, C.c_int64, C.c_int32]
        L.po_fixedbit_read_unchecked.restype = C.c_int32
        L.po_fixedbit_read_unchecked.argtypes = [C.c_void_p, C.c_int64, C.c_int32]
        L.po_fixedbit_read32.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p]
        L.po_fwd_read_dict_ids.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]
        L.po_roaring_serialize.restype = C.c_int64
        L.po_roaring_serialize.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int64]
        L.po_roaring_deserialize.restype = C.c_int64
        L.po_roaring_deserialize.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]
        L.po_inverted_index_build.restype = C.c_int64
        L.po_inverted_index_build.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int64]
        L.po_startree_info.restype = C.c_int32
        L.po_startree_info.argtypes = [C.c_void_p, C.c_int64, C.POINTER(C.c_int32), C.c_char_p, C.c_int32]
        L.po_startree_traverse.restype = C.c_int64
        L.po_startree_traverse.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.POINTER(_StarPredicate), C.c_int32,
                                           C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_uint32)]

        L.po_synth_fwd.argtypes = [C.c_uint64, C.c_int32, C.c_int64, C.c_int32, C.c_void_p, C.c_int32]
        L.po_synth_dict.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_void_p]

    # ---------------------------------------------------------------- benchmark table (twin of pb200_synth.cu)
    def synth_segment(self, name: str, num_docs: int, specs, threads: int = 0) -> sb.SegmentData:
        """The synthetic segment IndexSegment.synthetic(ctx, name, num_docs, specs) creates on the device, built on the
        CPU (same dictIds, same Pinot bytes; no inverted indexes).  specs: dicts with name, cardinality, seed,
        value_base=0, value_step=1."""
        threads = threads or (os.cpu_count() or 1)
        cols = []
        for s in specs:
            card = int(s["cardinality"])
            bits = sb.num_bits_per_value(card - 1)
            fwd = np.zeros((num_docs * bits + 7) // 8, dtype=np.uint8)
            self.lib.po_synth_fwd(int(s["seed"]), card, num_docs, bits, _ptr(fwd), threads)
            dct = np.zeros(4 * card, dtype=np.uint8)
            self.lib.po_synth_dict(card, int(s.get("value_base", 0)), int(s.get("value_step", 1)), _ptr(dct))
            vals = (int(s.get("value_base", 0)) + int(s.get("value_step", 1)) * np.arange(card, dtype=np.int64)).astype(np.int32)
            cols.append(sb.ColumnData(s["name"], sb.INT, True, bits, card, False, 4, fwd, dct, None, dict_values=vals))
        return sb.SegmentData(name, num_docs, cols)

    @staticmethod
    def row_ranges(seg: sb.SegmentData, parts: int):
        """Splits a segment of unsorted dict-encoded columns into `parts` consecutive row ranges WITHOUT copying: range
        starts are multiples of 32 rows, where every fixed-bit stream is word aligned (FixedBitIntReader.read32 groups).
        Used to run the single-threaded operator chain of the oracle on all host cores over one big segment; the
        sub-results share the dictionaries and are merged by dictId."""
        per = max(32, ((seg.num_docs + parts - 1) // parts + 31) // 32 * 32)
        out = []
        for start in range(0, seg.num_docs, per):
            n = min(per, seg.num_docs - start)
            cols = []
            for c in seg.columns:
                assert c.has_dictionary and not c.is_sorted and c.inv is None, "row_ranges: plain dict-encoded columns only"
                b0 = start * c.bits // 8
                cols.append(sb.ColumnData(c.name, c.data_type, True, c.bits, c.cardinality, False, c.dict_entry_bytes,
                                          c.fwd[b0: b0 + (n * c.bits + 7) // 8], c.dict, None, dict_values=c.dict_values))
            out.append(sb.SegmentData(f"{seg.name}[{start}:{start + n}]", n, cols))
        return out

    # ---------------------------------------------------------------- formats
    def bitset_write(self, values: np.ndarray, bits: int) -> np.ndarray:
        v = np.ascontiguousarray(values, dtype=np.int32)
        out = np.zeros((len(v) * bits + 7) // 8, dtype=np.uint8)
        self.lib.po_bitset_write(_ptr(out), 0, bits, len(v), _ptr(v))
        return out

    def bitset_read(self, buf: np.ndarray, index: int, bits: int) -> int:
        return self.lib.po_bitset_read(_ptr(buf), index, bits)

    def read_unchecked(self, buf: np.ndarray, index: int, bits: int) -> int:
        return self.lib.po_fixedbit_read_unchecked(_ptr(buf), index, bits)

    def read32(self, buf: np.ndarray, index: int, bits: int) -> np.ndarray:
        out = np.zeros(32, dtype=np.int32)
        self.lib.po_fixedbit_read32(_ptr(buf), index, bits, _ptr(out))
        return out

    def read_dict_ids(self, buf: np.ndarray, num_docs: int, bits: int, doc_ids: np.ndarray) -> np.ndarray:
        d = np.ascontiguousarray(doc_ids, dtype=np.int32)
        out = np.zeros(len(d), dtype=np.int32)
        self.lib.po_fwd_read_dict_ids(_ptr(buf), num_docs, bits, _ptr(d), len(d), _ptr(out))
        return out

    def roaring_serialize(self, values: np.ndarray, run_optimize: bool = True) -> np.ndarray:
        v = np.ascontiguousarray(values, dtype=np.uint32)
        n = self.lib.po_roaring_serialize(_ptr(v), len(v), int(run_optimize), None, 0)
        out = np.zeros(n, dtype=np.uint8)
        self.lib.po_roaring_serialize(_ptr(v), len(v), int(run_optimize), _ptr(out), n)
        return out

    def roaring_deserialize(self, buf: np.ndarray) -> np.ndarray:
        b = np.ascontiguousarray(buf, dtype=np.uint8)
        n = self.lib.po_roaring_deserialize(_ptr(b), len(b), None, 0)
        if n < 0:
            raise ValueError("malformed roaring bitmap")
        out = np.zeros(n, dtype=np.uint32)
        self.lib.po_roaring_deserialize(_ptr(b), len(b), _ptr(out), n)
        return out

    def inverted_index_build(self, dict_ids: np.ndarray, cardinality: int) -> np.ndarray:
        d = np.ascontiguousarray(dict_ids, dtype=np.int32)
        n = self.lib.po_inverted_index_build(_ptr(d), len(d), cardinality, None, 0)
        out = np.zeros(n, dtype=np.uint8)
        self.lib.po_inverted_index_build(_ptr(d), len(d), cardinality, _ptr(out), n)
        return out

    # ---------------------------------------------------------------- segments / queries
    def build_segment(self, name, columns, inverted=(), raw=(), raw_compression=None) -> sb.SegmentData:
        return sb.build_segment(name, columns, inverted=inverted, raw=raw, lib=self, raw_compression=raw_compression)

    @staticmethod
    def _c_segment(seg: sb.SegmentData):
        cols = (_Column * len(seg.columns))()
        for i, c in enumerate(seg.columns):
            fwd = c.fwd if getattr(c, "oracle_fwd", None) is None else c.oracle_fwd   # compressed raw chunks: decoded by chunk_codecs
            cols[i] = _Column(c.data_type, int(c.has_dictionary), c.bits, c.cardinality, int(c.is_sorted),
                              c.dict_entry_bytes, _ptr(fwd), len(fwd), _ptr(c.dict),
                              0 if c.dict is None else len(c.dict), _ptr(c.inv), 0 if c.inv is None else len(c.inv))
        return _Segment(seg.num_docs, len(seg.columns), cols), cols

    # ---------------------------------------------------------------- star-tree
    def startree_info(self, tree: np.ndarray):
        out = (C.c_int32 * 2)()
        names = C.create_string_buffer(4096)
        if self.lib.po_startree_info(_ptr(tree), len(tree), out, names, 4096) != 0:
            raise ValueError("malformed star-tree")
        dims = names.raw.split(b"\0")[: out[0]]
        return [d.decode() for d in dims], int(out[1])

    def startree_traverse(self, tree: np.ndarray, predicates: Dict[int, np.ndarray], group_by_dims, max_docs: int):
        """StarTreeFilterOperator.traverseStarTree: returns (sorted matched star-tree doc ids or None when empty,
        list of dimensions whose predicates remain to be applied)."""
        preds = (_StarPredicate * max(1, len(predicates)))()
        keep = []
        for i, (dim, ids) in enumerate(sorted(predicates.items())):
            arr = np.ascontiguousarray(np.sort(np.asarray(ids, dtype=np.int32)))
            keep.append(arr)
            preds[i] = _StarPredicate(int(dim), len(arr), _ptr(arr) if len(arr) else None)
        gb = np.ascontiguousarray(np.asarray(list(group_by_dims), dtype=np.int32))
        out = np.zeros(max_docs, dtype=np.int32)
        remaining = C.c_uint32(0)
        n = self.lib.po_startree_traverse(_ptr(tree), len(tree), len(predicates), preds, len(gb),
                                          _ptr(gb) if len(gb) else None, _ptr(out), max_docs, C.byref(remaining))
        if n == -2:
            raise ValueError("malformed star-tree")
        if n == -1:
            return None, []
        return out[:n].copy(), [d for d in range(32) if remaining.value >> d & 1]

    @staticmethod
    def _c_query(seg: sb.SegmentData, q: QueryContext, doc_ids: Optional[np.ndarray] = None):
        nodes = list(postfix(q.filter))
        if doc_ids is not None:  # AND(BitmapBasedFilterOperator(doc_ids), original filter)
            nodes = ["DOCIDS"] + nodes + ([Filter("AND", [None, None])] if nodes else [])
        lits: List[_Literal] = []
        keep = []  # keep byte strings alive

        def lit(col: sb.ColumnData, v):
            if col.data_type == sb.STRING:
                b = v.encode("utf-8") if isinstance(v, str) else bytes(v)
                keep.append(b)
                return _Literal(0, 0.0, b)
            # d = the literal rounded to double, i = the literal when it is an int64 (else 0): INT / LONG compare by
            # exact value (pinot_oracle.cpp cmp_integral)
            if isinstance(v, (int, np.integer)):
                iv = int(v)
                try:
                    d = float(iv)
                except OverflowError:
                    d = math.copysign(math.inf, iv)
                return _Literal(iv if -(1 << 63) <= iv < (1 << 63) else 0, d, None)
            d = float(v)
            return _Literal(int(d) if d.is_integer() and -2.0 ** 63 <= d < 2.0 ** 63 else 0, d, None)

        def encode(node_list):
            out = []
            for n in node_list:
                if isinstance(n, str):
                    out.append(_FilterNode(8, -1, 0, 0, 0, 0, 0, 0, 0))  # PO_DOCIDS
                    continue
                if isinstance(n, Filter):
                    out.append(_FilterNode(_TYPE_CODES[n.type], -1, len(n.children), 0, 0, 0, 0, 0, 0))
                    continue
                ci = seg.column_index(n.column)
                col = seg.columns[ci]
                off = len(lits)
                if n.type == "RANGE":
                    lits.append(lit(col, n.lower if n.lower is not None else 0))
                    lits.append(lit(col, n.upper if n.upper is not None else 0))
                    out.append(_FilterNode(_TYPE_CODES["RANGE"], ci, 0, int(n.lower_inclusive), int(n.upper_inclusive),
                                           int(n.lower is None), int(n.upper is None), 2, off))
                else:
                    for v in n.values:
                        lits.append(lit(col, v))
                    out.append(_FilterNode(_TYPE_CODES[n.type], ci, 0, 0, 0, 0, 0, len(n.values), off))
            return out
        enc = encode(nodes)
        c_nodes = (_FilterNode * max(1, len(enc)))(*enc)
        # FILTER (WHERE ...) clauses: one postfix tree per DISTINCT clause, concatenated
        agg_nodes, starts, counts, seen = [], [], [], {}
        for a in q.aggregations:
            f = getattr(a, "filter", None)
            if f is None:
                starts.append(0); counts.append(0)
                continue
            key = repr(f)
            if key not in seen:
                e = encode(list(postfix(f)))
                seen[key] = (len(agg_nodes), len(e))
                agg_nodes += e
            starts.append(seen[key][0]); counts.append(seen[key][1])
        c_agg_nodes = (_FilterNode * max(1, len(agg_nodes)))(*agg_nodes)
        c_starts = (C.c_int32 * max(1, len(starts)))(*starts)
        c_counts = (C.c_int32 * max(1, len(counts)))(*counts)
        c_lits = (_Literal * max(1, len(lits)))(*lits)
        gb = (C.c_int32 * max(1, len(q.group_by)))(*[seg.column_index(c) for c in q.group_by])
        aggs = (_Agg * max(1, len(q.aggregations)))()
        for i, a in enumerate(q.aggregations):
            aggs[i] = _Agg(_FN_CODES[a.function], -1 if a.column is None else seg.column_index(a.column))
        ids = None if doc_ids is None else np.ascontiguousarray(doc_ids, dtype=np.int32)
        cq = _Query(len(nodes), c_nodes, c_lits, len(q.group_by), gb, len(q.aggregations), aggs, q.num_groups_limit,
                    q.max_initial_result_holder_capacity, int(q.and_scan_reordering),
                    0 if ids is None else len(ids), _ptr(ids) if ids is not None and len(ids) else None,
                    c_agg_nodes, c_starts, c_counts)
        return cq, (c_nodes, c_lits, gb, aggs, keep, ids, c_agg_nodes, c_starts, c_counts)

    def execute(self, seg: sb.SegmentData, q: QueryContext, doc_ids: Optional[np.ndarray] = None) -> OracleResult:
        """== getOperator(query).nextBlock() on one segment (BaseQueriesTest.java:97-102).  `doc_ids` (star-tree
        traversal result) is AND-ed to the filter as a BitmapBasedFilterOperator."""
        cseg, _k1 = self._c_segment(seg)
        cq, _k2 = self._c_query(seg, q, doc_ids)
        r = self.lib.po_execute(C.byref(cseg), C.byref(cq))
        try:
            err = self.lib.po_result_error(r)
            if err:
                raise RuntimeError(err.decode())
            g = self.lib.po_result_num_groups(r)
            rows = 1 if g < 0 else g
            stats = (C.c_int64 * 4)()
            self.lib.po_result_stats(r, stats)
            k = len(q.group_by)
            keys = np.zeros((max(g, 0), k), dtype=np.int32)
            if g > 0 and k > 0:
                self.lib.po_result_group_keys(r, _ptr(keys))
            doubles, longs, distinct = [], [], {}
            for a, agg in enumerate(q.aggregations):
                d = np.zeros(rows, dtype=np.float64)
                l = np.zeros(rows, dtype=np.int64)
                if rows:
                    self.lib.po_result_agg_double(r, a, _ptr(d))
                    self.lib.po_result_agg_long(r, a, _ptr(l))
                doubles.append(d)
                longs.append(l)
                if agg.function == "DISTINCTCOUNT":
                    for grp in range(rows):
                        ids = np.zeros(int(l[grp]), dtype=np.int32)
                        self.lib.po_result_distinct(r, a, grp, _ptr(ids), len(ids))
                        distinct[(a, grp)] = ids
            raw_keys = {}
            for j, name in enumerate(q.group_by):
                n = self.lib.po_result_raw_key_values(r, j, None, None, 0)
                if n > 0:
                    d, l = np.zeros(n, dtype=np.float64), np.zeros(n, dtype=np.int64)
                    self.lib.po_result_raw_key_values(r, j, _ptr(d), _ptr(l), n)
                    raw_keys[j] = l if seg.column(name).data_type in (sb.INT, sb.LONG) else d
            raw_distinct = {}
            for a, agg in enumerate(q.aggregations):
                n = self.lib.po_result_raw_distinct_values(r, a, None, None, 0) if agg.function == "DISTINCTCOUNT" else 0
                if n > 0:
                    d, l = np.zeros(n, dtype=np.float64), np.zeros(n, dtype=np.int64)
                    self.lib.po_result_raw_distinct_values(r, a, _ptr(d), _ptr(l), n)
                    raw_distinct[a] = l if seg.column(agg.column).data_type in (sb.INT, sb.LONG) else d
            return OracleResult(g, REGIMES[self.lib.po_result_regime(r)],
                                bool(self.lib.po_result_groups_limit_reached(r)), tuple(stats), keys, doubles, longs,
                                distinct, raw_keys, raw_distinct)
        finally:
            self.lib.po_result_free(r)

    def filter_doc_ids(self, seg: sb.SegmentData, q: QueryContext):
        cseg, _k1 = self._c_segment(seg)
        cq, _k2 = self._c_query(seg, q)
        out = np.zeros(seg.num_docs, dtype=np.int32)
        entries = C.c_int64(0)
        n = self.lib.po_filter_doc_ids(C.byref(cseg), C.byref(cq), _ptr(out), len(out), C.byref(entries))
        return out[:n].copy(), int(entries.value)


_ORACLE: Optional[Oracle] = None


def oracle() -> Oracle:
    global _ORACLE
    if _ORACLE is None:
        _ORACLE = Oracle()
    return _ORACLE
