"""Python face of the host layer: the reference's plan-maker / operator interface for this path.

Names follow the reference so that tests read like its own (``pinot-core/src/test/java/org/apache/pinot/queries/
BaseQueriesTest.java:97-102``: ``PLAN_MAKER.makeSegmentPlanNode(new SegmentContext(segment), queryContext).run()``):

    ctx      = B200Context(device=0)
    segment  = IndexSegment.from_columns(ctx, "seg", num_docs, columns)          # ImmutableSegmentLoader.load
    operator = B200PlanMaker(ctx).make_segment_plan_node(segment, query).run()    # PlanMaker.makeSegmentPlanNode
    block    = operator.next_block()                                              # Operator.nextBlock()
    block.get_results() / block.group_keys / operator.get_execution_statistics()

All work happens in libpinot_b200.so (C++ plan maker above the C-ABI + CUDA kernels below it); this module only
marshals.  There is no CPU fallback: queries outside the accelerated set raise ``UnsupportedQueryError`` (the Java
``B200PlanMaker`` would call ``super.makeSegmentPlanNode`` there).
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from ._lib import UnsupportedQueryError  # noqa: F401  (re-export)
from .query import Filter, QueryContext, postfix


class B200Context:
    """One per (process, GPU): owns the CUDA context, stream pool and device memory pool."""

    def __init__(self, device: int = 0):
        self.lib = _lib.load()
        h = C.c_void_p()
        _lib.check(self.lib.pb200_init(device, C.byref(h)))
        self.handle = h
        self.device = device

    def device_info(self) -> Dict[str, int]:
        out = (C.c_int64 * 5)()
        _lib.check(self.lib.pb200_device_info(self.handle, out))
        return {"sm_count": out[0], "major": out[1], "minor": out[2], "total_mem_mb": out[3], "free_mem_mb": out[4]}

    def set_tuning(self, name: str, value: int) -> None:
        """pb200_tuning_set: launch knobs of the scan kernel (defaults come from PB200_* environment variables at init)."""
        _lib.check(self.lib.pb200_tuning_set(self.handle, name.encode(), int(value)))

    def last_phases(self) -> dict:
        """pb200_last_phases: host wall-clock (ms) of this thread's last pb200_execute by phase."""
        out = (C.c_double * 6)()
        _lib.check(self.lib.pb200_last_phases(out))
        return dict(zip(("plan", "launch", "device_wait", "results", "extract", "total"), (round(x, 4) for x in out)))

    def close(self):
        if self.handle:
            self.lib.pb200_shutdown(self.handle)
            self.handle = None


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class IndexSegment:
    """An immutable segment resident in HBM (+ host dictionaries). Mirrors ``IndexSegment`` / ``SegmentContext``."""

    def __init__(self, ctx: B200Context, handle, name: str):
        self.ctx = ctx
        self.handle = handle
        self.name = name
        L = ctx.lib
        self.num_docs = L.pb200h_segment_num_docs(handle)
        self.column_names = [L.pb200h_segment_column_name(handle, i).decode() for i in
                             range(L.pb200h_segment_num_columns(handle))]

    # ---- constructors -------------------------------------------------------------------------------------------
    @classmethod
    def from_columns(cls, ctx: B200Context, name: str, num_docs: int, columns: Sequence) -> "IndexSegment":
        """`columns`: objects with name, data_type, has_dictionary, bits, cardinality, is_sorted, dict_entry_bytes and
        numpy uint8 buffers fwd / dict / inv holding Pinot's index file bytes."""
        arr = (_lib.HColumn * len(columns))()
        keep = []
        for i, c in enumerate(columns):
            nm = c.name.encode()
            keep.append(nm)
            arr[i] = _lib.HColumn(nm, c.data_type, int(c.has_dictionary), c.bits, c.cardinality, int(c.is_sorted),
                                  c.dict_entry_bytes, _ptr(c.fwd), len(c.fwd), _ptr(c.dict),
                                  0 if c.dict is None else len(c.dict), _ptr(c.inv),
                                  0 if c.inv is None else len(c.inv))
        h = C.c_void_p()
        _lib.check(ctx.lib.pb200h_segment_create(ctx.handle, name.encode(), num_docs, len(columns), arr, C.byref(h)))
        return cls(ctx, h, name)

    @classmethod
    def synthetic(cls, ctx: B200Context, name: str, num_docs: int, columns: Sequence[dict]) -> "IndexSegment":
        """Generates dict-encoded INT columns directly in HBM (pb200_synth_segment).  Each column dict:
        {name, cardinality, seed, value_base=0, value_step=1, inverted=False}."""
        arr = (_lib.SynthCol * len(columns))()
        for i, c in enumerate(columns):
            arr[i] = _lib.SynthCol(c["cardinality"], c.get("value_base", 0), c.get("value_step", 1),
                                   int(c.get("inverted", False)), c["seed"])
        dev = C.c_void_p()
        _lib.check(ctx.lib.pb200_synth_segment(ctx.handle, name.encode(), num_docs, len(columns), arr, C.byref(dev)))
        names = (C.c_char_p * len(columns))(*[c["name"].encode() for c in columns])
        h = C.c_void_p()
        _lib.check(ctx.lib.pb200h_segment_adopt(ctx.handle, dev, num_docs, len(columns), names, C.byref(h)))
        return cls(ctx, h, name)

    @classmethod
    def load(cls, ctx: B200Context, index_dir: str) -> "IndexSegment":
        """ImmutableSegmentLoader.load(indexDir): reads metadata.properties + v1 / v3 index files from disk."""
        h = C.c_void_p()
        _lib.check(ctx.lib.pb200h_segment_load_dir(ctx.handle, index_dir.encode(), C.byref(h)))
        return cls(ctx, h, index_dir)

    def attach_star_tree(self, tree: np.ndarray, num_star_docs: int, dimensions: Sequence[str],
                         dimension_fwd: Sequence[np.ndarray], metrics: Sequence[tuple]) -> None:
        """StarTreeLoaderUtils.loadStarTreeV2 for one tree: `tree` = OffHeapStarTree bytes, per dimension (split order)
        the fixed-bit forward index of the star-tree docs, `metrics` = [(function, column or None, raw forward index
        bytes)] for the function-column pairs."""
        names = (C.c_char_p * len(dimensions))(*[d.encode() for d in dimensions])
        fwd = (C.c_void_p * len(dimensions))(*[a.ctypes.data for a in dimension_fwd])
        sizes = (C.c_uint64 * len(dimensions))(*[len(a) for a in dimension_fwd])
        arr = (_lib.HStarMetric * len(metrics))()
        keep = []
        for i, (fn, col, buf) in enumerate(metrics):
            nm = None if col is None else col.encode()
            keep.append((nm, buf))
            arr[i] = _lib.HStarMetric(_lib.AGG_CODES[fn], 0, nm, buf.ctypes.data, len(buf))
        _lib.check(self.ctx.lib.pb200h_startree_attach(self.ctx.handle, self.handle, _ptr(tree), len(tree), num_star_docs,
                                                       len(dimensions), names, fwd, sizes, len(metrics), arr))

    # ---- accessors ----------------------------------------------------------------------------------------------
    def column_index(self, name: str) -> int:
        return self.ctx.lib.pb200h_segment_column_index(self.handle, name.encode())

    def column_info(self, name: str) -> Dict[str, int]:
        out = (C.c_int32 * 6)()
        _lib.check(self.ctx.lib.pb200h_segment_column_info(self.handle, self.column_index(name), out))
        return dict(zip(("data_type", "has_dictionary", "bits", "cardinality", "is_sorted", "has_inverted"), out))

    def dictionary_value(self, column: str, dict_id: int):
        """Dictionary.getInternal(dictId)."""
        ci = self.column_index(column)
        info = self.column_info(column)
        d, l = C.c_double(), C.c_int64()
        buf = C.create_string_buffer(4096)
        _lib.check(self.ctx.lib.pb200h_dictionary_get(self.handle, ci, int(dict_id), C.byref(d), C.byref(l), buf, 4096))
        if info["data_type"] == _lib.STRING:
            return buf.value.decode("utf-8")
        return int(l.value) if info["data_type"] in (_lib.INT, _lib.LONG) else float(d.value)

    def read_index(self, column: str, which: str) -> np.ndarray:
        """Index file bytes as held on the device: which in {"fwd", "dict", "inv"}."""
        L = self.ctx.lib
        dev = L.pb200h_segment_device(self.handle)
        w = {"fwd": 0, "dict": 1, "inv": 2}[which]
        ci = self.column_index(column)
        n = L.pb200_segment_read_index(self.ctx.handle, dev, ci, w, None, 0)
        if n < 0:
            _lib.check(int(n))
        out = np.zeros(int(n), dtype=np.uint8)
        if n:
            r = L.pb200_segment_read_index(self.ctx.handle, dev, ci, w, _ptr(out), int(n))
            if r < 0:
                _lib.check(int(r))
        return out

    def bind_domain(self, domain: "DictionaryDomain") -> None:
        """Re-encodes the domain's columns into table-wide ids (pb200h_segment_bind_domain): afterwards this segment can
        be merged with the other bound segments on the device and across GPUs, by value."""
        _lib.check(self.ctx.lib.pb200h_segment_bind_domain(self.ctx.handle, self.handle, domain.handle))

    def local_ids(self, column: str) -> np.ndarray:
        """Ids of `column` that occur in this segment (bound: domain ids; unbound: 0..cardinality-1)."""
        L = self.ctx.lib
        dev, ci = L.pb200h_segment_device(self.handle), self.column_index(column)
        n = L.pb200_segment_local_ids(dev, ci, None, 0)
        out = np.zeros(int(n), dtype=np.int32)
        L.pb200_segment_local_ids(dev, ci, _ptr(out), int(n))
        return out

    def device_bytes(self) -> int:
        return int(self.ctx.lib.pb200_segment_device_bytes(self.ctx.lib.pb200h_segment_device(self.handle)))

    def destroy(self):
        if self.handle:
            self.ctx.lib.pb200h_segment_destroy(self.handle)
            self.handle = None


class SegmentCache:
    """HBM residency manager (pb200h_cache_*): segments on the device keyed by (name, CRC), byte budget, LRU eviction of
    segments no query holds -- TableDataManager + SegmentDataManager reference counting for device memory."""

    def __init__(self, ctx: B200Context, max_device_bytes: int = 0):
        self.ctx = ctx
        h = C.c_void_p()
        _lib.check(ctx.lib.pb200h_cache_create(ctx.handle, int(max_device_bytes), C.byref(h)))
        self.handle = h

    def acquire(self, name: str, crc: int, index_dir: Optional[str] = None, size_hint: int = 0) -> IndexSegment:
        h = C.c_void_p()
        _lib.check(self.ctx.lib.pb200h_cache_acquire(self.handle, name.encode(), int(crc),
                                                     None if index_dir is None else index_dir.encode(), int(size_hint), C.byref(h)))
        return IndexSegment(self.ctx, h, name)   # owned by the cache: release() it, never destroy()

    def release(self, segment: IndexSegment) -> None:
        _lib.check(self.ctx.lib.pb200h_cache_release(self.handle, segment.handle))
        segment.handle = None

    def evict(self, name: str, crc: int) -> None:
        _lib.check(self.ctx.lib.pb200h_cache_evict(self.handle, name.encode(), int(crc)))

    def stats(self) -> Dict[str, int]:
        out = (C.c_int64 * 6)()
        _lib.check(self.ctx.lib.pb200h_cache_stats(self.handle, out))
        return dict(zip(("segments", "bytes", "budget", "hits", "misses", "evictions"), [int(x) for x in out]))

    def close(self) -> None:
        if self.handle:
            self.ctx.lib.pb200h_cache_destroy(self.handle)
            self.handle = None


class DictionaryDomain:
    """Table-wide dictionaries (include/pinot_b200.h "domains"): the sorted union of per-segment dictionaries, the common
    id space that makes device-side and cross-GPU merges merges BY VALUE (GroupByCombineOperator.java:130-146)."""

    def __init__(self, ctx: B200Context, handle, columns: Sequence[str], column_ids: Sequence[int]):
        self.ctx, self.handle, self.columns, self.column_ids = ctx, handle, list(columns), list(column_ids)

    @classmethod
    def build(cls, ctx: B200Context, segments: Sequence[IndexSegment], columns: Sequence[str]) -> "DictionaryDomain":
        """Union over the given (still unbound) segments' own dictionaries."""
        names = (C.c_char_p * len(columns))(*[c.encode() for c in columns])
        segs = (C.c_void_p * len(segments))(*[s.handle for s in segments])
        h = C.c_void_p()
        _lib.check(ctx.lib.pb200h_domain_build(ctx.handle, segs, len(segments), len(columns), names, C.byref(h)))
        return cls(ctx, h, columns, [segments[0].column_index(c) for c in columns])

    @classmethod
    def from_dictionaries(cls, ctx: B200Context, columns: Sequence[str], column_ids: Sequence[int],
                          stored_types: Sequence[int], parts: Sequence[Sequence[np.ndarray]],
                          entry_bytes: Optional[Sequence[Sequence[int]]] = None) -> "DictionaryDomain":
        """parts[k] = the sorted dictionaries (Pinot's big-endian bytes, uint8 arrays) to union for column k -- e.g. the
        rank-local unions gathered from all GPUs."""
        arr = (_lib.DomainCol * len(columns))()
        keep = []
        for k in range(len(columns)):
            width = 8 if stored_types[k] in (_lib.LONG, _lib.DOUBLE) else 4
            ptrs = (C.c_void_p * len(parts[k]))(*[p.ctypes.data for p in parts[k]])
            if stored_types[k] == _lib.STRING:
                eb = (C.c_int32 * len(parts[k]))(*entry_bytes[k])
                cards = (C.c_int32 * len(parts[k]))(*[len(p) // w for p, w in zip(parts[k], entry_bytes[k])])
            else:
                eb = None
                cards = (C.c_int32 * len(parts[k]))(*[len(p) // width for p in parts[k]])
            keep.append((ptrs, cards, eb))
            arr[k] = _lib.DomainCol(column_ids[k], stored_types[k], len(parts[k]), 0, ptrs, cards, eb)
        h = C.c_void_p()
        _lib.check(ctx.lib.pb200_domain_create(ctx.handle, len(columns), arr, C.byref(h)))
        return cls(ctx, h, columns, column_ids)

    def info(self, column: str) -> Dict[str, int]:
        out = (C.c_int64 * 4)()
        _lib.check(self.ctx.lib.pb200_domain_column_info(self.handle, self.column_ids[self.columns.index(column)], out))
        return dict(zip(("stored_type", "cardinality", "bits", "entry_bytes"), [int(x) for x in out]))

    def dictionary_bytes(self, column: str) -> np.ndarray:
        """The domain dictionary in Pinot's dictionary-file encoding (big-endian sorted values / padded strings)."""
        ci = self.column_ids[self.columns.index(column)]
        n = self.ctx.lib.pb200_domain_dictionary(self.handle, ci, None, 0)
        if n < 0:
            _lib.check(int(n))
        out = np.zeros(int(n), dtype=np.uint8)
        self.ctx.lib.pb200_domain_dictionary(self.handle, ci, _ptr(out), int(n))
        return out

    def release(self):
        if self.handle:
            self.ctx.lib.pb200_domain_release(self.ctx.handle, self.handle)
            self.handle = None


@dataclass
class ExecutionStatistics:
    """core/operator/ExecutionStatistics.java"""
    num_docs_scanned: int
    num_entries_scanned_in_filter: int
    num_entries_scanned_post_filter: int
    num_total_docs: int


@dataclass
class ResultsBlock:
    """What an AggregationResultsBlock / GroupByResultsBlock is built from (intermediate results, dictId keys)."""
    num_groups: int  # -1: aggregation only
    regime: str
    groups_limit_reached: bool
    stats: ExecutionStatistics
    keys: np.ndarray  # [G, k] dictIds
    doubles: List[np.ndarray]
    longs: List[np.ndarray]
    dict_ids: List[np.ndarray]
    distinct: Dict[Tuple[int, int], np.ndarray] = field(default_factory=dict)
    device_ms: float = 0.0
    operator_kind: str = "AGGREGATION"
    handle: Optional[C.c_void_p] = None  # kept only for merged results (multi-GPU combine)
    count_carrier: bool = False  # the per-group row counts rode in an INT sum's reductions (pb200_plan.cpp)
    carrier_unsafe: bool = False  # deferred result: that sum may overflow in the cross-GPU reduce, rerun without carrier
    flag_slot: bool = False  # the int64 table block ends with this rank's unsafe verdict: all-reduce it with the tables

    def release(self, ctx: "B200Context") -> None:
        """Frees the native result of a block executed with keep_handle=True (or views=True: the arrays die with it)."""
        native = getattr(self, "_native", None)
        if native is not None:
            native.free()
            self.handle = None
            return
        if self.handle is not None:
            ctx.lib.pb200_result_free(self.handle)
            self.handle = None

    def get_results(self, query: QueryContext) -> List[object]:
        """AggregationResultsBlock.getResults(): Long for COUNT, Double for SUM/MIN/MAX, (sum, count) for AVG,
        set size for DISTINCTCOUNT -- row 0 (aggregation only)."""
        out = []
        for a, agg in enumerate(query.aggregations):
            if agg.function == "COUNT":
                out.append(int(self.longs[a][0]))
            elif agg.function == "AVG":
                out.append((float(self.doubles[a][0]), int(self.longs[a][0])))
            elif agg.function == "DISTINCTCOUNT":
                out.append(int(self.longs[a][0]))
            else:
                out.append(float(self.doubles[a][0]))
        return out


INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1


def numeric_literal(v) -> Tuple[int, float]:
    """(i, d) of pb200h_literal for a number: d = the literal rounded to double, i = the literal when it is an int64 (so
    (double)i == d), else 0 -- the host then compares INT / LONG values with the fraction `d` or knows the literal lies
    beyond int64 (a ctypes int64 field would wrap it silently)."""
    if isinstance(v, (int, np.integer)):
        v = int(v)
        try:
            d = float(v)
        except OverflowError:
            d = math.copysign(math.inf, v)
        return (v if INT64_MIN <= v <= INT64_MAX else 0), d
    d = float(v)
    return (int(d) if d.is_integer() and INT64_MIN <= d < 2.0 ** 63 else 0), d


def _marshal_query(q: QueryContext, merge: bool, reduce_world: int = 0, no_count_carrier: bool = False,
                   merged_docs_bound: int = 0):
    nodes = postfix(q.filter)
    keep: List[bytes] = []
    lits: List[_lib.HLiteral] = []

    def lit(v):
        if isinstance(v, str):
            b = v.encode("utf-8")
            keep.append(b)
            return _lib.HLiteral(0, 0.0, b)
        if isinstance(v, bytes):
            keep.append(v)
            return _lib.HLiteral(0, 0.0, v)
        return _lib.HLiteral(*numeric_literal(v), None)

    def encode(node_list):
        out = []
        for n in node_list:
            if isinstance(n, Filter):
                out.append(_lib.HFilterNode(_lib.FILTER_CODES[n.type], None, len(n.children), 0, 0, 0, 0, 0, 0))
                continue
            cname = n.column.encode()
            keep.append(cname)
            off = len(lits)
            if n.type == "RANGE":
                lits.append(lit(n.lower if n.lower is not None else 0))
                lits.append(lit(n.upper if n.upper is not None else 0))
                out.append(_lib.HFilterNode(_lib.FILTER_CODES["RANGE"], cname, 0, int(n.lower_inclusive),
                                            int(n.upper_inclusive), int(n.lower is None), int(n.upper is None), 2, off))
            else:
                for v in n.values:
                    lits.append(lit(v))
                out.append(_lib.HFilterNode(_lib.FILTER_CODES[n.type], cname, 0, 0, 0, 0, 0, len(n.values), off))
        return out
    enc = encode(nodes)
    c_nodes = (_lib.HFilterNode * max(1, len(enc)))(*enc)
    # FILTER (WHERE ...) clauses: one postfix tree per DISTINCT clause, concatenated (pb200h_query.agg_filter_*)
    agg_nodes, starts, counts, seen = [], [], [], {}
    for a in q.aggregations:
        f = getattr(a, "filter", None)
        if f is None:
            starts.append(0)
            counts.append(0)
            continue
        key = repr(f)
        if key not in seen:
            e = encode(postfix(f))
            seen[key] = (len(agg_nodes), len(e))
            agg_nodes += e
        starts.append(seen[key][0])
        counts.append(seen[key][1])
    c_agg_nodes = (_lib.HFilterNode * max(1, len(agg_nodes)))(*agg_nodes)
    c_starts = (C.c_int32 * max(1, len(starts)))(*starts)
    c_counts = (C.c_int32 * max(1, len(counts)))(*counts)
    c_lits = (_lib.HLiteral * max(1, len(lits)))(*lits)
    gb_names = [c.encode() for c in q.group_by]
    gb = (C.c_char_p * max(1, len(gb_names)))(*gb_names)
    aggs = (_lib.HAgg * max(1, len(q.aggregations)))()
    for i, a in enumerate(q.aggregations):
        nm = None if a.column is None else a.column.encode()
        keep.append(nm)
        aggs[i] = _lib.HAgg(_lib.AGG_CODES[a.function], nm)
    hq = _lib.HQuery(len(nodes), c_nodes, c_lits, len(q.group_by), gb, len(q.aggregations), aggs, q.num_groups_limit,
                     q.max_initial_result_holder_capacity, int(merge), int(not getattr(q, "use_star_tree", True)),
                     int(reduce_world), int(no_count_carrier), int(merged_docs_bound),
                     c_agg_nodes if agg_nodes else None, c_starts if agg_nodes else None, c_counts if agg_nodes else None)
    return hq, (c_nodes, c_lits, gb, gb_names, aggs, keep, c_agg_nodes, c_starts, c_counts)


def order_spec(q: QueryContext, merge: bool):
    """pb200_order_by of a GROUP BY query with an ORDER BY (None otherwise).  Trim: max(5 * LIMIT, option) rows when the
    option (min_server_group_trim_size for a merged result, min_segment_group_trim_size per segment) is > 0, else sorted
    without trimming -- Pinot's table capacity rule for the combine step."""
    from .sql import resolve_order_by
    if not q.is_group_by or not q.order_by:
        return None
    items = resolve_order_by(q)
    if len(items) > _lib.MAX_ORDER_BY:
        raise ValueError(f"ORDER BY has {len(items)} items, at most {_lib.MAX_ORDER_BY} are supported")
    option = q.min_server_group_trim_size if merge else q.min_segment_group_trim_size
    spec = _lib.OrderBy(len(items), max(5 * q.limit, option) if option > 0 else 0)
    for i, (kind, index, asc) in enumerate(items):
        spec.items[i] = _lib.OrderItem(_lib.ORDER_GROUP_BY if kind == "GROUP_BY" else _lib.ORDER_AGG, index, int(not asc))
    return spec


class _NativeResult:
    """Owner of a native pb200_result whose columns numpy arrays alias (views=True): freed with the block (or release())."""

    def __init__(self, lib, handle):
        self.lib, self.handle = lib, handle

    def free(self):
        if self.handle is not None:
            self.lib.pb200_result_free(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def _read_views(ctx: B200Context, handle, q: QueryContext, meta):
    """Zero-copy face (pb200_result_columns): numpy arrays over the pinned block the device extracted the groups into --
    what a JVM does with NewDirectByteBuffer.  Absent columns are read-only broadcast constants."""
    g = meta.num_groups
    rows = 1 if g < 0 else g
    k, na = len(q.group_by), len(q.aggregations)
    kp = C.c_void_p()
    dp, lp, ip = (C.c_void_p * na)(), (C.c_void_p * na)(), (C.c_void_p * na)()
    _lib.check(ctx.lib.pb200_result_columns(handle, C.byref(kp), dp, lp, ip))

    def wrap(ptr, n, ctype, dtype, neutral):
        if not ptr or n == 0:
            return np.broadcast_to(np.asarray(neutral, dtype=dtype), (n,))
        return np.frombuffer((ctype * n).from_address(ptr), dtype=dtype)
    keys = (wrap(kp.value, max(g, 0) * k, C.c_int32, np.int32, 0).reshape(max(g, 0), k) if (g > 0 and k > 0 and kp.value)
            else np.zeros((max(g, 0), k), dtype=np.int32))
    doubles = [wrap(dp[a], rows, C.c_double, np.float64, 0.0) for a in range(na)]
    longs = [wrap(lp[a], rows, C.c_int64, np.int64, 0) for a in range(na)]
    ids = [wrap(ip[a], rows, C.c_int32, np.int32, -1) for a in range(na)]
    return keys, doubles, longs, ids


def _read_result(ctx: B200Context, handle, q: QueryContext, kind: int, keep_handle: bool, views: bool = False) -> ResultsBlock:
    L = ctx.lib
    meta = _lib.ResultMeta()
    _lib.check(L.pb200_result_meta_get(handle, C.byref(meta)))
    g = meta.num_groups
    rows = 1 if g < 0 else g
    k = len(q.group_by)
    if views and not any(a.function == "DISTINCTCOUNT" for a in q.aggregations):
        keys, doubles, longs, ids = _read_views(ctx, handle, q, meta)
        stats = ExecutionStatistics(meta.num_docs_scanned, meta.num_entries_scanned_in_filter,
                                    meta.num_entries_scanned_post_filter, meta.num_total_docs)
        block = ResultsBlock(g, _lib.REGIMES[meta.regime], bool(meta.groups_limit_reached), stats, keys, doubles, longs,
                             ids, {}, meta.device_ms, _lib.OPERATOR_KINDS.get(kind, "AGGREGATION"))
        block.count_carrier = bool(meta.reserved & 1)
        block.carrier_unsafe = bool(meta.reserved & 2)
        block.flag_slot = bool(meta.reserved & 4)
        block._native = _NativeResult(L, handle)   # the arrays alias the result's pinned block: it lives as long as the block
        if keep_handle:
            block.handle = handle
        return block
    keys = np.zeros((max(g, 0), k), dtype=np.int32)
    na = len(q.aggregations)
    d_all = np.zeros((na, rows), dtype=np.float64)
    l_all = np.zeros((na, rows), dtype=np.int64)
    i_all = np.full((na, rows), -1, dtype=np.int32)
    if rows:  # one ABI round trip for keys and all intermediates
        _lib.check(L.pb200_result_fetch(handle, _ptr(keys) if (g > 0 and k > 0) else None, _ptr(d_all), _ptr(l_all), _ptr(i_all)))
    doubles, longs, ids, distinct = list(d_all), list(l_all), list(i_all), {}
    for a, agg in enumerate(q.aggregations):
        if agg.function == "DISTINCTCOUNT":
            for row in range(rows):
                buf = np.zeros(int(l_all[a][row]), dtype=np.int32)
                n = L.pb200_result_distinct(handle, a, row, _ptr(buf), len(buf))
                if n < 0:
                    _lib.check(int(n))
                distinct[(a, row)] = buf
    stats = ExecutionStatistics(meta.num_docs_scanned, meta.num_entries_scanned_in_filter,
                                meta.num_entries_scanned_post_filter, meta.num_total_docs)
    block = ResultsBlock(g, _lib.REGIMES[meta.regime], bool(meta.groups_limit_reached), stats, keys, doubles, longs,
                         ids, distinct, meta.device_ms, _lib.OPERATOR_KINDS.get(kind, "AGGREGATION"))
    block.count_carrier = bool(meta.reserved & 1)
    block.carrier_unsafe = bool(meta.reserved & 2)
    block.flag_slot = bool(meta.reserved & 4)
    if keep_handle:
        block.handle = handle
    else:
        L.pb200_result_free(handle)
    return block


class Operator:
    """GroupByOperator / AggregationOperator stand-in: next_block() may be called once."""

    def __init__(self, plan_maker: "B200PlanMaker", segment: IndexSegment, query: QueryContext):
        self._pm, self._segment, self._query = plan_maker, segment, query
        self._block: Optional[ResultsBlock] = None

    def next_block(self) -> ResultsBlock:
        if self._block is None:
            self._block = self._pm.execute_segments([self._segment], self._query)[0]
        return self._block

    def get_execution_statistics(self) -> ExecutionStatistics:
        return self.next_block().stats

    def get_index_segment(self) -> IndexSegment:
        return self._segment

    def to_explain_string(self) -> str:
        return self._pm.explain(self._segment, self._query)


class PlanNode:
    def __init__(self, plan_maker, segment, query):
        self._args = (plan_maker, segment, query)

    def run(self) -> Operator:
        return Operator(*self._args)


class B200PlanMaker:
    """``PlanMaker`` for this path (core/plan/maker/PlanMaker.java:37-67)."""

    def __init__(self, ctx: B200Context):
        self.ctx = ctx
        self.last_device_ms = 0.0  # CUDA-event time of the scan kernel(s) of the latest execute_segments call

    def make_segment_plan_node(self, segment: IndexSegment, query: QueryContext) -> PlanNode:
        return PlanNode(self, segment, query)

    def explain(self, segment: IndexSegment, query: QueryContext) -> str:
        hq, _keep = _marshal_query(query, False)
        buf = C.create_string_buffer(8192)
        n = self.ctx.lib.pb200h_explain(self.ctx.handle, C.byref(hq), segment.handle, buf, 8192)
        if n < 0:
            _lib.check(n)
        return buf.value.decode()

    def to_datatable(self, segment: IndexSegment, query: QueryContext, block: "ResultsBlock") -> bytes:
        """DataTableImplV4 bytes of a results block that still owns its handle (execute_segments(..., keep_handle=True) /
        finalized merged block): what the server would send to the broker for these rows."""
        if block.handle is None:
            raise ValueError("the block's native handle was released (execute with keep_handle=True)")
        hq, _keep = _marshal_query(query, False)
        L = self.ctx.lib
        n = L.pb200h_result_to_datatable(C.byref(hq), segment.handle, block.handle, None, 0)
        if n < 0:
            _lib.check(int(n))
        buf = C.create_string_buffer(int(n))
        r = L.pb200h_result_to_datatable(C.byref(hq), segment.handle, block.handle, buf, int(n))
        if r < 0:
            _lib.check(int(r))
        return buf.raw[: int(r)]

    def execute_segments(self, segments: Sequence[IndexSegment], query: QueryContext, merge: bool = False,
                         keep_handle: bool = False, reduce_world: int = 0, merged_docs_bound: int = 0,
                         no_count_carrier: bool = False, defer: Optional[bool] = None, views: bool = False,
                         ordered: bool = True) -> List[ResultsBlock]:
        """All segments of one query in ONE device submission (makeInstancePlan-level batching).  With merge=True the
        segments (sharing dictionaries) are combined on the device and one block is returned; with keep_handle=True as
        well, a group-by block comes back WITHOUT its groups extracted (PB200_Q_DEFER_FINALIZE): its dense device tables
        are meant to be reduced across GPUs (pinot_b200.distributed.combine_across_ranks), which extracts on the root.
        A GROUP BY query with an ORDER BY gets its rows ordered and trimmed by the library (order_spec; a deferred block
        when it is extracted); ordered=False returns every group in the library's row order."""
        # merge + keep_handle: the caller reduces the dense tables across GPUs first; groups are extracted afterwards
        # defer=False with keep_handle=True: extracted blocks that keep their native handle (to_datatable); release() them
        if defer is None:
            defer = merge and keep_handle and query.is_group_by
        # the marshalled (ctypes) form of a query is cached on the query object: a server compiles a query once and runs it
        # over many segments / steps
        mkey = (2 if defer else int(merge), int(reduce_world), bool(no_count_carrier), int(merged_docs_bound))
        cache = query.__dict__.setdefault("_pb200_marshalled", {})
        if mkey not in cache:
            cache[mkey] = _marshal_query(query, 2 if defer else merge, reduce_world, no_count_carrier, merged_docs_bound)
        hq, _keep = cache[mkey]
        n = len(segments)
        segs = (C.c_void_p * n)(*[s.handle for s in segments])
        nres = 1 if merge else n
        res = (C.c_void_p * nres)()
        kinds = (C.c_int32 * n)()
        spec = order_spec(query, merge) if ordered else None
        if spec is None:
            _lib.check(self.ctx.lib.pb200h_execute(self.ctx.handle, C.byref(hq), segs, n, res, kinds))
        else:
            _lib.check(self.ctx.lib.pb200h_execute_ordered(self.ctx.handle, C.byref(hq), C.byref(spec), segs, n, res, kinds))
        # views=True: the blocks' arrays alias the native results' pinned memory (no copy); keep the block alive while you
        # use them and drop it before the context closes
        blocks = [_read_result(self.ctx, C.c_void_p(res[i]), query, kinds[i if not merge else 0], keep_handle, views)
                  for i in range(nres)]
        self.last_device_ms = blocks[0].device_ms
        return blocks
