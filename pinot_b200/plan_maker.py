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
import json
import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from ._lib import UnsupportedQueryError  # noqa: F401  (re-export)
from .query import DISTINCT_SET_FUNCTIONS, MOMENT_FUNCTIONS, WITHTIME_FUNCTIONS, WITHTIME_TYPES, functions_where, Filter, Moments, QueryContext, postfix


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


def star_tree_config(dimensions: Sequence[str], function_pairs: Sequence[tuple], max_leaf_records: int = 10000,
                     skip_star_for: Sequence[str] = ()):
    """(pb200h_startree_config, the objects it points into).  Functions are upper-cased; one the library has no code
    for is passed as -1, which the library refuses as unsupported."""
    dims = [d.encode() for d in dimensions]
    skip = [d.encode() for d in skip_star_for]
    pairs = (_lib.HAgg * max(len(function_pairs), 1))()
    names = []
    for i, (fn, col) in enumerate(function_pairs):
        names.append(None if col is None else str(col).encode())
        pairs[i] = _lib.HAgg(_lib.AGG_CODES.get(str(fn).upper(), -1), names[-1])
    dim_arr = (C.c_char_p * max(len(dims), 1))(*dims)
    skip_arr = (C.c_char_p * max(len(skip), 1))(*skip)
    cfg = _lib.HStarTreeConfig(len(dims), dim_arr, len(skip), skip_arr if skip else None, len(function_pairs), pairs,
                               int(max_leaf_records))
    return cfg, (dims, skip, names, pairs, dim_arr, skip_arr)


def parse_star_tree_config(config) -> Dict[str, object]:
    """One StarTreeIndexConfig of a table config (JSON text or a dict) -> the keyword arguments of
    IndexSegment.build_star_tree.  Pairs come from "functionColumnPairs" ("SUM__m", "COUNT__*") and
    "aggregationConfigs" ([{"columnName": "m", "aggregationFunction": "SUM"}]); "maxLeafRecords" defaults to 10000."""
    if isinstance(config, str):
        try:
            config = json.loads(config)
        except json.JSONDecodeError as e:
            raise ValueError(f"star-tree config is not JSON: {e}") from None
    if not isinstance(config, dict):
        raise ValueError("star-tree config must be a JSON object")
    dims = config.get("dimensionsSplitOrder")
    if not isinstance(dims, list) or not dims or not all(isinstance(d, str) for d in dims):
        raise ValueError("star-tree config: dimensionsSplitOrder must be a non-empty list of column names")
    skip = config.get("skipStarNodeCreationForDimensions") or []
    if not isinstance(skip, list) or not all(isinstance(d, str) for d in skip):
        raise ValueError("star-tree config: skipStarNodeCreationForDimensions must be a list of column names")
    pairs = []
    for p in config.get("functionColumnPairs") or []:
        if not isinstance(p, str) or "__" not in p:
            raise ValueError(f"star-tree config: function-column pair {p!r} is not FUNCTION__column")
        fn, col = p.split("__", 1)
        pairs.append((fn.upper(), None if col == "*" else col))
    for a in config.get("aggregationConfigs") or []:
        if not isinstance(a, dict) or "aggregationFunction" not in a or "columnName" not in a:
            raise ValueError(f"star-tree config: aggregation config {a!r} needs columnName and aggregationFunction")
        pairs.append((str(a["aggregationFunction"]).upper(), None if a["columnName"] == "*" else a["columnName"]))
    if not pairs:
        raise ValueError("star-tree config: no functionColumnPairs / aggregationConfigs")
    leaf = config.get("maxLeafRecords", 10000)
    if not isinstance(leaf, int) or isinstance(leaf, bool):
        raise ValueError("star-tree config: maxLeafRecords must be an integer")
    return {"dimensions": dims, "function_pairs": list(dict.fromkeys(pairs)), "max_leaf_records": leaf,
            "skip_star_for": skip}


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

    def build_star_tree(self, dimensions: Sequence[str], function_pairs: Sequence[tuple], max_leaf_records: int = 10000,
                        skip_star_for: Sequence[str] = ()) -> Dict[str, object]:
        """Builds one star-tree of this segment on the device (pb200h_startree_build) and attaches it: `dimensions` =
        dimensionsSplitOrder, `function_pairs` = [(function, column)] with COUNT's column None or "*".  Returns the star
        docs, base docs and nodes of the tree and the milliseconds of each build phase."""
        cfg, _keep = star_tree_config(dimensions, function_pairs, max_leaf_records, skip_star_for)
        info = _lib.HStarTreeBuildInfo()
        _lib.check(self.ctx.lib.pb200h_startree_build(self.ctx.handle, self.handle, C.byref(cfg), C.byref(info)))
        return {"num_star_docs": int(info.num_star_docs), "num_base_docs": int(info.num_base_docs),
                "num_nodes": int(info.num_nodes), "phase_ms": dict(zip(_lib.STAR_BUILD_PHASES, list(info.phase_ms)))}

    def num_star_trees(self) -> int:
        """Star-trees of this segment, built or attached."""
        n = 0
        while self.ctx.lib.pb200h_startree_get(self.handle, n, None, None, None) == _lib.PB200_OK:
            n += 1
        return n

    def read_star_tree(self, index: int) -> Dict[str, object]:
        """The index-th star-tree, built or attached, read back: the OffHeapStarTree bytes, and per column of its star
        docs (dimensions: dictIds of the base dictionaries; count__*: int64; sum__m / min__m / max__m: float64) the
        values of every star doc."""
        L = self.ctx.lib
        tree, size, docs = C.c_void_p(), C.c_uint64(), C.c_void_p()
        _lib.check(L.pb200h_startree_get(self.handle, index, C.byref(tree), C.byref(size), C.byref(docs)))
        out = {"tree": np.ctypeslib.as_array(C.cast(tree, C.POINTER(C.c_uint8)), shape=(size.value,)).copy(), "columns": {}}
        seg = IndexSegment(self.ctx, docs, self.name + "$startree")  # owned by this segment: never destroyed here
        out["num_docs"] = seg.num_docs
        num_dims = int(np.frombuffer(out["tree"][16:20].tobytes(), dtype="<i4")[0])  # columns: dimensions, then metrics
        for i, name in enumerate(seg.column_names):
            info = seg.column_info(name)
            fwd = seg.read_index(name, "fwd")
            n, bits = seg.num_docs, info["bits"]
            bitstream = np.unpackbits(fwd)[: n * bits].reshape(n, bits).astype(np.int64)
            ids = bitstream @ (1 << np.arange(bits - 1, -1, -1, dtype=np.int64))
            if i >= num_dims:
                dtype = ">i8" if info["data_type"] == _lib.LONG else ">f8"
                out["columns"][name] = np.frombuffer(seg.read_index(name, "dict").tobytes(), dtype=dtype).astype(dtype[1:])[ids]
            else:
                out["columns"][name] = ids.astype(np.int32)
        return out

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

    def derive(self, expression: str) -> int:
        """Derives the column of a single-column expression (pb200h_segment_derive; a no-op when it exists) and returns
        its column id.  Queries derive the expressions they name by themselves; this does it ahead of them."""
        col = C.c_int32()
        _lib.check(self.ctx.lib.pb200h_segment_derive(self.ctx.handle, self.handle, expression.encode(), C.byref(col)))
        return col.value

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
    # PERCENTILE of per-segment results: (agg, row) -> (dictIds ascending, counts) of the row's non-zero histogram bins,
    # the intermediate a by-value merge adds up (cli.merge_blocks)
    histograms: Dict[Tuple[int, int], Tuple[np.ndarray, np.ndarray]] = field(default_factory=dict)
    # VAR / STDDEV: (agg, row) -> the row's exact Moments (pb200_result_moments), what a by-value merge adds up
    moments: Dict[Tuple[int, int], Moments] = field(default_factory=dict)

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

    def withtime(self, a: int, row: int, segment: "IndexSegment", column: str):
        """FIRST/LASTWITHTIME aggregation `a` in row `row`: (time value, data value) of the winning row, or None when the
        row has no matched doc.  The data value is looked up exactly through its dictId in `segment`'s dictionary of
        `column` (the block's segment; for a merged block any of its bound segments): STRING values and LONG values
        beyond 2^53 come back as stored."""
        d = int(self.dict_ids[a][row])
        return None if d < 0 else (int(self.longs[a][row]), segment.dictionary_value(column, d))

    def get_results(self, query: QueryContext, segment: Optional["IndexSegment"] = None) -> List[object]:
        """AggregationResultsBlock.getResults(): Long for COUNT, Double for SUM/MIN/MAX/PERCENTILE, (sum, count) for AVG,
        set size for DISTINCTCOUNT -- row 0 (aggregation only).  FIRST/LASTWITHTIME: with `segment` (the block's), the
        data value as stored (STRING included), -inf without a matched doc; without it the double column, which holds
        the dictId for a STRING column."""
        out = []
        for a, agg in enumerate(query.aggregations):
            if agg.function in WITHTIME_FUNCTIONS and segment is not None:
                v = self.withtime(a, 0, segment, agg.column)
                out.append(float("-inf") if v is None else v[1])
            elif agg.function == "COUNT":
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
    programs = 0   # a POST item names the next program of post_spec
    for i, (kind, index, asc) in enumerate(items):
        if kind == "POST":
            spec.items[i] = _lib.OrderItem(_lib.ORDER_POST, programs, int(not asc))
            programs += 1
            continue
        spec.items[i] = _lib.OrderItem(_lib.ORDER_GROUP_BY if kind == "GROUP_BY" else _lib.ORDER_AGG, index, int(not asc))
    return spec


def post_spec(q: QueryContext):
    """pb200_post_aggs of a GROUP BY query whose ORDER BY names post-aggregation expressions (None otherwise): their
    programs, in the order of those items (order_spec's POST items index it).  Expressions only in the SELECT list stay
    here: the caller computes them from the final values."""
    from .sql import resolve_order_by
    if not q.is_group_by or not q.order_by:
        return None
    programs = [q.post_aggregations[index].program for kind, index, _ in resolve_order_by(q) if kind == "POST"]
    if not programs:
        return None
    spec = _lib.PostAggs(len(programs), 0)
    for i, program in enumerate(programs):
        spec.programs[i].num_nodes = len(program)
        for j, n in enumerate(program):
            spec.programs[i].nodes[j] = _lib.PostNode(_lib.POST_CODES[n[0]], n[1] if n[0] == "AGG" else 0,
                                                      n[1] if n[0] == "LIT" else 0.0)
    return spec


def having_spec(q: QueryContext):
    """pb200_having of a query with HAVING (None otherwise): sql.resolve_having's postfix nodes as the C struct."""
    from .sql import resolve_having
    nodes = resolve_having(q)
    if not nodes:
        return None
    spec = _lib.Having(len(nodes), 0)
    for i, n in enumerate(nodes):
        op = _lib.HAVING_CODES[n[0]]
        if n[0] in ("AND", "OR"):
            spec.nodes[i] = _lib.HavingNode(op, n[1], 0, 0, 0.0, 0.0)
        elif n[0] == "NOT":
            spec.nodes[i] = _lib.HavingNode(op, 1, 0, 0, 0.0, 0.0)
        elif n[0] in ("EQ", "NEQ"):
            spec.nodes[i] = _lib.HavingNode(op, 0, n[1], 0, n[2], 0.0)
        else:
            _, a, lo, hi, lo_inc, hi_inc = n
            flags = ((_lib.HAVING_LO_UNBOUNDED if lo is None else 0) | (_lib.HAVING_HI_UNBOUNDED if hi is None else 0) |
                     (0 if lo_inc else _lib.HAVING_LO_EXCLUSIVE) | (0 if hi_inc else _lib.HAVING_HI_EXCLUSIVE))
            spec.nodes[i] = _lib.HavingNode(op, 0, a, flags, 0.0 if lo is None else lo, 0.0 if hi is None else hi)
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


def _read_result(ctx: B200Context, handle, q: QueryContext, kind: int, keep_handle: bool, views: bool = False,
                 histograms: bool = False) -> ResultsBlock:
    # histograms=True (per-segment blocks, the intermediates of a by-value merge): also PERCENTILE histograms, moments and
    # DISTINCTCOUNTHLL sets; otherwise a DISTINCTCOUNTHLL's set is never read, so the library never decodes it
    L = ctx.lib
    meta = _lib.ResultMeta()
    _lib.check(L.pb200_result_meta_get(handle, C.byref(meta)))
    g = meta.num_groups
    rows = 1 if g < 0 else g
    k = len(q.group_by)
    if views and not any(a.function in DISTINCT_SET_FUNCTIONS + ("PERCENTILE",) + MOMENT_FUNCTIONS or (a.function == "DISTINCTCOUNTHLL" and histograms)
                         for a in q.aggregations):
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
        if agg.function in DISTINCT_SET_FUNCTIONS:
            for row in range(rows):
                buf = np.zeros(int(l_all[a][row]), dtype=np.int32)
                n = L.pb200_result_distinct(handle, a, row, _ptr(buf), len(buf))
                if n < 0:
                    _lib.check(int(n))
                distinct[(a, row)] = buf
        elif agg.function == "DISTINCTCOUNTHLL" and histograms:   # its long column is the estimate: ask for the size
            for row in range(rows):
                n = L.pb200_result_distinct(handle, a, row, None, 0)
                if n < 0:
                    _lib.check(int(n))
                buf = np.zeros(int(n), dtype=np.int32)
                _lib.check(min(0, int(L.pb200_result_distinct(handle, a, row, _ptr(buf), len(buf)))))
                distinct[(a, row)] = buf
    hists = {}
    for a, agg in enumerate(q.aggregations):
        if agg.function == "PERCENTILE" and histograms:
            for row in range(rows):
                n = L.pb200_result_histogram(handle, a, row, None, None, 0)
                if n < 0:
                    _lib.check(int(n))
                hid, hcnt = np.zeros(int(n), dtype=np.int32), np.zeros(int(n), dtype=np.int64)
                _lib.check(min(0, int(L.pb200_result_histogram(handle, a, row, _ptr(hid), _ptr(hcnt), int(n)))))
                hists[(a, row)] = (hid, hcnt)
    moments = {}
    for a, agg in enumerate(q.aggregations):
        if agg.function in MOMENT_FUNCTIONS and histograms:   # per-segment blocks: what a by-value merge adds up
            n, cm, s1, lo, hi = C.c_int64(), C.c_int64(), C.c_uint64(), C.c_uint64(), C.c_uint64()
            cx, e = C.c_int32(), C.c_int32()
            for row in range(rows):
                _lib.check(L.pb200_result_moments(handle, a, row, C.byref(n), C.byref(cm), C.byref(cx), C.byref(e),
                                                  C.byref(s1), C.byref(lo), C.byref(hi)))
                moments[(a, row)] = Moments(n.value, cm.value, cx.value, e.value, s1.value, (hi.value << 64) | lo.value)
    stats = ExecutionStatistics(meta.num_docs_scanned, meta.num_entries_scanned_in_filter,
                                meta.num_entries_scanned_post_filter, meta.num_total_docs)
    block = ResultsBlock(g, _lib.REGIMES[meta.regime], bool(meta.groups_limit_reached), stats, keys, doubles, longs,
                         ids, distinct, meta.device_ms, _lib.OPERATOR_KINDS.get(kind, "AGGREGATION"))
    block.histograms = hists
    block.moments = moments
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
                         ordered: bool = True, sets: bool = False) -> List[ResultsBlock]:
        """All segments of one query in ONE device submission (makeInstancePlan-level batching).  With merge=True the
        segments (sharing dictionaries) are combined on the device and one block is returned; with keep_handle=True as
        well, a group-by block comes back WITHOUT its groups extracted (PB200_Q_DEFER_FINALIZE): its dense device tables
        are meant to be reduced across GPUs (pinot_b200.distributed.combine_across_ranks), which extracts on the root.
        A GROUP BY query with an ORDER BY gets its rows ordered and trimmed by the library (order_spec, with post_spec's
        programs for expressions over aggregations; a deferred block when it is extracted); ordered=False returns every group in the library's row order.  A query with HAVING gets
        its rows filtered by the library before that order when the call's result is final (merge=True, or one segment,
        and ordered); per-segment blocks of several segments come back unfiltered, for the caller's merge to filter.
        Per-segment blocks carry the intermediates of a by-value merge (DISTINCTCOUNTHLL sets among them); sets=True
        reads those of a merged block too."""
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
        post = post_spec(query) if ordered else None
        having = having_spec(query) if ordered and (merge or n == 1) else None
        for a in query.aggregations:
            if a.function == "DISTINCTCOUNTHLL" and a.arg == 0:   # the library reads an argument of 0 as the default 8
                raise UnsupportedQueryError(_lib.E_UNSUPPORTED, "DISTINCTCOUNTHLL with log2m 0 is not accelerated")
        # one argument per aggregation: the percentile of a PERCENTILE, the log2m of a DISTINCTCOUNTHLL
        numeric = functions_where(lambda f: f.arg in ("percentile", "log2m"))
        pct = [a.function in numeric for a in query.aggregations]
        if post is not None or any(a.function in WITHTIME_FUNCTIONS for a in query.aggregations):
            # FIRST/LASTWITHTIME: the time column and the type literal travel beside the query (pb200h_execute_agg_args);
            # ORDER BY expressions over aggregations: their programs (pb200h_execute_post)
            args = (_lib.HAggArg * len(pct))(*[
                _lib.HAggArg(float(a.arg) if is_p else 0.0,
                             a.time_column.encode() if a.function in WITHTIME_FUNCTIONS else None,
                             WITHTIME_TYPES[a.value_type] if a.function in WITHTIME_FUNCTIONS else 0)
                for a, is_p in zip(query.aggregations, pct)])
            if post is not None:
                _lib.check(self.ctx.lib.pb200h_execute_post(self.ctx.handle, C.byref(hq), C.byref(spec), args,
                                                            C.byref(having) if having is not None else None, C.byref(post),
                                                            segs, n, res, kinds))
            else:
                _lib.check(self.ctx.lib.pb200h_execute_agg_args(self.ctx.handle, C.byref(hq), C.byref(spec) if spec is not None else None,
                                                                args, C.byref(having) if having is not None else None, segs, n, res, kinds))
        elif having is not None:
            args = (C.c_double * max(1, len(pct)))(*[float(a.arg) if is_p else 0.0 for a, is_p in zip(query.aggregations, pct)])
            _lib.check(self.ctx.lib.pb200h_execute_having(self.ctx.handle, C.byref(hq), C.byref(spec) if spec is not None else None,
                                                          args, C.byref(having), segs, n, res, kinds))
        elif any(pct):
            # one argument per aggregation: the percentile of each PERCENTILE (pb200h_execute_args)
            args = (C.c_double * len(pct))(*[float(a.arg) if is_p else 0.0 for a, is_p in zip(query.aggregations, pct)])
            _lib.check(self.ctx.lib.pb200h_execute_args(self.ctx.handle, C.byref(hq), C.byref(spec) if spec is not None else None,
                                                        args, segs, n, res, kinds))
        elif spec is None:
            _lib.check(self.ctx.lib.pb200h_execute(self.ctx.handle, C.byref(hq), segs, n, res, kinds))
        else:
            _lib.check(self.ctx.lib.pb200h_execute_ordered(self.ctx.handle, C.byref(hq), C.byref(spec), segs, n, res, kinds))
        # views=True: the blocks' arrays alias the native results' pinned memory (no copy); keep the block alive while you
        # use them and drop it before the context closes
        blocks = [_read_result(self.ctx, C.c_void_p(res[i]), query, kinds[i if not merge else 0], keep_handle, views,
                               histograms=not merge or sets) for i in range(nres)]
        self.last_device_ms = blocks[0].device_ms
        return blocks

    def execute_selection(self, segments: Sequence[IndexSegment], query, merge: bool = False):
        """A selection query (sql.SelectionQuery) over the segments in ONE device submission: per segment its first
        `limit` matching docs in doc order (merge=True: one block, segments taken in submission order), or with an ORDER BY
        its top `limit` rows by value, ties by doc id (merge=True: the tops merged by value, ties by (segment, doc id)).  Returns a list of
        SelectionResultsBlock, one per segment, or one block when merged."""
        columns = query.columns if query.columns is not None else sorted(segments[0].column_names)
        if len(query.order_by) > _lib.MAX_ORDER_BY:
            raise ValueError(f"ORDER BY has {len(query.order_by)} items, at most {_lib.MAX_ORDER_BY} are supported")
        hq, _keep = _marshal_query(QueryContext(aggregations=[], filter=query.filter), merge)
        names = [c.encode() for c in columns]
        cnames = (C.c_char_p * max(1, len(names)))(*names)
        onames = [c.encode() for c, _ in query.order_by]
        sel = _lib.HSelection(len(columns), cnames, len(onames))
        for k, (name, (_, asc)) in enumerate(zip(onames, query.order_by)):
            sel.order[k] = _lib.HSelectOrder(name, int(not asc))
        sel.limit = int(query.limit)
        n = len(segments)
        segs = (C.c_void_p * n)(*[s.handle for s in segments])
        nres = 1 if merge else n
        res = (C.c_void_p * nres)()
        _lib.check(self.ctx.lib.pb200h_execute_selection(self.ctx.handle, C.byref(hq), C.byref(sel), segs, n, res))
        blocks = [_read_selection(self.ctx, C.c_void_p(res[i]), segments, columns) for i in range(nres)]
        self.last_device_ms = blocks[0].device_ms
        return blocks[0] if merge else blocks

    def execute_distinct(self, segments: Sequence[IndexSegment], query, merge: bool = False):
        """A DISTINCT query (sql.DistinctQuery) over the segments in ONE device submission: per segment its first `limit`
        distinct tuples in order of first occurrence, or with an ORDER BY its top `limit` tuples, ties by first
        occurrence.  merge=True: one block over all segments (every DISTINCT column bound to one domain; otherwise
        UnsupportedQueryError) -- merge_distinct_blocks combines per-segment blocks by value instead.  Returns a list of
        DistinctResultsBlock, one per segment, or one block when merged."""
        columns = list(query.columns)
        if len(query.order_by) > _lib.MAX_ORDER_BY:
            raise ValueError(f"ORDER BY has {len(query.order_by)} items, at most {_lib.MAX_ORDER_BY} are supported")
        hq, _keep = _marshal_query(QueryContext(aggregations=[], filter=query.filter), merge)
        names = [c.encode() for c in columns]
        cnames = (C.c_char_p * max(1, len(names)))(*names)
        onames = [c.encode() for c, _ in query.order_by]
        sel = _lib.HSelection(len(columns), cnames, len(onames))
        for k, (name, (_, asc)) in enumerate(zip(onames, query.order_by)):
            sel.order[k] = _lib.HSelectOrder(name, int(not asc))
        sel.limit = int(query.limit)
        n = len(segments)
        segs = (C.c_void_p * n)(*[s.handle for s in segments])
        nres = 1 if merge else n
        res = (C.c_void_p * nres)()
        _lib.check(self.ctx.lib.pb200h_execute_distinct(self.ctx.handle, C.byref(hq), C.byref(sel), segs, n, res))
        blocks = [_read_selection(self.ctx, C.c_void_p(res[i]), segments, columns, DistinctResultsBlock) for i in range(nres)]
        self.last_device_ms = blocks[0].device_ms
        return blocks[0] if merge else blocks


@dataclass
class SelectionResultsBlock:
    """What a SelectionResultsBlock is built from: the selected columns' values per row (INT / LONG as int64, FLOAT /
    DOUBLE as float64, STRING as str), the doc id and the segment (index into the submitted segments) of every row."""
    names: List[str]
    columns: List[np.ndarray]
    doc_ids: np.ndarray
    segment_index: np.ndarray
    stats: ExecutionStatistics
    device_ms: float = 0.0

    @property
    def num_rows(self) -> int:
        return len(self.doc_ids)


@dataclass
class DistinctResultsBlock(SelectionResultsBlock):
    """What a DistinctResultsBlock is built from: one row per distinct tuple, values typed as in a selection, doc_ids /
    segment_index = the tuple's first occurrence."""


def merge_distinct_blocks(blocks: Sequence[SelectionResultsBlock], order_by=(), limit: int = 10) -> DistinctResultsBlock:
    """By-value merge of per-segment DISTINCT blocks of one submission (segment_index refers to that submission): the
    union of their tuples, each with its earliest (segment, doc) occurrence, ordered by first occurrence or by `order_by`
    ([(column, ascending)], ties by first occurrence), then the first `limit`.  Exact, because each segment's block holds
    its own first (or top) `limit` tuples.  Floats are tuples' members by identity (one NaN, -0.0 apart from 0.0) and
    order by Double.compare (query.value_key / value_order), as in the reference's DISTINCT table."""
    from .query import value_key, value_order
    names = list(blocks[0].names)
    first: Dict[tuple, tuple] = {}
    for b in blocks:
        for i in range(b.num_rows):
            key = tuple(value_key(c[i].item() if hasattr(c[i], "item") else c[i]) for c in b.columns)
            occ = (int(b.segment_index[i]), int(b.doc_ids[i]))
            if key not in first or occ < first[key]:
                first[key] = occ
    rows = sorted(first.items(), key=lambda kv: kv[1])
    for col, asc in reversed(list(order_by)):   # stable passes, last item first
        k = names.index(col)
        rows.sort(key=lambda kv: value_order(kv[0][k]), reverse=not asc)
    rows = rows[:limit]
    columns = []
    for k, c in enumerate(blocks[0].columns):
        vals = [kv[0][k] for kv in rows]
        columns.append(np.array(vals, dtype=object) if c.dtype == object else np.array(vals, dtype=c.dtype))
    stats = ExecutionStatistics(*(sum(getattr(b.stats, f) for b in blocks) for f in
                                  ("num_docs_scanned", "num_entries_scanned_in_filter", "num_entries_scanned_post_filter", "num_total_docs")))
    return DistinctResultsBlock(names, columns, np.array([kv[1][1] for kv in rows], dtype=np.int32),
                                np.array([kv[1][0] for kv in rows], dtype=np.int32), stats, sum(b.device_ms for b in blocks[:1]))


def _read_selection(ctx: B200Context, handle, segments: Sequence[IndexSegment], columns: Sequence[str],
                    block_class=SelectionResultsBlock) -> SelectionResultsBlock:
    L = ctx.lib
    try:
        meta = _lib.ResultMeta()
        _lib.check(L.pb200_result_meta_get(handle, C.byref(meta)))
        rows = C.c_int64()
        docs, segi = C.c_void_p(), C.c_void_p()
        cols = (C.c_void_p * max(1, len(columns)))()
        _lib.check(L.pb200_result_selection(handle, C.byref(rows), C.byref(docs), C.byref(segi), cols))
        n = int(rows.value)

        def copy(ptr, ctype, dtype):
            if n == 0 or not ptr:
                return np.zeros(0, dtype=dtype)
            return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ctype)), shape=(n,)).astype(dtype, copy=True)
        doc_ids = copy(docs.value, C.c_int32, np.int32)
        seg_index = copy(segi.value, C.c_int32, np.int32)
        out = []
        for k, name in enumerate(columns):
            info = segments[0].column_info(name)
            if info["data_type"] in (_lib.FLOAT, _lib.DOUBLE):
                out.append(copy(cols[k], C.c_double, np.float64))
            elif info["data_type"] == _lib.STRING:   # dictIds of the row's segment -> the dictionary's strings
                ids = copy(cols[k], C.c_int64, np.int64)
                cache: Dict[Tuple[int, int], str] = {}
                vals = np.empty(n, dtype=object)
                for i in range(n):
                    key = (int(seg_index[i]), int(ids[i]))
                    if key not in cache:
                        cache[key] = segments[key[0]].dictionary_value(name, key[1])
                    vals[i] = cache[key]
                out.append(vals)
            else:
                out.append(copy(cols[k], C.c_int64, np.int64))
        stats = ExecutionStatistics(meta.num_docs_scanned, meta.num_entries_scanned_in_filter,
                                    meta.num_entries_scanned_post_filter, meta.num_total_docs)
        return block_class(list(columns), out, doc_ids, seg_index, stats, float(meta.device_ms))
    finally:
        L.pb200_result_free(handle)
