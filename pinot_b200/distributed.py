"""Multi-GPU combine: one process per GPU, segments sharded whole, ONE reduce of the per-GPU group tables.

What this replaces in the reference: the JVM-side merge of per-segment results blocks in ``GroupByCombineOperator``
(``core/operator/combine/GroupByCombineOperator.java:102-165`` -> ``IndexedTable.upsert`` with
``AggregationFunction.merge``) and ``AggregationResultsBlockMerger`` (``.../merger/AggregationResultsBlockMerger.java:34-44``).

Segments are independent units (the reference already runs one task per segment), so the data path needs no
collective: every rank scans its own segments with ``PB200_Q_MERGE_SEGMENTS`` (device-side combine into one dense table
keyed by raw dictId key -- a merge by VALUE because the shards share dictionaries: synthetic tables by construction, real
ones after ``DictionaryDomain`` binding, see ``global_domain``) and the tables meet exactly once:

    kind      contents                               reduce op        merge() it equals
    i64       COUNT(*) per group + integer SUMs       SUM              Count/Sum/Avg merge (a + b)
    f64       FLOAT/DOUBLE/LONG SUMs                  SUM              Sum/Avg merge
    u32max    MAX as (dictId + 1), 0 = empty          MAX              MaxAggregationFunction.merge
    u32min    MIN as dictId, 0xFFFFFFFF = empty       MIN              MinAggregationFunction.merge

A raw INT column's MIN / MAX entries hold value ^ 0x80000000 (MAX without the + 1): 0 and 0xFFFFFFFF are INT_MIN and
INT_MAX there as well as "empty", and the group's count, seen flag, count carrier or hash key says whether it exists.
The empty values are still the neutral elements of MAX / MIN, so the reduce is the same for both kinds.

``torch.distributed`` (NCCL over NVLink / NVSwitch) is plumbing only: the tensors handed to it alias the library's own
device buffers (``pb200_result_device_buffers``), nothing is copied.  The tables are O(groups), not O(rows): the
exchange is latency-bound (C4: 100 000 groups x (8+8+4) B = 2 MB per rank).

The control flow (``execute_and_combine``) talks to the tables through a small backend interface so that the SAME code is
exercised by the world_size-2 gloo test on CPU (tests/test_distributed_cpu.py, tables built from the oracle), by 2 and 3
simulated ranks on one GPU (tests/test_gpu_combine_loopback.py, ``DeviceBackend`` over an in-process collective) and by
the NCCL test on two GPUs (tests/test_gpu_multi.py).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence

from .query import (DISTINCT_SET_FUNCTIONS, MOMENT_FUNCTIONS, WITHTIME_FUNCTIONS, HllSet, distinct_final, functions_where, hll_final,
                    is_multi_column_expression, value_key)

# functions whose per-rank intermediate is a set of domain ids, united on the host
_SET_FUNCTIONS = DISTINCT_SET_FUNCTIONS + functions_where(lambda f: f.family == "DISTINCTCOUNTHLL")


KINDS = {"i64": 0, "f64": 1, "u32max": 2, "u32min": 3}
_TORCH_DTYPES = {"i64": "int64", "f64": "float64", "u32max": "int32", "u32min": "int32"}


def shard_segments(num_segments: int, world_size: int, rank: int) -> List[int]:
    """Whole segments per rank, contiguous and balanced (64 segments over 8 GPUs -> 8 each)."""
    base, extra = divmod(num_segments, world_size)
    start = rank * base + min(rank, extra)
    return list(range(start, start + base + (1 if rank < extra else 0)))


def reduce_buffers(buffers: Dict[str, "torch.Tensor"], dist, dst: int = 0) -> None:
    """In-place reduce of the four table kinds to rank `dst` (works on CPU tensors with gloo and CUDA with nccl).

    The two u32 tables are carried by int32 tensors (torch has no uint32 collectives): the top bit is flipped before and
    after the MAX / MIN reduce so that the signed order equals the unsigned one.
    """
    import torch
    for kind, t in buffers.items():
        if t is None or t.numel() == 0:
            continue
        if kind in ("i64", "f64"):
            dist.reduce(t, dst=dst, op=dist.ReduceOp.SUM)
        elif kind in ("u32max", "u32min"):
            # unsigned order == signed order after flipping the top bit: reduce in place, no widened copy
            t.bitwise_xor_(-2147483648)
            dist.reduce(t, dst=dst, op=dist.ReduceOp.MAX if kind == "u32max" else dist.ReduceOp.MIN)
            t.bitwise_xor_(-2147483648)
        else:
            raise KeyError(kind)


class _DeviceArray:
    """Minimal __cuda_array_interface__ carrier so torch can alias a raw device pointer without copying."""

    def __init__(self, ptr: int, n: int, typestr: str):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 3}


def device_buffers(ctx, block) -> Dict[str, "torch.Tensor"]:
    """torch views over the dense group-table buffers of a merged results block (needs keep_handle=True)."""
    import torch
    out = {}
    if block.handle is None:
        raise ValueError("results block was not executed with merge=True, keep_handle=True")
    for kind, code in KINDS.items():
        p, n = C.c_void_p(), C.c_int64()
        rc = ctx.lib.pb200_result_device_buffers(block.handle, code, C.byref(p), C.byref(n))
        if rc != 0:
            from . import _lib
            _lib.check(rc)
        if not p.value or n.value == 0:
            out[kind] = None
            continue
        typestr = {"i64": "<i8", "f64": "<f8", "u32max": "<i4", "u32min": "<i4"}[kind]
        out[kind] = torch.as_tensor(_DeviceArray(p.value, n.value, typestr), device=f"cuda:{ctx.device}")
    return out


class DeviceBackend:
    """The tables of libpinot_b200.so results (the product path)."""

    def __init__(self, plan_maker, views: bool = False):
        self.pm = plan_maker
        self.ctx = plan_maker.ctx
        self.views = views   # results on the root alias the pinned block (plan_maker._read_views) instead of being copied

    @property
    def native(self) -> bool:
        """True once init_comm gave the context its own NCCL communicator: the reduce then runs INSIDE the library
        (pb200_result_combine: one NCCL group + verdict + extraction on the library's stream, no torch tensors)."""
        return getattr(self.ctx, "comm_world", 0) > 1

    def combine_native(self, block, query, dst: int):
        """-> (result or None, retry).  pb200_comm.cu."""
        from . import _lib
        from .plan_maker import _read_result
        retry = C.c_int32(0)
        _lib.check(self.ctx.lib.pb200_result_combine(self.ctx.handle, block.handle, dst, C.byref(retry)))
        if retry.value:
            self.free(block)
            return None, True
        out = None
        if self.ctx.comm_rank == dst:
            out = _read_result(self.ctx, block.handle, query, 1, keep_handle=False, views=getattr(self, "views", False))
        else:
            self.ctx.lib.pb200_result_free(block.handle)
        block.handle = None
        return out, False

    def execute(self, segments, query, reduce_world: int, merged_docs_bound: int, no_count_carrier: bool):
        """-> a merged, NOT yet extracted results block (dense tables on the device) with .count_carrier / .carrier_unsafe"""
        return self.pm.execute_segments(segments, query, merge=True, keep_handle=True, reduce_world=reduce_world,
                                        merged_docs_bound=merged_docs_bound, no_count_carrier=no_count_carrier)[0]

    def buffers(self, block):
        return device_buffers(self.ctx, block)

    def flag_tensor(self, value: int):
        import torch
        return torch.tensor([value], dtype=torch.int32, device=f"cuda:{self.ctx.device}")

    def stats_tensor(self, block):
        """The block's four execution statistics as an int64 tensor on the device, for a SUM reduce."""
        import torch
        return torch.tensor(_stats_list(block.stats), dtype=torch.int64, device=f"cuda:{self.ctx.device}")

    def synchronize(self):
        import torch
        torch.cuda.synchronize(self.ctx.device)  # the extraction runs on the library's own stream

    def finish(self, block, query, is_root: bool):
        from . import _lib
        from .plan_maker import _read_result
        out = None
        if is_root:
            _lib.check(self.ctx.lib.pb200_result_finalize(self.ctx.handle, block.handle))
            out = _read_result(self.ctx, block.handle, query, 1, keep_handle=False, views=getattr(self, "views", False))
        else:
            self.ctx.lib.pb200_result_free(block.handle)
        block.handle = None
        return out

    def free(self, block):
        if block.handle is not None:
            self.ctx.lib.pb200_result_free(block.handle)
            block.handle = None


def combine_tables(backend, block, query, dist, dst: int = 0):
    """All ranks call this with their merged, unextracted block: reduce of the tables to `dst`, which extracts the groups.

    Count-carrying sums ("count carrier", pb200_plan.cpp: the per-group row count rides in the upper bits of an INT sum)
    add field by field in the same int64 reduce; whether that is safe is decided per rank BEFORE the reduce (the rank's
    largest sum field must leave room for the other ranks': block.carrier_unsafe) and agreed on with one 4-byte MAX
    all-reduce that travels with the tables.  Returns (result or None, retry): retry == True on EVERY rank iff some rank
    said unsafe -- then all ranks must run the query again without the carrier (the tables of all ranks must share one
    layout, so the fallback is collective)."""
    bufs = backend.buffers(block)
    # the execution statistics of the whole table (the broker sums them over servers), as the in-library combine does
    stats = backend.stats_tensor(block) if hasattr(backend, "stats_tensor") else None
    if stats is not None:
        dist.reduce(stats, dst=dst, op=dist.ReduceOp.SUM)
    flag = None
    if block.count_carrier and getattr(block, "flag_slot", False):
        # the verdict rides as the last element of the int64 block: one SUM all-reduce moves tables and verdicts together
        # (a separate 4-byte collective costs as much as the 1 MB one: both are latency bound)
        dist.all_reduce(bufs["i64"], op=dist.ReduceOp.SUM)
        flag = bufs["i64"][-1:]
        reduce_buffers({k: v for k, v in bufs.items() if k != "i64"}, dist, dst)
    else:
        if block.count_carrier:
            flag = backend.flag_tensor(1 if block.carrier_unsafe else 0)
            dist.all_reduce(flag, op=dist.ReduceOp.MAX)
        reduce_buffers(bufs, dist, dst)
    if flag is not None:
        unsafe = int(flag.item()) != 0   # host waits for the collectives queued before it
        if unsafe:
            backend.free(block)
            return None, True
    else:
        backend.synchronize()
    out = backend.finish(block, query, dist.get_rank() == dst)
    if out is not None and stats is not None:
        _set_stats(out, stats.tolist())
    return out, False


def _stats_list(stats) -> List[int]:
    return [stats.num_docs_scanned, stats.num_entries_scanned_in_filter, stats.num_entries_scanned_post_filter,
            stats.num_total_docs]


def _set_stats(block, values: Sequence[int]) -> None:
    (block.stats.num_docs_scanned, block.stats.num_entries_scanned_in_filter, block.stats.num_entries_scanned_post_filter,
     block.stats.num_total_docs) = (int(v) for v in values)


def execute_and_combine(plan_maker_or_backend, segments: Sequence, query, dist, dst: int = 0, merged_docs_bound: int = 0):
    """One query over the whole table: every rank scans its segments with the device-side combine, the per-GPU group tables
    are reduced ONCE to rank `dst`, which gets the results block of the whole table (others get None).  Every refusal
    below is raised on every rank before any collective is issued."""
    if getattr(query, "having", None) is not None:
        # HAVING filters final rows: no route here applies it to the whole table's rows (the dense tables are filtered at
        # extraction only on one GPU, the host merge would drop it): the caller filters the combined rows
        from ._lib import E_UNSUPPORTED, UnsupportedQueryError
        raise UnsupportedQueryError(E_UNSUPPORTED, "HAVING is not combined across GPUs")
    if any(a.function in WITHTIME_FUNCTIONS for a in query.aggregations):
        # the winning rows of different GPUs are compared by time value on the host: the caller merges per-GPU results
        from ._lib import E_UNSUPPORTED, UnsupportedQueryError
        raise UnsupportedQueryError(E_UNSUPPORTED, "FIRSTWITHTIME / LASTWITHTIME are not combined across GPUs")
    if any(a.function == "PERCENTILE" for a in query.aggregations):
        # per-GPU histograms are not reduced across GPUs: the caller runs the query per GPU and merges by value
        from ._lib import E_UNSUPPORTED, UnsupportedQueryError
        raise UnsupportedQueryError(E_UNSUPPORTED, "PERCENTILE is not combined across GPUs")
    if any(a.function in MOMENT_FUNCTIONS for a in query.aggregations):
        # per-GPU moments are not reduced across GPUs: the caller runs the query per GPU and merges them by value
        from ._lib import E_UNSUPPORTED, UnsupportedQueryError
        raise UnsupportedQueryError(E_UNSUPPORTED, "VAR/STDDEV is not combined across GPUs")
    if query.is_group_by and any(is_multi_column_expression(a.function, a.column) for a in query.aggregations):
        # the expression tables are not among the reduced table blocks: the caller runs the query per GPU and merges by key
        from ._lib import E_UNSUPPORTED, UnsupportedQueryError
        raise UnsupportedQueryError(E_UNSUPPORTED, "expression aggregations with GROUP BY are not combined across GPUs")
    backend = plan_maker_or_backend if hasattr(plan_maker_or_backend, "finish") else DeviceBackend(plan_maker_or_backend)
    world = dist.get_world_size()
    if any(a.function in _SET_FUNCTIONS for a in query.aggregations):
        return _combine_with_sets(backend, segments, query, dist, dst)
    if not query.is_group_by:
        return _combine_scalars(backend, segments, query, dist, dst)
    for no_carrier in (False, True):
        block = backend.execute(segments, query, world, merged_docs_bound, no_carrier)
        try:
            if getattr(backend, "native", False):
                out, retry = backend.combine_native(block, query, dst)
            else:
                out, retry = combine_tables(backend, block, query, dist, dst)
        except Exception as e:
            # Key spaces beyond the dense tables live in per-GPU HASH tables whose slots mean different keys on every rank:
            # not element-wise reducible.  Every rank gets this refusal before any collective was issued (the key space is the
            # domain's, identical everywhere), so all of them take the host route together: merge by key like the reference's
            # combine (IndexedTable.upsert).
            if "hash group tables" not in str(e):
                raise
            backend.free(block)
            return _combine_with_sets(backend, segments, query, dist, dst)
        if not retry:
            return out
    raise AssertionError("unreachable: the second pass carries no counts")


def _combine_with_sets(backend, segments, query, dist, dst):
    """Host-side merge BY KEY (also used for per-GPU hash group tables, see execute_and_combine).  Queries with DISTINCTCOUNT: the per-group dictId SETS are not one of the element-wise reducible table blocks (NCCL has
    no bitwise OR), so this path merges on the host like the reference's combine does (BaseDistinctAggregateAggregationFunction
    .merge :109-121 = set union): every rank extracts its combined block, the (key ids, intermediates, id sets) travel with
    all_gather_object and rank `dst` merges them by key.  Ids are only comparable across ranks when the key and DISTINCTCOUNT
    columns are bound to one dictionary domain (global_domain) -- the caller's precondition, as for every cross-GPU merge."""
    import numpy as np
    from .plan_maker import ResultsBlock
    # every group of every rank: a rank-level trim before this merge by key could drop a group of the global top rows
    # a DISTINCTCOUNTHLL's set is only read on request: the merged block's sets travel to the root
    hll = {"sets": True} if any(a.function == "DISTINCTCOUNTHLL" for a in query.aggregations) else {}
    block = backend.pm.execute_segments(segments, query, merge=True, ordered=False, **hll)[0]
    fns = [a.function for a in query.aggregations]
    rows = 1 if block.num_groups < 0 else block.num_groups
    mine = {}
    for g in range(rows):
        key = () if block.num_groups < 0 else tuple(int(x) for x in block.keys[g])
        mine[key] = [frozenset(int(d) for d in block.distinct[(a, g)]) if f in _SET_FUNCTIONS
                     else (float(block.doubles[a][g]), int(block.longs[a][g]), int(block.dict_ids[a][g])) for a, f in enumerate(fns)]
    stats = (block.stats.num_docs_scanned, block.stats.num_entries_scanned_in_filter, block.stats.num_entries_scanned_post_filter,
             block.stats.num_total_docs)
    everyone = [None] * dist.get_world_size()
    dist.all_gather_object(everyone, (mine, stats))
    if dist.get_rank() != dst:
        return None
    merged = {}
    for part, _ in everyone:
        for key, vals in part.items():
            cur = merged.get(key)
            if cur is None:
                merged[key] = list(vals)
                continue
            for a, f in enumerate(fns):
                if f in _SET_FUNCTIONS:
                    cur[a] = cur[a] | vals[a]
                elif f in ("COUNT", "SUM", "AVG"):
                    cur[a] = (cur[a][0] + vals[a][0], cur[a][1] + vals[a][1], -1)
                elif f == "MIN":
                    cur[a] = min(cur[a], vals[a], key=lambda t: t[0])
                else:
                    cur[a] = max(cur[a], vals[a], key=lambda t: t[0])
    keys_sorted = sorted(merged)   # raw-key order is not defined across tables: ascending ids, column 0 most significant
    def set_final(a, id_set):   # DISTINCTCOUNT / DISTINCTSUM / DISTINCTAVG / DISTINCTCOUNTHLL of a merged set of domain ids, exact
        if fns[a] == "DISTINCTCOUNT":
            return float(len(id_set))
        if fns[a] == "DISTINCTCOUNTHLL":
            agg = query.aggregations[a]
            members = HllSet((value_key(segments[0].dictionary_value(agg.column, d)) for d in id_set),   # -0.0 apart from 0.0
                             segments[0].column_info(agg.column)["data_type"])
            return hll_final(members, agg.arg, members.data_type)
        return float(distinct_final(fns[a], [segments[0].dictionary_value(query.aggregations[a].column, d) for d in id_set]))
    if query.is_group_by and query.order_by:
        keys_sorted = _order_and_trim(query, fns, keys_sorted, merged, set_final)
    n, k = len(keys_sorted), len(query.group_by)
    out_keys = np.asarray(keys_sorted, dtype=np.int32).reshape(n, k) if query.is_group_by else np.zeros((0, 0), dtype=np.int32)
    doubles, longs, ids, distinct = [], [], [], {}
    for a, f in enumerate(fns):
        d, l, i = np.zeros(max(n, 1)), np.zeros(max(n, 1), dtype=np.int64), np.full(max(n, 1), -1, dtype=np.int32)
        for g, key in enumerate(keys_sorted):
            v = merged[key][a]
            if f in _SET_FUNCTIONS:
                distinct[(a, g)] = np.asarray(sorted(v), dtype=np.int32)
                if f == "DISTINCTCOUNTHLL":   # the estimate in both columns, as the library returns it
                    est = set_final(a, v)
                    d[g], l[g] = float(est), est
                else:
                    d[g], l[g] = set_final(a, v), len(v)
            else:
                d[g], l[g], i[g] = v
        doubles.append(d[:n] if query.is_group_by else d); longs.append(l[:n] if query.is_group_by else l); ids.append(i[:n] if query.is_group_by else i)
    block.num_groups = n if query.is_group_by else -1
    block.keys, block.doubles, block.longs, block.dict_ids, block.distinct = out_keys, doubles, longs, ids, distinct
    block.stats.num_docs_scanned = sum(s[0] for _, s in everyone)
    block.stats.num_entries_scanned_in_filter = sum(s[1] for _, s in everyone)
    block.stats.num_entries_scanned_post_filter = sum(s[2] for _, s in everyone)
    block.stats.num_total_docs = sum(s[3] for _, s in everyone)
    return block


def _order_and_trim(query, fns, keys, merged, set_final):
    """The merged rows (`keys` ascending, column 0 most significant) in ORDER BY order, trimmed as the dense route trims a
    merged result (plan_maker.order_spec): one stable sort per item, last item first, so rows equal on every item keep
    the key order -- the library's tie rule.  Values compare in the reference's order (query.value_order); a key column
    compares by domain id, which is its value order."""
    from .plan_maker import order_spec
    from .query import post_eval, value_order
    from .sql import resolve_order_by

    def final(a, v):
        f = fns[a]
        if f in _SET_FUNCTIONS:
            return set_final(a, v)
        if f == "COUNT":
            return float(v[1])
        if f == "AVG":
            return v[0] / v[1] if v[1] else float("-inf")
        return v[0]
    rows = list(keys)
    for kind, index, asc in reversed(resolve_order_by(query)):
        if kind == "GROUP_BY":
            rows.sort(key=lambda key: key[index], reverse=not asc)
        elif kind == "POST":
            program = query.post_aggregations[index].program
            rows.sort(key=lambda key: value_order(post_eval(program, lambda a: float(final(a, merged[key][a])))), reverse=not asc)
        else:
            rows.sort(key=lambda key: value_order(float(final(index, merged[key][index]))), reverse=not asc)
    trim = order_spec(query, merge=True).trim_size
    return rows[:trim] if trim > 0 else rows


def _exact_sums(ctx, block, n: int) -> List[Optional[int]]:
    """Per aggregation of an aggregation-only block: the exact int64 sum behind an INT SUM / AVG, else None."""
    out = []
    for a in range(n):
        v = C.c_int64()
        rc = ctx.lib.pb200_result_exact_sum(block.handle, a, C.byref(v))
        if rc < 0:
            from . import _lib
            _lib.check(rc)
        out.append(v.value if rc == 1 else None)
    return out


def _combine_scalars(backend, segments, query, dist, dst):
    """Aggregation-only queries: a handful of scalars per rank (AggregationResultsBlockMerger.java:34-44)."""
    if getattr(backend, "native", False):   # the scalars meet inside the library too (pb200_comm.cu: combine_scalars)
        block = backend.pm.execute_segments(segments, query, merge=True, keep_handle=True, defer=False)[0]
        return backend.combine_native(block, query, dst)[0]
    import torch
    block = backend.pm.execute_segments(segments, query, merge=True, keep_handle=True, defer=False)[0]
    fns = [a.function for a in query.aggregations]
    n = len(fns)
    exact = _exact_sums(backend.ctx, block, n)
    block.release(backend.ctx)
    dev = f"cuda:{backend.ctx.device}"
    sums = torch.tensor([float(block.doubles[a][0]) if f in ("SUM", "AVG") else 0.0 for a, f in enumerate(fns)],
                        dtype=torch.float64, device=dev)
    # INT SUM / AVG add exactly and round once on the root: the ranks' doubles are rounded already, and rounded sums beyond
    # 2^53 do not add to the rounded total.  [exact sums | ranks that had one | counts | the four statistics]
    ints = torch.tensor([e or 0 for e in exact] + [int(e is not None) for e in exact] +
                        [int(block.longs[a][0]) for a in range(n)] + _stats_list(block.stats), dtype=torch.int64, device=dev)
    mins = torch.tensor([float(block.doubles[a][0]) if f == "MIN" else float("inf") for a, f in enumerate(fns)], dtype=torch.float64, device=dev)
    maxs = torch.tensor([float(block.doubles[a][0]) if f == "MAX" else float("-inf") for a, f in enumerate(fns)], dtype=torch.float64, device=dev)
    dist.reduce(sums, dst=dst, op=dist.ReduceOp.SUM)
    dist.reduce(ints, dst=dst, op=dist.ReduceOp.SUM)
    if "MIN" in fns:
        dist.reduce(mins, dst=dst, op=dist.ReduceOp.MIN)
    if "MAX" in fns:
        dist.reduce(maxs, dst=dst, op=dist.ReduceOp.MAX)
    if dist.get_rank() != dst:
        return None
    world = dist.get_world_size()
    sums, mins, maxs, ints = sums.cpu().numpy(), mins.cpu().numpy(), maxs.cpu().numpy(), [int(x) for x in ints.tolist()]
    for a, f in enumerate(fns):
        block.longs[a][0] = ints[2 * n + a]
        if f == "MIN":
            block.doubles[a][0] = mins[a]
        elif f == "MAX":
            block.doubles[a][0] = maxs[a]
        elif f in ("SUM", "AVG"):
            block.doubles[a][0] = float(ints[a]) if ints[n + a] == world else sums[a]
        else:
            block.doubles[a][0] = float(ints[2 * n + a])
        if f in ("MIN", "MAX"):
            block.dict_ids[a][0] = -1   # ids are rank local unless the segments are bound to one domain
    _set_stats(block, ints[3 * n:3 * n + 4])
    return block


def combine_across_ranks(plan_maker, block, query, dist, dst: int = 0):
    """Reduce + extraction of an already executed block (merge=True, keep_handle=True; executed WITHOUT reduce_world, i.e.
    with separate COUNT tables).  Rank `dst` gets the block of the whole table, others get None."""
    if getattr(block, "count_carrier", False) and dist.get_world_size() > 1:
        raise ValueError("a block whose counts ride in a sum must go through execute_and_combine (it sizes the packed fields "
                         "for all ranks and agrees on the fallback collectively)")
    out, _ = combine_tables(DeviceBackend(plan_maker), block, query, dist, dst)
    return out


def init_comm(ctx, dist) -> None:
    """Give the context its own NCCL communicator (pb200_comm_init): rank 0 creates the id, torch.distributed (any backend)
    only ships its 128 bytes.  After this execute_and_combine reduces inside the library."""
    from . import _lib
    world, rank = dist.get_world_size(), dist.get_rank()
    if world < 2 or getattr(ctx, "comm_world", 0) > 1:
        return
    box = [None]
    if rank == 0:
        buf = (C.c_ubyte * 128)()
        if ctx.lib.pb200_comm_unique_id(buf) == 0:
            box[0] = bytes(buf)
        else:   # e.g. no libnccl.so.2 for dlopen: tell the other ranks instead of leaving them in the broadcast
            box[0] = ("error", ctx.lib.pb200_last_error().decode())
    dist.broadcast_object_list(box, src=0)
    if isinstance(box[0], tuple):
        raise RuntimeError(f"pb200_comm_unique_id failed on rank 0: {box[0][1]}")
    _lib.check(ctx.lib.pb200_comm_init(ctx.handle, box[0], rank, world))
    ctx.comm_rank, ctx.comm_world = rank, world


def global_domain(ctx, segments: Sequence, columns: Sequence[str], dist):
    """Table-wide dictionaries across ALL ranks: every rank contributes the union of its own segments' dictionaries (built
    by the library), the unions are all-gathered as bytes, and every rank builds the same global domain from them and binds
    its segments.  After this the per-GPU tables share one id space: the reduce is a merge by value
    (GroupByCombineOperator.java:130-146).  Returns the DictionaryDomain (release it when the table is dropped)."""
    from . import _lib
    from .plan_maker import DictionaryDomain
    local = DictionaryDomain.build(ctx, segments, columns)
    mine = {c: (local.dictionary_bytes(c).tobytes(), local.info(c)) for c in columns}
    ids = list(local.column_ids)
    local.release()
    everyone: List[Optional[dict]] = [None] * dist.get_world_size()
    dist.all_gather_object(everyone, mine)
    import numpy as np
    parts, widths, types = [], [], []
    for c in columns:
        parts.append([np.frombuffer(e[c][0], dtype=np.uint8) for e in everyone])
        widths.append([e[c][1]["entry_bytes"] for e in everyone])
        types.append(mine[c][1]["stored_type"])
    dom = DictionaryDomain.from_dictionaries(ctx, columns, ids, types, parts, widths)
    for s in segments:
        s.bind_domain(dom)
    return dom
