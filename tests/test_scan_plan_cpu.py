"""CPU tests of the scan-launch planner (pb200::plan_scan, pinot_b200/csrc/pb200_plan.cpp): every decision pb200_execute
takes before it touches the device -- geometry, shared-memory layout, count carrier, table layouts, launch chunks and
refusals -- checked on segments made of column metadata alone (tests/host_probe/host_probe.cpp probe_plan_scan).

The named shapes pin the values the executor has always chosen for them on an H100 SXM (132 SMs, 232 448 bytes of
opt-in shared memory per block); the sweep checks the layout invariants the kernel relies on over a few thousand shapes."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from pinot_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

H100 = (132, 232_448)  # multiProcessorCount, sharedMemPerBlockOptin
F = dict(AND=0, OR=1, NOT=2, MATCH_ALL=3, EMPTY=4, SCAN_RANGE=5, SCAN_IN=6, SCAN_NOT_IN=7, INV_IN=8, INV_NOT_IN=9,
         DOC_RANGES=10, RAW_RANGE=11, DOC_MASK=12)
COUNT, SUM, MIN, MAX, AVG, DISTINCTCOUNT = range(6)
Q_PER_SEGMENT_FILTER, Q_MERGE, Q_DEFER_FINALIZE, Q_NO_COUNT_CARRIER = 1, 2, 4, 8
MAX_AGGS, MAX_LEAVES, MAX_STAGES, RES, SEG, CHUNK = 6, 8, 4, 40, 40, 4
VAL_DICT_I32, VAL_DICT_F32 = 1, 3
VARIANTS = {(6, 0, 1, 2), (8, 0, 1, 2), (8, 0, 0, 2), (6, 1, 0, 1), (8, 1, 0, 1), (6, 1, 0, 2), (8, 1, 0, 2)}

# probe_plan in host_probe.cpp, field by field (all int64)
PLAN_FIELDS = (
    [(n, 1) for n in ("warps", "ctas_per_sm", "stages", "stage_words", "tile_rows", "smem_bytes", "queue_off", "smem_table_off",
                      "queue_max", "sparse_max", "sparse_max_agg", "defer_agg", "conj", "num_slots", "num_leaves", "num_nodes",
                      "use_pipe", "smem_groups", "smem_copies", "smem_gstride", "smem_count", "smem_merged")]
    + [("smem_slot", MAX_AGGS), ("variant", 4), ("num_chunks", 1)]
    + [(n, CHUNK) for n in ("chunk_first_seg", "chunk_num_segs", "chunk_total_tiles", "chunk_grid")]
    + [("nres", 1), ("projected", 1), ("num_leaf_buffers", 1), ("in_filter", RES)]
    + [(n, RES) for n in ("hashed", "groups", "stride", "carrier_agg", "carrier_shift", "carrier_vmin", "need_count", "need_seen",
                          "exists_min", "exists_max", "reduce_world", "flag_slot", "tail_slots", "i64_elems", "f64_elems",
                          "u32max_elems", "u32min_elems")]
    + [("dwords", RES * MAX_AGGS), ("distinct_words", RES * MAX_AGGS)]
    + [(n, SEG) for n in ("seg_first_tile", "seg_num_tiles", "seg_stage_tx", "seg_num_agg_codes", "seg_num_defer_codes")]
    + [("seg_agg_code", SEG * MAX_AGGS)]
    + [(n, SEG * MAX_LEAVES) for n in ("seg_leaf_kind", "seg_leaf_cmp", "seg_leaf_negate", "seg_leaf_lo", "seg_leaf_span",
                                        "seg_leaf_slot")])


class ProbePlan(C.Structure):
    _fields_ = [(n, C.c_int64 if k == 1 else C.c_int64 * k) for n, k in PLAN_FIELDS]


class ProbeCol(C.Structure):
    _fields_ = [("fwd_kind", C.c_int32), ("stored_type", C.c_int32), ("bits", C.c_int32), ("cardinality", C.c_int32),
                ("dict_native", C.c_int32), ("dict_shared", C.c_int32), ("has_inv", C.c_int32), ("eligible", C.c_int32),
                ("dict_hash", C.c_uint64), ("dict_host", C.c_void_p), ("dict_host_bytes", C.c_uint64)]


@pytest.fixture(scope="module")
def probe():
    from pinot_b200.build import build
    build()
    src = os.path.join(HERE, "host_probe", "host_probe.cpp")
    out = os.path.join(HERE, "host_probe", "libhost_probe.so")
    libdir = os.path.join(ROOT, "pinot_b200")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(_lib.LIB_PATH)):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", f"-I{cuda_inc}", "-o", out, src, f"-L{libdir}",
                        "-lpinot_b200", f"-Wl,-rpath,{libdir}"], check=True)
    lib = C.CDLL(out)
    lib.probe_plan_size.restype = C.c_int64
    assert lib.probe_plan_size() == C.sizeof(ProbePlan)
    lib.probe_plan_scan.restype = C.c_int32
    lib.probe_plan_scan.argtypes = [C.c_int32, C.c_int32, C.POINTER(C.c_char_p), C.POINTER(C.c_int64), C.c_int32,
                                    C.POINTER(_lib.Query), C.POINTER(ProbeCol), C.c_int32, C.POINTER(C.c_int32), C.c_int32,
                                    C.c_int32, C.POINTER(ProbePlan)]
    core = C.CDLL(_lib.LIB_PATH)
    core.pb200_last_error.restype = C.c_char_p
    lib.last_error = lambda: core.pb200_last_error().decode()
    return lib


def bits_for(card):
    b = 1
    while b < 31 and (1 << b) < card:
        b += 1
    return b


def col(card, base=0, step=1, stored=_lib.INT, raw=False, device_dict=True, shared=False, inv=False, dict_id=0):
    """Column metadata of a dictionary-encoded column {base + step * i} (or a raw 32-bit INT column)."""
    if raw:
        return dict(kind=_lib.FWD_RAW_FIXEDBYTE, stored=stored, bits=32, card=card, native=False, shared=False, inv=False,
                    hash=0, host=None, cbuf=None)
    host = None
    if stored == _lib.INT and 0 < card <= 1 << 20:   # larger dictionaries come without host values (no count carrier)
        host = (base + step * np.arange(card, dtype=np.int64)).astype(np.int32).tobytes()
    return dict(kind=_lib.FWD_DICT_FIXEDBIT, stored=stored, bits=bits_for(card), card=card, native=device_dict and stored != _lib.STRING,
                shared=shared, inv=inv, hash=hash((card, base, step, stored, dict_id)) & (2**63 - 1), host=host,
                cbuf=C.create_string_buffer(host, len(host)) if host else None)


def node(op, column=0, children=0, lo=0, hi=0, ids=(), raw=(0.0, 0.0, 0)):
    return dict(op=F[op], column=column, children=children, lo=lo, hi=hi, ids=list(ids), raw=raw)


def make_query(filters, aggs, group_by=(), flags=0, limit=100_000, reduce_world=0, merged_docs_bound=0):
    """filters: one postfix node list, or one per segment (with Q_PER_SEGMENT_FILTER).  Returns (query, keep-alive)."""
    trees = filters if (flags & Q_PER_SEGMENT_FILTER) else [filters]
    nodes = [n for t in trees for n in t]
    keep = []
    fn = (_lib.FilterNode * max(len(nodes), 1))()
    for i, n in enumerate(nodes):
        ids = (C.c_int32 * max(len(n["ids"]), 1))(*n["ids"])
        keep.append(ids)
        fn[i] = _lib.FilterNode(n["op"], n["column"], n["children"], n["lo"], n["hi"], len(n["ids"]),
                                C.cast(ids, C.POINTER(C.c_int32)), n["raw"][0], n["raw"][1], n["raw"][2], 0)
    gb = (C.c_int32 * max(len(group_by), 1))(*group_by)
    ag = (_lib.Agg * max(len(aggs), 1))(*[_lib.Agg(f, c) for f, c in aggs])
    q = _lib.Query(len(trees[0]), len(group_by), len(aggs), limit, 10_000, flags, fn, gb, ag, reduce_world, 0, merged_docs_bound)
    keep += [fn, gb, ag]
    return q, keep


def plan(probe, seg_cols, num_docs, q, knobs=None, carrier=True, limits=H100):
    """seg_cols: one column list per segment.  Returns (rc, ProbePlan)."""
    knobs = knobs or {}
    ncols = len(seg_cols[0])
    cols = (ProbeCol * (len(seg_cols) * ncols))()
    for s, cs in enumerate(seg_cols):
        for k, c in enumerate(cs):
            host = c.get("cbuf")
            cols[s * ncols + k] = ProbeCol(c["kind"], c["stored"], c["bits"], c["card"], int(c["native"]), int(c["shared"]),
                                           int(c["inv"]), -1, c["hash"], C.cast(host, C.c_void_p) if host else None,
                                           len(c["host"]) if host else 0)
    names = (C.c_char_p * max(len(knobs), 1))(*[k.encode() for k in knobs])
    values = (C.c_int64 * max(len(knobs), 1))(*knobs.values())
    docs = (C.c_int32 * len(num_docs))(*num_docs)
    out = ProbePlan()
    rc = probe.probe_plan_scan(limits[0], limits[1], names, values, len(knobs), C.byref(q), cols, ncols, docs, len(num_docs),
                               int(carrier), C.byref(out))
    return rc, out


# ---------------------------------------------------------------------------------------------------------------------
# named shapes
# ---------------------------------------------------------------------------------------------------------------------
# the bench table's columns (bench.py CARDS / VALUE_BASE / VALUE_STEP): c3 10 000 values, c5 100 000, c6 1 000 000
C3, C5, C6 = col(10_000, 5, 3), col(100_000, 11, 7), col(1_000_000, 1, 2)
UPPER_TENTH = [node("SCAN_RANGE", 2, lo=899_999, hi=1_000_000)]     # c6 > value(899 998): the upper 10 % of the dictionary


def headline(probe, groups_col=C3, nseg=8, rows=100_000_000, **kw):
    """SELECT SUM(c5), COUNT(*) WHERE c6 > K GROUP BY <groups_col>, merged over nseg segments."""
    q, keep = make_query(UPPER_TENTH, [(SUM, 1), (COUNT, -1)], group_by=[0], flags=Q_MERGE)
    return plan(probe, [[groups_col, C5, C6]] * nseg, [rows] * nseg, q, **kw)


def test_headline_10000_groups_one_8_warp_cta_with_a_shared_table_and_no_count_array(probe):
    rc, p = headline(probe)
    assert rc == 0, probe.last_error()
    assert (p.warps, p.ctas_per_sm, p.stages, p.stage_words) == (8, 1, 2, 32 * 51)
    assert tuple(p.variant) == (8, 1, 0, 1)
    assert (p.smem_groups, p.smem_count, p.smem_gstride, p.smem_copies, p.smem_merged) == (10_000, 0, 10_001, 1, 1)
    assert list(p.smem_slot) == [0, -1, -1, -1, -1, -1]
    assert (p.smem_bytes, p.queue_off, p.smem_table_off) == (202_632, 106_240, 106_240 + 8 * 2048)
    assert p.smem_table_off + 10_001 * 4 * 2 <= p.smem_bytes <= H100[1]
    assert (p.carrier_agg[0], p.carrier_vmin[0], p.need_count[0], p.need_seen[0]) == (0, 11, 0, 0)
    assert p.carrier_shift[0] == (64 + (7 * 99_999).bit_length() + 1) // 2
    assert (p.hashed[0], p.groups[0], p.stride[0], p.i64_elems[0]) == (0, 10_000, 1, 10_000)
    assert (p.num_chunks, p.chunk_grid[0], p.chunk_total_tiles[0]) == (1, 132, 8 * -(-100_000_000 // 8192))


def test_1000_groups_two_6_warp_ctas_with_replicated_copies(probe):
    rc, p = headline(probe, groups_col=col(1_000, 0, 1))
    assert rc == 0, probe.last_error()
    assert (p.warps, p.ctas_per_sm, tuple(p.variant)) == (6, 2, (6, 1, 0, 2))
    assert (p.smem_groups, p.smem_gstride, p.smem_count, p.smem_copies) == (1_000, 1_001, 0, 2)
    assert (p.stages, p.smem_bytes) == (2, 102_288)
    assert p.chunk_grid[0] == 264


def test_16000_groups_global_table_with_stride(probe):
    rc, p = headline(probe, groups_col=col(16_000, 0, 1))
    assert rc == 0, probe.last_error()
    assert (p.smem_groups, p.warps, p.ctas_per_sm) == (0, 6, 2)
    assert (p.hashed[0], p.stride[0], p.groups[0]) == (0, 16, 256_000)   # 16 000 x 8 B x 16 stays within 2 MB
    assert p.carrier_agg[0] == 0 and p.i64_elems[0] == 256_000


def test_key_space_beyond_dense_max_is_a_hash_table(probe):
    big = col(1 << 20, 0, 1)
    q, keep = make_query([], [(SUM, 1), (COUNT, -1)], group_by=[0, 2], flags=Q_MERGE, limit=100_000)
    rc, p = plan(probe, [[big, C5, big]] * 2, [1_000_000] * 2, q)
    assert rc == 0, probe.last_error()
    assert (p.hashed[0], p.groups[0], p.stride[0], p.smem_groups) == (1, 1 << 18, 1, 0)
    assert (p.need_seen[0], p.carrier_agg[0]) == (0, 0)


def test_rows_too_wide_for_two_2_deep_rings_fall_back_to_one_cta(probe):
    wide = [col((1 << 20) + k, 0, 1) for k in range(4)]   # 4 x 21 bits = 84 bits per row
    q, keep = make_query([node("SCAN_RANGE", 0, lo=0, hi=10)], [(SUM, 1), (SUM, 2), (MAX, 3)])
    rc, p = plan(probe, [wide], [1_000_000], q)
    assert rc == 0, probe.last_error()
    assert (p.warps, p.ctas_per_sm, p.stages, tuple(p.variant)) == (6, 1, 3, (6, 0, 1, 2))
    assert p.chunk_grid[0] == 132


def test_c2_aggregation_only_defers_its_int_sum(probe):
    q, keep = make_query([node("SCAN_RANGE", 0, lo=3418, hi=6580), node("SCAN_RANGE", 2, lo=683_771, hi=1_000_000),
                          node("AND", children=2)], [(SUM, 1), (COUNT, -1)], flags=Q_MERGE)
    rc, p = plan(probe, [[C3, C5, C6]] * 8, [100_000_000] * 8, q)
    assert rc == 0, probe.last_error()
    assert (p.warps, p.ctas_per_sm, tuple(p.variant), p.defer_agg, p.conj) == (6, 2, (6, 0, 1, 2), 0, 1)
    assert (p.stages, p.sparse_max_agg, p.seg_num_defer_codes[0], p.seg_num_agg_codes[0]) == (2, 4, 0, 1)
    assert p.nres == 1 and p.chunk_grid[0] == 264


def test_carrier_refused_when_docs_times_range_reaches_2_to_the_63(probe):
    full = col(3, -(1 << 31), (1 << 31) - 1)                 # values -2^31, -1, 2^31 - 2: a 32-bit range
    q, keep = make_query([], [(SUM, 1), (COUNT, -1)], group_by=[0], flags=Q_MERGE | Q_DEFER_FINALIZE,
                         merged_docs_bound=1 << 32)         # 33 + 32 bits > 63
    rc, p = plan(probe, [[C3, full]] * 2, [1_000_000] * 2, q)
    assert rc == 0, probe.last_error()
    assert (p.carrier_agg[0], p.need_count[0], p.smem_count) == (-1, 1, 1)
    q, keep = make_query([], [(SUM, 1), (COUNT, -1)], group_by=[0], flags=Q_MERGE | Q_DEFER_FINALIZE,
                         merged_docs_bound=(1 << 31) - 1)   # 31 + 32 bits: admitted
    rc, p = plan(probe, [[C3, full]] * 2, [1_000_000] * 2, q)
    assert rc == 0 and (p.carrier_agg[0], p.carrier_shift[0], p.carrier_vmin[0]) == (0, 48, -(1 << 31))


def test_reduce_world_above_one_needs_a_bound_dictionary_for_the_carrier(probe):
    q, keep = make_query([], [(SUM, 1), (COUNT, -1)], group_by=[0], flags=Q_MERGE | Q_DEFER_FINALIZE, reduce_world=2)
    rc, p = plan(probe, [[C3, C5]] * 2, [1_000_000] * 2, q)
    assert rc == 0, probe.last_error()
    assert (p.carrier_agg[0], p.need_count[0], p.reduce_world[0], p.tail_slots[0], p.flag_slot[0]) == (-1, 1, 2, 5, 0)
    bound = col(100_000, 11, 7, shared=True)
    rc, p = plan(probe, [[C3, bound]] * 2, [1_000_000] * 2, q)
    assert rc == 0 and (p.carrier_agg[0], p.flag_slot[0], p.tail_slots[0]) == (0, 1, 5)
    assert p.i64_elems[0] == 10_000 + 5


def test_17_segments_launch_as_two_chunks_with_rebased_tiles(probe):
    docs = [1_000_000 + 7_000 * s for s in range(17)]
    q, keep = make_query(UPPER_TENTH, [(SUM, 1), (COUNT, -1)], group_by=[0])
    rc, p = plan(probe, [[C3, C5, C6]] * 17, docs, q)
    assert rc == 0, probe.last_error()
    tiles = [-(-d // (p.warps * 1024)) for d in docs]
    assert (p.num_chunks, p.chunk_first_seg[0], p.chunk_num_segs[0], p.chunk_first_seg[1], p.chunk_num_segs[1]) == (2, 0, 16, 16, 1)
    assert (p.chunk_total_tiles[0], p.chunk_total_tiles[1]) == (sum(tiles[:16]), tiles[16])
    assert [p.seg_first_tile[s] for s in range(17)] == [sum(tiles[:s]) for s in range(16)] + [0]
    assert (p.warps, p.ctas_per_sm) == (8, 1)   # the 10 000-group shared table
    assert (p.chunk_grid[0], p.chunk_grid[1]) == (132, min(132, tiles[16]))
    assert p.nres == 17 and p.in_filter[16] == docs[16]


# ---------------------------------------------------------------------------------------------------------------------
# refusals: the same code pb200_execute has always returned for them
# ---------------------------------------------------------------------------------------------------------------------
def _refusal(probe, cols, aggs, filters=(), group_by=(), flags=0, nseg=1, seg_cols=None, **kw):
    q, keep = make_query(list(filters), aggs, group_by=group_by, flags=flags, **kw)
    rc, _ = plan(probe, seg_cols or [cols] * nseg, [100_000] * len(seg_cols or [cols] * nseg), q)
    return rc, probe.last_error()


SMALL = col(100, 0, 1)


@pytest.mark.parametrize("case, code, message", [
    ("slots", _lib.E_UNSUPPORTED, "too many distinct columns"),
    ("leaves", _lib.E_UNSUPPORTED, "too many filter leaves"),
    ("nodes", _lib.E_UNSUPPORTED, "query exceeds device limits"),
    ("malformed", _lib.E_INVALID, "malformed postfix filter"),
    ("too_deep", _lib.E_UNSUPPORTED, "operands not supported"),
    ("unknown_op", _lib.E_INVALID, "unknown filter op"),
    ("unknown_fn", _lib.E_INVALID, "unknown aggregation function"),
    ("too_wide", _lib.E_UNSUPPORTED, "too wide for the shared-memory pipeline"),
    ("array_map", _lib.E_UNSUPPORTED, "ARRAY_MAP"),
    ("groups_limit", _lib.E_UNSUPPORTED, "too large for the device hash table"),
    ("distinct_budget", _lib.E_UNSUPPORTED, "exceed the device bitset budget"),
    ("distinct_raw", _lib.E_UNSUPPORTED, "DISTINCTCOUNT on raw column"),
    ("in_raw", _lib.E_UNSUPPORTED, "IN on raw column"),
    ("sum_string", _lib.E_UNSUPPORTED, "SUM/AVG over STRING"),
    ("merge_dicts", _lib.E_UNSUPPORTED, "different dictionary"),
    ("tree_shapes", _lib.E_INVALID, "must share their shape"),
])
def test_refusals(probe, case, code, message):
    many = [col(100 + k, 0, 1) for k in range(13)]
    if case == "slots":
        rc, err = _refusal(probe, many, [(SUM, k) for k in range(6)], [node("SCAN_RANGE", k + 6, lo=0, hi=5) for k in range(7)]
                           + [node("AND", children=7)])
    elif case == "leaves":
        rc, err = _refusal(probe, many, [(COUNT, -1)], [node("SCAN_RANGE", k, lo=0, hi=5) for k in range(9)] + [node("AND", children=9)])
    elif case == "nodes":
        rc, err = _refusal(probe, many, [(COUNT, -1)], [node("MATCH_ALL")] + [node("NOT")] * 16)
    elif case == "malformed":
        rc, err = _refusal(probe, [SMALL], [(COUNT, -1)], [node("SCAN_RANGE", 0, lo=0, hi=5), node("AND", children=2)])
    elif case == "too_deep":
        rc, err = _refusal(probe, many, [(COUNT, -1)], [node("SCAN_RANGE", k, lo=0, hi=5) for k in range(8)] + [node("AND", children=9)])
    elif case == "unknown_op":
        rc, err = _refusal(probe, [SMALL], [(COUNT, -1)], [dict(node("MATCH_ALL"), op=-1)])
    elif case == "unknown_fn":
        rc, err = _refusal(probe, [SMALL], [(6, 0)])
    elif case == "too_wide":
        rc, err = _refusal(probe, [col((1 << 30) + k) for k in range(12)], [(SUM, k) for k in range(6)],
                           [node("SCAN_RANGE", k + 6, lo=0, hi=5) for k in range(6)] + [node("AND", children=6)])
    elif case == "array_map":
        huge = col((1 << 31) - 1)
        rc, err = _refusal(probe, [huge, huge, huge, SMALL], [(COUNT, -1)], group_by=[0, 1, 2])
    elif case == "groups_limit":
        big = col(1 << 20)
        rc, err = _refusal(probe, [big, big], [(COUNT, -1)], group_by=[0, 1], limit=1 << 27)
    elif case == "distinct_budget":
        rc, err = _refusal(probe, [col(1 << 24), col(1000)], [(DISTINCTCOUNT, 1)], group_by=[0])
    elif case == "distinct_raw":
        rc, err = _refusal(probe, [SMALL, col(0, raw=True)], [(DISTINCTCOUNT, 1)])
    elif case == "in_raw":
        rc, err = _refusal(probe, [SMALL, col(0, raw=True)], [(COUNT, -1)], [node("SCAN_IN", 1, ids=[1, 2])])
    elif case == "sum_string":
        rc, err = _refusal(probe, [col(50, stored=_lib.STRING)], [(SUM, 0)])
    elif case == "merge_dicts":
        rc, err = _refusal(probe, None, [(COUNT, -1)], group_by=[0], flags=Q_MERGE,
                           seg_cols=[[col(100, dict_id=1)], [col(100, dict_id=2)]])
    else:
        rc, err = _refusal(probe, [SMALL, SMALL], [(COUNT, -1)],
                           [[node("SCAN_RANGE", 0, lo=0, hi=5), node("SCAN_RANGE", 1, lo=0, hi=5), node("AND", children=2)],
                            [node("SCAN_RANGE", 0, lo=0, hi=5), node("SCAN_RANGE", 1, lo=0, hi=5), node("OR", children=2)]],
                           flags=Q_PER_SEGMENT_FILTER, nseg=2)
    assert (rc, message in err) == (code, True), err


# ---------------------------------------------------------------------------------------------------------------------
# execution statistics
# ---------------------------------------------------------------------------------------------------------------------
def test_entries_scanned_per_segment_and_merged(probe):
    cols = [C3, C5, C6]
    docs = [100_000, 250_000, 70_000]
    trees = [[node("SCAN_RANGE", 2, lo=5, hi=900), node("SCAN_IN", 0, ids=[1, 5, 9]), node("AND", children=2)],
             [node("MATCH_ALL"), node("SCAN_IN", 0, ids=[2]), node("AND", children=2)],
             [node("DOC_RANGES", ids=[0, 10]), node("EMPTY"), node("AND", children=2)]]
    q, keep = make_query(trees, [(SUM, 1), (COUNT, -1)], group_by=[0], flags=Q_PER_SEGMENT_FILTER)
    rc, p = plan(probe, [cols] * 3, docs, q)
    assert rc == 0, probe.last_error()
    assert [p.in_filter[r] for r in range(3)] == [2 * docs[0], docs[1], 0]
    assert p.projected == 2                         # c3 (group) and c5 (agg); c6 only filters
    q, keep = make_query(trees, [(SUM, 1), (COUNT, -1)], group_by=[0], flags=Q_PER_SEGMENT_FILTER | Q_MERGE)
    rc, p = plan(probe, [cols] * 3, docs, q)
    assert rc == 0 and p.nres == 1 and p.in_filter[0] == 2 * docs[0] + docs[1]
    q, keep = make_query([node("SCAN_RANGE", 2, lo=5, hi=900)], [(COUNT, -1)])
    rc, p = plan(probe, [cols] * 3, docs, q)
    assert rc == 0 and [p.in_filter[r] for r in range(3)] == docs and p.projected == 0


# ---------------------------------------------------------------------------------------------------------------------
# invariants over a seeded sweep
# ---------------------------------------------------------------------------------------------------------------------
def _random_shape(rng):
    nseg = int(rng.choice([1, 1, 2, 3, 8, 16, 17, 33, 40]))
    ncols = int(rng.integers(1, 13))
    cols = []
    for k in range(ncols):
        r = rng.random()
        if r < 0.08:
            cols.append(col(0, raw=True))
        elif r < 0.12:
            cols.append(col(int(rng.integers(1, 500)), stored=_lib.STRING))
        else:
            bits = int(rng.integers(1, 32)) if rng.random() < 0.3 else int(rng.integers(1, 17))
            card = int(rng.integers(1 << (bits - 1), (1 << bits) + 1)) if bits > 1 else int(rng.integers(1, 3))
            card = min(card, (1 << 31) - 1)
            step = int(rng.choice([1, 3, 1000, 1 << 20]))
            base = int(rng.integers(-(1 << 31), (1 << 31) - step * (card - 1))) if step * (card - 1) < (1 << 32) - 1 else -(1 << 31)
            cols.append(col(card, base, step if step * (card - 1) < (1 << 32) else 1, shared=rng.random() < 0.3,
                            inv=card <= 1 << 16 and rng.random() < 0.3))
    docs = [int(rng.integers(1, 20_000_000)) for _ in range(nseg)]
    dict_cols = [k for k, c in enumerate(cols) if c["kind"] == _lib.FWD_DICT_FIXEDBIT and c["stored"] != _lib.STRING or
                 c["stored"] == _lib.STRING]
    ngb = int(rng.choice([0, 0, 1, 1, 1, 2, 3]))
    group_by = [int(x) for x in rng.choice(dict_cols, size=min(ngb, len(dict_cols)), replace=False)] if dict_cols else []
    aggs = []
    for _ in range(int(rng.integers(1, 7))):
        fn = int(rng.choice([COUNT, SUM, SUM, MIN, MAX, AVG, DISTINCTCOUNT]))
        aggs.append((fn, -1 if fn == COUNT else int(rng.integers(0, ncols))))
    leaves = []
    for _ in range(int(rng.integers(0, 5))):
        k = int(rng.integers(0, ncols))
        c = cols[k]
        r = rng.random()
        if c["kind"] == _lib.FWD_RAW_FIXEDBYTE:
            leaves.append(node("RAW_RANGE", k, raw=(float(rng.integers(-1000, 0)), float(rng.integers(0, 1000)), 0)))
        elif r < 0.5:
            lo = int(rng.integers(0, max(c["card"], 1)))
            leaves.append(node("SCAN_RANGE", k, lo=lo, hi=lo + int(rng.integers(0, max(c["card"], 1)))))
        elif r < 0.75 and c["bits"] <= 20:   # an IN leaf's bitmap covers every representable dictId of its column
            leaves.append(node("SCAN_IN" if rng.random() < 0.5 else "SCAN_NOT_IN", k,
                               ids=sorted({int(x) for x in rng.integers(0, max(c["card"], 1), size=int(rng.integers(1, 4)))})))
        elif r < 0.85 and c["inv"]:
            leaves.append(node("INV_IN", k, ids=[int(rng.integers(0, max(c["card"], 1)))]))
        elif r < 0.92:
            leaves.append(node("DOC_RANGES", ids=[0, 100]))
        else:
            leaves.append(node("MATCH_ALL"))
    filt = list(leaves)
    if len(leaves) > 1:
        if rng.random() < 0.5:
            filt.append(node("AND", children=len(leaves)))
        else:   # nested: (l0 OR l1) AND NOT(rest...)
            filt = [leaves[0], leaves[1], node("OR", children=2)] + leaves[2:]
            filt.append(node("AND", children=1 + len(leaves) - 2))
            if rng.random() < 0.5:
                filt.append(node("NOT"))
    flags = (Q_MERGE if rng.random() < 0.4 else 0)
    if flags & Q_MERGE and rng.random() < 0.3:
        flags |= Q_DEFER_FINALIZE
    knobs = {}
    if rng.random() < 0.5:
        for name, choices in (("warps", [6, 8]), ("ctas_per_sm", [1, 2]), ("stages", [0, 2, 3]), ("smem_copies", [0, 1, 2, 4, 32, 3]),
                              ("dense_max", [1 << 24, 1 << 16]), ("defer", [0, 1]), ("gb_defer", [0, 1]), ("pack_count", [0, 1]),
                              ("table_stride", [0, 1, 4]), ("smem_groups", [0, 1]), ("grid", [0, 0, 77]), ("always_count", [0, 1])):
            if rng.random() < 0.3:
                knobs[name] = int(rng.choice(choices))
    q = make_query(filt, aggs, group_by=group_by, flags=flags, limit=int(rng.choice([100, 100_000, 5_000_000])),
                   reduce_world=int(rng.choice([0, 1, 2, 8])), merged_docs_bound=int(rng.choice([0, 0, 1 << 33])))
    return [cols] * nseg, docs, q, knobs, dict(flags=flags, aggs=aggs, group_by=group_by)


def _bits(x):
    return int(x).bit_length()


def test_plan_invariants_over_a_seeded_sweep(probe):
    rng = np.random.default_rng(20261015)
    planned = refused = 0
    for i in range(3000):
        seg_cols, docs, (q, keep), knobs, shape = _random_shape(rng)
        rc, p = plan(probe, seg_cols, docs, q, knobs=knobs, carrier=bool(rng.random() < 0.9))
        if rc != 0:
            assert rc in (_lib.E_INVALID, _lib.E_UNSUPPORTED), (i, rc)
            refused += 1
            continue
        planned += 1
        ctx = (i, knobs, shape)
        group_by = bool(shape["group_by"])
        assert 2 <= p.stages <= MAX_STAGES, ctx
        assert p.smem_bytes <= H100[1] // p.ctas_per_sm, ctx
        assert p.queue_off + (p.warps * 2048 if group_by else 0) <= p.smem_table_off <= p.smem_bytes, ctx
        if p.smem_groups:
            nsum = sum(1 for a in range(MAX_AGGS) if p.smem_slot[a] >= 0)
            assert p.smem_gstride % 2 == 1 and p.smem_gstride >= p.smem_groups, ctx
            assert p.smem_table_off + p.smem_copies * p.smem_gstride * 4 * (p.smem_count + 2 * nsum) <= p.smem_bytes, ctx
            copies_knob = knobs.get("smem_copies", 0)
            if copies_knob == 0 or copies_knob & (copies_knob - 1) == 0:
                assert p.smem_copies in (1, 2, 4, 8, 16, 32), ctx
            if p.smem_count == 0:
                assert all(p.carrier_agg[r] >= 0 for r in range(p.nres)), ctx
        for r in range(p.nres if group_by else 0):
            a = p.carrier_agg[r]
            if a >= 0:
                c = shape["aggs"][a][1]
                segs = range(len(docs)) if shape["flags"] & Q_MERGE else [r]
                vals = [np.frombuffer(seg_cols[s][c]["host"], dtype=np.int32) for s in segs]
                rng_ = max(int(v[-1]) for v in vals) - min(int(v[0]) for v in vals)
                n = sum(docs[s] for s in segs)
                if shape["flags"] & Q_DEFER_FINALIZE:
                    n = q.merged_docs_bound if q.merged_docs_bound > 0 else n * max(q.reduce_world, 1)
                assert _bits(n) + _bits(rng_) <= 63, ctx
                assert p.carrier_vmin[r] == min(int(v[0]) for v in vals), ctx
            if p.stride[r] > 1:
                assert p.smem_groups == 0 and all(f != DISTINCTCOUNT for f, _ in shape["aggs"]), ctx
        for s in range(len(docs)):
            nd, na = p.seg_num_defer_codes[s], p.seg_num_agg_codes[s]
            assert nd <= 2 and (nd == 0 or group_by), ctx
            codes = [p.seg_agg_code[s * MAX_AGGS + k] for k in range(na)]
            for k, code in enumerate(codes):
                fn, vk = code >> 4 & 7, code >> 8 & 7
                if k >= na - nd:
                    assert fn in (MIN, MAX) or (fn in (SUM, AVG) and vk in (VAL_DICT_I32, VAL_DICT_F32)), ctx
            if not group_by and p.defer_agg >= 0:   # aggregation only: the deferred sum is the last code
                assert codes[-1] & 7 == p.defer_agg, ctx
                nd = 1
            head, tail = [c & 7 for c in codes[:na - nd]], [c & 7 for c in codes[na - nd:]]
            assert head == sorted(head) and tail == sorted(tail), ctx
        assert tuple(p.variant) in VARIANTS and p.variant[0] == p.warps, ctx
        for c in range(p.num_chunks):
            if knobs.get("grid", 0) > 0:
                assert p.chunk_grid[c] == knobs["grid"], ctx
            else:
                assert 1 <= p.chunk_grid[c] <= H100[0] * p.ctas_per_sm, ctx
        assert p.num_chunks == -(-len(docs) // 16), ctx
    assert planned > 1000 and refused > 100, (planned, refused)
