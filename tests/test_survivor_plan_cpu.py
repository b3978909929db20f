"""CPU tests of tests/survivor_plan.py: the designed segments are what they claim, and every query shape x tuning knobs that
tests/test_gpu_survivor_edges.py runs gets the plan it is meant to exercise there (pb200::plan_scan through the host probe
of tests/test_scan_plan_cpu.py, on the metadata of the very columns the GPU test loads).  When a planner change moves a
shape off its route, this file fails instead of the GPU test silently covering another path."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import survivor_plan as sp
from filter_ref import matching_docs_many
from pinot_b200 import _lib, sql
from pinot_b200.query import Filter, Predicate
from test_scan_plan_cpu import make_query, node, plan, probe  # noqa: F401
from test_scan_spec_plan_cpu import route as spec_route

HERE = os.path.dirname(os.path.abspath(__file__))

SEG_LEAF_DOCMASK = 4   # pb200_desc.h LeafKind: LEAF_DOCMASK


@pytest.fixture(scope="module")
def built(oracle):
    """{set name: [(Planned, host segment)]}: the first segments of each set the GPU test uses, and one of the long ones."""
    out = {}
    for name, plans in (("w6", sp.hand_over_plans(6)[:3] + sp.hand_over_plans(6)[-2:]),
                        ("w8", sp.hand_over_plans(8)[:3] + sp.hand_over_plans(8)[-2:]),
                        ("big", [sp.long_plan("big0", 73, 77)])):
        out[name] = []
        for k, p in enumerate(plans):
            pl = sp.build_columns(p, 1000 + k)
            out[name].append((pl, oracle.build_segment(p.name, pl.columns, inverted=["inv"], raw=["r"])))
    return out


# ---------------------------------------------------------------------------------------------------- the plan is what it claims
def test_designed_rows_are_the_filter_survivors(oracle, built):
    """matching_docs of `p1 = 1 AND p2 = 1`, of the first leaf alone and of `inv = 0 AND ...` gives the planned rows,
    slice by slice and lane by lane."""
    for name, segs in built.items():
        for pl, seg in segs:
            q_both, q_first, q_inv = (sql.parse(f"SELECT COUNT(*) FROM t WHERE {w}").filter
                                      for w in (sp.F, "p1 = 1", sp.FI))
            both, first, inv = matching_docs_many(oracle, seg, [q_both, q_first, q_inv])
            assert np.array_equal(both, pl.designed), pl.plan.name
            assert np.array_equal(first, pl.designed | pl.decoy), pl.plan.name
            assert np.array_equal(inv, pl.designed & ~pl.skipped), pl.plan.name
            for i, sl in enumerate(pl.plan.slices):
                lo, hi = i * sp.SLICE, min((i + 1) * sp.SLICE, seg.num_docs)
                lanes, pre = sp.per_lane(both[lo:hi]), sp.per_lane(first[lo:hi])
                assert lanes.sum() == sl.s, (pl.plan.name, i, sl)
                if sl.layout == "spread":
                    assert lanes.max() - lanes.min() <= 1, (pl.plan.name, i, sl)
                elif sl.layout == "one_lane":
                    assert lanes[sl.lane] == sl.s, (pl.plan.name, i, sl)
                else:
                    assert np.array_equal(np.nonzero(both[lo:hi])[0], np.arange(sl.s)), (pl.plan.name, i, sl)
                rows = hi - lo
                full = [min(32, rows - 32 * k) for k in range(32)]
                want = [max(int(lanes[k]), min(sl.pre, max(full[k], 0))) for k in range(32)]
                assert list(pre) == want, (pl.plan.name, i, sl)
                assert bool(sl.skipped) == bool(pl.skipped[lo]), (pl.plan.name, i)


def test_every_nonzero_edge_meets_every_successor_under_grid_1():
    """Under grid 1 each warp takes its slices in consecutive tiles: every non-zero S edge is followed in the same warp
    by a non-zero S, by S = 0, by a skipped slice, by the ragged last slice and by the segment's end, for W = 6 and 8."""
    for warps in (6, 8):
        seen = {s: set() for s in sp.NONZERO}
        for p in sp.hand_over_plans(warps):
            for sl, nxt in sp.successors(p, warps):
                if sl.s == 0 or sl.skipped:
                    continue
                seen.setdefault(sl.s, set()).add(nxt if isinstance(nxt, str) else "skipped" if nxt.skipped else "zero" if nxt.s == 0 else "nonzero")
        for s in sp.NONZERO:
            kinds = seen[s]
            assert kinds >= {"nonzero", "zero", "skipped", "ragged", "end"}, (warps, s, kinds)
        items = {(sl.s, sl.layout) for p in sp.hand_over_plans(warps) for sl in p.slices}
        assert items >= {(it.s, it.layout) for it in sp.all_items()}, warps


def test_segment_sizes_cover_the_tile_edges():
    sizes = [p.num_docs for p in sp.hand_over_plans(6)] + [p.num_docs for p in sp.hand_over_plans(8)]
    assert len(sp.hand_over_plans(6)) >= 17 and len(sp.hand_over_plans(8)) >= 17   # two launch chunks
    assert any(n % 1024 == 0 for n in sizes) and any(n % 1024 == 1 for n in sizes) and any(n % 1024 == 1023 for n in sizes)
    assert any(n % (6 * 1024) == 0 for n in sizes) and any(n % (8 * 1024) == 0 for n in sizes)
    assert max(sizes) <= 200_000 and sp.long_plan("big", 73, 77).num_docs <= 200_000


# ---------------------------------------------------------------------------------------------------- each route is the route it claims
def _probe_columns(seg):
    """test_scan_plan_cpu.col() records of the segment's columns as the device loads them: bit-packed dictIds (a sorted
    column too), raw INT kept raw."""
    out = []
    for k, c in enumerate(seg.columns):
        if not c.has_dictionary:
            out.append(dict(kind=_lib.FWD_RAW_FIXEDBYTE, stored=c.data_type, bits=32, card=c.cardinality, native=False,
                            shared=False, inv=False, hash=0, host=None, cbuf=None))
            continue
        host = np.asarray(c.dict_values).astype(np.int32).tobytes() if c.data_type == _lib.INT else None
        out.append(dict(kind=_lib.FWD_DICT_FIXEDBIT, stored=c.data_type,
                        bits=c.bits, card=c.cardinality, native=True, shared=False, inv=c.inv is not None and not c.is_sorted,
                        hash=hash((seg.name, c.name)) & (2**63 - 1), host=host,
                        cbuf=C.create_string_buffer(host, len(host)) if host else None))
    return out


def _probe_query(seg, q, flags=0):
    """The device form of a query over `seg`: EQ leaves -> SCAN_IN of one dictId (INV_IN on an inverted column)."""
    names = [c.name for c in seg.columns]
    nodes = []

    def walk(n):
        if isinstance(n, Filter):
            for ch in n.children:
                walk(ch)
            nodes.append(node(n.type, children=len(n.children)))
            return
        assert isinstance(n, Predicate) and n.type == "EQ", n
        c = seg.column(n.column)
        dict_id = int(np.searchsorted(np.asarray(c.dict_values), n.values[0]))
        nodes.append(node("INV_IN" if c.inv is not None else "SCAN_IN", names.index(n.column), ids=[dict_id]))
    if q.filter is not None:
        walk(q.filter)
    aggs = [(_lib.AGG_CODES[a.function], -1 if a.column is None else names.index(a.column)) for a in q.aggregations]
    return make_query(nodes, aggs, group_by=[names.index(g) for g in q.group_by], flags=flags, limit=q.num_groups_limit)


@pytest.fixture(scope="module")
def spec_probe(probe):
    """tests/spec_probe/spec_probe.cpp, built as tests/test_scan_spec_plan_cpu.py builds it (after `probe` built the
    library): whether plan_scan picks the kernel specialised for the shared-table shape."""
    src = os.path.join(HERE, "spec_probe", "spec_probe.cpp")
    out = os.path.join(HERE, "spec_probe", "libspec_probe.so")
    libdir = os.path.join(os.path.dirname(HERE), "pinot_b200")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(src), os.path.getmtime(_lib.LIB_PATH)):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", f"-I{cuda_inc}", "-o", out, src, f"-L{libdir}",
                        "-lpinot_b200", f"-Wl,-rpath,{libdir}"], check=True)
    lib = C.CDLL(out)
    lib.probe_spec_route.restype = C.c_int32
    return lib


def _route_plan(probe, seg, text, knobs, flags=0):
    q = sql.parse(text)
    hq, keep = _probe_query(seg, q, flags)
    rc, p = plan(probe, [_probe_columns(seg)], [seg.num_docs], hq, knobs=knobs)
    assert rc == 0, probe.last_error()
    return p


def _spec(spec_probe, seg, text, knobs):
    hq, keep = _probe_query(seg, sql.parse(text))
    r = spec_route(spec_probe, [_probe_columns(seg)], [seg.num_docs], hq, knobs=knobs)
    assert r[0] == 0
    return r[1]


def _fields(p, spec):
    """(W, SPEC, DEFER, smem_groups, smem_copies, hashed, num_defer_codes, defer_agg, sparse_max, sparse_max_agg,
    carrier_agg)"""
    return (p.variant[0], spec, p.variant[2], p.smem_groups, p.smem_copies, p.hashed[0], p.seg_num_defer_codes[0],
            p.defer_agg, p.sparse_max, p.sparse_max_agg, p.carrier_agg[0])


@pytest.mark.parametrize("rid, knobs, segset, queries", sp.ROUTES, ids=[r[0] for r in sp.ROUTES])
def test_route_plan(probe, spec_probe, built, rid, knobs, segset, queries):
    for text in queries:
        for pl, seg in built[segset]:
            got = _fields(_route_plan(probe, seg, text, knobs), _spec(spec_probe, seg, text, knobs))
            want = sp.EXPECTED_PLAN[(rid, text)]
            if want[3] is None:   # GROUP BY blk: a shared table of one entry per 16-row block
                assert got[3] == seg.column("blk").cardinality and got[4] >= 1, (rid, text, pl.plan.name, got)
                got = got[:3] + (None, None) + got[5:]
            assert got == want, (rid, text, pl.plan.name)


@pytest.mark.parametrize("knobs", [{}, {"spec": 0}])
def test_p1_leaf_runs_before_the_p2_leaf(probe, built, knobs):
    """The planner orders a conjunction by the matching fraction of the dictionary: p1 (1 of 4 dictIds) before p2 (1 of
    2), whatever their order in the query, after the doc mask of `inv = 0`.  So the decoys (p1 only) reach the p2 leaf.
    Seen through `p1 = 2 AND p2 = 0` (dictIds 2 and 0: the same fractions)."""
    pl, seg = built["w6"][0]
    for text in (sp.GB_SPEC, sp.GB_INV, sp.AGG_SUM, sp.MIX4):
        for a, b in (("p1 = 2", "p2 = 0"), ("p2 = 0", "p1 = 2")):
            p = _route_plan(probe, seg, text.replace("p1 = 1 AND p2 = 1", f"{a} AND {b}"), knobs)
            kinds = [p.seg_leaf_kind[l] for l in range(3 if "inv" in text else 2)]
            scan = [l for l, k in enumerate(kinds) if k != SEG_LEAF_DOCMASK]
            assert kinds[0] == SEG_LEAF_DOCMASK or "inv" not in text, (text, kinds)
            assert [p.seg_leaf_lo[l] for l in scan] == [2, 0] and [p.seg_leaf_span[l] for l in scan] == [1, 1], (text, a, b)


# ---------------------------------------------------------------------------------------------------- the hash table
def test_hash_copy_matches_splitmix64():
    """mix64_32 is the SplitMix64 finaliser: its first output from state 0 is mix(0x9E3779B97F4A7C15) =
    0xE220A8397B1DCDAF (low half 0x7B1DCDAF); the numpy copy agrees with the scalar one."""
    assert sp.mix64_32(0x9E3779B97F4A7C15) == 0x7B1DCDAF
    z = np.array([0, 1, 2047, 2048 * 2048 - 1, 123_456_789], dtype=np.int64)
    assert list(sp.mix64_32_np(z)) == [sp.mix64_32(int(x)) for x in z]


@pytest.mark.parametrize("limit", [300, 32_767, 32_768, 100_000])
def test_hash_capacity_and_wrapping_keys_match_the_plan(oracle, probe, limit):
    """A hashed two-column key (2 048 x 2 048 dictIds, dense_max 1): the plan's table has hash_capacity(limit) slots,
    and the chosen pairs' raw keys (column 0 least significant) hash into its last 16 slots."""
    cap = sp.hash_capacity(limit)
    assert cap >= 2 * (limit + 1) and cap >= 1 << 16 and cap & (cap - 1) == 0 and (cap == 1 << 16 or cap < 4 * (limit + 1))
    pairs = sp.keys_at_table_end(2048, 2048, limit, 48)
    assert len(set(pairs)) == 48
    for a, b in pairs:
        assert sp.mix64_32(sp.raw_key((a, b), (2048, 2048))) & (cap - 1) >= cap - 16
    pl = sp.hash_segment_columns(sp.distinct_pairs(pairs, 2048, 300), 2048, 11)
    seg = oracle.build_segment("hash_probe", pl.columns, inverted=["inv"], raw=["r"])
    for text in (f"SELECT SUM(v), COUNT(*) FROM t WHERE {sp.F} GROUP BY ha, hb", "SELECT MIN(v) FROM t GROUP BY ha, hb"):
        q = sql.parse(text, num_groups_limit=limit)
        hq, keep = _probe_query(seg, q)
        rc, p = plan(probe, [_probe_columns(seg)], [seg.num_docs], hq, knobs={"dense_max": 1})
        assert rc == 0, probe.last_error()
        assert (p.hashed[0], p.groups[0], p.smem_groups) == (1, cap, 0), text
    # the designed rows carry exactly the pairs, the last two in the pipelined last batch (queue entries 128, 129)
    rows = np.nonzero(pl.designed)[0]
    got = list(zip(pl.columns["ha"][rows].tolist(), pl.columns["hb"][rows].tolist()))
    assert set(got) == set(sp.distinct_pairs(pairs, 2048, 300))
    assert rows[-2] % 1024 == 128 and rows[-1] % 1024 == 129
    assert got[-2] not in got[:-2] and got[-1] not in got[:-2]
