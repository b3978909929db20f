"""-m gpu, one GPU: the cross-GPU combine (pinot_b200.distributed.execute_and_combine) end to end, with 2 and 3 simulated
ranks over the loopback collective (tests/loopback_dist.py), against the exact reference.

Every rank is set up as a deployment sets up one GPU: its own B200Context on cuda:0, its own segments (per-segment
dictionaries that differ, a different number of segments per rank, sizes 1, 8 193 and ragged tails), its own parsed
query, and a table-wide dictionary domain from global_domain.  The tensors the combine reduces are the library's own
device tables (device_buffers); the loopback reduces them with torch in rank order.  A recording DeviceBackend tells
which route each query took:

  dense    the per-rank dense tables are reduced (count carrier in the int64 block, its verdict in the i64 tail)
  host     DISTINCTCOUNT, or per-GPU hash tables: rows merged by key on the root
  scalars  aggregation only

Every result on the root is held to the exact reference over the union of all ranks' segments (exact_ref.check_exact)
and to the oracle's per-segment tables merged by value (reduce_util.combine); non-root ranks get None.  Statistics:
documents scanned and total documents equal the oracle's sums; the entries scanned in and after the filter, which count
the device plan's own work, equal the sums of each rank's single-GPU results.

The in-library NCCL combine (pb200_result_combine) runs at world size 1 only: a communicator of one rank, with tables
sized for a reduce over two (tail and flag slot).  A real two-rank NCCL reduce needs two GPUs (tests/test_gpu_multi.py).
"""
import contextlib
import ctypes as C

import numpy as np
import pytest

from exact_ref import check_exact
from gpu_util import assert_tables_equal, oracle_table, to_device, tuned
from loopback_dist import run_ranks, values
from pinot_b200 import _lib, sql
from pinot_b200.distributed import DeviceBackend, execute_and_combine, global_domain
from pinot_b200.plan_maker import B200Context, B200PlanMaker, order_spec
from reduce_util import combine
from test_gpu_order_by import assert_rows, ordered_reference

pytestmark = pytest.mark.gpu

INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1
DOMAIN = ["k", "j", "s", "fk", "v", "l", "f", "d", "t3", "hv"]
# per rank: segment sizes (ranks hold different numbers of segments)
SIZES = {0: [1, 8_193, 20_011], 1: [5_003, 8_194], 2: [12_345, 3]}
# k = 1000 + rank * 10 + i: groups that only one rank has; k = 5000 / 5001: one row in all of the table, on rank 1,
# whose raw INT is INT_MIN / INT_MAX
STRS = np.array([f"s{i:02d}".encode() for i in range(20)])


def _segment(oracle, rank, i, n):
    rng = np.random.default_rng(1000 + 17 * rank + i)

    def pool(values, size):   # a per-segment dictionary: a different subset of the column's values in every segment
        return np.asarray(values)[np.sort(rng.choice(len(values), size=min(size, len(values)), replace=False))]

    def pick(p):
        return p[rng.integers(0, len(p), size=n)]
    pk = np.concatenate([pool(np.arange(60) * 3 - 50, 30 + 5 * i + 3 * rank), 1000 + rank * 10 + np.arange(4)])
    cols = {"k": pick(pk).astype(np.int32),
            "j": rng.integers(0, 7, size=n).astype(np.int32),
            "s": pick(pool(STRS, 12 + i)),
            "fk": pick(pool(np.arange(16, dtype=np.float32) / np.float32(4.0) - np.float32(2.0), 9 + rank)),
            "v": pick(pool(np.arange(2000) - 1000, 300)).astype(np.int32),
            "l": pick(pool(np.arange(10_000, dtype=np.int64) * 1_000_003 - (1 << 40), 40)),
            "f": pick(pool((np.arange(300) / 8.0 - 10.0).astype(np.float32), 25 + i)),
            "d": pick(pool(np.round(np.random.default_rng(7).standard_normal(500) * 1e6, 3), 60)),
            "t3": rng.integers(0, 3, size=n).astype(np.int32),
            # heavy on rank 0 only: a count-carrying SUM(hv) overflows a small sum field there and nowhere else
            "hv": (pick(np.arange(10)) + (1_000_000 if rank == 0 else 0)).astype(np.int32),
            "ri": rng.integers(-50_000, 50_000, size=n).astype(np.int32)}
    cols["ri"][rng.random(n) < 0.01] = INT_MIN
    cols["ri"][rng.random(n) < 0.01] = INT_MAX
    if rank == 1 and i == 0:
        cols["k"][:2] = [5000, 5001]
        cols["ri"][:2] = [INT_MIN, INT_MAX]
    return oracle.build_segment(f"cl{rank}s{i}", cols, raw=["ri"])


class RecordingBackend(DeviceBackend):
    """DeviceBackend that records the route of every execution and the carrier state of every dense pass."""

    def __init__(self, pm):
        super().__init__(pm)
        self.routes, self.passes = [], []
        inner, rec = pm, self

        class _PlanMaker:
            ctx = pm.ctx

            def execute_segments(self, segments, query, **kw):
                rec.routes.append("host" if kw.get("ordered") is False else "dense" if kw.get("reduce_world") else "scalars")
                blocks = inner.execute_segments(segments, query, **kw)
                if rec.routes[-1] == "dense":
                    b = blocks[0]
                    rec.passes.append(dict(no_carrier=kw["no_count_carrier"], carrier=b.count_carrier,
                                           unsafe=b.carrier_unsafe, flag_slot=b.flag_slot))
                return blocks
        self.pm = _PlanMaker()


class Cluster:
    def __init__(self, oracle, world):
        self.world = world
        self.hosts = [[_segment(oracle, r, i, n) for i, n in enumerate(SIZES[r])] for r in range(world)]
        self.ctxs = [B200Context(0) for _ in range(world)]
        self.pms = [B200PlanMaker(c) for c in self.ctxs]
        self.devs = []
        for c, hs in zip(self.ctxs, self.hosts):
            with tuned(c, raw_dict_max=0):   # "ri" stays a raw 32-bit column
                self.devs.append([to_device(c, h) for h in hs])
        self.doms = values(run_ranks(world, lambda dist: global_domain(self.ctxs[dist.get_rank()], self.devs[dist.get_rank()],
                                                                       DOMAIN, dist)))
        self.all_hosts = [h for hs in self.hosts for h in hs]
        self.total_docs = sum(h.num_docs for h in self.all_hosts)

    def close(self):
        for devs in self.devs:
            for d in devs:
                d.destroy()
        for dom in self.doms:
            dom.release()
        for c in self.ctxs:
            c.close()

    @contextlib.contextmanager
    def tuned(self, **knobs):
        with contextlib.ExitStack() as stack:
            for c in self.ctxs:
                stack.enter_context(tuned(c, **knobs))
            yield


@pytest.fixture(scope="module", params=[2, 3], ids=["world2", "world3"])
def cluster(request, oracle):
    cl = Cluster(oracle, request.param)
    yield cl
    cl.close()


def parse(text, **options):
    return sql.parse(text, num_groups_limit=1_000_000, **options)


def combine_all(cl, text, merged_docs_bound=0, **options):
    """execute_and_combine on every rank, each with its own parsed query and recording backend -> (per-rank outcomes,
    backends)."""
    backends = [RecordingBackend(pm) for pm in cl.pms]

    def body(dist):
        r = dist.get_rank()
        q = parse(text, **options)
        got = execute_and_combine(backends[r], cl.devs[r], q, dist, dst=0, merged_docs_bound=merged_docs_bound)
        assert (got is None) == (r != 0), r
        return got
    outcomes = run_ranks(cl.world, body)
    return outcomes, backends


def decode(cl, q, got):
    """The root's block as {key values: [per aggregation]} (reduce_util's form), ids decoded through the domain."""
    seg = cl.devs[0][0]
    rows = 1 if got.num_groups < 0 else got.num_groups
    table = {}
    for g in range(rows):
        key = () if got.num_groups < 0 else tuple(seg.dictionary_value(c, int(got.keys[g, j])) for j, c in enumerate(q.group_by))
        vals = []
        for a, agg in enumerate(q.aggregations):
            fn = agg.function
            vals.append(int(got.longs[a][g]) if fn == "COUNT" else
                        (float(got.doubles[a][g]), int(got.longs[a][g])) if fn == "AVG" else
                        frozenset(seg.dictionary_value(agg.column, int(d)) for d in got.distinct[(a, g)]) if fn == "DISTINCTCOUNT"
                        else float(got.doubles[a][g]))
        assert key not in table, key
        table[key] = vals
    return table


def check(oracle, cl, text, routes, **kw):
    """Runs `text` on every rank and holds the root's result to both references; every rank took `routes`."""
    outcomes, backends = combine_all(cl, text, **kw)
    got = values(outcomes)[0]
    q = parse(text)
    what = f"world {cl.world}: {text}"
    for r, b in enumerate(backends):
        assert b.routes == routes, (what, r, b.routes)
    table = decode(cl, q, got)
    check_exact(oracle, cl.all_hosts, q, table, what)
    parts = [oracle_table(h, q, r) for h in cl.all_hosts for r in [oracle.execute(h, q)]]
    assert_tables_equal(q, table, combine([a.function for a in q.aggregations], parts), what)
    check_stats(oracle, cl, q, got, what)
    return got, backends


def check_stats(oracle, cl, q, got, what):
    mine = [pm.execute_segments(devs, q, merge=True, ordered=False)[0].stats for pm, devs in zip(cl.pms, cl.devs)]
    ref = [oracle.execute(h, q).stats for h in cl.all_hosts]
    st = got.stats
    assert st.num_docs_scanned == sum(s[0] for s in ref), (what, "docs scanned", st.num_docs_scanned)
    assert st.num_total_docs == sum(s[3] for s in ref) == cl.total_docs, (what, "total docs", st.num_total_docs)
    assert st.num_entries_scanned_in_filter == sum(s.num_entries_scanned_in_filter for s in mine), (what, "in filter")
    assert st.num_entries_scanned_post_filter == sum(s.num_entries_scanned_post_filter for s in mine), (what, "post filter")


# ------------------------------------------------------------------------------------------------------------- dense
CARRIER_Q = "SELECT SUM(v), COUNT(*), MAX(l), MIN(f) FROM t WHERE v > -900 GROUP BY k, j"


@pytest.mark.parametrize("knobs", [{}, {"smem_groups": 0}, {"table_stride": 4}, {"gb_defer": 0}],
                         ids=["smem", "global", "stride4", "gb_defer0"])
@pytest.mark.parametrize("bound", ["given", "zero"])
def test_dense_count_carrier(oracle, cluster, knobs, bound):
    """The counts ride in SUM(v) and the verdict in the i64 tail: one pass on every rank, exact."""
    mdb = cluster.total_docs if bound == "given" else 0
    for text in (CARRIER_Q, "SELECT SUM(v), AVG(v) FROM t GROUP BY s"):
        with cluster.tuned(**knobs):
            got, backends = check(oracle, cluster, text, ["dense"], merged_docs_bound=mdb)
        for b in backends:
            assert [p["no_carrier"] for p in b.passes] == [False]
            assert b.passes[0]["carrier"] and b.passes[0]["flag_slot"] and not b.passes[0]["unsafe"], b.passes
        assert got.count_carrier


def test_carrier_off(oracle, cluster):
    with cluster.tuned(pack_count=0):
        got, backends = check(oracle, cluster, CARRIER_Q, ["dense"])
    for b in backends:
        assert len(b.passes) == 1 and not b.passes[0]["carrier"] and not b.passes[0]["flag_slot"], b.passes
    assert not got.count_carrier


def test_carrier_unsafe_on_one_rank(oracle, cluster):
    """A 24-bit sum field: rank 0's SUM(hv) (values near 10^6) cannot be proven to fit, the other ranks' can.  The verdict
    is agreed on: every rank reruns without the carrier, and the result is exact."""
    with cluster.tuned(pack_shift=24):
        got, backends = check(oracle, cluster, "SELECT SUM(hv), COUNT(*) FROM t GROUP BY k", ["dense", "dense"])
    for r, b in enumerate(backends):
        assert [p["no_carrier"] for p in b.passes] == [False, True], (r, b.passes)
        assert b.passes[0]["carrier"] and b.passes[0]["unsafe"] == (r == 0), (r, b.passes)
    assert not got.count_carrier


@pytest.mark.parametrize("text", [
    "SELECT MIN(v), MAX(v), MIN(l), MAX(l), MIN(ri), MAX(ri) FROM t GROUP BY k",
    "SELECT MIN(f), MAX(f), MIN(d), MAX(d), MAX(ri), COUNT(*) FROM t WHERE t3 != 1 GROUP BY k, fk",
    "SELECT MIN(ri), MAX(ri) FROM t WHERE k >= 1000 GROUP BY k",   # groups of one rank; k 5000 / 5001: one raw extreme
], ids=["int_long_raw", "float_double", "one_rank_groups"])
def test_min_max(oracle, cluster, text):
    got, _ = check(oracle, cluster, text, ["dense"])
    if "k >= 1000" in text:
        table = decode(cluster, parse(text), got)
        assert table[(5000,)] == [float(INT_MIN), float(INT_MIN)] and table[(5001,)] == [float(INT_MAX), float(INT_MAX)]
        assert len(table) == 4 * cluster.world + 2


def test_f64_sums(oracle, cluster):
    check(oracle, cluster, "SELECT SUM(l), SUM(f), SUM(d), AVG(d), AVG(f), COUNT(*) FROM t GROUP BY j, t3", ["dense"])


# -------------------------------------------------------------------------------------------------------- host route
def test_hash_tables_take_the_host_route(oracle, cluster):
    with cluster.tuned(dense_max=1):
        check(oracle, cluster, "SELECT SUM(v), COUNT(*), MAX(f), MIN(ri), AVG(l) FROM t WHERE v > 0 GROUP BY k, j, s",
              ["dense", "host"])


@pytest.mark.parametrize("text", [
    "SELECT DISTINCTCOUNT(v), DISTINCTCOUNT(s), SUM(v), MAX(d) FROM t GROUP BY j",
    "SELECT DISTINCTCOUNT(k), DISTINCTCOUNT(fk), COUNT(*), SUM(v), MIN(ri) FROM t WHERE v > 0",
], ids=["group_by", "aggregation_only"])
def test_distinctcount(oracle, cluster, text):
    check(oracle, cluster, text, ["host"])


# ------------------------------------------------------------------------------------------------- aggregation only
@pytest.mark.parametrize("text", [
    "SELECT COUNT(*), SUM(v), AVG(v), MIN(l), MIN(ri), MAX(ri) FROM t WHERE j < 5",
    "SELECT SUM(l), AVG(f), MIN(f), MAX(v), COUNT(*) FROM t",
    # matches rows of rank 0 only: the other ranks' MIN / MAX stay +-inf
    "SELECT COUNT(*), SUM(v), MIN(v), MAX(l), MIN(ri), MAX(d) FROM t WHERE k BETWEEN 1000 AND 1009",
], ids=["filtered", "all_rows", "one_rank_matches"])
def test_scalars(oracle, cluster, text):
    check(oracle, cluster, text, ["scalars"])


def _big_sum_cluster(oracle, world):
    """SUM of INT values near INT_MAX: rank 0 sums to 2^53 + 1 (two segments), rank 1 to 2^53 + 5, rank 2 to 1."""
    n = 1 << 22
    parts = {0: [np.full(n // 2, INT_MAX), np.r_[np.full(n // 2, INT_MAX), 4_194_305]],
             1: [np.r_[np.full(n, INT_MAX), 4_194_309]],
             2: [np.array([1])]}
    hosts, ctxs, devs = [], [], []
    for r in range(world):
        hs = [oracle.build_segment(f"big{r}_{i}", {"b": p.astype(np.int32), "g": np.zeros(len(p), dtype=np.int32)})
              for i, p in enumerate(parts[r])]
        assert sum(int(p.astype(np.int64).sum()) for p in parts[r]) == {0: (1 << 53) + 1, 1: (1 << 53) + 5, 2: 1}[r]
        hosts.append(hs)
        ctxs.append(B200Context(0))
        devs.append([to_device(ctxs[-1], h) for h in hs])
    return hosts, ctxs, devs


@pytest.mark.parametrize("world", [2, 3])
def test_int_sums_beyond_2_53(oracle, world):
    """Each rank's rounded sum is exact only to 2^53: the total must be float(exact), on the scalar and the dense route."""
    hosts, ctxs, devs = _big_sum_cluster(oracle, world)
    try:
        doms = values(run_ranks(world, lambda dist: global_domain(ctxs[dist.get_rank()], devs[dist.get_rank()], ["b", "g"], dist)))
        exact = (1 << 54) + 6 + (1 if world == 3 else 0)
        count = sum(h.num_docs for hs in hosts for h in hs)
        assert float(exact) == 2.0 ** 54 + 8
        for text, route in (("SELECT SUM(b), AVG(b), COUNT(*) FROM t", "scalars"),
                            ("SELECT SUM(b), AVG(b), COUNT(*) FROM t GROUP BY g", "dense")):
            backends = [RecordingBackend(B200PlanMaker(c)) for c in ctxs]
            got = values(run_ranks(world, lambda dist: execute_and_combine(
                backends[dist.get_rank()], devs[dist.get_rank()], parse(text), dist)))[0]
            assert backends[0].routes[0] == route
            assert got.num_groups == (-1 if route == "scalars" else 1)
            assert float(got.doubles[0][0]) == float(exact), (text, float(got.doubles[0][0]).hex(), float(exact).hex())
            assert float(got.doubles[1][0]) == float(exact) and int(got.longs[1][0]) == count, text
            assert int(got.longs[2][0]) == count and got.stats.num_docs_scanned == count, text
        for d in doms:
            d.release()
    finally:
        for ds in devs:
            for d in ds:
                d.destroy()
        for c in ctxs:
            c.close()


# ----------------------------------------------------------------------------------------------------------- ORDER BY
def device_rows(cl, q, got):
    seg = cl.devs[0][0]
    out = []
    for g in range(got.num_groups):
        key = tuple(seg.dictionary_value(c, int(got.keys[g, j])) for j, c in enumerate(q.group_by))
        vals = []
        for a, agg in enumerate(q.aggregations):
            if agg.function in ("COUNT", "DISTINCTCOUNT"):
                vals.append(int(got.longs[a][g]))
            elif agg.function == "AVG":
                n = int(got.longs[a][g])
                vals.append(float(got.doubles[a][g]) / n if n else float("-inf"))
            else:
                vals.append(float(got.doubles[a][g]))
        out.append((key, vals))
    return out


@pytest.mark.parametrize("text,routes,knobs", [
    ("SELECT COUNT(*), MAX(t3), MIN(t3) FROM t GROUP BY k, j ORDER BY MAX(t3) DESC, MIN(t3) LIMIT 7", ["dense"], {}),
    ("SELECT SUM(v), COUNT(*) FROM t GROUP BY s, t3 ORDER BY t3 DESC, COUNT(*) LIMIT 4", ["dense"], {}),
    ("SELECT COUNT(*), MAX(t3), DISTINCTCOUNT(t3) FROM t GROUP BY k, j ORDER BY MAX(t3) DESC, DISTINCTCOUNT(t3) LIMIT 7",
     ["host"], {}),
    ("SELECT COUNT(*), MIN(t3), SUM(v) FROM t GROUP BY k, j ORDER BY MIN(t3), k DESC LIMIT 5", ["dense", "host"],
     {"dense_max": 1}),
], ids=["dense_ties", "dense_key_item", "distinctcount", "hash"])
@pytest.mark.parametrize("trim_option", [0, 1, 5000])
def test_order_by_limit_with_ties(oracle, cluster, text, routes, knobs, trim_option):
    """Rows in ORDER BY order, ties by key ascending, trimmed to max(5 * LIMIT, min_server_group_trim_size) (option 0:
    not trimmed) -- the same rows on the dense and the host route."""
    q = parse(text, min_server_group_trim_size=trim_option)
    trim = order_spec(q, merge=True).trim_size
    with cluster.tuned(**knobs):
        outcomes, backends = combine_all(cluster, text, min_server_group_trim_size=trim_option)
        got = values(outcomes)[0]
        check_stats(oracle, cluster, q, got, text)
    assert all(b.routes == routes for b in backends), [b.routes for b in backends]
    want = ordered_reference(oracle, cluster.all_hosts, q)
    if trim_option == 1:
        assert 0 < trim < len(want)
    assert_rows(device_rows(cluster, q, got), want, trim, f"world {cluster.world}: {text} trim={trim}")


# ---------------------------------------------------------------------------------------------------------- refusals
@pytest.mark.parametrize("text,knobs", [
    ("SELECT SUM(v), COUNT(*) FROM t GROUP BY k HAVING COUNT(*) > 3", {}),
    ("SELECT DISTINCTCOUNT(v) FROM t GROUP BY j HAVING DISTINCTCOUNT(v) > 2", {}),
    ("SELECT SUM(v) FROM t GROUP BY k, j HAVING SUM(v) > 0", {"dense_max": 1}),
    ("SELECT SUM(v), COUNT(*) FROM t GROUP BY k HAVING MAX(l) > 0 ORDER BY COUNT(*) LIMIT 3", {}),
    ("SELECT PERCENTILE(v, 50) FROM t GROUP BY j", {}),
    ("SELECT PERCENTILE(v, 90), COUNT(*) FROM t", {}),
    ("SELECT VAR_POP(v) FROM t GROUP BY j", {}),
    ("SELECT STDDEV_SAMP(v) FROM t", {}),
    ("SELECT LASTWITHTIME(v, l, 'INT') FROM t GROUP BY j", {}),
    ("SELECT FIRSTWITHTIME(v, l, 'INT') FROM t", {}),
], ids=["having_dense", "having_distinctcount", "having_hash", "having_order_by", "percentile_gb", "percentile",
        "var_gb", "stddev", "lastwithtime", "firstwithtime"])
def test_refusals_come_before_any_collective(cluster, text, knobs):
    with cluster.tuned(**knobs):
        outcomes, backends = combine_all(cluster, text)
    for r, o in enumerate(outcomes):
        assert isinstance(o.error, _lib.UnsupportedQueryError), (text, r, repr(o.error))
        assert o.calls == [], (text, r, o.calls)
        assert backends[r].routes == [], (text, r, backends[r].routes)


# ------------------------------------------------------------------------------------------ native combine, world 1
def test_native_combine_at_world_1(oracle, cluster):
    """pb200_result_combine over a one-rank NCCL communicator: tables sized for a reduce over two ranks (tail and flag
    slot), the verdict read from the tail, the speculative extraction, the retry and the scalar combine.  This is not a
    two-rank NCCL reduce."""
    if cluster.world != 2:
        pytest.skip("runs once")
    ctx, pm, devs, hosts = cluster.ctxs[0], cluster.pms[0], cluster.devs[0], cluster.hosts[0]
    L = ctx.lib
    buf = (C.c_ubyte * 128)()
    rc = L.pb200_comm_unique_id(buf)
    if rc == _lib.E_UNSUPPORTED:
        pytest.skip(L.pb200_last_error().decode())
    _lib.check(rc)
    _lib.check(L.pb200_comm_init(ctx.handle, bytes(buf), 0, 1))
    ctx.comm_rank = 0
    try:
        be = DeviceBackend(pm)

        def single(text, got):
            q = parse(text)
            table = decode(cluster, q, got)
            check_exact(oracle, hosts, q, table, f"native: {text}")
            want = combine([a.function for a in q.aggregations], [oracle_table(h, q, oracle.execute(h, q)) for h in hosts])
            assert_tables_equal(q, table, want, f"native: {text}")
            assert got.stats.num_docs_scanned == sum(oracle.execute(h, q).stats[0] for h in hosts)
            assert got.stats.num_total_docs == sum(h.num_docs for h in hosts)

        q = parse(CARRIER_Q)
        block = be.execute(devs, q, 2, 0, False)
        assert block.count_carrier and block.flag_slot and not block.carrier_unsafe
        got, retry = be.combine_native(block, q, 0)
        assert not retry
        single(CARRIER_Q, got)

        text = "SELECT SUM(hv), COUNT(*) FROM t GROUP BY k"
        q = parse(text)
        with tuned(ctx, pack_shift=24):
            block = be.execute(devs, q, 2, 0, False)
            assert block.count_carrier and block.carrier_unsafe
            got, retry = be.combine_native(block, q, 0)
            assert retry and got is None and block.handle is None
            block = be.execute(devs, q, 2, 0, True)
            assert not block.count_carrier
            got, retry = be.combine_native(block, q, 0)
        assert not retry
        single(text, got)

        text = "SELECT COUNT(*), SUM(v), AVG(v), MIN(ri), MAX(d), SUM(d) FROM t WHERE j < 5"
        q = parse(text)
        block = pm.execute_segments(devs, q, merge=True, keep_handle=True, defer=False)[0]
        exact = C.c_int64()
        assert L.pb200_result_exact_sum(block.handle, 1, C.byref(exact)) == 1
        assert L.pb200_result_exact_sum(block.handle, 5, C.byref(exact)) == 0   # DOUBLE: summed in double
        got, retry = be.combine_native(block, q, 0)
        assert not retry and got.num_groups == -1
        single(text, got)
    finally:
        L.pb200_comm_shutdown(ctx.handle)
        del ctx.comm_rank
