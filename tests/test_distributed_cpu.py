"""world_size-2 gloo tests (CPU) of the multi-GPU host logic: segment sharding and the table reduce semantics."""
import os

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from pinot_b200.distributed import reduce_buffers, shard_segments


def test_shard_segments_covers_everything_once():
    for n, w in [(64, 8), (8, 8), (7, 2), (3, 4), (1, 1), (0, 2)]:
        got = [shard_segments(n, w, r) for r in range(w)]
        flat = [s for part in got for s in part]
        assert flat == list(range(n))
        assert max(len(p) for p in got) - min(len(p) for p in got) <= 1


def _worker(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    rng = np.random.default_rng(100 + rank)
    G = 1000
    count = rng.integers(0, 5, size=G)
    sums = rng.integers(-10**12, 10**12, size=G) * (count > 0)
    fsum = rng.random(G) * (count > 0)
    mx = np.where(count > 0, rng.integers(0, 2**31 - 2, size=G) + 1, 0).astype(np.uint32)      # dictId + 1, 0 = empty
    mn = np.where(count > 0, rng.integers(0, 2**32 - 2, size=G), 0xFFFFFFFF).astype(np.uint32)  # raw order-preserving
    np.savez(os.path.join(out_dir, f"in{rank}.npz"), count=count, sums=sums, fsum=fsum, mx=mx, mn=mn)
    bufs = {"i64": torch.from_numpy(np.concatenate([count, sums]).astype(np.int64)),
            "f64": torch.from_numpy(fsum.copy()),
            "u32max": torch.from_numpy(mx.view(np.int32).copy()),
            "u32min": torch.from_numpy(mn.view(np.int32).copy())}
    reduce_buffers(bufs, dist, dst=0)
    if rank == 0:
        np.savez(os.path.join(out_dir, "out.npz"), i64=bufs["i64"].numpy(), f64=bufs["f64"].numpy(),
                 mx=bufs["u32max"].numpy().view(np.uint32), mn=bufs["u32min"].numpy().view(np.uint32))
    dist.destroy_process_group()


def test_reduce_buffers_world_size_2(tmp_path):
    world = 2
    port = 29500 + (os.getpid() % 2000)
    mp.spawn(_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    ins = [np.load(tmp_path / f"in{r}.npz") for r in range(world)]
    out = np.load(tmp_path / "out.npz")
    G = 1000
    assert np.array_equal(out["i64"][:G], sum(i["count"] for i in ins))          # COUNT merge = a + b
    assert np.array_equal(out["i64"][G:], sum(i["sums"] for i in ins))           # SUM merge (exact integers)
    assert np.allclose(out["f64"], sum(i["fsum"] for i in ins), rtol=1e-12)
    assert np.array_equal(out["mx"], np.maximum(ins[0]["mx"], ins[1]["mx"]))     # MAX merge, 0 = empty loses
    assert np.array_equal(out["mn"], np.minimum(ins[0]["mn"], ins[1]["mn"]))     # MIN merge, 0xFFFFFFFF = empty loses


# ------------------------------------------------------------------------------------------------------------------
# execute_and_combine end to end on CPU: the control flow of pinot_b200.distributed (flag all-reduce, table reduce,
# collective fallback) over tables built from the ORACLE's per-segment results in the device library's table layout
# (raw-key dense tables, count carrier in the upper bits of the first INT sum), against the oracle-side merge by value.
# ------------------------------------------------------------------------------------------------------------------
class _Block:
    def __init__(self, bufs, count_carrier, carrier_unsafe, layout):
        self.bufs, self.count_carrier, self.carrier_unsafe, self.layout = bufs, count_carrier, carrier_unsafe, layout


class OracleBackend:
    """Stands in for DeviceBackend on a GPU-less box: same interface, tables computed by the CPU oracle."""

    def __init__(self, oracle, force_shift=0):
        self.oracle, self.force_shift = oracle, force_shift
        self.passes = []

    def execute(self, segments, query, reduce_world, merged_docs_bound, no_count_carrier):
        from reduce_util import normalise
        fns = [a.function for a in query.aggregations]
        cards = [segments[0].column(c).cardinality for c in query.group_by]
        groups = int(np.prod(cards))
        need_count = any(f in ("COUNT", "AVG") for f in fns)
        has_minmax = any(f in ("MIN", "MAX") for f in fns)
        carrier = -1
        if not no_count_carrier and (need_count or not has_minmax):
            carrier = next((a for a, ag in enumerate(query.aggregations) if ag.function in ("SUM", "AVG")), -1)
        # the library's field sizing (pb200_plan.cpp "count carrier"): balanced fields from the dictionary's value range
        dv = segments[0].column(query.aggregations[carrier].column).dict_values if carrier >= 0 else np.zeros(1, dtype=np.int64)
        vmin, rbits = int(dv.min()), int(int(dv.max()) - int(dv.min())).bit_length()
        shift = self.force_shift or (64 + rbits + 1) // 2
        count = np.zeros(groups, dtype=np.int64)
        isum = {a: np.zeros(groups, dtype=np.int64) for a, f in enumerate(fns) if f in ("SUM", "AVG")}
        gmax = {a: np.zeros(groups, dtype=np.uint32) for a, f in enumerate(fns) if f == "MAX"}
        gmin = {a: np.full(groups, 0xFFFFFFFF, dtype=np.uint32) for a, f in enumerate(fns) if f == "MIN"}
        for seg in segments:
            r = self.oracle.execute(seg, query)
            raw = np.zeros(r.num_groups, dtype=np.int64)
            mult = 1
            for j, c in enumerate(cards):
                raw += r.keys[:, j].astype(np.int64) * mult
                mult *= c
            # per-group row counts of this segment (COUNT(*) with the same filter and keys)
            from pinot_b200 import sql as _sql
            cq = _sql.parse("SELECT COUNT(*) FROM t" + (" WHERE " + query.text.split(" WHERE ", 1)[1] if " WHERE " in query.text else
                            " GROUP BY " + query.text.split(" GROUP BY ", 1)[1]))
            rc = self.oracle.execute(seg, cq)
            craw = np.zeros(rc.num_groups, dtype=np.int64)
            mult = 1
            for j, c in enumerate(cards):
                craw += rc.keys[:, j].astype(np.int64) * mult
                mult *= c
            np.add.at(count, craw, rc.longs[0])
            for a, f in enumerate(fns):
                col = query.aggregations[a].column
                if f in ("SUM", "AVG"):
                    np.add.at(isum[a], raw, np.rint(r.doubles[a]).astype(np.int64))
                elif f in ("MAX", "MIN"):   # tables hold dictIds (+1 for MAX): value -> id through the sorted dictionary
                    ids = np.searchsorted(seg.column(col).dict_values, r.doubles[a]).astype(np.uint32)
                    if f == "MAX":
                        np.maximum.at(gmax[a], raw, ids + 1)
                    else:
                        np.minimum.at(gmin[a], raw, ids)
        unsafe = False
        i64 = []
        if carrier >= 0:
            f_field = isum[carrier] - count * vmin
            assert (f_field >= 0).all()
            unsafe = bool((f_field > ((1 << shift) - 1) // reduce_world).any() or (count > ((1 << (64 - shift)) - 1) // reduce_world).any())
            isum[carrier] = (f_field + (count << shift)) if not unsafe else np.zeros(groups, dtype=np.int64)  # unsafe: garbage anyway
        elif need_count or not has_minmax:
            i64.append(count)
        i64 += [isum[a] for a in sorted(isum)]
        bufs = {"i64": torch.from_numpy(np.concatenate(i64)) if i64 else None, "f64": None,
                "u32max": torch.from_numpy(np.concatenate([gmax[a] for a in sorted(gmax)]).view(np.int32).copy()) if gmax else None,
                "u32min": torch.from_numpy(np.concatenate([gmin[a] for a in sorted(gmin)]).view(np.int32).copy()) if gmin else None}
        self.passes.append("carrier" if carrier >= 0 else "plain")
        return _Block(bufs, carrier >= 0, unsafe, dict(groups=groups, cards=cards, carrier=carrier, shift=shift, vmin=vmin,
                                                        has_count=carrier < 0 and (need_count or not has_minmax),
                                                        sums=sorted(isum), maxs=sorted(gmax), mins=sorted(gmin), seg=segments[0]))

    def buffers(self, block):
        return block.bufs

    def flag_tensor(self, value):
        return torch.tensor([value], dtype=torch.int32)

    def synchronize(self):
        pass

    def free(self, block):
        block.bufs = None

    def finish(self, block, query, is_root):
        if not is_root:
            return None
        L, G = block.layout, block.layout["groups"]
        i64 = block.bufs["i64"].numpy() if block.bufs["i64"] is not None else np.zeros(0, dtype=np.int64)
        off = 0
        count = None
        if L["has_count"]:
            count, off = i64[:G], G
        sums = {}
        for a in L["sums"]:
            sums[a] = i64[off:off + G]
            off += G
        if L["carrier"] >= 0:
            packed = sums[L["carrier"]]
            count = packed >> L["shift"]
            sums[L["carrier"]] = (packed & ((1 << L["shift"]) - 1)) + count * L["vmin"]
        mx = block.bufs["u32max"].numpy().view(np.uint32) if block.bufs["u32max"] is not None else None
        mn = block.bufs["u32min"].numpy().view(np.uint32) if block.bufs["u32min"] is not None else None
        exists = (count > 0) if count is not None else (mx[:G] > 0 if mx is not None else mn[:G] != 0xFFFFFFFF)
        out, seg = {}, L["seg"]
        for g in np.nonzero(exists)[0]:
            raw, key = int(g), []
            for c, name in zip(L["cards"], query.group_by):
                key.append(seg.value_of(name, raw % c))
                raw //= c
            vals = []
            for a, ag in enumerate(query.aggregations):
                f = ag.function
                if f == "COUNT":
                    vals.append(int(count[g]))
                elif f == "SUM":
                    vals.append(float(sums[a][g]))
                elif f == "AVG":
                    vals.append((float(sums[a][g]), int(count[g])))
                elif f == "MAX":
                    vals.append(float(seg.value_of(ag.column, int(mx[L["maxs"].index(a) * G + g]) - 1)))
                else:
                    vals.append(float(seg.value_of(ag.column, int(mn[L["mins"].index(a) * G + g]))))
            out[tuple(key)] = vals
        return out


def _combine_worker(rank, world, port, out_dir, force_shift):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import pickle
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from oracle.pinot_oracle import oracle as get_oracle
    from pinot_b200 import sql
    from pinot_b200.distributed import execute_and_combine
    from reduce_util import combine, normalise
    o = get_oracle()
    rng = np.random.default_rng(31 + rank)

    def seg(i, n):   # shared dictionaries: every value occurs in every segment
        k = np.concatenate([np.arange(40), rng.integers(0, 40, size=n - 40)]).astype(np.int32) * 3
        j = np.concatenate([np.arange(40) % 6, rng.integers(0, 6, size=n - 40)]).astype(np.int32)
        v = np.concatenate([np.arange(40) * 25 - 500, rng.integers(0, 40, size=n - 40) * 25 - 500]).astype(np.int32)
        return o.build_segment(f"r{rank}s{i}", {"k": k, "j": j, "v": v})
    segs = [seg(i, n) for i, n in enumerate([3000, 700 + 50 * rank, 4096])]
    report = {}
    for text in ("SELECT SUM(v), COUNT(*) FROM t WHERE v > -400 GROUP BY k",
                 "SELECT AVG(v), MAX(v), MIN(k) FROM t GROUP BY k, j",
                 "SELECT SUM(v), MAX(k) FROM t WHERE j < 5 GROUP BY j",
                 "SELECT SUM(v) FROM t GROUP BY k"):
        q = sql.parse(text)
        q.text = text
        backend = OracleBackend(o, force_shift)
        got = execute_and_combine(backend, segs, q, dist, dst=0)
        mine = [normalise(s, q, r.num_groups, r.keys, r.doubles, r.longs, r.distinct) for s in segs for r in [o.execute(s, q)]]
        everyone = [None] * world
        dist.all_gather_object(everyone, mine)
        if rank == 0:
            want = combine([a.function for a in q.aggregations], [t for part in everyone for t in part])
            report[text] = (got == want, backend.passes, len(want))
        else:
            assert got is None
            report[text] = (True, backend.passes, 0)
    pickle.dump(report, open(os.path.join(out_dir, f"report{rank}.pkl"), "wb"))
    dist.destroy_process_group()


import pytest  # noqa: E402


@pytest.mark.parametrize("force_shift", [0, 8])
def test_execute_and_combine_world_size_2(tmp_path, force_shift):
    """force_shift 8: an 8-bit sum field overflows on every rank -> both ranks agree (MAX all-reduce) to rerun without the
    count carrier; results are exact either way and equal the oracle-side merge by value of all 6 segments."""
    import pickle
    world = 2
    port = 31500 + (os.getpid() % 1500) + force_shift
    mp.spawn(_combine_worker, args=(world, port, str(tmp_path), force_shift), nprocs=world, join=True)
    reports = [pickle.load(open(tmp_path / f"report{r}.pkl", "rb")) for r in range(world)]
    for text, (ok, passes, n) in reports[0].items():
        assert ok, text
        assert n > 0
        # every rank took the same number of passes (a rank-local retry would deadlock the collectives)
        assert passes == reports[1][text][1], (text, passes, reports[1][text][1])
        if "COUNT" in text or "AVG" in text or text.endswith("GROUP BY k"):
            assert passes == (["carrier", "plain"] if force_shift else ["carrier"]), (text, passes)
