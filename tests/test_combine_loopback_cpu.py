"""The loopback collective (tests/loopback_dist.py) on CPU: torch.distributed semantics, the execute_and_combine flow of
tests/test_distributed_cpu.py over it (same results and passes as under gloo), and failure without hanging."""
import os
import pickle
import threading
import time

import numpy as np
import pytest
import torch

import test_distributed_cpu as gloo_tests
from loopback_dist import LoopbackAborted, run_ranks, values
from pinot_b200.distributed import reduce_buffers


def _tables(rank, G=777):
    rng = np.random.default_rng(500 + rank)
    count = rng.integers(0, 5, size=G)
    return dict(count=count,
                sums=rng.integers(-10**15, 10**15, size=G) * (count > 0),
                fsum=rng.standard_normal(G) * 1e9 * (count > 0),
                mx=np.where(count > 0, rng.integers(0, 2**32 - 1, size=G, dtype=np.int64) + 1, 0).astype(np.uint32),
                mn=np.where(count > 0, rng.integers(0, 2**32 - 1, size=G, dtype=np.int64), 0xFFFFFFFF).astype(np.uint32))


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("dst", [0, 1])
def test_reduce_buffers_match_numpy(world, dst):
    ins = [_tables(r) for r in range(world)]

    def rank(dist):
        t = ins[dist.get_rank()]
        bufs = {"i64": torch.from_numpy(np.concatenate([t["count"], t["sums"]]).astype(np.int64)),
                "f64": torch.from_numpy(t["fsum"].copy()),
                "u32max": torch.from_numpy(t["mx"].view(np.int32).copy()),
                "u32min": torch.from_numpy(t["mn"].view(np.int32).copy())}
        reduce_buffers(bufs, dist, dst=dst)
        return {k: v.numpy().copy() for k, v in bufs.items()}, list(dist.calls)

    outs = values(run_ranks(world, rank))
    G = len(ins[0]["count"])
    fsum = ins[0]["fsum"].copy()
    for t in ins[1:]:
        fsum = fsum + t["fsum"]            # rank order: the same rounding as the loopback's
    for r, (got, calls) in enumerate(outs):
        assert calls == ["reduce"] * 4
        if r != dst:   # torch: reduce leaves the other ranks' tensors as they were
            mine = ins[r]
            assert np.array_equal(got["i64"], np.concatenate([mine["count"], mine["sums"]]))
            assert np.array_equal(got["u32max"].view(np.uint32), mine["mx"])
            assert np.array_equal(got["u32min"].view(np.uint32), mine["mn"])
            continue
        assert np.array_equal(got["i64"][:G], sum(t["count"] for t in ins))
        assert np.array_equal(got["i64"][G:], sum(t["sums"] for t in ins))
        assert np.array_equal(got["f64"], fsum)
        assert np.array_equal(got["u32max"].view(np.uint32), np.maximum.reduce([t["mx"] for t in ins]))
        assert np.array_equal(got["u32min"].view(np.uint32), np.minimum.reduce([t["mn"] for t in ins]))


def test_all_reduce_objects_and_broadcast():
    def rank(dist):
        r = dist.get_rank()
        t = torch.tensor([r + 1, -r], dtype=torch.int64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        everyone = [None] * dist.get_world_size()
        mine = {"rank": r, "payload": [r] * 3}
        dist.all_gather_object(everyone, mine)
        mine["payload"].append(99)         # pickled on the way: the peers' copies do not change
        box = [("id", r)]
        dist.broadcast_object_list(box, src=2)
        return t.tolist(), everyone, box, dist.get_world_size()

    for t, everyone, box, world in values(run_ranks(3, rank)):
        assert t == [3, 0] and world == 3
        assert everyone == [{"rank": i, "payload": [i] * 3} for i in range(3)]
        assert box == [("id", 2)]


class _PerThreadDist:
    """torch.distributed as test_distributed_cpu's worker sees it: each thread gets its own loopback rank."""

    local = threading.local()

    def init_process_group(self, *args, **kwargs):
        pass

    def destroy_process_group(self):
        pass

    def __getattr__(self, name):
        return getattr(self.local.dist, name)


@pytest.mark.parametrize("force_shift", [0, 8])
def test_oracle_backend_flow_matches_gloo(tmp_path, monkeypatch, force_shift):
    """test_distributed_cpu's execute_and_combine worker, run once over gloo processes and once over loopback threads:
    the reports (result equals the oracle merge, passes taken per query, group counts) must be identical."""
    world = 2
    gloo_dir, loop_dir = tmp_path / "gloo", tmp_path / "loop"
    gloo_dir.mkdir()
    loop_dir.mkdir()
    port = 35500 + (os.getpid() % 1500) + force_shift
    import torch.multiprocessing as mp
    mp.spawn(gloo_tests._combine_worker, args=(world, port, str(gloo_dir), force_shift), nprocs=world, join=True)

    for k in ("MASTER_ADDR", "MASTER_PORT", "RANK", "WORLD_SIZE"):   # the worker sets them: restore afterwards
        monkeypatch.setenv(k, os.environ.get(k, ""))
    monkeypatch.setattr(gloo_tests, "dist", _PerThreadDist())

    def rank(dist):
        _PerThreadDist.local.dist = dist
        gloo_tests._combine_worker(dist.get_rank(), world, 0, str(loop_dir), force_shift)

    values(run_ranks(world, rank))
    for r in range(world):
        gloo = pickle.load(open(gloo_dir / f"report{r}.pkl", "rb"))
        loop = pickle.load(open(loop_dir / f"report{r}.pkl", "rb"))
        assert loop == gloo, r
        for text, (ok, passes, n) in loop.items():
            assert ok, text
            if r == 0:
                assert n > 0, text


def test_a_failing_rank_fails_every_rank_without_hanging():
    def rank(dist):
        if dist.get_rank() == 1:
            raise ValueError("rank 1 fails before its first collective")
        dist.all_reduce(torch.zeros(4))
        return "unreachable"

    t0 = time.monotonic()
    out = run_ranks(3, rank, timeout=30.0)
    assert time.monotonic() - t0 < 10.0     # the abort wakes the peers at once, not at the timeout
    assert isinstance(out[1].error, ValueError)
    assert all(isinstance(out[r].error, LoopbackAborted) for r in (0, 2))
    assert out[0].calls == out[2].calls == ["all_reduce"] and out[1].calls == []
    with pytest.raises(ValueError):
        values(out)


def test_a_late_rank_times_out():
    def rank(dist):
        if dist.get_rank() == 0:
            time.sleep(1.5)
            return "late"
        dist.all_reduce(torch.zeros(1))

    t0 = time.monotonic()
    out = run_ranks(2, rank, timeout=0.5)
    assert time.monotonic() - t0 < 10.0
    assert out[0].value == "late" and out[0].error is None
    assert isinstance(out[1].error, LoopbackAborted)
