"""CPU tests of the sharing map of a mixed aggregation query: which aggregation's state each aggregation reads
(pb200::plan_scan's ds_rep, hll_rep, pct_rep, mom_first and limb) and which sum carries a result's counts, checked on
segments made of column metadata alone (tests/host_probe/host_probe.cpp probe_plan_sharing).

The rule is restated here, independently of the planner:

* an aggregation's owner is the earliest aggregation before it over the same column whose state it may share:
  DISTINCTSUM / DISTINCTAVG / DISTINCTCOUNTHLL read the bitset of the first DISTINCTCOUNT or reader of their column (a
  reader's owner is the owner of that first one); DISTINCTCOUNTHLLs share one estimate per (column, log2m); PERCENTILEs
  of one column share the first one's histogram; VAR / STDDEV of one column share one set of moments;
* VAR / STDDEV append three internal INT SUMs (the K, H, L limbs) per column behind the caller's aggregations, and the
  caller's aggregations plus those sums must be 6 or fewer;
* the count carrier is the first INT dictionary SUM / AVG of the caller's, never a limb sum.

The shapes are the pinned ones of tests/test_gpu_mixed_aggs.py and a seeded random draw biased towards repeated columns."""
import ctypes as C
import random

import pytest

from pinot_b200 import _lib
from test_scan_plan_cpu import H100, ProbeCol, col, make_query, probe  # noqa: F401  (probe: the fixture)

A = _lib.AGG_CODES
MAX_AGGS, RES = 6, 40
MOMENTS = ("VARPOP", "VARSAMP", "STDDEVPOP", "STDDEVSAMP")
DISTINCT_VALUE = ("DISTINCTSUM", "DISTINCTAVG")
HLL_DEFAULT_LOG2M = 8

# columns: 0 g (INT, 10 values: the group key), 1 x, 2 y (INT), 3 z (LONG), 4 w (DOUBLE), 5 t (INT time), 6 s (STRING)
COLS = [col(10), col(500, -1000, 7), col(300, 5, 3), col(400, stored=_lib.LONG), col(200, stored=_lib.DOUBLE),
        col(1000, 1_700_000, 60), col(30, stored=_lib.STRING)]
G, X, Y, Z, W, T, S = range(7)
NUMERIC = (X, Y, Z, W)
INT_COLS = (X, Y)


class ProbeSharing(C.Structure):
    _fields_ = ([(n, C.c_int64) for n in ("num_user_aggs", "num_aggs", "nres")]
                + [(n, C.c_int64 * MAX_AGGS) for n in ("function", "column", "ds_rep", "hll_log2m", "hll_rep", "pct_rep",
                                                       "mom_first", "limb")]
                + [("carrier_agg", C.c_int64 * RES)])


@pytest.fixture(scope="module")
def sharing(probe):  # noqa: F811
    probe.probe_sharing_size.restype = C.c_int64
    assert probe.probe_sharing_size() == C.sizeof(ProbeSharing)
    probe.probe_plan_sharing.restype = C.c_int32
    probe.probe_plan_sharing.argtypes = [C.c_int32, C.c_int32, C.POINTER(C.c_char_p), C.POINTER(C.c_int64), C.c_int32,
                                         C.POINTER(_lib.Query), C.POINTER(C.c_double), C.POINTER(_lib.AggArg), C.POINTER(ProbeCol),
                                         C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.POINTER(ProbeSharing)]
    return probe


def run(probe, aggs, group_by=(G,), nseg=1, flags=0, docs=100_000, knobs=None):
    """aggs: (function name, column or -1, arg) with arg PERCENTILE's p, DISTINCTCOUNTHLL's log2m (0: default) or the
    time column of FIRST/LASTWITHTIME.  Returns (rc, ProbeSharing)."""
    q, keep = make_query([], [(A[f], c) for f, c, _ in aggs], group_by=list(group_by), flags=flags)
    args = (C.c_double * MAX_AGGS)(*[float(x) if f in ("PERCENTILE", "DISTINCTCOUNTHLL") else 0.0 for f, _, x in aggs])
    wt = (_lib.AggArg * MAX_AGGS)(*[_lib.AggArg(0.0, x if "WITHTIME" in f else -1, COLS[c]["stored"] if "WITHTIME" in f else 0)
                                    for f, c, x in aggs])
    ncols = len(COLS)
    cols = (ProbeCol * (nseg * ncols))()
    for s in range(nseg):
        for k, c in enumerate(COLS):
            host = c.get("cbuf")
            cols[s * ncols + k] = ProbeCol(c["kind"], c["stored"], c["bits"], c["card"], int(c["native"]), int(c["shared"]),
                                           0, 1 if k in NUMERIC else -1, c["hash"], C.cast(host, C.c_void_p) if host else None,
                                           len(c["host"]) if host else 0)
    knobs = knobs or {}
    names = (C.c_char_p * max(len(knobs), 1))(*[k.encode() for k in knobs])
    values = (C.c_int64 * max(len(knobs), 1))(*knobs.values())
    nd = (C.c_int32 * nseg)(*([docs] * nseg))
    out = ProbeSharing()
    rc = probe.probe_plan_sharing(*H100, names, values, len(knobs), C.byref(q), args, wt, cols, ncols, nd, nseg, 1, C.byref(out))
    del keep
    return rc, out


def expected(aggs, group_by=True):
    """The sharing map by the rule of the module docstring: a dict of the probe's fields, or None when the query is over
    the 6-aggregation cap."""
    n = len(aggs)
    plan = [(f, c) for f, c, _ in aggs]
    mom_first = [-1] * n
    for a, (f, c, _) in enumerate(aggs):
        if f not in MOMENTS:
            continue
        b = next((b for b in range(a) if aggs[b][1] == c and mom_first[b] >= 0), -1)
        if b >= 0:
            mom_first[a] = mom_first[b]
        else:
            mom_first[a] = len(plan)
            plan += [("SUM", c)] * 3
    if len(plan) > MAX_AGGS:
        return None
    m = len(plan)
    limb = [-1] * m
    for a in range(n):
        if mom_first[a] >= 0:
            for j in range(3):
                limb[mom_first[a] + j] = j
    ds_rep, hll_rep, pct_rep, log2m = [-1] * m, [-1] * m, [-1] * m, [0] * m
    for a, (f, c, x) in enumerate(aggs):
        earlier = [b for b in range(a) if aggs[b][1] == c]
        if f in DISTINCT_VALUE or f == "DISTINCTCOUNTHLL":
            b = next((b for b in earlier if aggs[b][0] in ("DISTINCTCOUNT", "DISTINCTCOUNTHLL") + DISTINCT_VALUE), -1)
            ds_rep[a] = a if b < 0 else b if aggs[b][0] == "DISTINCTCOUNT" else ds_rep[b]
        if f == "DISTINCTCOUNTHLL":
            log2m[a] = int(x) or HLL_DEFAULT_LOG2M
            hll_rep[a] = next((b for b in earlier if aggs[b][0] == "DISTINCTCOUNTHLL" and log2m[b] == log2m[a]), a)
        if f == "PERCENTILE":
            pct_rep[a] = next((b for b in earlier if aggs[b][0] == "PERCENTILE"), a)
    # the carrier: the first INT dictionary SUM / AVG of the caller's, when the table keeps counts or marks groups
    carrier = -1
    if group_by:
        candidate = next((a for a, (f, c, _) in enumerate(aggs) if f in ("SUM", "AVG") and c in INT_COLS), -1)
        need_count = any(f in ("COUNT", "AVG") + MOMENTS for f, _, _ in aggs)
        marker = any(f in ("MIN", "MAX") for f, _, _ in aggs)
        if need_count or not marker:
            carrier = candidate
    return dict(num_user_aggs=n, num_aggs=m, function=[A[f] for f, _ in plan], column=[c for _, c in plan], ds_rep=ds_rep,
                hll_log2m=log2m, hll_rep=hll_rep, pct_rep=pct_rep, mom_first=mom_first, limb=limb, carrier=carrier)


def check(probe, aggs, group_by=True, what=""):
    rc, out = run(probe, aggs, group_by=(G,) if group_by else ())
    want = expected(aggs, group_by)
    if want is None:
        assert rc == _lib.E_UNSUPPORTED, (what, aggs, rc)
        assert "VAR/STDDEV" in probe.last_error(), (what, probe.last_error())
        return None
    assert rc == 0, (what, aggs, probe.last_error())
    n, m = want["num_user_aggs"], want["num_aggs"]
    assert (out.num_user_aggs, out.num_aggs) == (n, m), (what, aggs)
    for field in ("function", "column", "ds_rep", "hll_log2m", "hll_rep", "pct_rep", "limb"):
        assert list(getattr(out, field))[:m] == want[field], (what, field, aggs, list(getattr(out, field))[:m])
    assert list(out.mom_first)[:n] == want["mom_first"], (what, aggs, list(out.mom_first))
    if group_by:
        assert out.carrier_agg[0] == want["carrier"], (what, aggs, out.carrier_agg[0])
        assert out.carrier_agg[0] < 0 or want["limb"][out.carrier_agg[0]] < 0, (what, "the carrier is a limb sum")
    return out


PINNED = [
    [("PERCENTILE", X, 10), ("PERCENTILE", X, 90), ("PERCENTILE", Y, 50)],
    [("DISTINCTSUM", X, 0), ("DISTINCTCOUNT", X, 0), ("DISTINCTAVG", X, 0), ("DISTINCTCOUNTHLL", X, 0)],
    [("DISTINCTCOUNT", X, 0), ("DISTINCTSUM", X, 0), ("DISTINCTAVG", X, 0), ("DISTINCTCOUNTHLL", X, 0)],
    [("DISTINCTCOUNTHLL", X, 0), ("DISTINCTCOUNTHLL", X, 8), ("DISTINCTCOUNTHLL", X, 12)],
    [("STDDEVPOP", X, 0), ("VARSAMP", X, 0), ("PERCENTILE", X, 50)],
    [("STDDEVPOP", X, 0), ("VARSAMP", X, 0), ("LASTWITHTIME", X, T)],
    [("VARPOP", X, 0), ("STDDEVSAMP", X, 0), ("SUM", Y, 0)],
    [("VARPOP", X, 0), ("STDDEVSAMP", X, 0), ("SUM", Y, 0), ("COUNT", -1, 0)],
    [("VARPOP", X, 0), ("VARPOP", Y, 0)],
    [("VARPOP", X, 0), ("SUM", X, 0)],
    [("VARPOP", Z, 0), ("SUM", Y, 0), ("AVG", X, 0)],
    [("DISTINCTAVG", Y, 0), ("PERCENTILE", Y, 50), ("PERCENTILE", Y, 75), ("DISTINCTCOUNTHLL", Y, 12), ("FIRSTWITHTIME", Y, T)],
    [("DISTINCTCOUNTHLL", S, 0), ("DISTINCTCOUNT", S, 0), ("DISTINCTCOUNTHLL", S, 8), ("MIN", S, 0)],
    [("SUM", X, 0), ("VARPOP", X, 0), ("DISTINCTCOUNTHLL", X, 0)],
]


@pytest.mark.parametrize("group_by", [True, False], ids=["group_by", "aggregation_only"])
def test_pinned_shapes(sharing, group_by):
    for i, aggs in enumerate(PINNED):
        check(sharing, aggs, group_by, f"shape {i}")


def test_owners_of_the_pinned_shapes(sharing):
    """The sharing the pinned shapes exist for, spelled out."""
    pct = check(sharing, PINNED[0])
    assert list(pct.pct_rep)[:3] == [0, 0, 2]
    for order, rep in ((PINNED[1], [0, -1, 0, 0]), (PINNED[2], [-1, 0, 0, 0])):
        assert list(check(sharing, order).ds_rep)[:4] == rep
    hll = check(sharing, PINNED[3])
    assert list(hll.hll_rep)[:3] == [0, 0, 2] and list(hll.hll_log2m)[:3] == [8, 8, 12]
    var = check(sharing, PINNED[4])
    assert list(var.mom_first)[:3] == [3, 3, -1] and list(var.limb)[:6] == [-1, -1, -1, 0, 1, 2]
    assert check(sharing, PINNED[6]).num_aggs == 6
    assert check(sharing, PINNED[9]).carrier_agg[0] == 1   # the caller's SUM(x), not a limb sum of x
    var_sum = check(sharing, PINNED[13])   # a SUM over the column of the limb sums, before them: the carrier
    assert list(var_sum.mom_first)[:3] == [-1, 3, -1] and var_sum.carrier_agg[0] == 0


@pytest.mark.parametrize("aggs", [PINNED[7], PINNED[8],
                                  [("VARPOP", X, 0), ("VARPOP", Y, 0), ("STDDEVSAMP", Z, 0)],
                                  [("STDDEVPOP", X, 0), ("COUNT", -1, 0), ("SUM", Y, 0), ("MIN", Y, 0)]],
                         ids=["4+3", "2+6", "3+9", "4+3_stddev"])
def test_moment_cap_refusals(sharing, aggs):
    assert expected(aggs) is None
    check(sharing, aggs)


# the functions that share state weigh more; VAR / STDDEV less (four of them would put most draws over the cap)
FNS = {"COUNT": 2, "SUM": 3, "MIN": 2, "MAX": 2, "AVG": 2, "DISTINCTCOUNT": 4, "PERCENTILE": 6, "VARPOP": 1, "VARSAMP": 1,
       "STDDEVPOP": 1, "STDDEVSAMP": 1, "FIRSTWITHTIME": 2, "LASTWITHTIME": 2, "DISTINCTSUM": 4, "DISTINCTAVG": 4,
       "DISTINCTCOUNTHLL": 6}


def draw(rng, k):
    """k aggregations over two columns per query (an INT one and any numeric one), so that most functions share a column
    with another."""
    pool = [rng.choice(INT_COLS), rng.choice(NUMERIC)]
    out = []
    for f in rng.choices(list(FNS), weights=list(FNS.values()), k=k):
        if f == "COUNT":
            out.append((f, -1, 0))
            continue
        # DISTINCTSUM / DISTINCTAVG: the grid check needs the host dictionary the metadata carries for INT only
        c = pool[0] if f in DISTINCT_VALUE else rng.choice(pool)
        arg = {"PERCENTILE": rng.choice([0, 10, 50, 90, 100]), "DISTINCTCOUNTHLL": rng.choice([0, 4, 8, 12]),
               "FIRSTWITHTIME": T, "LASTWITHTIME": T}.get(f, 0)
        out.append((f, c, arg))
    return out


@pytest.mark.parametrize("group_by", [True, False], ids=["group_by", "aggregation_only"])
def test_random_shapes(sharing, group_by):
    rng = random.Random(20261018)
    refused = shared = 0
    for i in range(600):
        aggs = draw(rng, rng.randint(1, 6))
        out = check(sharing, aggs, group_by, f"draw {i}")
        if out is None:
            refused += 1
        elif any(out.ds_rep[a] not in (-1, a) or out.hll_rep[a] not in (-1, a) or out.pct_rep[a] not in (-1, a)
                 for a in range(out.num_user_aggs)):
            shared += 1
    assert refused > 20 and shared > 100, (refused, shared)
