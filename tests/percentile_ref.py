"""Value-space reference of PERCENTILE(col, p): the doc set from tests/filter_ref.py, the column's stored values at those
docs (exact_ref.column_values), sorted, and PercentileAggregationFunction.extractFinalResult's index rule
(restated below, independently of the product's copy).  Groups come from the group-by columns' values.  It never looks at the product's
histograms or dictIds.

Values are sorted in the column's own type and converted to double afterwards: the conversion is monotone, so this is the
reference's "convert, then sort" order, and the selected stored value also names the dictId a dictionary column must
return (a LONG beyond 2^53 is then checked exactly).  NaN and -0.0 are held by tests/float_edges_ref.py."""
from __future__ import annotations

from typing import Dict, List, Sequence

import numpy as np

from exact_ref import column_values
from filter_ref import matching_docs


def percentile_index(n: int, p: float) -> int:
    """PercentileAggregationFunction.extractFinalResult's index among n > 0 sorted values, restated here (not taken from
    the product): the largest at p == 100, otherwise (int)((double)n * p / 100.0), clamped to n - 1."""
    return n - 1 if p == 100.0 else min(int(float(n) * float(p) / 100.0), n - 1)


def _key_value(v):
    return v.decode("utf-8") if isinstance(v, bytes) else (v.item() if hasattr(v, "item") else v)


def group_values(oracle, segs: Sequence, flt, group_by: Sequence[str], column: str) -> Dict[tuple, np.ndarray]:
    """{group key values: the column's stored values over the group's matched rows, sorted ascending} over all segments
    (aggregation only: the one key (), present even without a matched row)."""
    parts: Dict[tuple, List[np.ndarray]] = {} if group_by else {(): []}
    for seg in segs:
        docs = np.nonzero(matching_docs(oracle, seg, flt))[0]
        vals = column_values(oracle, seg, column, docs)
        if not group_by:
            parts[()].append(vals)
            continue
        code = np.zeros(len(docs), dtype=np.int64)
        uniq = []
        for g in group_by:
            u, inv = np.unique(column_values(oracle, seg, g, docs), return_inverse=True)
            code = code * len(u) + inv
            uniq.append(u)
        keys, ginv = np.unique(code, return_inverse=True)
        order = np.argsort(ginv, kind="stable")
        bounds = np.searchsorted(ginv[order], np.arange(len(keys) + 1))
        for k, c in enumerate(keys):
            key = []
            for u in reversed(uniq):
                key.append(_key_value(u[c % len(u)]))
                c //= len(u)
            parts.setdefault(tuple(reversed(key)), []).append(vals[order[bounds[k]:bounds[k + 1]]])
    return {k: np.sort(np.concatenate(v)) if v else np.zeros(0) for k, v in parts.items()}


def pick(values: np.ndarray, p: float):
    """The selected stored value of PERCENTILE over sorted `values` (None when empty)."""
    return None if len(values) == 0 else values[percentile_index(len(values), p)]


def percentile(values: np.ndarray, p: float) -> float:
    """PERCENTILE's final result over sorted `values`: -inf when empty."""
    v = pick(values, p)
    return float("-inf") if v is None else float(v)
