"""PERCENTILE over the oracle's operator chain: the reference's PercentileAggregationFunction restated on top of the
oracle (oracle/pinot_oracle.cpp, the C++ restatement of the Java filter operators and forward-index readers), which itself
has no percentile operator.

    FilterOperator tree -> DocIdSet         oracle.filter_doc_ids (the reference's leaf / AND / OR / NOT operators)
    ProjectionOperator -> values            exact_ref.column_values (the oracle's FixedBitIntReader and dictionaries)
    aggregate                               per group a DoubleArrayList: every value converted to double, in doc order
    extractFinalResult                      Arrays.sort, then the index rule (restated here: n = 0 -> -inf,
                                            p == 100 -> the largest, else (int)((double)n * p / 100.0), clamped)

It shares nothing with tests/percentile_ref.py's doc-set computation (value-space filters) or its sort (in the column's
own type), and nothing with the product."""
from __future__ import annotations

from typing import Dict, Sequence

import numpy as np

from exact_ref import column_values
from pinot_b200.query import QueryContext


def _final(values: list, p: float) -> float:
    if not values:
        return float("-inf")
    values = sorted(values)   # Arrays.sort(double[]) for values without NaN / -0.0
    n = len(values)
    if p == 100.0:
        return values[-1]
    return values[min(int(float(n) * float(p) / 100.0), n - 1)]


def _key(v):
    return v.decode("utf-8") if isinstance(v, bytes) else (v.item() if hasattr(v, "item") else v)


def percentiles(oracle, segs: Sequence, flt, group_by: Sequence[str], column: str, ps: Sequence[float]) -> Dict[tuple, list]:
    """{group key values: [PERCENTILE(column, p) for p in ps]} over the segments (aggregation only: the key ())."""
    lists: Dict[tuple, list] = {} if group_by else {(): []}
    for seg in segs:
        docs, _ = oracle.filter_doc_ids(seg, QueryContext(aggregations=[], filter=flt))
        docs = np.sort(docs).astype(np.int64)
        vals = [float(v) for v in column_values(oracle, seg, column, docs)]
        keys = [column_values(oracle, seg, g, docs) for g in group_by]
        for i, v in enumerate(vals):
            lists.setdefault(tuple(_key(k[i]) for k in keys), []).append(v)
    return {k: [_final(v, p) for p in ps] for k, v in lists.items()}
