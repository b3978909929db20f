"""Expected rows of a DISTINCT query (SELECT DISTINCT columns WHERE ... [ORDER BY columns] LIMIT n), from column values
alone.

The doc set comes from filter_ref (the filter evaluated on stored values), the values from exact_ref.column_values.  The
distinct tuples of a result are those of its matching docs (per segment: that segment's; merged: all segments'), each
with its first occurrence in (segment index, doc id) order.  Without ORDER BY they are ordered by first occurrence; with
ORDER BY by the items' values (DESC reversed), ties by first occurrence.  Then the first `limit`."""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np

from exact_ref import column_values
from filter_ref import matching_docs
from selection_ref import _typed


def _ordered(segi, docs, values, columns, order_by):
    """Indexes of the distinct tuples' first occurrences among the rows (in (segment, doc) order), ordered."""
    if len(docs) == 0:
        return np.zeros(0, dtype=np.int64)
    ranks = np.stack([np.unique(v, return_inverse=True)[1].reshape(-1) for v in values], axis=1)
    _, first = np.unique(ranks, axis=0, return_index=True)
    first = np.sort(first)                                   # by first occurrence
    keys = []
    for col, asc in order_by:
        r = ranks[first, columns.index(col)].astype(np.int64)
        keys.append(r if asc else -r)
    if keys:
        first = first[np.lexsort([np.arange(len(first))] + keys[::-1])]
    return first


def expected(oracle, segs: Sequence, flt, columns: Sequence[str], limit: Optional[int], merge: bool, order_by=()) -> List[dict]:
    """One dict {doc_ids, segment_index, columns, matched} per result (one when merged).  order_by: [(column, ascending)];
    limit None: every distinct tuple."""
    columns, order_by = list(columns), list(order_by)
    parts = []
    for s, seg in enumerate(segs):
        docs = np.flatnonzero(matching_docs(oracle, seg, flt)).astype(np.int64)
        parts.append((s, docs, [column_values(oracle, seg, c, docs) for c in columns]))
    groups = [parts] if merge else [[p] for p in parts]
    out = []
    for g in groups:
        docs = np.concatenate([d for _, d, _ in g])
        segi = np.concatenate([np.full(len(d), s, dtype=np.int64) for s, d, _ in g])
        values = [np.concatenate([v[k] for _, _, v in g]) for k in range(len(columns))]
        idx = _ordered(segi, docs, values, columns, order_by)[:limit]
        out.append(dict(doc_ids=docs[idx], segment_index=segi[idx], columns=[_typed(v[idx]) for v in values], matched=len(docs)))
    return out


def merge_by_value(results: Sequence[dict], columns: Sequence[str], order_by=(), limit: int = 10) -> dict:
    """The by-value merge of per-segment results: the union of their tuples with the earliest (segment, doc), ordered as
    above, first `limit` -- equal to the merged result because each segment's result holds its own first `limit`."""
    columns = list(columns)
    first = {}
    for r in results:
        for i in range(len(r["doc_ids"])):
            key = tuple(c[i] for c in r["columns"])
            occ = (int(r["segment_index"][i]), int(r["doc_ids"][i]))
            if key not in first or occ < first[key]:
                first[key] = occ
    rows = sorted(first.items(), key=lambda kv: kv[1])
    for col, asc in reversed(list(order_by)):
        k = columns.index(col)
        rows.sort(key=lambda kv: kv[0][k], reverse=not asc)
    rows = rows[:limit]
    cols = []
    for k in range(len(columns)):
        like = results[0]["columns"][k]
        cols.append(np.array([kv[0][k] for kv in rows], dtype=like.dtype))
    return dict(doc_ids=np.array([kv[1][1] for kv in rows], dtype=np.int64),
                segment_index=np.array([kv[1][0] for kv in rows], dtype=np.int64), columns=cols,
                matched=sum(r["matched"] for r in results))
