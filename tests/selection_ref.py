"""Expected rows of a selection query (SELECT columns WHERE ... [ORDER BY columns] LIMIT n), from column values alone.

The doc set comes from filter_ref (the filter evaluated on stored values), the values from exact_ref.column_values.
Selection only (SelectionOnlyOperator): per segment the first `limit` matching docs in doc-id order.  Merged over several
segments: segments in submission order, each contributing a doc-order prefix of its matches, `limit` rows in all.
ORDER BY (SelectionOrderByOperator): np.lexsort over the order values (value order; DESC reversed) with the doc id as
the last key -- merged, (segment index, doc id) -- then the first `limit` rows."""
from __future__ import annotations

from typing import List, Sequence

import numpy as np

from exact_ref import column_values
from filter_ref import matching_docs


def _typed(values: np.ndarray) -> np.ndarray:
    """What the product returns per stored type: int64, float64, or str (STRING dictionary entries without padding)."""
    if values.dtype.kind in ("S", "a"):
        return np.array([v.rstrip(b"\0").decode("utf-8") for v in values], dtype=object)
    if values.dtype.kind == "f":
        return values.astype(np.float64)
    return values.astype(np.int64)


def segment_rows(oracle, seg, flt, columns: Sequence[str], limit: int):
    """(doc ids, [values per column], matched docs) of one segment."""
    match = matching_docs(oracle, seg, flt)
    docs = np.flatnonzero(match)[:limit].astype(np.int64)
    return docs, [_typed(column_values(oracle, seg, c, docs)) for c in columns], int(match.sum())


def _ordered(oracle, segs: Sequence, flt, columns: Sequence[str], order_by, limit: int, merge: bool) -> List[dict]:
    parts = []
    for s, seg in enumerate(segs):
        docs = np.flatnonzero(matching_docs(oracle, seg, flt)).astype(np.int64)
        parts.append((s, docs, [column_values(oracle, seg, c, docs) for c, _ in order_by]))
    groups = [parts] if merge else [[p] for p in parts]
    out = []
    for g in groups:
        docs = np.concatenate([d for _, d, _ in g])
        segi = np.concatenate([np.full(len(d), s, dtype=np.int64) for s, d, _ in g])
        keys = []
        for k, (_, asc) in enumerate(order_by):
            vals = np.concatenate([v[k] for _, _, v in g])
            rank = np.unique(vals, return_inverse=True)[1].astype(np.int64).reshape(-1)   # value order, equal values equal
            keys.append(rank if asc else -rank)
        idx = np.lexsort([docs, segi] + keys[::-1])[:limit] if len(docs) else np.zeros(0, dtype=np.int64)
        cols = []
        for c in columns:
            vals = np.concatenate([column_values(oracle, segs[s], c, d) for s, d, _ in g]) if len(docs) else np.zeros(0)
            cols.append(_typed(vals[idx]) if len(docs) else _typed(column_values(oracle, segs[g[0][0]], c, docs)))
        out.append(dict(doc_ids=docs[idx], segment_index=segi[idx], columns=cols, matched=len(docs)))
    return out


def expected(oracle, segs: Sequence, flt, columns: Sequence[str], limit: int, merge: bool, order_by=()) -> List[dict]:
    """One dict {doc_ids, segment_index, columns, matched} per result (one when merged).  order_by: [(column, ascending)]."""
    if order_by:
        return _ordered(oracle, segs, flt, columns, list(order_by), limit, merge)
    per = [segment_rows(oracle, seg, flt, columns, limit) for seg in segs]
    if not merge:
        return [dict(doc_ids=d, segment_index=np.full(len(d), s, dtype=np.int64), columns=v, matched=m)
                for s, (d, v, m) in enumerate(per)]
    docs, segi, cols, left = [], [], [[] for _ in columns], limit
    for s, (d, v, _) in enumerate(per):
        k = min(left, len(d))
        docs.append(d[:k])
        segi.append(np.full(k, s, dtype=np.int64))
        for i in range(len(columns)):
            cols[i].append(v[i][:k])
        left -= k
    return [dict(doc_ids=np.concatenate(docs), segment_index=np.concatenate(segi),
                 columns=[np.concatenate(c) if c else np.zeros(0) for c in cols], matched=sum(m for _, _, m in per))]


def assert_rows_equal(block, want: dict, what: str = "") -> None:
    """Device rows == reference rows: doc ids, segments and every value, in order (floats compared bit for bit)."""
    assert np.array_equal(block.doc_ids.astype(np.int64), want["doc_ids"]), (what, block.doc_ids[:20], want["doc_ids"][:20])
    assert np.array_equal(block.segment_index.astype(np.int64), want["segment_index"]), what
    for name, got, exp in zip(block.names, block.columns, want["columns"]):
        assert len(got) == len(exp), (what, name)
        if exp.dtype == object:
            assert list(got) == list(exp), (what, name)
        else:
            assert got.dtype == exp.dtype, (what, name, got.dtype, exp.dtype)
            assert np.array_equal(got.view(np.int64), exp.view(np.int64)), (what, name, got[:10], exp[:10])
