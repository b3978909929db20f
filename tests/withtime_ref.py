"""Per-row reference of FIRSTWITHTIME / LASTWITHTIME(v, t, 'T') from stored column values (DESIGN.md section 3.13).

The doc set comes from tests/filter_ref.py and the values from exact_ref.column_values; nothing here looks at the
product's keys, dictIds or tables.  Rows are visited in the call's row order -- segments in submission order, then doc
id -- and a sequential scan keeps the winner: LAST replaces it on t >= best (the last tied row wins), FIRST only on
t < best (the first tied row wins).  A group without a matched row (aggregation only: the one key ()) maps to None."""
from __future__ import annotations

from typing import Dict, Optional, Sequence, Tuple

import numpy as np

from exact_ref import column_values
from filter_ref import matching_docs


def _py(v):
    return v.decode("utf-8") if isinstance(v, bytes) else (v.item() if hasattr(v, "item") else v)


def withtime(oracle, segs: Sequence, flt, group_by: Sequence[str], function: str, v: str, t: str,
             time_of=None) -> Dict[tuple, Optional[Tuple[int, object]]]:
    """{group key values: (time value, data value) of the winning row, or None}.  time_of(seg_index, times) maps the
    stored time values of a segment to the time the query compares (e.g. DATETRUNC); default: the values themselves."""
    last = function == "LASTWITHTIME"
    out: Dict[tuple, Optional[Tuple[int, object]]] = {} if group_by else {(): None}
    for si, seg in enumerate(segs):
        docs = np.nonzero(matching_docs(oracle, seg, flt))[0]
        if not len(docs):
            continue
        tv = column_values(oracle, seg, t, docs)
        if time_of is not None:
            tv = time_of(si, tv)
        vv = column_values(oracle, seg, v, docs)
        keys = [column_values(oracle, seg, g, docs) for g in group_by]
        for i in range(len(docs)):
            key = tuple(_py(k[i]) for k in keys)
            cur = out.get(key)
            ti = int(tv[i])
            if cur is None or (ti >= cur[0] if last else ti < cur[0]):
                out[key] = (ti, _py(vv[i]))
    return out
