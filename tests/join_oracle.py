"""numpy restatement of the GPU bucket join over several key columns with a filter below each side -- what
hs_bucket_join_where is compared against.

Per bucket, each side's rows are taken in oracle.index_rows order on the key columns (bucket, then the keys ascending
nulls first, then the source row), which is the order of the index files and of the engine's re-sort of multi-file
buckets.  Rows with a null in any key column, or where a predicate of their side fails (filter_oracle.predicate_mask), are
dropped.  The key tuples of both sides are then rank-encoded jointly into int64 codes that keep their order, and
oracle.merge_join on the codes gives the pairs in the engine's order: (bucket, left sorted position, right sorted
position).
"""
from typing import Dict, Optional, Sequence, Tuple

import numpy as np

import filter_oracle as F
from oracle import oracle as O


def _ranks(values: np.ndarray) -> np.ndarray:
    """Dense order-preserving ranks of one column (object arrays of bytes compare as unsigned bytes)."""
    if values.dtype == object:
        uniq = sorted(set(values.tolist()))
        pos = {v: i for i, v in enumerate(uniq)}
        return np.array([pos[v] for v in values.tolist()], dtype=np.int64)
    return np.unique(values, return_inverse=True)[1].astype(np.int64).reshape(-1)


def tuple_codes(columns: Sequence[np.ndarray]) -> np.ndarray:
    """int64 codes of the rows' key tuples: equal tuples get equal codes, and codes ascend with the tuples."""
    code = np.zeros(len(columns[0]), dtype=np.int64)
    for c in columns:
        r = _ranks(c)
        code = _ranks(code * (int(r.max(initial=0)) + 1) + r)  # re-ranked after every column: never overflows
    return code


def _valid(valids, name, n):
    v = (valids or {}).get(name)
    return np.ones(n, dtype=bool) if v is None else np.asarray(v, dtype=bool)


def bucket_join(left: Dict[str, np.ndarray], right: Dict[str, np.ndarray], nb: int, left_keys: Sequence[str],
                right_keys: Sequence[str], left_predicates=(), right_predicates=(), left_valids=None, right_valids=None
                ) -> Tuple[np.ndarray, np.ndarray]:
    """(left rows, right rows) of every output pair, in the engine's output order.  Tables are {name: numpy array} (object
    arrays of bytes for strings); valids are {name: bool array} for nullable columns."""
    sides = []
    for cols, keys, preds, valids in ((left, left_keys, left_predicates, left_valids),
                                      (right, right_keys, right_predicates, right_valids)):
        n = len(cols[keys[0]])
        kvalid = {k: np.asarray(valids[k]).astype(np.uint8) for k in keys if valids and k in valids}
        perm, offs, _ = O.index_rows(cols, list(keys), [], nb, kvalid or None)
        keep = np.ones(n, dtype=bool)
        for k in keys:
            keep &= _valid(valids, k, n)
        if preds:
            keep &= F.predicate_mask(cols, list(preds), {c: v for c, v in (valids or {}).items()})
        sides.append((perm, offs, keep))
    # one joint code per row of either side
    nl = len(left[left_keys[0]])
    joint = [np.concatenate([np.asarray(left[lk]), np.asarray(right[rk])]) for lk, rk in zip(left_keys, right_keys)]
    if any(c.dtype == object for c in joint):
        joint = [np.array(c.tolist(), dtype=object) if c.dtype == object else c for c in joint]
    codes = tuple_codes(joint)
    lcode, rcode = codes[:nl], codes[nl:]
    (lperm, loffs, lkeep), (rperm, roffs, rkeep) = sides
    out_l, out_r = [], []
    for b in range(nb):
        lp = lperm[loffs[b]:loffs[b + 1]]
        rp = rperm[roffs[b]:roffs[b + 1]]
        lp, rp = lp[lkeep[lp]], rp[rkeep[rp]]
        a, c = O.merge_join(lcode[lp], rcode[rp])
        out_l.append(lp[a])
        out_r.append(rp[c])
    return np.concatenate(out_l).astype(np.int64), np.concatenate(out_r).astype(np.int64)
