"""numpy restatement of the GPU left semi / left anti bucket join (hs_bucket_join_exists), Spark 3.1's
SortMergeJoinExec with joinType LeftSemi / LeftAnti.

Per bucket, each side's rows are taken in oracle.index_rows order on the key columns, as in join_oracle.  A left row is
a candidate when its side's filter holds; a right row can match when its filter holds and no key column is null.  The
key tuples of both sides get joint codes (join_oracle.tuple_codes).  Semi keeps a candidate left row whose key has no
null and whose code some matchable right row of the same bucket shares; anti keeps every other candidate left row,
null-key rows included (a null key matches nothing, and an unmatched row is output).  The kept left rows come out once
each, in (bucket, left sorted position) order.
"""
from typing import Dict, Sequence

import numpy as np

import filter_oracle as F
import join_oracle as J
from oracle import oracle as O


def exists_join(left: Dict[str, np.ndarray], right: Dict[str, np.ndarray], nb: int, left_keys: Sequence[str],
                right_keys: Sequence[str], how: str, left_predicates=(), right_predicates=(), left_valids=None,
                right_valids=None, left_mask=None, right_mask=None) -> np.ndarray:
    """The left rows a semi (how="semi") or anti (how="anti") join outputs, in the engine's order.  Tables are {name:
    numpy array} (object arrays of bytes for strings); valids are {name: bool array} for nullable columns; predicates
    are filter_oracle.predicate_mask's; left_mask / right_mask (bool per row) AND further filters onto a side, for the
    filter forms predicate_mask does not state."""
    assert how in ("semi", "anti")
    sides = []
    for cols, keys, preds, valids, extra in ((left, left_keys, left_predicates, left_valids, left_mask),
                                             (right, right_keys, right_predicates, right_valids, right_mask)):
        n = len(cols[keys[0]])
        kvalid = {k: np.asarray(valids[k]).astype(np.uint8) for k in keys if valids and k in valids}
        perm, offs, _ = O.index_rows(cols, list(keys), [], nb, kvalid or None)
        keep = np.ones(n, dtype=bool)
        if preds:
            keep &= F.predicate_mask(cols, list(preds), {c: v for c, v in (valids or {}).items()})
        if extra is not None:
            keep &= np.asarray(extra, dtype=bool)
        key_ok = np.ones(n, dtype=bool)
        for k in keys:
            key_ok &= J._valid(valids, k, n)
        sides.append((perm, offs, keep, key_ok))
    nl = len(left[left_keys[0]])
    joint = [np.concatenate([np.asarray(left[lk]), np.asarray(right[rk])]) for lk, rk in zip(left_keys, right_keys)]
    joint = [np.array(c.tolist(), dtype=object) if c.dtype == object else c for c in joint]
    codes = J.tuple_codes(joint)
    lcode, rcode = codes[:nl], codes[nl:]
    (lperm, loffs, lkeep, lkey_ok), (rperm, roffs, rkeep, rkey_ok) = sides
    out = []
    for b in range(nb):
        lp = lperm[loffs[b]:loffs[b + 1]]
        rp = rperm[roffs[b]:roffs[b + 1]]
        lp, rp = lp[lkeep[lp]], rp[rkeep[rp] & rkey_ok[rp]]
        matched = np.isin(lcode[lp], rcode[rp]) & lkey_ok[lp]
        out.append(lp[matched] if how == "semi" else lp[~matched])
    return np.concatenate(out).astype(np.int64) if out else np.empty(0, dtype=np.int64)
