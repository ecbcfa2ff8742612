"""numpy restatement of the GPU left, right and full outer bucket joins (hs_bucket_join_outer), Spark 3.1's
SortMergeJoinExec with joinType LeftOuter / RightOuter / FullOuter over a filter below each side.

Per bucket, each side's rows are taken in oracle.index_rows order on the key columns, as in join_oracle.  A row that
fails its side's filter is gone: not output on a preserved side, matching nothing on the other.  A row with a null in
any key column matches nothing.  The key tuples of both sides get joint codes (join_oracle.tuple_codes).

- left: every left row once per matching right row, in right sorted order, or once with no right row; (bucket, left
  sorted position, right sorted position) order.
- right: the mirror image, (bucket, right sorted position, left sorted position).
- full: per bucket, the bucket's left-outer rows, then its right rows that matched nothing, in right sorted order.

A missing row is -1.
"""
from typing import Dict, Sequence, Tuple

import numpy as np

import filter_oracle as F
import join_oracle as J
from oracle import oracle as O


def _probe(pp: np.ndarray, pcode: np.ndarray, pkey_ok: np.ndarray, tp: np.ndarray, tcode: np.ndarray):
    """(probe row, target row or -1) for the probe positions pp against the matchable target positions tp (ascending
    codes): each probe row with its matches in target order, or once with -1."""
    tc = tcode[tp]
    c = pcode[pp]
    lo, hi = np.searchsorted(tc, c, "left"), np.searchsorted(tc, c, "right")
    n = np.where(pkey_ok[pp], hi - lo, 0)
    reps = np.maximum(n, 1)
    prow = np.repeat(pp, reps)
    start = np.repeat(np.cumsum(reps) - reps, reps)
    j = np.arange(len(prow)) - start            # rank of the pair inside its probe row's run
    first = np.repeat(lo, reps)
    matched = np.repeat(n > 0, reps)
    trow = np.full(len(prow), -1, dtype=np.int64)
    trow[matched] = tp[(first + j)[matched]]
    return prow.astype(np.int64), trow


def outer_join(left: Dict[str, np.ndarray], right: Dict[str, np.ndarray], nb: int, left_keys: Sequence[str],
               right_keys: Sequence[str], how: str, left_predicates=(), right_predicates=(), left_valids=None,
               right_valids=None, left_mask=None, right_mask=None) -> Tuple[np.ndarray, np.ndarray]:
    """(left rows, right rows) of every output row in the engine's order, -1 where a side is padded.  how is "left",
    "right" or "full"; the other arguments are join_exists_oracle.exists_join's."""
    assert how in ("left", "right", "full")
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
        sides.append((np.asarray(perm, dtype=np.int64), offs, keep, key_ok))
    nl = len(left[left_keys[0]])
    joint = [np.concatenate([np.asarray(left[lk]), np.asarray(right[rk])]) for lk, rk in zip(left_keys, right_keys)]
    joint = [np.array(c.tolist(), dtype=object) if c.dtype == object else c for c in joint]
    codes = J.tuple_codes(joint)
    code = (codes[:nl], codes[nl:])
    out_l, out_r = [], []
    for b in range(nb):
        pos = []
        for perm, offs, keep, _ in sides:
            p = perm[offs[b]:offs[b + 1]]
            pos.append(p[keep[p]])
        lp, rp = pos
        lok, rok = sides[0][3], sides[1][3]
        if how == "right":
            r, l = _probe(rp, code[1], rok, lp[lok[lp]], code[0])
            out_l.append(l)
            out_r.append(r)
            continue
        l, r = _probe(lp, code[0], lok, rp[rok[rp]], code[1])
        out_l.append(l)
        out_r.append(r)
        if how == "full":
            lmatch = lp[lok[lp]]
            unmatched = rp[~(rok[rp] & np.isin(code[1][rp], code[0][lmatch]))]
            out_l.append(np.full(len(unmatched), -1, dtype=np.int64))
            out_r.append(unmatched.astype(np.int64))
    if not out_l:
        return np.empty(0, dtype=np.int64), np.empty(0, dtype=np.int64)
    return np.concatenate(out_l).astype(np.int64), np.concatenate(out_r).astype(np.int64)
