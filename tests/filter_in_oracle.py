"""numpy restatement of Spark 3.1's In, and of an Or of ranges on one column, beside filter_oracle's conjunctions.

`k IN (v1, ..., vn)` is `k = v1 OR ... OR k = vn`, every `=` evaluated as filter_oracle.compare evaluates it (the wider
type decides, NaN equals NaN, -0.0 equals 0.0); a range is filter_oracle.predicate_mask of one predicate.  A null row is
never selected.  A term is (column, values, ranges) with ranges as (lo, lo_strict, hi, hi_strict), the shape
Context.filter_scan_any takes.
"""
import numpy as np

import filter_oracle as F


def term_mask(columns, term, valids=None) -> np.ndarray:
    valids = valids or {}
    name, values, ranges = term
    v = columns[name]
    m = np.zeros(len(v), dtype=bool)
    for x in (values.tolist() if isinstance(values, np.ndarray) else values):
        if x is None:
            continue
        m |= F.compare(v, x) == 0
    for lo, ls, hi, hs in ranges:
        m |= F.predicate_mask({name: v}, [(name, lo, ls, hi, hs)])
    if name in valids:
        m &= np.asarray(valids[name], dtype=bool)
    return m


def mask(columns, predicates, terms, valids=None) -> np.ndarray:
    """Rows where every predicate and every term holds."""
    m = F.predicate_mask(columns, predicates, valids)
    for t in terms:
        m &= term_mask(columns, t, valids)
    return m
