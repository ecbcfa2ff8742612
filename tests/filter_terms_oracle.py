"""numpy restatement of Spark 3.1's Not, IsNull / IsNotNull, EqualNullSafe, StringStartsWith / EndsWith / Contains and Like
in three-valued logic, built on filter_oracle / filter_in_oracle's comparisons.

Every term gives two masks over the rows, (true, unknown); false is neither.  A row is selected when every AND-ed term is
true.  Terms are tuples:
  ("in", c, values)                 In; a None in the list makes a value outside it unknown
  ("range", c, lo, ls, hi, hs)      a comparison range (filter_oracle's predicate)
  ("isnull", c) / ("isnotnull", c)
  ("eqns", c, v)                    EqualNullSafe: a null row is false; v None is IsNull
  ("startswith" | "endswith" | "contains", c, p)   bytes; the empty pattern matches every non-null value
  ("like", c, pattern)              escape '\\'; matched on the decoded UTF-8 text, as Spark matches a String
  ("not", term), ("or", [terms])
A null row gives unknown for every comparison and pattern.
"""
import re

import numpy as np

import filter_in_oracle as FI
import filter_oracle as F


def like_regex(pattern: str) -> str:
    """A LIKE pattern as a Python regex (StringUtils.escapeLikeRegex); raises ValueError with Spark's message."""
    out, i = [], 0
    while i < len(pattern):
        ch = pattern[i]
        if ch == "\\":
            if i + 1 == len(pattern):
                raise ValueError(f"the pattern '{pattern}' is invalid, it is not allowed to end with the escape character")
            nx = pattern[i + 1]
            if nx not in "_%\\":
                raise ValueError(f"the pattern '{pattern}' is invalid, the escape character is not allowed to precede '{nx}'")
            out.append(re.escape(nx))
            i += 2
            continue
        out.append("." if ch == "_" else (".*" if ch == "%" else re.escape(ch)))
        i += 1
    return "(?s)" + "".join(out)


def _as_bytes(v):
    return v.encode("utf-8") if isinstance(v, str) else bytes(v)


def evaluate(columns, term, valids=None):
    """(true, unknown) masks of one term."""
    valids = valids or {}
    kind = term[0]
    if kind == "not":
        t, u = evaluate(columns, term[1], valids)
        return ~t & ~u, u
    if kind == "or":
        parts = [evaluate(columns, x, valids) for x in term[1]]
        t = np.logical_or.reduce([p[0] for p in parts])
        return t, ~t & np.logical_or.reduce([p[1] for p in parts])
    c = term[1]
    v = columns[c]
    valid = np.asarray(valids[c], dtype=bool) if c in valids else np.ones(len(v), dtype=bool)
    null = ~valid
    if kind == "isnull":
        return null.copy(), np.zeros(len(v), bool)
    if kind == "isnotnull":
        return valid.copy(), np.zeros(len(v), bool)
    if kind == "eqns":
        if term[2] is None:
            return null.copy(), np.zeros(len(v), bool)
        return (F.compare(v, term[2]) == 0) & valid, np.zeros(len(v), bool)
    if kind == "in":
        hit = FI.term_mask({c: v}, (c, [x for x in term[2] if x is not None], [])) & valid
        miss_unknown = any(x is None for x in term[2])
        return hit, null | (valid & ~hit & miss_unknown)
    if kind == "range":
        hit = F.predicate_mask({c: v}, [(c,) + tuple(term[2:])]) & valid
        return hit, null.copy()
    p = _as_bytes(term[2]) if kind != "like" else term[2]
    if kind == "startswith":
        hit = np.array([x.startswith(p) for x in v], dtype=bool)
    elif kind == "endswith":
        hit = np.array([x.endswith(p) for x in v], dtype=bool)
    elif kind == "contains":
        hit = np.array([p in x for x in v], dtype=bool)
    elif kind == "like":
        rx = re.compile(like_regex(p))
        hit = np.array([rx.fullmatch(x.decode("utf-8")) is not None for x in v], dtype=bool)
    else:
        raise ValueError(kind)
    return hit & valid, null.copy()


def mask(columns, terms, valids=None, predicates=()):
    """Rows where every term is true (and every filter_oracle predicate holds)."""
    m = F.predicate_mask(columns, list(predicates), valids) if predicates else np.ones(len(next(iter(columns.values()))), bool)
    for t in terms:
        m &= evaluate(columns, t, valids)[0]
    return m
