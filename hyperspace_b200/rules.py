"""Index selection (the conditions of FilterIndexRule / JoinIndexRule) and the physical operators that run on the GPU.

Restated from the reference's driver-side rule layer (no Catalyst here; the conditions are the same, the plan shapes
are the linear ``Project?(Filter?(Relation))`` and ``Join(linear, linear)`` the reference's rules accept):
  * CandidateIndexCollector / FileSignatureFilter  -- index/rules/CandidateIndexCollector.scala:28-60,
    index/rules/FileSignatureFilter.scala:33-192 (exact signature match, or Hybrid Scan's appended/deleted byte ratios)
  * FilterIndexRule / FilterIndexRanker             -- index/covering/FilterIndexRule.scala:33-174, FilterIndexRanker.scala:28-65
  * JoinIndexRule / JoinIndexRanker                 -- index/covering/JoinIndexRule.scala:47-720, JoinIndexRanker.scala:28-95
  * transformPlanToUseIndex / Hybrid Scan           -- index/covering/CoveringIndexRuleUtils.scala:55-288
Physical execution is the C ABI: hs_filter_scan_expr (K1 + K7) and hs_bucket_join_expr (K1 + K8), which takes the join
type (inner, left semi / left anti, left / right / full outer).
"""
from __future__ import annotations

import os
import re
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import log_entry as LE
from .session import FilterNode, JoinNode, Predicate, ProjectNode, RelationNode, spark_values

_BUCKET_RE = re.compile(r"_(\d+)(?:\..*)?$")  # Spark BucketingUtils.getBucketId


def bucket_id_of(file_name: str) -> int:
    m = _BUCKET_RE.search(os.path.basename(file_name))
    if not m:
        raise LE.HyperspaceException(f"cannot parse a bucket id from {file_name}")
    return int(m.group(1))


def index_signature(rel: RelationNode) -> str:
    """IndexSignatureProvider (index/IndexSignatureProvider.scala:33-51) = md5(fileBasedSignature + planSignature); the
    plan of a bare relation is the single node "LogicalRelation" (PlanSignatureProvider.scala:28-44)."""
    file_sig = LE.md5_hex(rel.signature)
    plan_sig = LE.md5_hex("LogicalRelation")
    return LE.md5_hex(file_sig + plan_sig)


def active_indexes(session) -> List[LE.IndexLogEntry]:
    root = LE.PathResolver(session.conf).system_path
    out = []
    if os.path.isdir(root):
        for name in sorted(os.listdir(root)):
            e = LE.IndexLogManager(os.path.join(root, name)).get_latest_stable_log()
            if e is not None and e.state == LE.States.ACTIVE:
                out.append(e)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# candidate collection
# ---------------------------------------------------------------------------------------------------------------------

@dataclass
class Candidate:
    entry: LE.IndexLogEntry
    appended: List[Tuple[str, int, int]]   # source files not covered by the index (Hybrid Scan)
    deleted_ids: List[int]                 # lineage ids of indexed source files that no longer exist
    common_bytes: int


def _candidate(session, rel: RelationNode, e: LE.IndexLogEntry) -> Optional[Candidate]:
    cols = {c.lower() for c in rel.column_names}
    if not all(c.lower() in cols for c in e.indexedColumns + [c for c in e.includedColumns if c != LE.DATA_FILE_NAME_ID]):
        return None  # ColumnSchemaFilter
    cur = {LE.FileInfo(u, s, m) for u, s, m in rel.files}
    indexed = {f: f.id for f in e.source_file_infos}
    # quick refresh bookkeeping: files recorded in Update are already known appended / deleted
    sig_match = any(s.value == index_signature(rel) for s in e.signatures)
    if sig_match and not e.appended_files and not e.deleted_files:
        return Candidate(e, [], [], sum(f.size for f in indexed))
    if sig_match:
        # refreshIndex(mode = "quick") recorded the appended / deleted source files in Update and re-signed the entry: the
        # reference then applies the Hybrid Scan transformation from those recorded files whether or not
        # spark.hyperspace.index.hybridscan.enabled is set (CoveringIndexRuleUtils.scala:68-84, RefreshQuickAction.scala:32-80)
        recorded_deleted = e.deleted_files
        if not recorded_deleted or e.has_lineage_column:
            common = cur & set(indexed)
            return Candidate(e, sorted((f.name, f.size, f.modifiedTime) for f in e.appended_files),
                             sorted(f.id for f in recorded_deleted), sum(f.size for f in common))
    if not session.conf.hybrid_scan_enabled:
        return None
    common = cur & set(indexed)
    if not common:
        return None
    appended = [f for f in cur if f not in indexed]
    deleted = [f for f in indexed if f not in cur]
    if deleted and not e.has_lineage_column:
        return None
    cur_bytes = sum(f.size for f in cur) or 1
    idx_bytes = sum(f.size for f in indexed) or 1
    if sum(f.size for f in appended) / cur_bytes > session.conf.hybrid_scan_appended_ratio:
        return None
    if sum(f.size for f in deleted) / idx_bytes > session.conf.hybrid_scan_deleted_ratio:
        return None
    return Candidate(e, sorted((f.name, f.size, f.modifiedTime) for f in appended), sorted(indexed[f] for f in deleted),
                     sum(f.size for f in common))


def candidates_for(session, rel: RelationNode) -> List[Candidate]:
    out = []
    for e in active_indexes(session):
        c = _candidate(session, rel, e)
        if c is not None:
            out.append(c)
    return out


def _covers(e: LE.IndexLogEntry, columns: Sequence[str]) -> bool:
    have = {c.lower() for c in e.indexedColumns + e.includedColumns}
    return all(c.lower() in have for c in columns)


# ---------------------------------------------------------------------------------------------------------------------
# linear plan extraction
# ---------------------------------------------------------------------------------------------------------------------

@dataclass
class Linear:
    relation: RelationNode
    predicate: Optional[Predicate]
    project: Optional[List[str]]

    @property
    def output(self) -> List[str]:
        return self.project if self.project is not None else self.relation.column_names

    def referenced(self) -> List[str]:
        cols = list(self.output)
        if self.predicate:
            cols += [c for c in self.predicate.columns if c not in cols]
        return cols


def _linear(plan) -> Optional[Linear]:
    project = None
    pred = None
    node = plan
    if isinstance(node, ProjectNode):
        project = node.columns
        node = node.child
    if isinstance(node, FilterNode):
        pred = node.predicate
        node = node.child
        while isinstance(node, FilterNode):
            pred = pred & node.predicate
            node = node.child
    if isinstance(node, ProjectNode) and project is None:
        project = node.columns
        node = node.child
    if isinstance(node, RelationNode):
        return Linear(node, pred, project)
    return None


# ---------------------------------------------------------------------------------------------------------------------
# physical operators
# ---------------------------------------------------------------------------------------------------------------------

def _file_images(files: Sequence[str]):
    from . import _native

    return [_native.FileImage(path=LE.from_uri(f)) for f in files]


def _concat(parts: List[Dict[str, np.ndarray]], columns: List[str]) -> Dict[str, np.ndarray]:
    parts = [p for p in parts if p]
    if not parts:
        return {c: np.empty(0) for c in columns}
    return {c: np.concatenate([p[c] for p in parts]) for c in columns}


def _host_column(d: np.ndarray) -> np.ndarray:
    """A result column copied out of the batch; string / binary columns (object arrays of bytes) become text when every
    value is UTF-8 and stay bytes otherwise."""
    if d.dtype != object:
        return d.copy()
    try:
        return np.array([v.decode("utf-8") for v in d], dtype=object)
    except UnicodeDecodeError:
        return d.copy()


def _terms_text(pred) -> str:
    """The disjunction terms, column comparisons and expression comparisons of a filter for explain(), long lists cut
    short: `k IN (1, 2, 3, ... 997 more)`, `(a < b)`, `((a + b) < c)`."""
    anys = pred.disjunctions() if pred else []
    cmps = pred.comparisons() if pred else []
    exprs = pred.expressions() if pred else []
    return "".join(f", where=({a})" for a in anys + cmps + exprs)


class ScanExec:
    """Filter / projection over a relation: index-only scan, Hybrid Scan, or plain source scan -- hs_filter_scan_expr with
    the filter's comparisons with literals as its predicates, its disjunctions (isin, |) as its terms, its comparisons
    between two columns as its compares and its comparisons of arithmetic expressions as its exprs."""

    def __init__(self, session, lin: Linear, cand: Optional[Candidate]):
        self.session, self.lin, self.cand = session, lin, cand

    def describe(self) -> str:
        if self.cand is None:
            return f"GpuSourceScan(files={len(self.lin.relation.files)}, predicate={self.lin.predicate}{_terms_text(self.lin.predicate)})"
        e = self.cand.entry
        extra = ""
        if self.cand.appended or self.cand.deleted_ids:
            extra = f", hybridScan(appended={len(self.cand.appended)}, deletedIds={self.cand.deleted_ids})"
        return (f"GpuIndexScan(Hyperspace(Type: CI, Name: {e.name}, LogVersion: {e.id}), files={len(e.index_files)}{extra}"
                f"{_terms_text(self.lin.predicate)})")

    def _scan(self, files, key, out_cols, sorted_on_key, deleted_ids=(), buckets=None, num_buckets=0):
        preds = self.lin.predicate.conjuncts() if self.lin.predicate else []
        terms = [a.as_native() for a in self.lin.predicate.disjunctions()] if self.lin.predicate else []
        cmps = [c.as_native() for c in self.lin.predicate.comparisons()] if self.lin.predicate else []
        exprs = [e.as_native() for e in self.lin.predicate.expressions()] if self.lin.predicate else []
        # file_buckets only where the files are bucketed on the key alone
        batch, _ = self.session.gpu.filter_scan_expr(files, key, out_cols, preds, terms, cmps, exprs, sorted_on_key=sorted_on_key,
                                                     deleted_file_ids=list(deleted_ids), file_buckets=buckets, num_buckets=num_buckets)
        types = dict(self.lin.relation.schema)
        out = {n: spark_values(_host_column(d), types.get(n)) for n, d, _ in batch.columns}
        batch.free()
        return out

    def execute(self) -> Dict[str, np.ndarray]:
        out_cols = self.lin.output
        if self.cand is None:
            return self._scan(_file_images([f[0] for f in self.lin.relation.files]), None, out_cols, False)
        e = self.cand.entry
        first = e.indexedColumns[0]
        pred_cols = self.lin.predicate.columns if self.lin.predicate else []
        key = next((c for c in pred_cols if c.lower() == first.lower()), first)
        parts = []
        # a point lookup on the key of a single-column index reads only the files of the points' buckets
        terms = self.lin.predicate.disjunctions() if self.lin.predicate else []
        buckets = [bucket_id_of(f) for f in e.index_files] if terms and len(e.indexedColumns) == 1 else None
        nb = e.numBuckets if buckets is not None else 0
        if self.cand.deleted_ids:  # NOT (_data_file_id IN deleted): CoveringIndexRuleUtils.scala:244-253
            parts.append(self._scan(_file_images(e.index_files), key, out_cols, False, self.cand.deleted_ids, buckets, nb))
        else:  # index files are sorted on the first indexed column: binary search when the filter bounds it
            parts.append(self._scan(_file_images(e.index_files), key, out_cols, key in pred_cols, (), buckets, nb))
        if self.cand.appended:     # appended source files are scanned raw and unioned: CoveringIndexRuleUtils.scala:191-212
            parts.append(self._scan(_file_images([f[0] for f in self.cand.appended]), None, out_cols, False))
        return _concat(parts, out_cols)


# JoinNode.how of the outer joins -> join_type of Context.bucket_join_expr
_OUTER = {"leftouter": "left", "rightouter": "right", "fullouter": "full"}
_JOIN_TYPE = {"inner": "inner", "leftsemi": "semi", "leftanti": "anti", **_OUTER}


class BucketJoinExec:
    """Join of two index scans bucket by bucket (no exchange), or of two on-the-fly bucketed sides when no index applies.
    ``keys`` are the (left, right) key pairs in the order both sides are bucketed and sorted on: the left index's indexed
    columns when the indexes serve, the condition's order otherwise; None when the condition is not a one-to-one equi-join
    between the two sides, which the GPU join cannot run.  A filter below a side becomes that side's predicates.  ``how``
    is "inner", "leftsemi" / "leftanti" (left rows only, each at most once), or "leftouter" / "rightouter" / "fullouter"
    (rows padded with nulls where the other side has no match); hs_bucket_join_expr runs them all."""

    def __init__(self, session, left: Linear, right: Linear, keys: Optional[List[Tuple[str, str]]], lcand: Optional[Candidate],
                 rcand: Optional[Candidate], condition: Optional[List[Tuple[str, str]]] = None, how: str = "inner"):
        self.session, self.left, self.right, self.keys, self.lcand, self.rcand = session, left, right, keys, lcand, rcand
        self.condition = condition if condition is not None else keys
        self.how = how

    def describe(self) -> str:
        def side(c, lin):
            if c is None:
                return f"GpuShuffle(files={len(lin.relation.files)})"
            return f"Hyperspace(Type: CI, Name: {c.entry.name}, LogVersion: {c.entry.id})"

        keys = ", ".join(f"{l} = {r}" for l, r in (self.keys or self.condition or []))
        filters = "".join(f", {n}Filter={lin.predicate.conjuncts()}{_terms_text(lin.predicate)}"
                          for n, lin in (("left", self.left), ("right", self.right)) if lin.predicate)
        jt = {"leftsemi": ", joinType=LeftSemi", "leftanti": ", joinType=LeftAnti", "leftouter": ", joinType=LeftOuter",
              "rightouter": ", joinType=RightOuter", "fullouter": ", joinType=FullOuter"}.get(self.how, "")
        return (f"GpuBucketJoin({side(self.lcand, self.left)}, {side(self.rcand, self.right)}, keys=[{keys}]{jt}{filters}, "
                "exchange=none)")

    def _side(self, lin: Linear, cand: Optional[Candidate], keys: List[str], nb: int):
        """(file images, bucket ids, temporaries to free)."""
        from . import _native

        ctx = self.session.gpu
        temps = []
        low = {k.lower() for k in keys}
        cols = [c for c in lin.referenced() if c.lower() not in low]
        if cand is None:
            res, _ = ctx.create_index(_file_images([f[0] for f in lin.relation.files]), keys, cols, nb, output=_native.HS_OUT_DEVICE)
            temps.append(res)
            return res.as_sources(), [f.bucket for f in res.files], temps
        files = list(cand.entry.index_files)
        images = _file_images(files)
        buckets = [bucket_id_of(f) for f in files]
        if cand.deleted_ids:
            raise LE.HyperspaceException("join over an index with deleted source files needs refreshIndex first")
        if cand.appended:  # BucketUnion(index scan, repartitioned appended rows): CoveringIndexRuleUtils.scala:256-284
            res, _ = ctx.create_index(_file_images([f[0] for f in cand.appended]), keys, cols, nb, output=_native.HS_OUT_DEVICE)
            temps.append(res)
            images += res.as_sources()
            buckets += [f.bucket for f in res.files]
        return images, buckets, temps

    def execute(self) -> Dict[str, np.ndarray]:
        if self.keys is None:
            raise LE.HyperspaceException(f"join condition {self.condition} is not a one-to-one equi-join between the two sides")
        nb = self.lcand.entry.numBuckets if self.lcand else (self.rcand.entry.numBuckets if self.rcand else self.session.conf.num_buckets)
        lkeys, rkeys = [l for l, _ in self.keys], [r for _, r in self.keys]
        li, lb, lt = self._side(self.left, self.lcand, lkeys, nb)
        ri, rb, rt = self._side(self.right, self.rcand, rkeys, nb)
        try:
            lp = self.left.predicate.conjuncts() if self.left.predicate else []
            rp = self.right.predicate.conjuncts() if self.right.predicate else []
            lt_, rt_ = ([a.as_native() for a in lin.predicate.disjunctions()] if lin.predicate else [] for lin in (self.left, self.right))
            lc_, rc_ = ([c.as_native() for c in lin.predicate.comparisons()] if lin.predicate else [] for lin in (self.left, self.right))
            lx_, rx_ = ([e.as_native() for e in lin.predicate.expressions()] if lin.predicate else [] for lin in (self.left, self.right))
            right_out = [] if self.how in ("leftsemi", "leftanti") else self.right.output
            batch, _ = self.session.gpu.bucket_join_expr(li, lb, ri, rb, nb, lkeys, rkeys, self.left.output, right_out,
                                                         _JOIN_TYPE[self.how], lp, rp, lt_, rt_, lc_, rc_, lx_, rx_)
        finally:
            for t in lt + rt:
                t.free()
        out: Dict[str, np.ndarray] = {}
        nleft = len(self.left.output)
        for i, (n, d, v) in enumerate(batch.columns):
            name = n if n not in out else f"{n}_right"
            types = dict((self.left if i < nleft else self.right).relation.schema)
            out[name] = spark_values(_host_column(d), types.get(n))
            if self.how in _OUTER and v is not None:  # an outer join's nulls: masked where the column is not valid
                out[name] = np.ma.MaskedArray(out[name], mask=np.asarray(v) == 0)
        batch.free()
        return out


# ---------------------------------------------------------------------------------------------------------------------
# the rules
# ---------------------------------------------------------------------------------------------------------------------

def rank_filter_candidates(session, cands: Sequence[Candidate]) -> Optional[Candidate]:
    """FilterIndexRanker.rank (covering/FilterIndexRanker.scala:43-64): the smallest index wins; under Hybrid Scan the index
    with the most source bytes in common with the relation wins instead (first one on a tie, like Scala's maxBy/minBy)."""
    if not cands:
        return None
    if session.conf.hybrid_scan_enabled:
        return max(cands, key=lambda c: c.common_bytes)
    return min(cands, key=lambda c: c.entry.index_files_size_in_bytes)


def rank_join_pairs(session, pairs: Sequence[Tuple[Candidate, Candidate]]) -> List[Tuple[Candidate, Candidate]]:
    """JoinIndexRanker.rank (covering/JoinIndexRanker.scala:52-90), best pair first: pairs with equal bucket counts come
    before unequal ones; among equal-bucket pairs more buckets is better -- unless Hybrid Scan is on and the pairs differ in
    common source bytes, then more common bytes is better; unequal-bucket pairs keep their order (more common bytes first
    under Hybrid Scan).  Stable, like Scala's sortWith on a Seq."""
    import functools

    hybrid = session.conf.hybrid_scan_enabled

    def before(p1, p2) -> bool:
        (l1, r1), (l2, r2) = p1, p2
        c1, c2 = l1.common_bytes + r1.common_bytes, l2.common_bytes + r2.common_bytes
        eq1, eq2 = l1.entry.numBuckets == r1.entry.numBuckets, l2.entry.numBuckets == r2.entry.numBuckets
        if eq1 and eq2:
            if not hybrid or c1 == c2:
                return l1.entry.numBuckets > l2.entry.numBuckets
            return c1 > c2
        if eq1:
            return True
        if eq2:
            return False
        return (not hybrid) or c1 > c2

    def cmp(p1, p2) -> int:
        if before(p1, p2):
            return -1
        if before(p2, p1):
            return 1
        return 0

    # Scala: indexPairs.sortWith(before) = a stable sort under Ordering.fromLessThan(before), restated literally
    return sorted(pairs, key=functools.cmp_to_key(cmp))


def filter_index_rule(session, lin: Linear) -> Optional[Candidate]:
    """FilterIndexRule: the first indexed column must appear in the filter, and the index must cover every referenced
    column (FilterIndexRule.scala:60-103); ranked by rank_filter_candidates."""
    if not lin.predicate:
        return None
    fcols = {c.lower() for c in lin.predicate.columns}
    good = [c for c in candidates_for(session, lin.relation)
            if c.entry.indexedColumns[0].lower() in fcols and _covers(c.entry, lin.referenced())]
    return rank_filter_candidates(session, good)


def join_key_pairs(left: Linear, right: Linear, pairs: Sequence[Tuple[str, str]]) -> Optional[List[Tuple[str, str]]]:
    """JoinAttributeFilter (JoinIndexRule.scala:164-170, 262-301): every equality must compare a column of the left side
    with one of the right side, in either orientation, and the columns must map one to one; repeated equalities collapse
    (names match case-insensitively).  Returns the (left, right) pairs in condition order, or None."""
    lcols = {c.lower(): c for c in left.relation.column_names}
    rcols = {c.lower(): c for c in right.relation.column_names}
    out, seen, l2r, r2l = [], set(), {}, {}
    for a, b in pairs:
        if a.lower() in lcols and b.lower() in rcols:
            l, r = lcols[a.lower()], rcols[b.lower()]
        elif b.lower() in lcols and a.lower() in rcols:
            l, r = lcols[b.lower()], rcols[a.lower()]
        else:
            return None  # both columns on one side (or unknown)
        if l2r.setdefault(l.lower(), r.lower()) != r.lower() or r2l.setdefault(r.lower(), l.lower()) != l.lower():
            return None  # not one-to-one
        if (l.lower(), r.lower()) not in seen:
            seen.add((l.lower(), r.lower()))
            out.append((l, r))
    return out


def join_index_rule(session, left: Linear, right: Linear, keys: Sequence[Tuple[str, str]]):
    """JoinIndexRule over the (left, right) key pairs of join_key_pairs: JoinColumnFilter -- an index's indexed columns
    equal its side's key columns as a set, and it covers every column its side references, filter columns included
    (JoinIndexRule.scala:399-463); JoinRankFilter -- a pair is compatible only when the right index's indexed columns are
    the left index's, mapped through the keys, in the same order (JoinIndexRule.scala:569-616); pairs ranked by
    rank_join_pairs.  The GPU merge join needs both sides bucketed alike, so only the best EQUAL-bucket pair is used (the
    reference would re-shuffle one side of an unequal pair; here the query then runs without indexes)."""
    # (an index whose source lost files would need the lineage NOT-IN filter below the merge join, which the GPU join does
    # not apply: such a candidate is skipped and the query falls back to the next pair / to no index, as the fail-open rule
    # layer of the reference would -- ApplyHyperspace.scala:57-64)
    lset, rset = {l.lower() for l, _ in keys}, {r.lower() for _, r in keys}
    l2r = {l.lower(): r.lower() for l, r in keys}
    lc = [c for c in candidates_for(session, left.relation)
          if {x.lower() for x in c.entry.indexedColumns} == lset and len(c.entry.indexedColumns) == len(lset)
          and _covers(c.entry, left.referenced()) and not c.deleted_ids]
    rc = [c for c in candidates_for(session, right.relation)
          if {x.lower() for x in c.entry.indexedColumns} == rset and len(c.entry.indexedColumns) == len(rset)
          and _covers(c.entry, right.referenced()) and not c.deleted_ids]

    # Spark's analyzer puts a Cast on one side when the key types differ, and a condition over a Cast is not the plain
    # attribute equality the rule asks for (JoinIndexRule.scala:143-163): no index then.  It also matters physically:
    # hashInt and hashLong (and hashUnsafeBytes) send equal values to different buckets.
    def key_type(lin: Linear, key: str):
        return next((t for n, t in lin.relation.schema if n.lower() == key.lower()), None)

    if any(key_type(left, l) != key_type(right, r) for l, r in keys):
        return None

    def compatible(a: Candidate, b: Candidate) -> bool:
        return [l2r[x.lower()] for x in a.entry.indexedColumns] == [x.lower() for x in b.entry.indexedColumns]

    ranked = rank_join_pairs(session, [(a, b) for a in lc for b in rc if compatible(a, b)])
    if not ranked or ranked[0][0].entry.numBuckets != ranked[0][1].entry.numBuckets:
        return None
    return ranked[0]


def plan_query(session, plan):
    """ApplyHyperspace + physical planning: returns an operator with describe() / execute()."""
    enabled = session.isHyperspaceEnabled()
    node = plan
    post_project = None
    if isinstance(node, ProjectNode) and isinstance(node.child, JoinNode):
        post_project = node.columns
        node = node.child
    if isinstance(node, JoinNode):
        l, r = _linear(node.left), _linear(node.right)
        if l is None or r is None:
            raise LE.HyperspaceException("only joins of linear plans (Project?(Filter?(Relation))) are handled")
        keys = join_key_pairs(l, r, node.pairs)
        semi_or_anti = node.how in ("leftsemi", "leftanti")
        if semi_or_anti:  # the right side of a semi / anti join is only probed: it outputs its keys, its filter is read
            r = Linear(r.relation, r.predicate, [b for _, b in keys] if keys else [])
        if post_project is not None:  # column pruning: each side outputs only what the final projection needs + its keys
            lout, rout = l.output, r.output
            lneed = [c for c in post_project if c in lout]
            rneed = [c for c in post_project if c not in lout and c in rout]
            if semi_or_anti and rneed:
                raise LE.HyperspaceException(f"a left semi / anti join outputs left columns only: cannot resolve {rneed}")
            missing = [c for c in post_project if c not in lout and c not in rout]
            if missing:
                raise LE.HyperspaceException(f"cannot resolve columns {missing}")
            # the filter stays on its side: its columns are read, not output
            lk = [a for a, _ in keys] if keys else []
            rk = [b for _, b in keys] if keys else []
            l = Linear(l.relation, l.predicate, lneed + [k for k in lk if k not in lneed])
            r = Linear(r.relation, r.predicate, rneed + [k for k in rk if k not in rneed])
        pair = join_index_rule(session, l, r, keys) if enabled and keys else None
        if pair:  # both sides bucketed and sorted in the left index's column order
            order = [x.lower() for x in pair[0].entry.indexedColumns]
            keys = sorted(keys, key=lambda p: order.index(p[0].lower()))
        op = BucketJoinExec(session, l, r, keys, pair[0] if pair else None, pair[1] if pair else None, list(node.pairs), node.how)
        if post_project is not None:
            return _Projected(op, post_project)
        return op
    lin = _linear(plan)
    if lin is None:
        raise LE.HyperspaceException("unsupported plan shape for the GPU engine")
    cand = filter_index_rule(session, lin) if enabled else None
    return ScanExec(session, lin, cand)


class _Projected:
    def __init__(self, op, columns):
        self.op, self.columns = op, columns

    def describe(self):
        return f"Project({self.columns}) <- {self.op.describe()}"

    def execute(self):
        res = self.op.execute()
        return {c: res[c] for c in self.columns}
