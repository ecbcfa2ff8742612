// read_side.cu -- K7 sorted range select and K8 per-bucket merge join over decoded index buckets.
//
// K7 replaces the FileSourceScanExec + pushed Filter Spark runs after FilterIndexRule.applyIndex swaps the source
// relation for the index files (index/covering/FilterIndexRule.scala:135-149).  Index files are sorted on the key, so a
// range predicate is two binary searches per file instead of a predicate over every row.
// K8 replaces the bucketed scan + SortMergeJoinExec (no ShuffleExchangeExec) Spark plans after
// JoinIndexRule.applyIndex (index/covering/JoinIndexRule.scala:653-687): bucket b of the left index joins bucket b of
// the right index; every left row binary-searches its match range in the right bucket, a scan turns match counts into
// output offsets, and a second kernel emits the (left row, right row) pairs in (left, right) order.  The key tuples of
// 1-8 columns are compared column by column (k_join_count).
#include "column_expr.h"
#include "device_utils.cuh"
#include "kernels.h"

namespace hs {

namespace {

// ---- predicate evaluation (kernels.h: PredRange) -------------------------------------------------------------------
// value i of a column of type KT against a bound: -1 / 0 / +1.  Numeric values are compared as sort_encode(KT, value)
// with an encoded bound (Spark's order: NaN greatest, -0.0 == 0.0); strings as references in UTF8String byte order.
template <int KT>
__device__ __forceinline__ int cmp_bound(const void* __restrict__ col, int64_t i, uint64_t bound) {
  if constexpr (KT == HS_TYPE_STRING) {
    return string_compare(((const uint64_t*)col)[i], bound);
  } else {
    uint64_t raw;
    if constexpr (KT == HS_TYPE_INT32 || KT == HS_TYPE_FLOAT) raw = ((const uint32_t*)col)[i];
    else raw = ((const uint64_t*)col)[i];
    const uint64_t e = sort_encode(KT, raw);
    return e < bound ? -1 : (e > bound ? 1 : 0);
  }
}

// first row of the ascending rows [b, b + n) with cmp_bound(row, bound) >= t (segment-relative)
template <int KT>
__device__ __forceinline__ int64_t first_at_least(const void* col, int64_t b, int64_t n, uint64_t bound, int t) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = lo + ((hi - lo) >> 1);
    if (cmp_bound<KT>(col, b + mid, bound) < t) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// K7 window search, one thread per (sorted file, range) work item: bounds[2w] = first row inside the range, bounds[2w+1] =
// first row above it.  Numeric bounds are inclusive (strictness is folded in on the host); string bounds carry their
// strictness.
template <int KT>
__global__ void k_range_bounds(const void* __restrict__ keys, const PredRange* __restrict__ ranges,
                               const uint64_t* __restrict__ seg_offsets, const uint2* __restrict__ work, int64_t nwork,
                               int64_t* __restrict__ bounds) {
  const int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= nwork) return;
  const uint2 sr = work[w];
  const PredRange r = ranges[sr.y];
  const int64_t b = (int64_t)seg_offsets[sr.x], n = (int64_t)seg_offsets[sr.x + 1] - b;
  int64_t first = r.has_lo ? first_at_least<KT>(keys, b, n, r.lo, r.lo_strict ? 1 : 0) : 0;
  int64_t last = r.has_hi ? first_at_least<KT>(keys, b, n, r.hi, r.hi_strict ? 0 : 1) : n;
  if (last < first) last = first;
  bounds[2 * w] = first;
  bounds[2 * w + 1] = last;
}

// one thread per output row: the window holding output position o is found by binary search over the windows' output
// offsets, so millions of windows of 0-2 rows cost no more than a few long ones
__global__ void k_ranges_to_indices(const int64_t* __restrict__ win, const uint64_t* __restrict__ out_offsets, int64_t nwin,
                                    int64_t n_out, uint32_t* __restrict__ out_idx) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; o < n_out; o += stride) {
    int64_t lo = 0, hi = nwin - 1;  // last window with out_offsets[w] <= o
    while (lo < hi) {
      const int64_t mid = hi - ((hi - lo) >> 1);
      if (out_offsets[mid] <= (uint64_t)o) lo = mid;
      else hi = mid - 1;
    }
    out_idx[o] = (uint32_t)(win[2 * lo] + (o - (int64_t)out_offsets[lo]));
  }
}

template <int KT>
__device__ __forceinline__ bool in_range(const void* col, int64_t i, const PredRange& r) {
  if (r.has_lo && cmp_bound<KT>(col, i, r.lo) < (r.lo_strict ? 1 : 0)) return false;
  if (r.has_hi && cmp_bound<KT>(col, i, r.hi) > (r.hi_strict ? -1 : 0)) return false;
  return true;
}

// the predicate on row i: its range, or (set form) one binary search for the first range of the set not below the value
template <int KT>
__device__ __forceinline__ bool holds(const PredDesc& d, int64_t i) {
  if (!d.set) return in_range<KT>(d.data, i, d.r);
  int64_t lo = 0, hi = d.n_set;
  while (lo < hi) {
    const int64_t mid = lo + ((hi - lo) >> 1);
    const PredRange& r = d.set[mid];
    if (r.has_hi && cmp_bound<KT>(d.data, i, r.hi) > (r.hi_strict ? -1 : 0)) lo = mid + 1;
    else hi = mid;
  }
  return lo < d.n_set && in_range<KT>(d.data, i, d.set[lo]);
}

// The residual conjunction, one thread per candidate row: mask[i] = every predicate holds for row cand[i] (row i without a
// candidate list).  Inside a window the candidates are consecutive rows, so the predicate columns are read coalesced.
__global__ void k_predicate_mask(const __grid_constant__ PredSet ps, const uint32_t* __restrict__ cand, int64_t n,
                                 uint32_t* __restrict__ mask) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int64_t row = cand ? (int64_t)cand[i] : i;
    bool ok = true;
    for (int p = 0; p < ps.n && ok; p++) {
      const PredDesc& d = ps.p[p];
      if (d.valid && !d.valid[row]) {  // a null satisfies no comparison; a null test or NOT (c <=> v) says so in null_true
        ok = d.null_true != 0;
        continue;
      }
      switch (d.r.type) {
        case HS_TYPE_INT32: ok = holds<HS_TYPE_INT32>(d, row); break;
        case HS_TYPE_INT64: ok = holds<HS_TYPE_INT64>(d, row); break;
        case HS_TYPE_FLOAT: ok = holds<HS_TYPE_FLOAT>(d, row); break;
        case HS_TYPE_DOUBLE: ok = holds<HS_TYPE_DOUBLE>(d, row); break;
        default: ok = holds<HS_TYPE_STRING>(d, row); break;
      }
    }
    mask[i] = ok ? 1u : 0u;
  }
}

// The pattern terms, one thread per candidate row: clears mask[i] where one of them does not hold for row cand[i] (row i
// without a candidate list).  A thread matches its row's whole value; rows already dropped by k_predicate_mask are skipped.
// Measured (DESIGN.md section 6), the string scans are bound by the key decode, not by this kernel, on short values; on
// 1 KB values a warp per value would coalesce the loads that a thread per row does not.
__global__ void k_pattern_mask(const __grid_constant__ PatternSet ps, const uint32_t* __restrict__ cand, int64_t n,
                               uint32_t* __restrict__ mask) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (!mask[i]) continue;
    const int64_t row = cand ? (int64_t)cand[i] : i;
    bool ok = true;
    for (int p = 0; p < ps.n && ok; p++) {
      const PatternDesc& d = ps.p[p];
      if (d.valid && !d.valid[row]) {
        ok = d.null_true != 0;
        continue;
      }
      const uint64_t ref = d.refs[row];
      ok = pattern_matches(ref_ptr(ref), ref_len(ref), d.items, d.fail, d.segs, d.nseg, d.whole != 0) != (d.negate != 0);
    }
    if (!ok) mask[i] = 0;
  }
}

// The comparisons between two columns, one thread per candidate row: clears mask[i] where one of them does not hold for
// row cand[i] (row i without a candidate list); rows already dropped by k_predicate_mask or k_pattern_mask are skipped.
// Inside a window the candidates are consecutive rows, so both columns of a comparison are read coalesced.
__global__ void __launch_bounds__(256, 8) k_compare_mask(const __grid_constant__ CompareSet cs, const uint32_t* __restrict__ cand, int64_t n,
                               uint32_t* __restrict__ mask) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (!mask[i]) continue;
    const int64_t row = cand ? (int64_t)cand[i] : i;
    bool ok = true;
    for (int p = 0; p < cs.n && ok; p++) ok = compare_holds(cs.p[p], row);
    if (!ok) mask[i] = 0;
  }
}

// The expression comparisons, one thread per candidate row: clears mask[i] where one of them does not hold for row
// cand[i] (row i without a candidate list); rows already dropped by the earlier masks are skipped.  The evaluator's value
// stack is indexed at run time, so it lives in local memory (DESIGN.md section 6 gives ptxas' frame); the programs and
// their columns are read through the set's device arrays, the same addresses in every thread.
__global__ void __launch_bounds__(256, 8) k_expr_mask(const __grid_constant__ ExprSet es, const uint32_t* __restrict__ cand, int64_t n,
                                                      uint32_t* __restrict__ mask) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (!mask[i]) continue;
    const int64_t row = cand ? (int64_t)cand[i] : i;
    bool ok = true;
    for (int p = 0; p < es.n && ok; p++) ok = expr_holds(es.descs[p], es.insts, es.cols, row);
    if (!ok) mask[i] = 0;
  }
}

// k_expr_mask for programs with function instructions (column_expr.h: expr_holds<true>): calendar fields, string
// references and the string domain.  A kernel of its own, so that arithmetic-only programs keep k_expr_mask's code.
__global__ void __launch_bounds__(256, 8) k_func_mask(const __grid_constant__ ExprSet es, const uint32_t* __restrict__ cand, int64_t n,
                                                      uint32_t* __restrict__ mask) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (!mask[i]) continue;
    const int64_t row = cand ? (int64_t)cand[i] : i;
    bool ok = true;
    for (int p = 0; p < es.n && ok; p++) ok = expr_holds<true>(es.descs[p], es.insts, es.cols, row);
    if (!ok) mask[i] = 0;
  }
}

// a key value at position p, read at its type's width: int32 sign-extended, int64 as it is, a string as its reference
template <int KT>
__device__ __forceinline__ int64_t key_value(const void* col, int64_t p) {
  if constexpr (KT == HS_TYPE_INT32) return ((const int32_t*)col)[p];
  else return ((const int64_t*)col)[p];
}

// -1 / 0 / +1: integers as signed values, strings in UTF8String byte order
template <int KT>
__device__ __forceinline__ int compare_keys(int64_t a, int64_t b) {
  if constexpr (KT == HS_TYPE_STRING) return string_compare((uint64_t)a, (uint64_t)b);
  else return a < b ? -1 : (a > b ? 1 : 0);
}

// key column k of left position i against right position j
__device__ __forceinline__ int compare_column(const JoinKeyCols& l, int64_t i, const JoinKeyCols& r, int64_t j, int k) {
  switch (r.type[k]) {
    case HS_TYPE_INT32: return compare_keys<HS_TYPE_INT32>(key_value<HS_TYPE_INT32>(l.col[k], i), key_value<HS_TYPE_INT32>(r.col[k], j));
    case HS_TYPE_INT64: return compare_keys<HS_TYPE_INT64>(key_value<HS_TYPE_INT64>(l.col[k], i), key_value<HS_TYPE_INT64>(r.col[k], j));
    default: return compare_keys<HS_TYPE_STRING>(key_value<HS_TYPE_STRING>(l.col[k], i), key_value<HS_TYPE_STRING>(r.col[k], j));
  }
}

// the segment of position i: the last s with seg[s] <= i, by binary search over the (few hundred) segment offsets
__device__ __forceinline__ int segment_of(const uint64_t* __restrict__ seg, int nseg, int64_t i) {
  int lo = 0, hi = nseg;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (seg[mid] <= (uint64_t)i) lo = mid;
    else hi = mid;
  }
  return lo;
}

// the left tuple at position i, its leading value l0 held in a register, against right position j
template <int KT0>
__device__ __forceinline__ int compare_tuple(int64_t l0, const JoinKeyCols& lk, int64_t i, const JoinKeyCols& rk, int64_t j) {
  int c = compare_keys<KT0>(l0, key_value<KT0>(rk.col[0], j));
  for (int k = 1; k < rk.n && c == 0; k++) c = compare_column(lk, i, rk, j, k);
  return c;
}

// the first of the right positions [rb, rb + rn) whose tuple is >= the left tuple at i, relative to rb (rn: none is)
template <int KT0>
__device__ __forceinline__ int64_t lower_bound_tuple(int64_t l0, const JoinKeyCols& lk, int64_t i, const JoinKeyCols& rk, int64_t rb,
                                                     int64_t rn) {
  int64_t x = 0, y = rn;
  while (x < y) {
    const int64_t mid = x + ((y - x) >> 1);
    if (compare_tuple<KT0>(l0, lk, i, rk, rb + mid) > 0) x = mid + 1;
    else y = mid;
  }
  return x;
}

// One thread per left position; the segment of a position is found by segment_of.  The right positions of a bucket are
// ascending on the key tuples, so the matches of a left position are the range between two lexicographic binary
// searches.  The leading key column, KT0 its type, decides almost every step: its left value stays in a register and its
// comparison is compiled in, so a step is one load and a branch-free compare.  The later columns are compared only where
// the leading ones tie.
template <int KT0>
__device__ __forceinline__ void join_count_rows(const JoinKeyCols& lk, const uint64_t* __restrict__ lseg, const JoinKeyCols& rk,
                                                const uint64_t* __restrict__ rseg, int nseg, int64_t nl,
                                                uint32_t* __restrict__ counts, uint32_t* __restrict__ first_match) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nl; i += stride) {
    const int lo = segment_of(lseg, nseg, i);
    const int64_t l0 = key_value<KT0>(lk.col[0], i);
    auto compare = [&](int64_t j) { return compare_tuple<KT0>(l0, lk, i, rk, j); };
    const int64_t rb = (int64_t)rseg[lo], rn = (int64_t)rseg[lo + 1] - rb;
    const int64_t f = lower_bound_tuple<KT0>(l0, lk, i, rk, rb, rn);  // first right row >= the left tuple
    int64_t x = 0, y = rn;  // first right row > the left tuple (from the start again: the same path, so cached)
    while (x < y) {
      const int64_t mid = x + ((y - x) >> 1);
      if (compare(rb + mid) >= 0) x = mid + 1;
      else y = mid;
    }
    counts[i] = (uint32_t)(x - f);
    first_match[i] = (uint32_t)(rb + f);
  }
}

__global__ void k_join_count(const __grid_constant__ JoinKeyCols lk, const uint64_t* __restrict__ lseg,
                             const __grid_constant__ JoinKeyCols rk, const uint64_t* __restrict__ rseg, int nseg, int64_t nl,
                             uint32_t* __restrict__ counts, uint32_t* __restrict__ first_match) {
  switch (lk.type[0]) {
    case HS_TYPE_INT32: join_count_rows<HS_TYPE_INT32>(lk, lseg, rk, rseg, nseg, nl, counts, first_match); break;
    case HS_TYPE_INT64: join_count_rows<HS_TYPE_INT64>(lk, lseg, rk, rseg, nseg, nl, counts, first_match); break;
    default: join_count_rows<HS_TYPE_STRING>(lk, lseg, rk, rseg, nseg, nl, counts, first_match); break;
  }
}

// The semi / anti join's probe, one thread per left position: one lower-bound search in the right bucket, then one
// equality test at the position it finds.  A left position with a null in any key column (lv) matches nothing.
// keep[i] = 1 where the match is what keep_match asks for (1: a match, semi; 0: none, anti).
template <int KT0>
__device__ __forceinline__ void join_exists_rows(const JoinKeyCols& lk, const JoinKeyValid& lv, const uint64_t* __restrict__ lseg,
                                                 const JoinKeyCols& rk, const uint64_t* __restrict__ rseg, int nseg, int64_t nl,
                                                 uint32_t keep_match, uint32_t* __restrict__ keep) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nl; i += stride) {
    bool null = false;
    for (int k = 0; k < lv.n; k++) null |= lv.valid[k] != nullptr && lv.valid[k][i] == 0;
    uint32_t match = 0;
    if (!null) {
      const int s = segment_of(lseg, nseg, i);
      const int64_t l0 = key_value<KT0>(lk.col[0], i);
      const int64_t rb = (int64_t)rseg[s], rn = (int64_t)rseg[s + 1] - rb;
      const int64_t f = lower_bound_tuple<KT0>(l0, lk, i, rk, rb, rn);
      match = f < rn && compare_tuple<KT0>(l0, lk, i, rk, rb + f) == 0;
    }
    keep[i] = match == keep_match;
  }
}

__global__ void k_join_exists(const __grid_constant__ JoinKeyCols lk, const __grid_constant__ JoinKeyValid lv,
                              const uint64_t* __restrict__ lseg, const __grid_constant__ JoinKeyCols rk,
                              const uint64_t* __restrict__ rseg, int nseg, int64_t nl, uint32_t keep_match,
                              uint32_t* __restrict__ keep) {
  switch (lk.type[0]) {
    case HS_TYPE_INT32: join_exists_rows<HS_TYPE_INT32>(lk, lv, lseg, rk, rseg, nseg, nl, keep_match, keep); break;
    case HS_TYPE_INT64: join_exists_rows<HS_TYPE_INT64>(lk, lv, lseg, rk, rseg, nseg, nl, keep_match, keep); break;
    default: join_exists_rows<HS_TYPE_STRING>(lk, lv, lseg, rk, rseg, nseg, nl, keep_match, keep); break;
  }
}

// the matches of left position i are right positions [first_match[i], + counts[i]); both go through their side's
// permutation (nullptr: the identity) to rows
__global__ void k_join_emit(const uint32_t* __restrict__ counts, const uint32_t* __restrict__ first_match,
                            const uint64_t* __restrict__ out_offsets, int64_t nl, const uint32_t* __restrict__ lperm,
                            const uint32_t* __restrict__ rperm, uint32_t* __restrict__ out_lrow, uint32_t* __restrict__ out_rrow) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nl; i += stride) {
    const uint32_t c = counts[i];
    const uint64_t o = out_offsets[i];
    const uint32_t f = first_match[i];
    const uint32_t lrow = lperm ? lperm[i] : (uint32_t)i;
    for (uint32_t j = 0; j < c; j++) {
      out_lrow[o + j] = lrow;
      out_rrow[o + j] = rperm ? rperm[f + j] : f + j;
    }
  }
}

// The outer joins' probe, one thread per position of the preserved (probing) side: k_join_exists' key-validity test and
// equality test at the lower bound, then, where that matches, k_join_count's search for the end of the match range.  A
// position with a null in any key column (pv), or with no match, is output once with the other side padded: counts[i] =
// max(matches, 1), and first_match[i] = kNoRow where there is no match.
template <int KT0>
__device__ __forceinline__ void join_count_outer_rows(const JoinKeyCols& pk, const JoinKeyValid& pv, const uint64_t* __restrict__ pseg,
                                                      const JoinKeyCols& tk, const uint64_t* __restrict__ tseg, int nseg, int64_t np,
                                                      uint32_t* __restrict__ counts, uint32_t* __restrict__ first_match) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < np; i += stride) {
    bool null = false;
    for (int k = 0; k < pv.n; k++) null |= pv.valid[k] != nullptr && pv.valid[k][i] == 0;
    uint32_t count = 1, first = kNoRow;
    if (!null) {
      const int s = segment_of(pseg, nseg, i);
      const int64_t p0 = key_value<KT0>(pk.col[0], i);
      const int64_t tb = (int64_t)tseg[s], tn = (int64_t)tseg[s + 1] - tb;
      const int64_t f = lower_bound_tuple<KT0>(p0, pk, i, tk, tb, tn);
      if (f < tn && compare_tuple<KT0>(p0, pk, i, tk, tb + f) == 0) {
        int64_t x = 0, y = tn;  // first position > the tuple (from the start again: the same path, so cached)
        while (x < y) {
          const int64_t mid = x + ((y - x) >> 1);
          if (compare_tuple<KT0>(p0, pk, i, tk, tb + mid) >= 0) x = mid + 1;
          else y = mid;
        }
        count = (uint32_t)(x - f);
        first = (uint32_t)(tb + f);
      }
    }
    counts[i] = count;
    first_match[i] = first;
  }
}

__global__ void k_join_count_outer(const __grid_constant__ JoinKeyCols pk, const __grid_constant__ JoinKeyValid pv,
                                   const uint64_t* __restrict__ pseg, const __grid_constant__ JoinKeyCols tk,
                                   const uint64_t* __restrict__ tseg, int nseg, int64_t np, uint32_t* __restrict__ counts,
                                   uint32_t* __restrict__ first_match) {
  switch (pk.type[0]) {
    case HS_TYPE_INT32: join_count_outer_rows<HS_TYPE_INT32>(pk, pv, pseg, tk, tseg, nseg, np, counts, first_match); break;
    case HS_TYPE_INT64: join_count_outer_rows<HS_TYPE_INT64>(pk, pv, pseg, tk, tseg, nseg, np, counts, first_match); break;
    default: join_count_outer_rows<HS_TYPE_STRING>(pk, pv, pseg, tk, tseg, nseg, np, counts, first_match); break;
  }
}

// The outer joins' pairs: preserved position i (row pperm[i]) with each of its matches, the searched positions
// [first_match[i], + counts[i]) (rows tperm[...]), or once with kNoRow when first_match[i] is kNoRow.  shift (FullOuter,
// else nullptr): every output position of bucket b moves up by shift[b], the rows placed before the bucket's own
// (k_join_place_unmatched); the bucket of i is found by segment_of over pseg.
__global__ void k_join_emit_outer(const uint32_t* __restrict__ counts, const uint32_t* __restrict__ first_match,
                                  const uint64_t* __restrict__ out_offsets, const uint64_t* __restrict__ pseg,
                                  const uint64_t* __restrict__ shift, int nseg, int64_t np, const uint32_t* __restrict__ pperm,
                                  const uint32_t* __restrict__ tperm, uint32_t* __restrict__ out_prow, uint32_t* __restrict__ out_trow) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < np; i += stride) {
    uint64_t o = out_offsets[i];
    if (shift) o += shift[segment_of(pseg, nseg, i)];
    const uint32_t prow = pperm ? pperm[i] : (uint32_t)i;
    const uint32_t f = first_match[i];
    if (f == kNoRow) {
      out_prow[o] = prow;
      out_trow[o] = kNoRow;
      continue;
    }
    const uint32_t c = counts[i];
    for (uint32_t j = 0; j < c; j++) {
      out_prow[o + j] = prow;
      out_trow[o + j] = tperm ? tperm[f + j] : f + j;
    }
  }
}

// FullOuter's right rows that match nothing: urow[r], of global rank r in (bucket, right sorted position) order, goes to
// output position base[b] + r with its left row kNoRow; b is the bucket holding rank r (ucum: the nseg + 1 ranks at which
// the buckets start), base[b] the number of left-outer rows in buckets 0..b.
__global__ void k_join_place_unmatched(const uint32_t* __restrict__ urow, int64_t nu, const uint64_t* __restrict__ ucum,
                                       const uint64_t* __restrict__ base, int nseg, uint32_t* __restrict__ out_lrow,
                                       uint32_t* __restrict__ out_rrow) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nu; r += stride) {
    const uint64_t o = base[segment_of(ucum, nseg, r)] + (uint64_t)r;
    out_lrow[o] = kNoRow;
    out_rrow[o] = urow[r];
  }
}

// The gathers of a side an outer join pads: row idx[i], or a null (value 0, validity 0) where idx[i] is kNoRow.  The
// validity is always written; valid nullptr: the column has no nulls.
template <typename T>
__global__ void k_gather_padded(const T* __restrict__ src, const uint8_t* __restrict__ valid, const uint32_t* __restrict__ idx,
                                int64_t n, T* __restrict__ out, uint8_t* __restrict__ out_valid) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint32_t r = idx[i];
    const bool pad = r == kNoRow;
    out[i] = pad ? T(0) : src[r];
    out_valid[i] = pad ? 0 : (valid ? valid[r] : 1);
  }
}

// k_string_lengths over a padded side: a padded value has length 0 and validity 0
__global__ void k_string_lengths_padded(const uint64_t* __restrict__ refs, const uint8_t* __restrict__ valid,
                                        const uint32_t* __restrict__ idx, int64_t n, uint32_t* __restrict__ lens,
                                        uint8_t* __restrict__ out_valid) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint32_t r = idx[i];
    const uint8_t v = r == kNoRow ? 0 : (valid ? valid[r] : 1);
    lens[i] = v ? ref_len(refs[r]) : 0u;
    out_valid[i] = v;
  }
}

// k_copy_strings over a padded side: padded values (and nulls) copy nothing
__global__ void k_copy_strings_padded(const uint64_t* __restrict__ refs, const uint8_t* __restrict__ valid,
                                      const uint32_t* __restrict__ idx, int64_t n, const uint64_t* __restrict__ offsets,
                                      uint8_t* __restrict__ out) {
  const unsigned lane = threadIdx.x & 31;
  const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
    const uint32_t r = idx[i];
    if (r == kNoRow || (valid && !valid[r])) continue;
    const uint64_t ref = refs[r];
    const uint8_t* src = ref_ptr(ref);
    uint8_t* dst = out + offsets[i];
    for (uint32_t j = lane, len = ref_len(ref); j < len; j += 32) dst[j] = src[j];
  }
}

// ---- exclusive scan uint32 -> uint64 (three kernels; block of 256 threads x 8 items) --------------------------------
constexpr int kScanThreads = 256;
constexpr int kScanItems = 8;
constexpr int kScanTile = kScanThreads * kScanItems;

__global__ void __launch_bounds__(kScanThreads) k_scan_block_sums(const uint32_t* __restrict__ in, int64_t n,
                                                                   unsigned long long* __restrict__ block_sums) {
  __shared__ unsigned long long s[kScanThreads / 32];
  const int64_t base = (int64_t)blockIdx.x * kScanTile;
  unsigned long long v = 0;
  for (int k = 0; k < kScanItems; k++) {
    const int64_t i = base + k * kScanThreads + threadIdx.x;
    if (i < n) v += in[i];
  }
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
    for (int w = 0; w < kScanThreads / 32; w++) t += s[w];
    block_sums[blockIdx.x] = t;
  }
}

// one CTA of 1024 threads: each thread owns a contiguous slice of the block sums
__global__ void __launch_bounds__(1024) k_scan_block_offsets(unsigned long long* __restrict__ block_sums, int64_t nblocks,
                                                              unsigned long long* __restrict__ total_out) {
  __shared__ unsigned long long s[1025];
  const int64_t per = (nblocks + 1023) / 1024;
  const int64_t b0 = (int64_t)threadIdx.x * per, b1 = min(b0 + per, nblocks);
  unsigned long long local = 0;
  for (int64_t b = b0; b < b1; b++) local += block_sums[b];
  s[threadIdx.x] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long run = 0;
    for (int i = 0; i < 1024; i++) {
      const unsigned long long v = s[i];
      s[i] = run;
      run += v;
    }
    s[1024] = run;
  }
  __syncthreads();
  unsigned long long run = s[threadIdx.x];
  for (int64_t b = b0; b < b1; b++) {
    const unsigned long long v = block_sums[b];
    block_sums[b] = run;
    run += v;
  }
  if (threadIdx.x == 0) *total_out = s[1024];
}

__global__ void __launch_bounds__(kScanThreads) k_scan_apply(const uint32_t* __restrict__ in, int64_t n,
                                                              const unsigned long long* __restrict__ block_offsets,
                                                              uint64_t* __restrict__ out) {
  __shared__ uint32_t warp_sums[40];
  const int64_t base = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanItems;
  uint32_t x[kScanItems];
  uint32_t local = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; k++) {
    x[k] = (base + k < n) ? in[base + k] : 0;
    local += x[k];
  }
  uint32_t pre = block_exclusive_scan(local, warp_sums, nullptr);
  unsigned long long run = block_offsets[blockIdx.x] + pre;
#pragma unroll
  for (int k = 0; k < kScanItems; k++) {
    if (base + k < n) out[base + k] = run;
    run += x[k];
  }
}

__global__ void k_not_in_mask(const int64_t* __restrict__ ids, int64_t n, const int64_t* __restrict__ deleted,
                              int ndeleted, uint32_t* __restrict__ mask) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int64_t id = ids[i];
    bool hit = false;
    for (int d = 0; d < ndeleted; d++) hit |= deleted[d] == id;
    if (hit) mask[i] = 0;
  }
}

__global__ void k_compact(const uint32_t* __restrict__ mask, const uint64_t* __restrict__ offsets, int64_t n,
                          const uint32_t* __restrict__ cand, uint32_t* __restrict__ out_idx) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    if (mask[i]) out_idx[offsets[i]] = cand ? cand[i] : (uint32_t)i;
}

inline int grid_for(hs_ctx* ctx, int64_t n, int threads, int per_sm) {
  int64_t want = ceil_div(n, threads);
  int64_t cap = (int64_t)ctx->sm_count * per_sm;
  return (int)std::max<int64_t>(1, std::min(want, cap));
}

__global__ void k_string_lengths(const uint64_t* __restrict__ refs, const uint8_t* __restrict__ valid,
                                 const uint32_t* __restrict__ idx, int64_t n, uint32_t* __restrict__ lens) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint32_t r = idx[i];
    lens[i] = (!valid || valid[r]) ? ref_len(refs[r]) : 0u;
  }
}

// one warp per output value: short values are a single coalesced pass, long ones loop
__global__ void k_copy_strings(const uint64_t* __restrict__ refs, const uint8_t* __restrict__ valid,
                               const uint32_t* __restrict__ idx, int64_t n, const uint64_t* __restrict__ offsets,
                               uint8_t* __restrict__ out) {
  const unsigned lane = threadIdx.x & 31;
  const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
    const uint32_t r = idx[i];
    if (valid && !valid[r]) continue;
    const uint64_t ref = refs[r];
    const uint8_t* src = ref_ptr(ref);
    uint8_t* dst = out + offsets[i];
    for (uint32_t j = lane, len = ref_len(ref); j < len; j += 32) dst[j] = src[j];
  }
}

}  // namespace

void launch_string_lengths(hs_ctx* ctx, const uint64_t* refs, const uint8_t* valid, const uint32_t* idx, int64_t n,
                           uint32_t* lens) {
  if (n == 0) return;
  k_string_lengths<<<grid_for(ctx, n, 256, 16), 256, 0, ctx->stream>>>(refs, valid, idx, n, lens);
  HS_LAUNCH_CHECK(ctx);
}

void launch_copy_strings(hs_ctx* ctx, const uint64_t* refs, const uint8_t* valid, const uint32_t* idx, int64_t n,
                         const uint64_t* offsets, uint8_t* out) {
  if (n == 0) return;
  k_copy_strings<<<grid_for(ctx, n * 32, 256, 16), 256, 0, ctx->stream>>>(refs, valid, idx, n, offsets, out);
  HS_LAUNCH_CHECK(ctx);
}

void launch_range_bounds(hs_ctx* ctx, const void* keys, int ranges_type, const PredRange* ranges, const uint64_t* seg_offsets,
                         const uint2* work, int64_t nwork, int64_t* bounds) {
  KernelScope _ks(ctx, "k_range_bounds", nwork);
  if (nwork == 0) return;
  const unsigned grid = (unsigned)ceil_div(nwork, 128);
  switch (ranges_type) {
    case HS_TYPE_INT32: k_range_bounds<HS_TYPE_INT32><<<grid, 128, 0, ctx->stream>>>(keys, ranges, seg_offsets, work, nwork, bounds); break;
    case HS_TYPE_INT64: k_range_bounds<HS_TYPE_INT64><<<grid, 128, 0, ctx->stream>>>(keys, ranges, seg_offsets, work, nwork, bounds); break;
    case HS_TYPE_FLOAT: k_range_bounds<HS_TYPE_FLOAT><<<grid, 128, 0, ctx->stream>>>(keys, ranges, seg_offsets, work, nwork, bounds); break;
    case HS_TYPE_DOUBLE: k_range_bounds<HS_TYPE_DOUBLE><<<grid, 128, 0, ctx->stream>>>(keys, ranges, seg_offsets, work, nwork, bounds); break;
    case HS_TYPE_STRING: k_range_bounds<HS_TYPE_STRING><<<grid, 128, 0, ctx->stream>>>(keys, ranges, seg_offsets, work, nwork, bounds); break;
    default: fail(HS_EUNSUPPORTED, "range search over a column of type %d", ranges_type);
  }
  HS_LAUNCH_CHECK(ctx);
}

void launch_windows_to_indices(hs_ctx* ctx, const int64_t* win, const uint64_t* out_offsets, int64_t nwin, int64_t n_out,
                               uint32_t* out_idx) {
  k_ranges_to_indices<<<grid_for(ctx, n_out, 256, 16), 256, 0, ctx->stream>>>(win, out_offsets, nwin, n_out, out_idx);
  HS_LAUNCH_CHECK(ctx);
}

void launch_predicate_mask(hs_ctx* ctx, const PredSet& preds, const uint32_t* cand, int64_t n, uint32_t* mask) {
  KernelScope _ks(ctx, "k_predicate_mask");
  if (n == 0) return;
  k_predicate_mask<<<grid_for(ctx, n, 256, 16), 256, 0, ctx->stream>>>(preds, cand, n, mask);
  HS_LAUNCH_CHECK(ctx);
}

void launch_pattern_mask(hs_ctx* ctx, const PatternSet& pats, const uint32_t* cand, int64_t n, uint32_t* mask) {
  if (pats.n == 0) return;
  KernelScope _ks(ctx, "k_pattern_mask");
  if (n == 0) return;
  k_pattern_mask<<<grid_for(ctx, n, 256, 16), 256, 0, ctx->stream>>>(pats, cand, n, mask);
  HS_LAUNCH_CHECK(ctx);
}

void launch_compare_mask(hs_ctx* ctx, const CompareSet& cmps, const uint32_t* cand, int64_t n, uint32_t* mask) {
  if (cmps.n == 0) return;
  KernelScope _ks(ctx, "k_compare_mask");
  if (n == 0) return;
  k_compare_mask<<<grid_for(ctx, n, 256, 16), 256, 0, ctx->stream>>>(cmps, cand, n, mask);
  HS_LAUNCH_CHECK(ctx);
}

void launch_expr_mask(hs_ctx* ctx, const ExprSet& exprs, const uint32_t* cand, int64_t n, uint32_t* mask) {
  if (exprs.n == 0) return;
  KernelScope _ks(ctx, "k_expr_mask");
  if (n == 0) return;
  k_expr_mask<<<grid_for(ctx, n, 256, 16), 256, 0, ctx->stream>>>(exprs, cand, n, mask);
  HS_LAUNCH_CHECK(ctx);
}

void launch_func_mask(hs_ctx* ctx, const ExprSet& funcs, const uint32_t* cand, int64_t n, uint32_t* mask) {
  if (funcs.n == 0) return;
  KernelScope _ks(ctx, "k_func_mask");
  if (n == 0) return;
  k_func_mask<<<grid_for(ctx, n, 256, 16), 256, 0, ctx->stream>>>(funcs, cand, n, mask);
  HS_LAUNCH_CHECK(ctx);
}

void launch_join_count(hs_ctx* ctx, const JoinKeyCols& lkeys, const uint64_t* lseg, const JoinKeyCols& rkeys,
                       const uint64_t* rseg, int nseg, int64_t nl, uint32_t* counts, uint32_t* first_match) {
  KernelScope _ks(ctx, "k_join_count");
  if (nl == 0) return;
  k_join_count<<<grid_for(ctx, nl, 256, 16), 256, 0, ctx->stream>>>(lkeys, lseg, rkeys, rseg, nseg, nl, counts, first_match);
  HS_LAUNCH_CHECK(ctx);
}

void launch_join_emit(hs_ctx* ctx, const uint32_t* counts, const uint32_t* first_match, const uint64_t* out_offsets,
                      int64_t nl, const uint32_t* lperm, const uint32_t* rperm, uint32_t* out_lrow, uint32_t* out_rrow) {
  KernelScope _ks(ctx, "k_join_emit");
  if (nl == 0) return;
  k_join_emit<<<grid_for(ctx, nl, 256, 16), 256, 0, ctx->stream>>>(counts, first_match, out_offsets, nl, lperm, rperm,
                                                                      out_lrow, out_rrow);
  HS_LAUNCH_CHECK(ctx);
}

void exclusive_scan_u32_u64(hs_ctx* ctx, const uint32_t* in, int64_t n, uint64_t* out) {
  // out has n+1 entries; out[n] = total
  const int64_t nblocks = std::max<int64_t>(1, ceil_div(n, kScanTile));
  Buf<unsigned long long> block_sums(ctx, (size_t)nblocks);
  k_scan_block_sums<<<(unsigned)nblocks, kScanThreads, 0, ctx->stream>>>(in, n, block_sums.get());
  HS_LAUNCH_CHECK(ctx);
  k_scan_block_offsets<<<1, 1024, 0, ctx->stream>>>(block_sums.get(), nblocks, (unsigned long long*)(out + n));
  HS_LAUNCH_CHECK(ctx);
  if (n > 0) {
    k_scan_apply<<<(unsigned)nblocks, kScanThreads, 0, ctx->stream>>>(in, n, block_sums.get(), out);
    HS_LAUNCH_CHECK(ctx);
  }
}

void launch_join_exists(hs_ctx* ctx, const JoinKeyCols& lkeys, const JoinKeyValid& lvalid, const uint64_t* lseg,
                        const JoinKeyCols& rkeys, const uint64_t* rseg, int nseg, int64_t nl, bool keep_match, uint32_t* keep) {
  KernelScope _ks(ctx, "k_join_exists");
  if (nl == 0) return;
  k_join_exists<<<grid_for(ctx, nl, 256, 16), 256, 0, ctx->stream>>>(lkeys, lvalid, lseg, rkeys, rseg, nseg, nl,
                                                                       keep_match ? 1u : 0u, keep);
  HS_LAUNCH_CHECK(ctx);
}

void launch_join_count_outer(hs_ctx* ctx, const JoinKeyCols& pkeys, const JoinKeyValid& pvalid, const uint64_t* pseg,
                             const JoinKeyCols& tkeys, const uint64_t* tseg, int nseg, int64_t np, uint32_t* counts,
                             uint32_t* first_match) {
  KernelScope _ks(ctx, "k_join_count_outer");
  if (np == 0) return;
  k_join_count_outer<<<grid_for(ctx, np, 256, 16), 256, 0, ctx->stream>>>(pkeys, pvalid, pseg, tkeys, tseg, nseg, np, counts,
                                                                            first_match);
  HS_LAUNCH_CHECK(ctx);
}

void launch_join_emit_outer(hs_ctx* ctx, const uint32_t* counts, const uint32_t* first_match, const uint64_t* out_offsets,
                            const uint64_t* pseg, const uint64_t* shift, int nseg, int64_t np, const uint32_t* pperm,
                            const uint32_t* tperm, uint32_t* out_prow, uint32_t* out_trow) {
  KernelScope _ks(ctx, "k_join_emit_outer");
  if (np == 0) return;
  k_join_emit_outer<<<grid_for(ctx, np, 256, 16), 256, 0, ctx->stream>>>(counts, first_match, out_offsets, pseg, shift, nseg, np,
                                                                           pperm, tperm, out_prow, out_trow);
  HS_LAUNCH_CHECK(ctx);
}

void launch_join_place_unmatched(hs_ctx* ctx, const uint32_t* urow, int64_t nu, const uint64_t* ucum, const uint64_t* base,
                                 int nseg, uint32_t* out_lrow, uint32_t* out_rrow) {
  KernelScope _ks(ctx, "k_join_place_unmatched");
  if (nu == 0) return;
  k_join_place_unmatched<<<grid_for(ctx, nu, 256, 16), 256, 0, ctx->stream>>>(urow, nu, ucum, base, nseg, out_lrow, out_rrow);
  HS_LAUNCH_CHECK(ctx);
}

void launch_gather_padded(hs_ctx* ctx, const void* src, const uint8_t* valid, const uint32_t* idx, int64_t n, int width, void* out,
                          uint8_t* out_valid) {
  KernelScope _ks(ctx, "k_gather_padded");
  if (n == 0) return;
  const int grid = grid_for(ctx, n, 256, 16);
  switch (width) {
    case 8: k_gather_padded<uint64_t><<<grid, 256, 0, ctx->stream>>>((const uint64_t*)src, valid, idx, n, (uint64_t*)out, out_valid); break;
    case 4: k_gather_padded<uint32_t><<<grid, 256, 0, ctx->stream>>>((const uint32_t*)src, valid, idx, n, (uint32_t*)out, out_valid); break;
    case 1: k_gather_padded<uint8_t><<<grid, 256, 0, ctx->stream>>>((const uint8_t*)src, valid, idx, n, (uint8_t*)out, out_valid); break;
    default: fail(HS_EINVAL, "gather: unsupported width %d", width);
  }
  HS_LAUNCH_CHECK(ctx);
}

void launch_string_lengths_padded(hs_ctx* ctx, const uint64_t* refs, const uint8_t* valid, const uint32_t* idx, int64_t n,
                                  uint32_t* lens, uint8_t* out_valid) {
  if (n == 0) return;
  k_string_lengths_padded<<<grid_for(ctx, n, 256, 16), 256, 0, ctx->stream>>>(refs, valid, idx, n, lens, out_valid);
  HS_LAUNCH_CHECK(ctx);
}

void launch_copy_strings_padded(hs_ctx* ctx, const uint64_t* refs, const uint8_t* valid, const uint32_t* idx, int64_t n,
                                const uint64_t* offsets, uint8_t* out) {
  if (n == 0) return;
  k_copy_strings_padded<<<grid_for(ctx, n * 32, 256, 16), 256, 0, ctx->stream>>>(refs, valid, idx, n, offsets, out);
  HS_LAUNCH_CHECK(ctx);
}

int64_t compact_rows(hs_ctx* ctx, const uint32_t* mask, int64_t n, const uint32_t* cand, Buf<uint32_t>* kept,
                     Buf<uint64_t>* offsets) {
  Buf<uint64_t> own_offsets;
  if (!offsets) offsets = &own_offsets;
  offsets->alloc(ctx, n + 1);
  exclusive_scan_u32_u64(ctx, mask, n, offsets->get());
  uint64_t count = 0;
  copy_d2h(ctx, &count, offsets->get() + n, 8);
  sync_stream(ctx);
  kept->alloc(ctx, std::max<uint64_t>(1, count));
  if (n > 0) {
    k_compact<<<grid_for(ctx, n, 256, 16), 256, 0, ctx->stream>>>(mask, offsets->get(), n, cand, kept->get());
    HS_LAUNCH_CHECK(ctx);
  }
  return (int64_t)count;
}

int64_t select_rows(hs_ctx* ctx, const RowFilter& filter, const uint32_t* cand, int64_t n, const int64_t* file_ids,
                    const int64_t* deleted, int ndeleted, Buf<uint32_t>* kept, Buf<uint64_t>* offsets) {
  Buf<uint32_t> mask(ctx, std::max<int64_t>(1, n));
  launch_predicate_mask(ctx, filter.preds, cand, n, mask.get());
  launch_pattern_mask(ctx, filter.pats, cand, n, mask.get());
  launch_compare_mask(ctx, filter.cmps, cand, n, mask.get());
  launch_expr_mask(ctx, filter.exprs, cand, n, mask.get());
  launch_func_mask(ctx, filter.funcs, cand, n, mask.get());
  Buf<int64_t> d_deleted;
  if (n > 0 && ndeleted > 0) {
    d_deleted.alloc(ctx, ndeleted);
    copy_h2d(ctx, d_deleted.get(), deleted, sizeof(int64_t) * ndeleted);
    k_not_in_mask<<<grid_for(ctx, n, 256, 16), 256, 0, ctx->stream>>>(file_ids, n, d_deleted.get(), ndeleted, mask.get());
    HS_LAUNCH_CHECK(ctx);
  }
  return compact_rows(ctx, mask.get(), n, cand, kept, offsets);
}

}  // namespace hs
