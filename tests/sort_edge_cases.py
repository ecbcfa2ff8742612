"""Key-sort inputs placed exactly on either side of the limits at which the GPU sort changes path, and a numpy restatement
of how sort_rows() (hyperspace_b200/csrc/radix_sort.cu) chooses that path.

Every limit the sort turns on is restated once below, with the line of radix_sort.cu it mirrors.  A change that moves a
limit changes the constant here; tests/test_sort_edge_cases_host.py then says whether every boundary case still sits
where it claims to (the right bucket, sub-bucket and run sizes around the new limit), without a GPU.

A case is a function returning (cols, valids, nb, expected_path): the key columns, their validity arrays (or None), the
number of buckets and the path sort_rows must take with its default settings, one of PATHS.  CLAIMS[name] lists what
the case is built to put on a boundary; analyse() measures it from the oracle's order.  With several key columns the
path is that of the last key column, which is sorted first and straight from the raw column.

Keys are built in their sort encoding (sort_encode in device_utils.cuh, restated by encode()): the MSD digit, the
k_local_sort prefix and the k_fix_runs prefix are bit ranges of the encoded key, so a case writes those bits directly.
The row order is random; rows that share a prefix get their low bits in descending load order, so that every such run
has to be reversed.
"""
import functools

import numpy as np

from oracle import oracle as O

# ---- the limits ------------------------------------------------------------------------------------------------------
LOCAL_CAP = 12288                          # kLocalSortCap (radix_sort.cu:404): rows of one k_local_sort work item
MSD_MAX_SEG = int(0.85 * 256 * LOCAL_CAP)  # = 2 673 868: largest bucket that tries the MSD pass (radix_sort.cu:836)
SORT_TILE = 4096                           # kSortTile (kernels.h:208): tiles start at their bucket's first row
MAX_RUN = 64                               # kLocalMaxRun (radix_sort.cu:412) and kFixMaxRun (radix_sort.cu:269)

PATHS = ("raw_local", "msd_local", "lsd_fixup", "lsd_full", "materialise")


def want_bytes(max_seg: int) -> int:
    """High bytes the tie fix-up sorts on (radix_sort.cu:780-781): enough that the largest bucket spreads over more
    prefixes than twice its rows, at least 2."""
    w = 2
    while w < 8 and max_seg / 256.0 ** w > 0.5:
        w += 1
    return w


def local_prefix_low(count: int, varying: int) -> int:
    """Lowest bit of the prefix k_local_sort radix-sorts an item of `count` rows on (radix_sort.cu:503-507); rows that
    share bits [low, 64) form the runs it insertion-sorts, or re-sorts the item for when one is longer than MAX_RUN."""
    top = varying.bit_length() - 1
    pbits = 1
    while (1 << pbits) < 2 * count:
        pbits += 1
    ndig = (min(pbits, top + 1) + 7) // 8
    return max(0, top + 1 - 8 * ndig)


def msd_shift(varying: int) -> int:
    """Shift of the MSD digit: the 8 bits ending at the highest varying bit of the encoded keys (radix_sort.cu:837,
    63 - clz(varying) - 7)."""
    return max(0, varying.bit_length() - 1 - 7)


def fix_low_bit(varying: int, max_seg: int) -> int:
    """Lowest bit of the k_fix_runs prefix: the lowest of the top want_bytes varying bytes (radix_sort.cu:813-818,846)."""
    seen, low = 0, 0
    for b in range(7, -1, -1):
        if (varying >> (8 * b)) & 0xFF:
            seen += 1
            if seen == want_bytes(max_seg):
                low = b
    return 8 * low


# ---- sort_encode ------------------------------------------------------------------------------------------------------
def encode(col: np.ndarray) -> np.ndarray:
    """sort_encode (device_utils.cuh) of a column as uint64: order-preserving, -0.0 -> 0.0 and every NaN -> the canonical
    one (greatest)."""
    col = np.ascontiguousarray(col)
    if col.dtype == np.int32:
        return (col.view(np.uint32) ^ np.uint32(0x80000000)).astype(np.uint64)
    if col.dtype == np.int64:
        return col.view(np.uint64) ^ np.uint64(1 << 63)
    if col.dtype == np.float32:
        b = col.view(np.uint32).copy()
        mag = b & np.uint32(0x7FFFFFFF)
        b[mag == 0] = 0
        b[mag > 0x7F800000] = 0x7FC00000
        return np.where(b >> np.uint32(31) == 1, ~b, b | np.uint32(0x80000000)).astype(np.uint64)
    if col.dtype == np.float64:
        b = col.view(np.uint64).copy()
        mag = b & np.uint64(0x7FFFFFFFFFFFFFFF)
        b[mag == 0] = 0
        b[mag > np.uint64(0x7FF0000000000000)] = np.uint64(0x7FF8000000000000)
        return np.where(b >> np.uint64(63) == 1, ~b, b | np.uint64(1 << 63))
    raise TypeError(f"unhandled key dtype {col.dtype}")


def varying_bits(enc: np.ndarray) -> int:
    if len(enc) == 0:
        return 0
    return int(np.bitwise_or.reduce(enc)) ^ int(np.bitwise_and.reduce(enc))


def _runs(prefix: np.ndarray):
    """(start, length) of every maximal run of two or more equal values."""
    if len(prefix) < 2:
        return []
    edge = np.flatnonzero(prefix[1:] != prefix[:-1]) + 1
    starts = np.concatenate([[0], edge])
    lens = np.diff(np.concatenate([starts, [len(prefix)]]))
    keep = lens >= 2
    return list(zip(starts[keep].tolist(), lens[keep].tolist()))


@functools.lru_cache(maxsize=None)
def case_data(name: str):
    return CASES[name]()


@functools.lru_cache(maxsize=None)
def analyse(name: str) -> dict:
    """Where the oracle's order puts case `name` relative to every limit above, and the path sort_rows takes for it,
    with the default settings ('path') and under HS_LSD_SORT=1 ('lsd_path')."""
    cols, valids, nb, _ = case_data(name)
    n = len(cols[0])
    b = O.bucket_ids(cols, nb, valids)
    perm, offs = O.sort_perm(cols, nb, b, valids)
    sizes = np.diff(offs)
    max_seg = max(1, int(sizes.max()) if n else 1)
    enc = encode(cols[-1])
    var = varying_bits(enc)
    nbytes = sum(1 for i in range(8) if (var >> (8 * i)) & 0xFF)
    nullable_last = valids is not None and valids[-1] is not None
    a = dict(n=n, perm=perm, sizes=sizes, offs=offs, max_seg=max_seg, varying=var, nbytes=nbytes, sub_sizes=None, items=[],
             local_runs=[], fix_runs=[], constant_items=0)
    s_enc = enc[perm] if n else enc
    shift = msd_shift(var)
    if nbytes > 2 and max_seg > LOCAL_CAP:
        digit = (enc >> np.uint64(shift)) & np.uint64(0xFF)
        a["sub_sizes"] = np.bincount(b.astype(np.int64) * 256 + digit.astype(np.int64), minlength=nb * 256).reshape(nb, 256)
    msd_ok = (nbytes > 2 and max_seg <= MSD_MAX_SEG and int(a["sub_sizes"].max()) <= LOCAL_CAP) if a["sub_sizes"] is not None else False

    def path(lsd_only):
        if var == 0:
            return "materialise"
        if not nullable_last and not lsd_only:
            if max_seg <= LOCAL_CAP:
                return "raw_local"
            if msd_ok:
                return "msd_local"
        return "lsd_fixup" if nbytes > want_bytes(max_seg) else "lsd_full"

    a["path"], a["lsd_path"] = path(False), path(True)
    # k_local_sort work items (radix_sort.cu:657-664 whole buckets, 681-694 consecutive whole sub-buckets) and their runs
    if a["path"] == "raw_local":
        a["items"] = [(int(offs[g]), int(sizes[g])) for g in range(nb) if sizes[g]]
    elif a["path"] == "msd_local":
        for g in range(nb):
            start, count = int(offs[g]), 0
            for d in range(256):
                sz = int(a["sub_sizes"][g, d])
                if count + sz > LOCAL_CAP:
                    a["items"].append((start, count))
                    start, count = start + count, 0
                count += sz
            if count:
                a["items"].append((start, count))
    if len(cols) > 1:
        return a  # the runs below are those of a lone key column, sorted in its own order
    for start, count in a["items"]:
        keys = s_enc[start:start + count]
        v = varying_bits(keys)
        if v == 0:
            a["constant_items"] += 1
            continue
        low = local_prefix_low(count, v)
        if v & ((1 << low) - 1) == 0:
            continue  # nothing below the prefix: no runs to sort
        for s, ln in _runs(keys >> np.uint64(low)):
            where = "first" if s == 0 else ("last" if s + ln == count else "inside")
            a["local_runs"].append(dict(pos=start + s, len=ln, where=where, reversed=_reversed(perm, start + s, ln),
                                        ties=len(np.unique(keys[s:s + ln])) < ln))
    # k_fix_runs runs: rows of one bucket that share the top want_bytes varying bytes
    if a["path"] == "lsd_fixup" or a["lsd_path"] == "lsd_fixup":
        low = fix_low_bit(var, max_seg)
        a["fix_low"] = low
        prefix = s_enc >> np.uint64(low)
        nonempty = [g for g in range(nb) if sizes[g]]
        for i, g in enumerate(nonempty):
            lo, hi = int(offs[g]), int(offs[g + 1])
            for s, ln in _runs(prefix[lo:hi]):
                kinds = set()
                if s // SORT_TILE != (s + ln - 1) // SORT_TILE:
                    kinds.add("crossing")
                else:
                    kinds.add("inside")
                if s % SORT_TILE == 0 and s > 0:
                    kinds.add("tile_start")
                if s + ln == hi - lo:
                    kinds.add("bucket_end")
                    nxt = nonempty[i + 1] if i + 1 < len(nonempty) else None
                    if (hi - lo) % SORT_TILE == 0 and nxt is not None and prefix[int(offs[nxt])] == prefix[hi - 1]:
                        kinds.add("next_bucket")
                a["fix_runs"].append(dict(pos=lo + s, len=ln, kinds=kinds, reversed=_reversed(perm, lo + s, ln)))
    return a


def _reversed(perm, pos, ln) -> bool:
    """The run's rows sit in the sorted order against their load order: the sort has to move every one of them."""
    return bool(np.all(np.diff(perm[pos:pos + ln]) < 0))


# ---- case builders ----------------------------------------------------------------------------------------------------
def _dec64(e: np.ndarray) -> np.ndarray:
    """int64 keys whose sort encoding is e."""
    return (np.asarray(e, dtype=np.uint64) ^ np.uint64(1 << 63)).view(np.int64)


def _grouped_keys(groups, low: int, rng, nb: int = 1, ties=()):
    """int64 keys, in random load order, made of `groups` = [(bucket, prefix, length)]: every row of a group has the
    encoded key prefix << low | l, its low bits l distinct (in pairs of equal ones for the group indices in `ties`) and
    descending in load order.  With nb > 1, the low bits are drawn until the key hashes into the group's bucket."""
    n = sum(g[2] for g in groups)
    pos = rng.permutation(n)
    keys = np.empty(n, dtype=np.int64)
    at = 0
    for gi, (bucket, prefix, length) in enumerate(groups):
        want = (length + 1) // 2 if gi in ties else length
        lows = np.empty(0, dtype=np.uint64)
        while len(lows) < want:
            cand = np.unique(rng.integers(0, 1 << low, size=4 * want + 64, dtype=np.uint64))
            if nb > 1:
                k = _dec64((np.uint64(prefix) << np.uint64(low)) | cand)
                cand = cand[O.bucket_ids([k], nb) == bucket]
            lows = np.union1d(lows, cand)
        lows = np.sort(rng.choice(lows, want, replace=False))[::-1]
        if gi in ties:
            lows = np.repeat(lows, 2)[:length]
        p = np.sort(pos[at:at + length])
        keys[p] = _dec64((np.uint64(prefix) << np.uint64(low)) | lows)
        at += length
    return keys


def _spread(lengths, width: int, base: int = 0):
    """Groups for runs of the given lengths in sorted order, on prefixes spread evenly over [0, 2^width) under `base`
    (so that the prefix's top bit varies)."""
    g = len(lengths)
    assert g <= 1 << width
    return [(0, (base << width) | (j * ((1 << width) - 1) // max(1, g - 1)), ln) for j, ln in enumerate(lengths)]


def _pad(total: int, most: int = 56):
    """Run lengths of at most `most` rows (below MAX_RUN) that add up to total."""
    q, r = divmod(total, most)
    return [most] * q + ([r] if r else [])


def _random_in_buckets(sizes, nb, rng, draw):
    """Keys drawn by draw(rng, m) with exactly sizes[b] rows in bucket b, in random order."""
    need = np.asarray(sizes)
    out, have = [], np.zeros(nb, dtype=np.int64)
    while (have < need).any():
        k = draw(rng, int(max(need.sum(), 1000)) * 2)
        bk = O.bucket_ids([k], nb)
        for bucket in np.flatnonzero(have < need):
            sel = k[bk == bucket][: need[bucket] - have[bucket]]
            out.append(sel)
            have[bucket] += len(sel)
    keys = np.concatenate(out) if out else np.empty(0, dtype=np.int64)
    return keys[rng.permutation(len(keys))]


def _uniform64(rng, m):
    return rng.integers(-2**63, 2**63 - 1, size=m, dtype=np.int64, endpoint=True)


def _on_digits(sizes, rng):
    """int64 keys with exactly sizes[d] rows whose encoded top byte is d (random below it), in random order."""
    d = np.repeat(np.arange(256, dtype=np.uint64), sizes)
    e = (d << np.uint64(56)) | rng.integers(0, 1 << 56, size=len(d), dtype=np.uint64)
    return _dec64(e[rng.permutation(len(e))])


CASES = {}
CLAIMS = {}


def case(**claims):
    def reg(fn):
        CASES[fn.__name__] = fn
        CLAIMS[fn.__name__] = claims
        return fn
    return reg


# ---- raw-path capacity ------------------------------------------------------------------------------------------------
@case(max_bucket=LOCAL_CAP)
def raw_bucket_at_cap():
    return [_uniform64(np.random.default_rng(1), LOCAL_CAP)], None, 1, "raw_local"


@case(max_bucket=LOCAL_CAP + 1)
def raw_bucket_over_cap():
    return [_uniform64(np.random.default_rng(2), LOCAL_CAP + 1)], None, 1, "msd_local"


@case(max_bucket=LOCAL_CAP, empty_between=True)
def raw_200_buckets_largest_at_cap():
    rng = np.random.default_rng(3)
    sizes = rng.integers(1, 3000, size=200)
    sizes[1::4] = 0
    sizes[[6, 150]] = LOCAL_CAP
    return [_random_in_buckets(sizes, 200, rng, _uniform64)], None, 200, "raw_local"


@case(n=1)
def one_row_4096_buckets():
    return [np.array([-123456789], dtype=np.int64)], None, 4096, "materialise"  # one row: no varying bit


@case(n=0)
def empty_input():
    return [np.empty(0, dtype=np.int64)], None, 4, "materialise"


# ---- MSD sub-buckets (nb = 1; the encoded keys span both halves, so the MSD digit is their top byte) ------------------
def _digit_sizes(special, rest):
    s = np.full(256, rest, dtype=np.int64)
    for d, v in special.items():
        s[d] = v
    return s


@case(max_sub=LOCAL_CAP, item_sizes=[LOCAL_CAP])
def msd_sub_bucket_at_cap():
    return [_on_digits(_digit_sizes({0x42: LOCAL_CAP}, 40), np.random.default_rng(10))], None, 1, "msd_local"


@case(max_sub=LOCAL_CAP + 1)
def msd_sub_bucket_over_cap():
    return [_on_digits(_digit_sizes({0x42: LOCAL_CAP + 1}, 40), np.random.default_rng(11))], None, 1, "lsd_fixup"


@case(max_sub=4096, item_sizes=[LOCAL_CAP, LOCAL_CAP])
def msd_items_exactly_full():
    """Three sub-buckets of 4096 fill an item exactly, twice."""
    sizes = _digit_sizes({d: 4096 for d in range(6)}, 20)
    return [_on_digits(sizes, np.random.default_rng(12))], None, 1, "msd_local"


@case(max_sub=4097, item_sizes=[8192])
def msd_items_one_row_over():
    """The third sub-bucket holds one row more: the item closes after two sub-buckets and the third straddles row
    12 288 of the bucket."""
    sizes = _digit_sizes({0: 4096, 1: 4096, 2: 4097, 3: 4096, 4: 4096, 5: 4096}, 20)
    return [_on_digits(sizes, np.random.default_rng(13))], None, 1, "msd_local"


@case(item_sizes=[LOCAL_CAP])
def msd_bucket_on_one_digit():
    """Bucket 1 has every row on one MSD digit (12 288 rows, a single full item); bucket 0 spreads its rows."""
    rng = np.random.default_rng(14)
    spread = _random_in_buckets([20000, 0], 2, rng, _uniform64)
    one = _random_in_buckets([0, LOCAL_CAP], 2, rng,
                             lambda r, m: _dec64((np.uint64(0x37) << np.uint64(56)) | r.integers(0, 1 << 56, size=m, dtype=np.uint64)))
    k = np.concatenate([spread, one])
    return [k[rng.permutation(len(k))]], None, 2, "msd_local"


# ---- MSD ceiling ------------------------------------------------------------------------------------------------------
def _ceiling_keys(n, seed):
    rng = np.random.default_rng(seed)
    return _on_digits(np.bincount(np.arange(n) % 256, minlength=256), rng)


@case(max_bucket=MSD_MAX_SEG)
def msd_bucket_at_ceiling():
    return [_ceiling_keys(MSD_MAX_SEG, 20)], None, 1, "msd_local"


@case(max_bucket=MSD_MAX_SEG + 1)
def msd_bucket_over_ceiling():
    return [_ceiling_keys(MSD_MAX_SEG + 1, 21)], None, 1, "lsd_fixup"


# ---- varying bytes ----------------------------------------------------------------------------------------------------
@case(nbytes=2)
def two_varying_bytes():
    rng = np.random.default_rng(30)
    r = rng.integers(0, 1 << 16, size=100_000, dtype=np.uint64)
    return [_dec64((np.uint64(0x5A) << np.uint64(56)) | (r << np.uint64(24)))], None, 1, "lsd_full"


@case(nbytes=3)
def three_varying_bytes():
    rng = np.random.default_rng(31)
    r = rng.integers(0, 1 << 24, size=100_000, dtype=np.uint64)
    return [_dec64((np.uint64(0x5A) << np.uint64(56)) | (r << np.uint64(16)))], None, 1, "msd_local"


@case(nbytes=0, max_bucket=5000)
def all_equal_below_cap():
    return [np.full(5000, 0x1234, dtype=np.int64)], None, 1, "materialise"


@case(nbytes=0, max_bucket=50_000)
def all_equal_above_cap():
    return [np.full(50_000, -77, dtype=np.float64)], None, 1, "materialise"


@case(constant_items=1)
def constant_bucket_among_varying():
    rng = np.random.default_rng(32)
    k = _random_in_buckets([3000, 3000, 0, 3000], 4, rng, _uniform64)
    const = _random_in_buckets([0, 0, 1, 0], 4, rng, _uniform64)
    k = np.concatenate([k, np.repeat(const, 3000)])
    return [k[rng.permutation(len(k))]], None, 4, "raw_local"


@case(constant_items=1)
def constant_bucket_in_msd_pass():
    rng = np.random.default_rng(33)
    k = _random_in_buckets([20000, 0], 2, rng, _uniform64)
    const = _random_in_buckets([0, 1], 2, rng, _uniform64)
    k = np.concatenate([k, np.repeat(const, 5000)])
    return [k[rng.permutation(len(k))]], None, 2, "msd_local"


# ---- k_local_sort runs ------------------------------------------------------------------------------------------------
# Raw path: one bucket of 8000 rows spanning the whole key range; k_local_sort's prefix is then bits [48, 64).
# MSD path: the run item is the sub-bucket of digit 0x10 (8000 rows, bit 55 varying): prefix bits [40, 64).  Two more
# sub-buckets (0x90: 8000 rows, 0xF0: 3000) make a second item.
_ITEM = 8000


def _raw_runs(lengths, seed, ties=()):
    low = local_prefix_low(_ITEM, 1 << 63)
    rng = np.random.default_rng(seed)
    return [_grouped_keys(_spread(lengths, 64 - low), low, rng, ties=ties)], None, 1, "raw_local"


def _msd_runs(lengths, seed, ties=()):
    low = local_prefix_low(_ITEM, 1 << 55)
    rng = np.random.default_rng(seed)
    item = _grouped_keys(_spread(lengths, 56 - low, base=0x10), low, rng, ties=ties)
    other = _on_digits(_digit_sizes({0x90: 8000, 0xF0: 3000}, 0), rng)
    k = np.empty(len(item) + len(other), dtype=np.int64)
    at = np.zeros(len(k), dtype=bool)
    at[rng.choice(len(k), len(item), replace=False)] = True  # the item's rows keep their load order
    k[at], k[~at] = item, other
    return [k], None, 1, "msd_local"


def _layout(runs_first, run_mid, runs_last, total=_ITEM):
    """Run lengths in sorted order: optional runs at the first slot, in the middle and at the last slot, single rows
    between them."""
    fill = total - sum(runs_first) - sum(run_mid) - sum(runs_last)
    a = fill // 2
    return list(runs_first) + [1] * a + list(run_mid) + [1] * (fill - a) + list(runs_last)


@case(local_runs=[(64, "first"), (64, "inside"), (64, "last")], max_local_run=64)
def local_runs_of_64_raw():
    return _raw_runs(_layout([64], [64], [64]), 40)


@case(local_runs=[(65, "inside")])
def local_run_of_65_raw():
    return _raw_runs(_layout([], [65], []), 41)


@case(local_runs=[(65, "first")], ties=True)
def local_run_of_65_with_ties_first_raw():
    return _raw_runs(_layout([65], [], []), 42, ties=(0,))


@case(local_runs=[(65, "last")])
def local_run_of_65_last_raw():
    lengths = _layout([], [], [65])
    return _raw_runs(lengths, 43)


@case(local_runs=[(64, "first"), (64, "inside"), (64, "last")], max_local_run=64)
def local_runs_of_64_msd():
    return _msd_runs(_layout([64], [64], [64]), 44)


@case(local_runs=[(65, "inside")], ties=True)
def local_run_of_65_with_ties_msd():
    lengths = _layout([], [65], [])
    return _msd_runs(lengths, 45, ties=(lengths.index(65),))


# ---- k_fix_runs runs ----------------------------------------------------------------------------------------------------
# Encoded keys (0x80 | g) << 56 | b2 << 16 | low16 with g in {0, 1}: four varying bytes (7, 2, 1, 0).  The MSD digit
# (bits 49..56) holds only g, so the g = 0 sub-bucket (more than 12 288 rows) sends the bucket to the fix-up, whose prefix
# is (g, b2): bits [16, 64) for buckets of up to 32 768 rows.  Every (g, b2) group is a run of at most 56 rows apart from
# the ones a case places.
_FIX_ROWS = 13000


def _fix_groups(lengths0, lengths1, bucket=0, b2_start=0):
    groups = [(bucket, (0x80 << 40) | (b2_start + j), ln) for j, ln in enumerate(lengths0)]
    groups += [(bucket, (0x81 << 40) | j, ln) for j, ln in enumerate(lengths1)]
    assert b2_start + len(lengths0) <= 256 and len(lengths1) <= 256
    return groups


def _fix_case(before, run, seed, lengths1=(1,)):
    """A run of `run` rows starting at row `before` of the bucket, among g = 0 runs that add up to _FIX_ROWS rows."""
    lengths0 = _pad(before) + [run] + _pad(_FIX_ROWS - before - run)
    rng = np.random.default_rng(seed)
    return [_grouped_keys(_fix_groups(lengths0, list(lengths1)), 16, rng)], None, 1, "lsd_fixup"


@case(fix_runs=[(64, "inside")], max_fix_run=64)
def fix_runs_of_64_inside_tiles():
    lengths0 = _pad(1000) + [64] + _pad(5000) + [64] + _pad(_FIX_ROWS - 6128)
    return [_grouped_keys(_fix_groups(lengths0, [1]), 16, np.random.default_rng(50))], None, 1, "lsd_fixup"


@case(fix_runs=[(65, "inside")])
def fix_run_of_65_inside_a_tile():
    return _fix_case(2000, 65, 51)


@case(fix_runs=[(64, "crossing")], max_fix_run=64)
def fix_run_of_64_across_tiles():
    return _fix_case(SORT_TILE - 20, 64, 52)


@case(fix_runs=[(65, "crossing")], max_fix_run=65)
def fix_run_of_65_across_tiles():
    return _fix_case(2 * SORT_TILE - 30, 65, 53)


@case(fix_runs=[(64, "tile_start")], max_fix_run=64)
def fix_run_at_tile_row_0():
    return _fix_case(SORT_TILE, 64, 54)


@case(fix_runs=[(64, "bucket_end")], max_fix_run=64)
def fix_run_at_bucket_end():
    return _fix_case(100, 10, 55, lengths1=_pad(300) + [64])


@case(fix_runs=[(30, "next_bucket")], max_fix_run=56)
def fix_run_into_next_bucket():
    """Bucket 0 holds 8192 rows (two full tiles) and ends with a run of 30; bucket 1 begins with 30 rows of the same
    prefix.  They are two runs: one sorted across the bucket edge mixes the buckets' rows."""
    lengths0 = _pad(2 * SORT_TILE - 30) + [30]
    shared = len(lengths0) - 1
    groups = _fix_groups(lengths0, [], bucket=0)
    groups += _fix_groups([30], _pad(_FIX_ROWS), bucket=1, b2_start=shared)
    return [_grouped_keys(groups, 16, np.random.default_rng(56), nb=2)], None, 2, "lsd_fixup"


# ---- encoding edges -----------------------------------------------------------------------------------------------------
_F64_SPECIAL = np.array([
    0x7FF8000000000000, 0x7FF8000000000123, 0xFFF8000000000000, 0xFFF80000DEADBEEF,  # quiet NaNs, both signs, payloads
    0x7FF0000000000001, 0x7FF4000000000000, 0xFFF0000000000001, 0xFFF7FFFFFFFFFFFF,  # signalling NaNs
    0x0000000000000000, 0x8000000000000000, 0x7FF0000000000000, 0xFFF0000000000000,  # +-0.0, +-inf
    0x0000000000000001, 0x800FFFFFFFFFFFFF, 0x0010000000000000, 0x8000000000000001,  # subnormals, smallest normal
    0x7FEFFFFFFFFFFFFF, 0xFFEFFFFFFFFFFFFF,                                          # largest finite
], dtype=np.uint64).view(np.float64)
_F32_SPECIAL = np.array([
    0x7FC00000, 0x7FC00123, 0xFFC00000, 0xFFC0BEEF, 0x7F800001, 0x7FA00000, 0xFF800001, 0xFFBFFFFF,
    0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x00000001, 0x807FFFFF, 0x00800000, 0x80000001,
    0x7F7FFFFF, 0xFF7FFFFF,
], dtype=np.uint32).view(np.float32)
_I64_SPECIAL = np.array([-2**63, -2**63 + 1, -1, 0, 1, 2**63 - 2, 2**63 - 1], dtype=np.int64)
_I32_SPECIAL = np.array([-2**31, -2**31 + 1, -1, 0, 1, 2**31 - 2, 2**31 - 1], dtype=np.int32)


def _random_of(dtype, rng, m):
    if dtype == np.int64:
        return _uniform64(rng, m)
    if dtype == np.int32:
        return rng.integers(-2**31, 2**31 - 1, size=m, dtype=np.int32, endpoint=True)
    if dtype == np.float64:
        return rng.standard_normal(m) * 10.0 ** rng.uniform(-300, 300, size=m)
    return (rng.standard_normal(m) * 10.0 ** rng.uniform(-30, 30, size=m)).astype(np.float32)


def _one_digit_of(dtype, rng, m):
    """m values that share the MSD digit of a spread column of their type."""
    if dtype == np.int64:
        return (np.int64(0x37) << np.int64(56)) | rng.integers(0, 1 << 56, size=m, dtype=np.int64)
    if dtype == np.int32:
        return (np.int32(0x37) << np.int32(24)) | rng.integers(0, 1 << 24, size=m, dtype=np.int32)
    return (1.0 + rng.random(m)).astype(dtype)


_SPECIALS = {np.int64: _I64_SPECIAL, np.int32: _I32_SPECIAL, np.float64: _F64_SPECIAL, np.float32: _F32_SPECIAL}


def _edges(dtype, size, seed):
    """Every special value of the type 20 times at random places among random values; size: 'raw' (4 buckets of about
    5000 rows), 'msd' (one bucket of 30 000) or 'fix' (the same, 13 000 of them on one MSD digit)."""
    rng = np.random.default_rng(seed)
    sp = np.repeat(_SPECIALS[dtype], 20)
    n = 20_000 if size == "raw" else 30_000
    parts = [sp, _random_of(dtype, rng, n - len(sp) - (13_000 if size == "fix" else 0))]
    if size == "fix":
        parts.append(_one_digit_of(dtype, rng, 13_000))
    k = np.concatenate(parts).astype(dtype)
    k = k[rng.permutation(len(k))]
    path = {"raw": "raw_local", "msd": "msd_local", "fix": "lsd_fixup"}[size]
    return [k], None, 4 if size == "raw" else 1, path


def _register_edges():
    seed = 70
    for dt, tag in ((np.int64, "int64"), (np.int32, "int32"), (np.float64, "float64"), (np.float32, "float32")):
        for size in ("raw", "msd", "fix"):
            fn = functools.partial(_edges, dt, size, seed)
            fn.__name__ = f"{tag}_edges_{size}"
            case(specials=True)(fn)
            seed += 1


# ---- several columns and nulls --------------------------------------------------------------------------------------
def _nulls_zeroed(v, valid):
    return np.where(valid, v, 0).astype(v.dtype)  # decoded nulls hold 0


@case()
def multi_nullable_first_column():
    rng = np.random.default_rng(60)
    n = 20_000
    valid = rng.random(n) > 0.3
    a = _nulls_zeroed(rng.integers(0, 10, size=n, dtype=np.int32), valid)
    return [a, _uniform64(rng, n)], [valid.astype(np.uint8), None], 4, "raw_local"


@case(specials=True)
def multi_float_first_column_nan_payloads():
    """A low-cardinality double first column whose NaNs (every payload, both signs) and zeros (both signs) tie: the
    int64 second column orders them."""
    rng = np.random.default_rng(61)
    n = 20_000
    vals = np.concatenate([_F64_SPECIAL, [1.5, -2.25]])
    return [vals[rng.integers(0, len(vals), size=n)], _uniform64(rng, n)], None, 4, "raw_local"


@case()
def multi_nullable_last_column():
    rng = np.random.default_rng(62)
    n = 20_000
    valid = rng.random(n) > 0.2
    b = _nulls_zeroed(_uniform64(rng, n), valid)
    return [rng.integers(0, 10, size=n, dtype=np.int32), b], [None, valid.astype(np.uint8)], 4, "lsd_fixup"


@case(specials=True)
def multi_three_columns():
    rng = np.random.default_rng(63)
    n = 40_000
    f = np.concatenate([_F32_SPECIAL, np.float32([0.5, 7.0])])
    cols = [rng.integers(0, 4, size=n, dtype=np.int32), f[rng.integers(0, len(f), size=n)], _uniform64(rng, n)]
    return cols, None, 8, "raw_local"


_register_edges()
