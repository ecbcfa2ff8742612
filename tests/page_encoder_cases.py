"""Source tables placed where the index page encoder changes path, a Python restatement of the encoder's choices per
column, and an independent walker that checks every page of an index file byte for byte.

The encoder (hyperspace_b200/csrc/engine.cu: layout_segments / write_segments, dict_encode.cu, gather_encode.cu and the
page prefixes of parquet_meta.h) decides per column whether to dictionary-encode it, samples the column in three
stages to find out, batches the dictionary columns eight to a launch, and lays the pages out by rows_per_page and
rows_per_row_group.  Every limit it turns on is restated once below with the source line it mirrors;
tests/test_page_encoder_host.py checks each line against the source and checks, without a GPU, that every case has
the shape it claims (measured from the data in the order the encoder sees it: the stable bucket partition).
tests/test_gpu_page_encoder.py builds every case and walks every page of every file.

A case is a function returning a Case: the source images, the decoded columns in file order (numpy; strings as
object arrays of bytes), their validity, the bucket count, the included columns and the create_index keywords.
CLAIMS[name] lists what the case is built to put on a boundary.

plan(name) restates the encoder's choice per column: dictionary or not, the rule that decided it, the dictionary (in
sort_dictionary's order), its bit width, and where the hash set came from -- the data, sampled in stages; the
source's dictionary pages, whose union is taken as it is (entries the data never uses included); or the codes of a
carried column, whose dictionary is that same union.

walk(image) parses a file with parquet_shapes.read_struct and decodes every page, rejecting what the encoder never
writes (a bit width other than bits_for(dictionary size), an index run that is not one bit-packed run over the page,
non-zero padding).  check_file() then compares every page body with the bytes expect_pages() builds from the oracle's
rows, and every chunk's metadata with what it counted.
"""
import functools
import io
import struct
from dataclasses import dataclass, field
from typing import Dict, List

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

import parquet_shapes as S
import sort_edge_cases as E
from oracle import oracle as O

# ---- the limits ------------------------------------------------------------------------------------------------------
MAX_DICT_ENTRIES = S.MAX_DICT_ENTRIES  # kMaxDictEntries (kernels.h:323): bit width <= 16
STAGE1_ROWS = 1 << 14          # engine.cu:1192: the first sample (also DictProbe's, engine.cu:960)
STAGE2_ROWS = 1 << 18          # engine.cu:1228: the second sample
EARLY_DROP_ROWS = 1 << 20      # engine.cu:1224: only tables above this many rows drop a column after stage 1 ...
EARLY_DROP_FRACTION = 0.95     # engine.cu:1224: ... whose first STAGE1_ROWS rows are more than this fraction distinct
PAYS_OFF = 0.9                 # engine.cu:152: dictionary bytes at most this fraction of the PLAIN bytes
SORT_TILE = 4096               # kSortTile (kernels.h:225): rows_per_page is rounded up to a multiple
DEFAULT_PAGE_ROWS = 131072     # engine.cu:1093
DEFAULT_RG_ROWS = 4194304      # engine.cu:1297; rounded down to a multiple of the page, at least one page (engine.cu:1298)
MAX_CARRIED = S.MAX_CARRIED    # kMaxCarried (engine.h:44): carried columns per build (4-slot code records)
AGREE_CAP = S.AGREE_CAP        # kAgreeCap (engine.cu:599): largest source union a carried column may have
MAP_BATCH = 8                  # engine.cu:1542: dictionary columns per k_dict_map / k_dict_pack launch ...
RECORD_SLOTS_SMALL = 4         # dict_encode.cu:312: ... in 4-slot records for up to 4 columns, 8-slot ones above
ALIGN_SEARCH_BYTES = 24        # parquet_meta.h:359: extra definition-level bytes tried to align PLAIN values
EMPTY = 0xFFFFFFFFFFFFFFFF     # dict_encode.cu:17: the hash sets' empty marker (a value the set tracks in state[2])

# (value, file, line, text on that line): the host test reads each line
SOURCE_LINES = [
    (MAX_DICT_ENTRIES, "kernels.h", 323, "constexpr uint32_t kMaxDictEntries = {};"),
    (STAGE1_ROWS, "engine.cu", 1192, "const int64_t mini = std::min<int64_t>(total_rows, 1 << 14);"),
    (STAGE1_ROWS, "engine.cu", 960, "pr->mini = std::min<int64_t>(part.nrows, 1 << 14);"),
    (STAGE2_ROWS, "engine.cu", 1228, "const int64_t sample = std::min<int64_t>(total_rows, 1 << 18);"),
    (EARLY_DROP_ROWS, "engine.cu", 1224, "if (total_rows > (1 << 20) && st[0] + st[2] > 0.95 * mini) {"),
    (EARLY_DROP_FRACTION, "engine.cu", 1224, "st[0] + st[2] > 0.95 * mini"),
    (PAYS_OFF, "engine.cu", 152, "return ndict > 0 && ndict <= kMaxDictEntries && dict_bytes <= 0.9 * plain_bytes;"),
    (None, "engine.cu", 151, "const double dict_bytes = (double)total_rows * bw / 8.0 + (double)ndict * width * std::max(1, nseg);"),
    (None, "engine.cu", 157, "while ((1u << bw) < ndict) bw++;"),
    (None, "engine.cu", 127, "return ea != eb ? ea < eb : a < b;"),
    (SORT_TILE, "kernels.h", 225, "constexpr int kSortTile = {};"),
    (DEFAULT_PAGE_ROWS, "engine.cu", 1093, "int64_t P = req.rows_per_page > 0 ? req.rows_per_page : {};"),
    (None, "engine.cu", 1094, "P = (int64_t)round_up((size_t)P, kSortTile);"),
    (DEFAULT_RG_ROWS, "engine.cu", 1297, ": (req.rows_per_row_group > 0 ? req.rows_per_row_group : {});"),
    (None, "engine.cu", 1298, "RG = std::max<int64_t>(P, RG / P * P);"),
    (MAX_CARRIED, "engine.h", 44, "constexpr int kMaxCarried = {};"),
    (AGREE_CAP, "engine.cu", 599, "constexpr uint32_t kAgreeCap = {};"),
    (MAP_BATCH, "engine.cu", 1542, "for (size_t b0 = 0; b0 < dcols.size(); b0 += {}) {{"),
    (RECORD_SLOTS_SMALL, "dict_encode.cu", 315, "const int slots = map_args.ncols <= {0} ? {0} : 8;"),
    (ALIGN_SEARCH_BYTES, "parquet_meta.h", 359, "for (int extra = 0; extra <= {} && best.first < 0; extra++) {{"),
    (None, "engine.cu", 799, "(flags[1 + c] & 2u)"),
    (None, "engine.cu", 814, "dc.dict_ready = dc.dict_state[1] == 0 && dc.dict_state[0] <= kMaxDictEntries;"),
    (None, "dict_encode.cu", 187, "for (int w = 0; w < kWords; w++) r[j][w] = 0;  // padding indices of the last group are zero"),
]

# Parquet physical types of the index columns, by numpy dtype (strings: BYTE_ARRAY)
PTYPE = {np.dtype(np.int32): S.INT32, np.dtype(np.int64): S.INT64, np.dtype(np.float32): S.FLOAT,
         np.dtype(np.float64): S.DOUBLE}


def bits_for(ndict: int) -> int:
    """engine.cu:155-159: at least 1."""
    bw = 1
    while (1 << bw) < ndict:
        bw += 1
    return bw


def raw_bits(col: np.ndarray) -> np.ndarray:
    """The encoder's 64-bit view of a 4- or 8-byte column (4-byte values zero-extended: int32 -1 is not EMPTY)."""
    col = np.ascontiguousarray(col)
    return col.view(np.uint32).astype(np.uint64) if col.dtype.itemsize == 4 else col.view(np.uint64)


def from_raw(raw: np.ndarray, dtype) -> np.ndarray:
    dtype = np.dtype(dtype)
    raw = np.asarray(raw, dtype=np.uint64)
    if dtype.itemsize == 4:
        return (raw & np.uint64(0xFFFFFFFF)).astype(np.uint32).view(dtype)
    return raw.view(dtype)


def sort_dictionary(raw: np.ndarray, dtype) -> np.ndarray:
    """sort_dictionary (engine.cu:124-129): the column's order (sort_encode), then the raw bits.  EMPTY sorts as the
    value it is (for 8-byte columns: the all-ones NaN or int64 -1)."""
    raw = np.asarray(raw, dtype=np.uint64)
    if len(raw) == 0:
        return raw
    typed = from_raw(raw, dtype)
    enc = E.encode(typed)
    return raw[np.lexsort((raw, enc))]


# ---- cases -----------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    images: List[bytes]
    cols: Dict[str, np.ndarray]              # file order; strings: object arrays of bytes
    valids: Dict[str, np.ndarray]            # nullable columns only
    nb: int
    included: List[str]
    kw: dict = field(default_factory=dict)   # create_index keywords (rows_per_page, rows_per_row_group, dictionary)
    notes: dict = field(default_factory=dict)  # what the builder placed where (checked by the host test)


CASES = {}
CLAIMS = {}


def case(**claims):
    def reg(fn):
        CASES[fn.__name__] = fn
        CLAIMS[fn.__name__] = claims
        return fn
    return reg


@functools.lru_cache(maxsize=None)
def case_data(name) -> Case:
    return CASES[name]()


def _rng(seed):
    return np.random.default_rng(seed)


def _keys(n, seed):
    """Distinct int64 keys in random order, three varying bytes: the sort needs no tie fix-up, which would gather the
    pages a second time."""
    return _rng(seed).permutation(n).astype(np.int64) + 10**9


def partition_order(keys, nb):
    """Row order of the partitioned table, which the dictionary stages sample: stable by bucket."""
    return np.argsort(O.bucket_ids([keys], nb), kind="stable")


def _table(cols, valids):
    arrays = {}
    for c, v in cols.items():
        mask = None if c not in valids else ~valids[c]
        if v.dtype == object:
            arrays[c] = pa.array([x.decode() for x in v], type=pa.string(), mask=mask)
        else:
            arrays[c] = pa.array(v, mask=mask)
    return pa.table(arrays)


def _images(cols, valids=None, files=1, **write_kw):
    """Source files written by pyarrow (uncompressed, v1 pages, PLAIN unless use_dictionary says otherwise)."""
    valids = valids or {}
    t = _table(cols, valids)
    kw = dict(compression="NONE", use_dictionary=False, data_page_version="1.0")
    kw.update(write_kw)
    n = t.num_rows
    out = []
    for f in range(files):
        sink = io.BytesIO()
        pq.write_table(t.slice(f * n // files, (f + 1) * n // files - f * n // files), sink, **kw)
        out.append(sink.getvalue())
    return out


def _distinct(dtype, m, rng, exclude_empty=True):
    """m distinct values of the type (no NaN; for 8-byte types not the EMPTY bits unless asked)."""
    dtype = np.dtype(dtype)
    out = np.empty(0, dtype=dtype)
    while len(out) < m:
        if dtype.kind == "f":
            cand = (rng.standard_normal(2 * m + 16) * 1e6).astype(dtype)
        else:
            info = np.iinfo(dtype)
            cand = rng.integers(info.min, info.max, size=2 * m + 16, dtype=dtype, endpoint=True)
        out = np.unique(np.concatenate([out, cand]))
        if dtype.kind == "f":
            out = out[~np.isnan(out)]
        if exclude_empty and dtype.itemsize == 8:
            out = out[raw_bits(out) != np.uint64(EMPTY)]
    return rng.permutation(out)[:m]


def _every_value(dictionary, n, rng):
    """n rows drawn from `dictionary`, each of its values at least once, in random order."""
    m = len(dictionary)
    assert m <= n
    ix = np.concatenate([np.arange(m), rng.integers(0, m, size=n - m)])
    return dictionary[rng.permutation(ix)]


def _in_partition_order(seq, order):
    """The column whose rows, read in partition order, are `seq`."""
    out = np.empty_like(seq)
    out[order] = seq
    return out


# ---- bit widths ------------------------------------------------------------------------------------------------------
_WIDTH_TYPES = [np.int32, np.int64, np.float32, np.float64]


@case(distinct={f"d{m}": m for m in sorted({1 << k for k in range(13)} | {(1 << k) + 1 for k in range(13)})},
      dict_columns=26, map_launches=4)
def bit_widths_1_to_13():
    """2^k and 2^k + 1 distinct values for k = 0..12 (bit widths 1..13, each at its top and one past it), the four
    value types in turn, and int32 -1 (0xFFFFFFFF: not the empty marker at width 4) among 16 values."""
    n, nb = 200_000, 4
    rng = _rng(1)
    cols = {"k": _keys(n, 1)}
    for i, m in enumerate(sorted({1 << k for k in range(13)} | {(1 << k) + 1 for k in range(13)})):
        cols[f"d{m}"] = _every_value(_distinct(_WIDTH_TYPES[i % 4], m, rng), n, rng)
    d = _distinct(np.int32, 16, rng)
    d[0] = -1
    cols["m1"] = _every_value(d, n, rng)
    return Case(_images(cols, row_group_size=100_000), cols, {}, nb, [c for c in cols if c != "k"], dict(rows_per_page=65536))


def _stage_column(order, n, rng, first_new_at, few=10, late=None):
    """In partition order: `few` values from row 0, then new values from row first_new_at on (each new value first
    seen there), then the same mixture.  late: one value placed at first_new_at only."""
    base = np.arange(few, dtype=np.int64) * 1000 + 7
    seq = base[rng.integers(0, few, size=n)]
    if late is not None:
        seq[first_new_at] = late
    else:
        new = np.arange(few, dtype=np.int64) * 1000 + 8
        seq[first_new_at:first_new_at + few] = new
        tail = n - (first_new_at + few)
        seq[first_new_at + few:] = np.concatenate([base, new])[rng.integers(0, 2 * few, size=tail)]
    return _in_partition_order(seq, order)


@case(distinct={"d8192": 8192, "d8193": 8193, "d16384": 16384, "d16385": 16385, "d32768": 32768, "d32769": 32769,
                "d65536": 65536, "d65537": 65537, "e65535": 65536, "e65536": 65537},
      first_new={"s2": 20_000, "s3": 300_000, "late_empty": 500_000}, burst=("burst", STAGE2_ROWS),
      empty_marker=["e65535", "e65536", "late_empty"], rows_over=STAGE2_ROWS, default_layout=True)
def bit_widths_14_to_16_limits_and_stages():
    """600 K int64 rows in 4 buckets (the default page and row-group sizes: two pages per file).  Bit widths 13..16 at
    2^k and 2^k + 1 distinct values; 65 536 (width 16) and 65 537 (PLAIN); 65 535 values plus ~0 (a 65 536-entry
    dictionary) and 65 536 plus ~0 (PLAIN); a burst of 300 K new values after a quiet first 256 K rows, which
    overflows while the whole grid inserts (the count may pass the limit without the flag: PLAIN either way);
    values first seen in sampling stage 2 and stage 3, and ~0 first seen in stage 3."""
    n, nb = 600_000, 4
    rng = _rng(2)
    k = _keys(n, 2)
    order = partition_order(k, nb)
    cols = {"k": k}
    for m in (8192, 8193, 16384, 16385, 32768, 32769, 65536, 65537):
        cols[f"d{m}"] = _every_value(_distinct(np.int64, m, rng), n, rng)
    for m in (65535, 65536):
        d = np.concatenate([_distinct(np.int64, m, rng), np.array([-1], dtype=np.int64)])
        cols[f"e{m}"] = _every_value(d, n, rng)
    quiet = np.arange(5, dtype=np.int64)[rng.integers(0, 5, size=STAGE2_ROWS)]
    loud = _distinct(np.int64, n - STAGE2_ROWS, rng)
    cols["burst"] = _in_partition_order(np.concatenate([quiet, loud]), order)
    cols["s2"] = _stage_column(order, n, rng, 20_000)
    cols["s3"] = _stage_column(order, n, rng, 300_000)
    cols["late_empty"] = _stage_column(order, n, rng, 500_000, late=-1)
    return Case(_images(cols, row_group_size=200_000), cols, {}, nb, [c for c in cols if c != "k"], {})


@case(rows_over=EARLY_DROP_ROWS, stage1_distinct={"drop": 15565, "keep": 15564})
def early_drop_over_2_20_rows():
    """1.1 M rows: a column whose first 16 K rows (partition order) hold 15 565 distinct values -- more than 95 % --
    is dropped after stage 1 although it has only those values overall (the documented early drop, pinned here), and
    one with 15 564 is dictionary-encoded (width 14)."""
    n, nb = 1_100_000, 4
    rng = _rng(3)
    k = _keys(n, 3)
    order = partition_order(k, nb)
    cols = {"k": k}
    for name, m in (("drop", 15565), ("keep", 15564)):
        d = _distinct(np.int64, m, rng)
        head = np.concatenate([d, d[rng.integers(0, m, size=STAGE1_ROWS - m)]])
        seq = np.concatenate([rng.permutation(head), d[rng.integers(0, m, size=n - STAGE1_ROWS)]])
        cols[name] = _in_partition_order(seq, order)
    return Case(_images(cols, row_group_size=400_000), cols, {}, nb, ["drop", "keep"], {})


@case(specials=True)
def float_specials():
    """Double dictionaries with -0.0, 0.0, NaN payloads and the all-ones NaN (the empty marker's bits), float ones with
    -0.0, 0.0 and NaN payloads: one entry per bit pattern, in sort_dictionary's order."""
    n, nb = 50_000, 4
    rng = _rng(4)
    d64 = np.array([0x8000000000000000, 0, 0x7FF8000000000000, 0x7FF0000000000001, 0xFFF8000000000000,
                    0x7FFFFFFFFFFFFFFF, EMPTY, 0x3FF8000000000000, 0xC000000000000000, 0x7FF0000000000000,
                    0xFFF0000000000000, 0x0000000000000001], dtype=np.uint64).view(np.float64)
    d32 = np.array([0x80000000, 0, 0x7FC00000, 0x7F800001, 0xFFC00000, 0xFFFFFFFF, 0x3FC00000, 0x7F800000,
                    0xFF800000], dtype=np.uint32).view(np.float32)
    cols = {"k": _keys(n, 4), "f64": _every_value(d64, n, rng), "f32": _every_value(d32, n, rng)}
    return Case(_images(cols), cols, {}, nb, ["f64", "f32"], {})


@case(distinct={"pay5226": 5226, "pay5227": 5227})
def pays_off_edge():
    """The 0.9 rule at its edge: 30 000 int64 rows in 4 buckets, width 13: 5 226 distinct values pay off, 5 227 do not."""
    n, nb = 30_000, 4
    rng = _rng(11)
    cols = {"k": _keys(n, 11)}
    for m in (5226, 5227):
        cols[f"pay{m}"] = _every_value(_distinct(np.int64, m, rng), n, rng)
    return Case(_images(cols), cols, {}, nb, ["pay5226", "pay5227"], dict(rows_per_page=8192))


# ---- dictionary columns per launch -----------------------------------------------------------------------------------
def _dict_columns(ndict, ncarried, seed):
    n, nb = 30_000, 4
    rng = _rng(seed)
    cols = {"k": _keys(n, seed)}
    for i in range(ncarried + ndict):
        t = np.int32 if i % 2 else np.int64
        cols[f"c{i}"] = _every_value(_distinct(t, 3 + 7 * i, rng), n, rng)
    included = [c for c in cols if c != "k"]
    images = _images(cols, use_dictionary=included[:ncarried] or False, row_group_size=10_000)
    return Case(images, cols, {}, nb, included, dict(rows_per_page=8192))


def _register_dict_columns():
    for nd in (1, 4, 5, 8, 9, 12):
        for nc in (0, MAX_CARRIED):
            name = f"dict_columns_{nd}" + (f"_beside_{nc}_carried" if nc else "")

            def fn(nd=nd, nc=nc, seed=100 + nd + 20 * nc):
                return _dict_columns(nd, nc, seed)
            fn.__name__ = name
            case(mapped=nd, carried=nc, map_launches=-(-nd // MAP_BATCH))(fn)


_register_dict_columns()


# ---- source dictionary pages -----------------------------------------------------------------------------------------
def _dict_file(rows, k, cols):
    """A file of `rows` rows: k PLAIN, then per (name, dictionary, indices) a dictionary-encoded int64 column."""
    out = [S.Col("k", S.INT64, True, [S.Chunk([S.Page(rows=rows, values=k)])])]
    for name, d, ix in cols:
        out.append(S.Col(name, S.INT64, True, [S.Chunk([S.Page(rows=rows, enc=S.RLE_DICTIONARY, idx=S.runs_of(ix))], dict=d)]))
    return S.write_file(S.FileSpec(out))


@case(union={"u": 300, "w": 8193, "x": 65537, "z": 65536}, used={"u": 200, "x": 300}, carried=["u"])
def source_dictionaries():
    """Three files whose chunk dictionaries are taken as the hash set: u holds 300 entries of which the data uses 200
    (carried; the index dictionary keeps all 300), w a union of 8 193 (too many to carry; built from the pages), z a
    union of 65 536 (built from the pages, does not pay off), x a union of 65 537 of which 300 are used (the pages
    overflow: the data is sampled instead)."""
    rows, nfiles, nb = 20_000, 3, 4
    rng = _rng(5)
    k = _keys(rows * nfiles, 5)
    du = _distinct(np.int64, 300, rng)
    dw = _distinct(np.int64, 8193, rng)
    dz = _distinct(np.int64, 65536, rng)
    dx = _distinct(np.int64, 65537, rng)
    images, vals = [], {c: [] for c in "uwxz"}
    for f in range(nfiles):
        kf = k[f * rows:(f + 1) * rows]
        parts = {}
        iu = rng.integers(0, 200, size=rows)
        iu[:200] = np.arange(200)
        parts["u"] = (du, iu)
        sw = np.array_split(np.arange(8193), nfiles)[f]
        iw = rng.integers(0, len(sw), size=rows)
        iw[:len(sw)] = np.arange(len(sw))
        parts["w"] = (dw[sw], iw)
        sz = np.array_split(np.arange(65536), nfiles)[f]
        parts["z"] = (dz[sz], rng.integers(0, len(sz), size=rows))
        sx = np.array_split(np.arange(65537), nfiles)[f]
        ix = rng.integers(0, 100, size=rows)
        ix[:100] = np.arange(100)
        parts["x"] = (dx[sx], ix)
        images.append(_dict_file(rows, kf, [(c, parts[c][0], parts[c][1]) for c in "uwxz"]))
        for c in "uwxz":
            vals[c].append(parts[c][0][parts[c][1]])
    cols = {"k": k, **{c: np.concatenate(vals[c]) for c in "uwxz"}}
    return Case(images, cols, {}, nb, ["u", "w", "x", "z"], dict(rows_per_page=8192))


# ---- nullable and string columns -------------------------------------------------------------------------------------
@case(null_rows_in_bucket0=[4095, 4096], all_null_page=(1, 1), all_null_column="allnull")
def nullable_and_strings():
    """Columns that are never dictionary-encoded however few values they hold: nullable ones (nulls at sorted rows
    4095 / 4096 of bucket 0, i.e. on a tile and page edge; every row of bucket 1's second page null; an all-null
    column) and strings (non-null and nullable), beside a non-null dictionary column, 4096-row pages."""
    n, nb = 30_000, 3
    rng = _rng(6)
    k = _keys(n, 6)
    perm, offs, _ = O.index_rows({"k": k}, ["k"], [], nb)
    few = np.arange(5, dtype=np.int64) * 3
    cols = {"k": k, "d": few[rng.integers(0, 5, size=n)], "nv": few[rng.integers(0, 5, size=n)],
            "ne": rng.integers(-1000, 1000, size=n).astype(np.int32), "allnull": np.zeros(n, dtype=np.int64),
            "s": np.array([b"s%d" % i for i in rng.integers(0, 4, size=n)], dtype=object),
            "ns": np.array([b"str-%d" % i * (i % 3) for i in rng.integers(0, 50, size=n)], dtype=object)}
    valids = {"nv": rng.random(n) > 0.3, "ne": np.ones(n, bool), "allnull": np.zeros(n, bool), "ns": rng.random(n) > 0.5}
    valids["ne"][perm[offs[0] + 4095]] = False
    valids["ne"][perm[offs[0] + 4096]] = False
    valids["ne"][perm[offs[1] + 4096:offs[1] + 8192]] = False
    for c, v in valids.items():
        if cols[c].dtype != object:
            cols[c] = np.where(v, cols[c], 0).astype(cols[c].dtype)
        else:
            cols[c] = np.array([x if ok else b"" for x, ok in zip(cols[c], v)], dtype=object)
    return Case(_images(cols, valids), cols, valids, nb, ["d", "nv", "ne", "allnull", "s", "ns"], dict(rows_per_page=4096))


# ---- page and row-group layout ---------------------------------------------------------------------------------------
def _sized_buckets(sizes, seed):
    """Distinct int64 keys whose buckets (len(sizes) of them) hold exactly sizes[b] rows, in random order."""
    nb = len(sizes)
    rng = _rng(seed)
    pool = rng.permutation(np.unique(rng.integers(0, 1 << 24, size=20 * sum(sizes) + 1000, dtype=np.int64)))
    b = O.bucket_ids([pool], nb)
    parts = [pool[b == i][:s] for i, s in enumerate(sizes)]
    assert all(len(p) == s for p, s in zip(parts, sizes))
    return rng.permutation(np.concatenate(parts))


def _layout_columns(k, rng, nullable=True):
    n = len(k)
    cols = {"k": k, "d3": np.arange(5, dtype=np.int32)[rng.integers(0, 5, size=n)],
            "d9": _every_value(_distinct(np.int64, 300, rng), n, rng),
            "p64": rng.integers(-2**62, 2**62, size=n, dtype=np.int64),
            "p32": rng.integers(-2**31, 2**31 - 1, size=n, dtype=np.int32),
            "pf64": rng.standard_normal(n)}
    valids = {}
    if nullable:
        cols["n64"] = rng.integers(0, 1 << 40, size=n, dtype=np.int64)
        valids["n64"] = rng.random(n) > 0.25
        cols["n64"] = np.where(valids["n64"], cols["n64"], 0)
    return cols, valids


PAGE_EDGE_SIZES = [4095, 4096, 4097, 0, 4098, 4099, 4100, 4101, 4102, 4103]


@case(bucket_rows=PAGE_EDGE_SIZES, last_group_rows=set(range(1, 8)))
def page_edges():
    """Buckets of P - 1, P and P + 1 rows (P = 4096), an empty bucket beside them, and buckets whose last page's last
    group of eight holds 1..7 rows; dictionary, PLAIN (4- and 8-byte) and nullable columns."""
    rng = _rng(7)
    k = _sized_buckets(PAGE_EDGE_SIZES, 7)
    cols, valids = _layout_columns(k, rng)
    return Case(_images(cols, valids), cols, valids, len(PAGE_EDGE_SIZES), [c for c in cols if c != "k"],
                dict(rows_per_page=4096))


@case(page_rows=8192, rg_rows=16384)
def pages_not_a_multiple_of_the_tile():
    """rows_per_page = 5000 (rounded up to 8192) and rows_per_row_group = 20 000 (not a multiple of the page: 16 384)."""
    rng = _rng(8)
    k = _keys(100_000, 8)
    cols, valids = _layout_columns(k, rng)
    return Case(_images(cols, valids), cols, valids, 2, [c for c in cols if c != "k"],
                dict(rows_per_page=5000, rows_per_row_group=20_000))


@case(page_rows=4096, rg_rows=4096)
def row_group_below_the_page():
    """rows_per_row_group = 3000 below rows_per_page = 4096: one page per row group."""
    rng = _rng(9)
    k = _keys(30_000, 9)
    cols, valids = _layout_columns(k, rng)
    return Case(_images(cols, valids), cols, valids, 2, [c for c in cols if c != "k"],
                dict(rows_per_page=4096, rows_per_row_group=3000))


@case(plain_page_offsets_mod8=set(range(8)), unaligned_pages=True)
def tiny_buckets():
    """3000 rows in 200 buckets: PLAIN pages of a few rows at every file offset modulo 8 (each file's PLAIN chunks follow
    a string chunk of random length), many too small for any run split within ALIGN_SEARCH_BYTES to align their values."""
    rng = _rng(10)
    n = 3000
    cols = {"k": _keys(n, 10), "s": np.array([b"x" * int(i) for i in rng.integers(0, 40, size=n)], dtype=object),
            "p64": rng.integers(-2**62, 2**62, size=n, dtype=np.int64),
            "p32": rng.integers(-2**31, 2**31 - 1, size=n, dtype=np.int32), "pf32": rng.standard_normal(n).astype(np.float32)}
    return Case(_images(cols), cols, {}, 200, ["s", "p64", "p32", "pf32"], {})


COMPRESSED_CASES = ["page_edges", "nullable_and_strings", "dict_columns_9_beside_4_carried", "pages_not_a_multiple_of_the_tile"]


# ---- the encoder's choices, restated ---------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def source_dictionaries_of(name):
    """Per column: (every page dictionary-encoded, union of the chunk dictionaries as raw bits, rows) of the sources."""
    c = case_data(name)
    pages, _ = S.measure(c.images)
    out = {}
    for col in c.cols:
        pcs = [p for p in pages if p["col"] == col]
        out[col] = dict(all_dict=bool(pcs) and all(p["enc"] in (S.PLAIN_DICTIONARY, S.RLE_DICTIONARY) for p in pcs),
                        union=set())
    for img in c.images:
        flen = struct.unpack_from("<I", img, len(img) - 8)[0]
        fm, _ = S.read_struct(img, len(img) - 8 - flen)
        leaves = fm[2][1:]
        for rg in fm[4]:
            for ci, cc in enumerate(rg[1]):
                md = cc[3]
                if 11 not in md:
                    continue
                h, q = S.read_struct(img, md[11])
                assert h[1] == S.DICTIONARY_PAGE and md[4] == S.UNCOMPRESSED
                w = S.WIDTH[leaves[ci][1]]
                vals = np.frombuffer(img[q:q + h[3]], dtype=np.uint32 if w == 4 else np.uint64).astype(np.uint64)
                out[leaves[ci][4].decode()]["union"] |= set(vals.tolist())
    return out, pages


def _sample(raw, n):
    """The three stages of layout_segments (engine.cu:1178-1239) over the column's raw bits in partition order:
    (rule, k_dict_build launches as (fewest, most))."""
    mini = min(n, STAGE1_ROWS)

    def distinct(a):
        u = np.unique(a)
        e = int(len(u) > 0 and u[-1] == np.uint64(EMPTY))
        return len(u) - e, e

    d, e = distinct(raw[:mini])
    if n > EARLY_DROP_ROWS and d + e > EARLY_DROP_FRACTION * mini:
        return "early_drop", (1, 1)
    launches, over, sample = 1, False, min(n, STAGE2_ROWS)
    if sample > mini:
        launches += 1
        over = distinct(raw[:sample])[0] > MAX_DICT_ENTRIES
    if over and sample < n:
        # the count may pass the limit without the flag (dict_encode.cu:51-54): stage 3 may then run too; the result is
        # PLAIN either way, since more than kMaxDictEntries values never pay off
        return "overflow", (launches, launches + 1)
    if sample < n:
        launches += 1
        over = distinct(raw)[0] > MAX_DICT_ENTRIES
    return ("overflow" if over else "sampled"), (launches, launches)


@functools.lru_cache(maxsize=None)
def plan(name, carry=True):
    """The encoder's choice for every index column: {column: dict(dictionary, rule, source, values, bw, launches)}.
    rule: 'nullable' / 'string' (never dictionary-encoded), 'early_drop', 'overflow', 'no_pay' (the 0.9 rule), or
    'pays_off'.  source: 'data', 'pages' (the union of the source dictionaries) or 'carried' (the same union)."""
    c = case_data(name)
    srcd, pages = source_dictionaries_of(name)
    order = partition_order(c.cols["k"], c.nb)
    n = len(c.cols["k"])
    use_dict = c.kw.get("dictionary", True)
    carried = []
    if carry and use_dict and c.nb <= 1024:  # api.cu:607-613: the fused partition carries codes up to 1024 buckets
        carried = S.carried(pages, {col: srcd[col]["union"] for col in c.cols}, c.included, c.nb)
    out = {}
    for col in ["k"] + c.included:
        v = c.cols[col]
        p = dict(dictionary=False, rule=None, source="data", values=None, bw=None, launches=(0, 0),
                 carried=col in carried, width=8 if v.dtype == object else v.dtype.itemsize)
        out[col] = p
        nullable = col in c.valids and not c.valids[col].all()
        if v.dtype == object:
            p["rule"] = "string"
            continue
        union = srcd[col]["union"]
        from_pages = srcd[col]["all_dict"] and len(union - {EMPTY}) <= MAX_DICT_ENTRIES
        if nullable:
            p["rule"] = "nullable"
            continue
        raw = raw_bits(v)
        if col in carried or (use_dict and from_pages):
            p["source"] = "carried" if col in carried else "pages"
            values = np.array(sorted(union), dtype=np.uint64)
        else:
            if not use_dict:
                p["launches"] = (1, 1)  # DictProbe runs behind the partition whatever the setting (engine.cu:898)
                p["rule"] = "disabled"
                continue
            rule, p["launches"] = _sample(raw[order], n)
            if rule != "sampled":
                p["rule"] = rule
                continue
            values = np.unique(raw)
        p["values"] = sort_dictionary(values, v.dtype)
        ndict = len(values)
        p["bw"] = bits_for(ndict)
        if not S.dictionary_pays_off(ndict, p["width"], n, c.nb):
            p["rule"] = "no_pay"
            continue
        p["rule"], p["dictionary"] = "pays_off", True
    return out


def expected_launches(name, carry=True):
    """Kernel launches the plan implies: k_dict_build (fewest, most), k_dict_map, k_dict_pack, and whether
    k_dict_build_from_pages runs."""
    pl = plan(name, carry)
    lo = sum(p["launches"][0] for p in pl.values())
    hi = sum(p["launches"][1] for p in pl.values())
    mapped = sum(1 for p in pl.values() if p["dictionary"] and not p["carried"])
    ncarried = sum(1 for p in pl.values() if p["carried"])
    maps = -(-mapped // MAP_BATCH)
    return dict(k_dict_build=(lo, hi), k_dict_map=maps, k_dict_pack=maps + (1 if ncarried else 0),
                from_pages=any(p["source"] in ("pages", "carried") for p in pl.values()))


def layout_sizes(kw):
    """(rows per page, rows per row group) of create_index keywords (engine.cu:1093-1094, 1296-1298)."""
    P = kw.get("rows_per_page", 0) or DEFAULT_PAGE_ROWS
    P = -(-P // SORT_TILE) * SORT_TILE
    RG = kw.get("rows_per_row_group", 0) or DEFAULT_RG_ROWS
    return P, max(P, RG // P * P)


def plain_alignment_possible(page_offset, n, width):
    """write_plain_page_prefix's search (parquet_meta.h:347-388), restated: is there a split of the n ones into runs,
    within ALIGN_SEARCH_BYTES extra bytes, after which the values start 8-byte aligned?"""
    for extra in range(ALIGN_SEARCH_BYTES + 1):
        for medium in range(extra // 3 + 1):
            rest = extra - 3 * medium
            if rest % 2:
                continue
            small = rest // 2
            if n - small - 64 * medium < 1:
                continue
            defs = _def_runs(n, small, medium)
            hdr = _data_page_header(len(defs) + 4 + n * width, n, S.PLAIN)
            if (page_offset + len(hdr) + 4 + len(defs)) % 8 == 0:
                return True
    return False


def _def_runs(n, small, medium):
    runs = [n - small - 64 * medium] + [1] * small + [64] * medium
    return b"".join(S.varint(r << 1) + b"\x01" for r in runs)


def _data_page_header(body_len, n, enc, stored=None):
    w = S.ThriftWriter()
    w.i32(1, S.DATA_PAGE).i32(2, body_len).i32(3, body_len if stored is None else stored)
    w.begin(5).i32(1, n).i32(2, enc).i32(3, S.RLE).i32(4, S.RLE).end()
    return bytes(w.end().b)


# ---- the page walker -------------------------------------------------------------------------------------------------
class PageError(AssertionError):
    pass


def _decompress(codec, body, size):
    if codec == S.UNCOMPRESSED:
        return bytes(body)
    if codec == S.SNAPPY:
        return pa.decompress(body, size, codec="snappy", asbytes=True)
    if codec == 2:
        return pa.decompress(body, size, codec="gzip", asbytes=True)
    if codec == 5:  # Hadoop's Lz4Codec framing: [BE group size]([BE block size][block])...; one block per group here
        out, p = bytearray(), 0
        while p < len(body):
            usz, csz = struct.unpack_from(">II", body, p)
            out += pa.Codec("lz4_raw").decompress(bytes(body[p + 8:p + 8 + csz]), decompressed_size=usz, asbytes=True)
            p += 8 + csz
        return bytes(out)
    raise PageError(f"codec {codec} not handled")


def _runs_exact(b, p, end, bw, n, where):
    """One bit-packed run of ceil(n/8) groups filling b[p:end] exactly, padding zero: the n values."""
    h, q = S._read_varint(b, p)
    groups = (n + 7) // 8
    if h != (groups << 1) | 1:
        raise PageError(f"{where}: run header {h:#x} at byte {p}, expected one bit-packed run of {groups} groups")
    if end - q != groups * bw:
        raise PageError(f"{where}: {end - q} bytes of packed values, expected {groups * bw}")
    bits = np.unpackbits(np.frombuffer(b[q:end], dtype=np.uint8), bitorder="little").reshape(-1, bw).astype(np.uint64)
    vals = (bits << np.arange(bw, dtype=np.uint64)).sum(axis=1).astype(np.uint64) if bw else np.zeros(groups * 8, np.uint64)
    if vals[n:].any():
        slot = n + int(np.flatnonzero(vals[n:])[0])
        raise PageError(f"{where}: padding of the last group is not zero (value {int(vals[slot])} at slot {slot}, "
                        f"byte {q + slot * bw // 8} of the page body)")
    return vals[:n], q


def walk(image, name="file"):
    """Every page of a file: [dict(rg, col, ptype, kind, offset, hdr, hdr_len, body (decompressed), ...)] plus the
    footer; the structure the encoder writes is enforced, the values are decoded (dictionary pages: 'values'; data
    pages: 'valid', and 'indices' or 'values' raw bytes)."""
    img = bytes(image)
    if img[:4] != b"PAR1" or img[-4:] != b"PAR1":
        raise PageError(f"{name}: bad magic")
    flen = struct.unpack_from("<I", img, len(img) - 8)[0]
    fm, _ = S.read_struct(img, len(img) - 8 - flen)
    leaves = fm[2][1:]
    pages = []
    for g, rg in enumerate(fm[4]):
        for ci, cc in enumerate(rg[1]):
            md = cc[3]
            leaf = leaves[ci]
            ptype, cname, W = leaf[1], leaf[4].decode(), S.WIDTH[leaf[1]]
            start = md.get(11, md[9])
            p, end = start, start + md[7]
            dict_count = None
            while p < end:
                where = f"{name}: row group {g}, column {cname}, page {sum(1 for x in pages if x['rg'] == g and x['col'] == cname)}"
                h, q = S.read_struct(img, p)
                usize, csize = h[2], h[3]
                body = _decompress(md[4], img[q:q + csize], usize)
                if len(body) != usize:
                    raise PageError(f"{where}: body holds {len(body)} bytes, header says {usize}")
                rec = dict(rg=g, col=cname, ptype=ptype, offset=p, hdr=h, hdr_len=q - p, body=body, stored=csize,
                           body_offset=q, where=where)
                if h[1] == S.DICTIONARY_PAGE:
                    dict_count = h[7][1]
                    if usize != dict_count * W:
                        raise PageError(f"{where}: dictionary page of {usize} bytes for {dict_count} entries")
                    rec.update(kind="dict", values=np.frombuffer(body, dtype=np.uint32 if W == 4 else np.uint64).astype(np.uint64))
                elif h[1] == S.DATA_PAGE:
                    n, enc = h[5][1], h[5][2]
                    rec.update(kind="data", n=n, enc=enc)
                    def_len = struct.unpack_from("<I", body, 0)[0]
                    runs = S._level_runs(body, 4, 4 + def_len, n)
                    rec["def_runs"] = runs
                    rec["valid"] = S._level_values(runs, n).astype(bool)
                    if len(rec["valid"]) != n:
                        raise PageError(f"{where}: definition levels cover {len(rec['valid'])} of {n} rows")
                    at = 4 + def_len
                    rec["values_at"] = at
                    if enc in (S.PLAIN_DICTIONARY, S.RLE_DICTIONARY):
                        if dict_count is None:
                            raise PageError(f"{where}: dictionary data page without a dictionary page")
                        bw = body[at]
                        if bw != bits_for(dict_count):
                            raise PageError(f"{where}: bit width byte {bw} at byte {at}, expected {bits_for(dict_count)} "
                                            f"for {dict_count} entries")
                        nvalid = int(rec["valid"].sum())
                        rec["bw"] = bw
                        rec["indices"], _ = _runs_exact(body, at + 1, len(body), bw, nvalid, where)
                        if len(rec["indices"]) and rec["indices"].max() >= dict_count:
                            raise PageError(f"{where}: index {int(rec['indices'].max())} past the dictionary")
                    else:
                        rec["values"] = body[at:]
                else:
                    raise PageError(f"{where}: page type {h[1]}")
                pages.append(rec)
                p = q + csize
            if p != end:
                raise PageError(f"{name}: row group {g}, column {cname}: pages end at {p}, the chunk at {end}")
    return fm, pages


def _first_diff(got, want, where):
    if got == want:
        return
    m = min(len(got), len(want))
    a, b = np.frombuffer(got[:m], np.uint8), np.frombuffer(want[:m], np.uint8)
    d = np.flatnonzero(a != b)
    if len(d):
        i = int(d[0])
        raise PageError(f"{where}: byte {i} of the page body is {got[i]:#04x}, expected {want[i]:#04x}")
    raise PageError(f"{where}: page body has {len(got)} bytes, expected {len(want)}")


def _plain_values(v, width):
    if v.dtype == object:
        return b"".join(struct.pack("<I", len(x)) + x for x in v)
    return np.ascontiguousarray(v).tobytes()


def _bitpack(values, bw, n):
    groups = (n + 7) // 8
    padded = np.zeros(groups * 8, dtype=np.uint64)
    padded[:n] = values
    return S.bitpack(padded, bw)


def expect_pages(name, bucket_rows, carry=True):
    """The pages of one bucket's file, in file order: [(row group, column, kind, header checks, expected body or None,
    extra)] from the oracle's rows (bucket_rows: source row numbers in sorted order)."""
    c = case_data(name)
    pl = plan(name, carry)
    P, RG = layout_sizes(c.kw)
    n = len(bucket_rows)
    out = []
    for g, r0 in enumerate(range(0, n, RG)):
        r1 = min(n, r0 + RG)
        for col in ["k"] + c.included:
            p = pl[col]
            v = c.cols[col][bucket_rows[r0:r1]]
            valid = c.valids[col][bucket_rows[r0:r1]] if col in c.valids else np.ones(r1 - r0, bool)
            W = p["width"]
            if p["dictionary"]:
                dv = p["values"]
                body = from_raw(dv, c.cols[col].dtype).tobytes()
                out.append(dict(rg=g, col=col, kind="dict", n=len(dv), body=body))
                by_bits = np.argsort(dv, kind="stable")
                at = np.searchsorted(dv[by_bits], raw_bits(v))
                assert (dv[by_bits][np.minimum(at, len(dv) - 1)] == raw_bits(v)).all(), f"{col}: a value outside the dictionary"
                idx = by_bits[at].astype(np.uint64)
            for p0 in range(0, r1 - r0, P):
                p1 = min(r1 - r0, p0 + P)
                m = p1 - p0
                if p["dictionary"]:
                    defs = S.varint(m << 1) + b"\x01"
                    body = (struct.pack("<I", len(defs)) + defs + bytes([p["bw"]]) + S.varint((((m + 7) // 8) << 1) | 1)
                            + _bitpack(idx[p0:p1], p["bw"], m))
                    out.append(dict(rg=g, col=col, kind="data", n=m, enc=S.PLAIN_DICTIONARY, body=body))
                elif p["rule"] in ("nullable", "string"):
                    ok = valid[p0:p1]
                    groups = (m + 7) // 8
                    hv = S.varint((groups << 1) | 1)
                    bits = np.zeros(groups * 8, np.uint8)
                    bits[:m] = ok
                    defs = hv + np.packbits(bits, bitorder="little").tobytes()
                    body = struct.pack("<I", len(defs)) + defs + _plain_values(v[p0:p1][ok], W)
                    out.append(dict(rg=g, col=col, kind="data", n=m, enc=S.PLAIN, body=body, nulls=int(m - ok.sum())))
                else:
                    out.append(dict(rg=g, col=col, kind="data", n=m, enc=S.PLAIN, body=None,
                                    values=_plain_values(v[p0:p1], W), plain_width=W))
    return out


def check_file(image, name, bucket_rows, file_name="file", carry=True, codec=S.UNCOMPRESSED):
    """Walks one index file and checks every page against expect_pages and every chunk's metadata against the walk.
    Returns the walked pages (with 'aligned' / 'can_align' on PLAIN pages)."""
    c = case_data(name)
    fm, pages = walk(image, file_name)
    want = expect_pages(name, bucket_rows, carry)
    got_kinds = [(x["rg"], x["col"], x["kind"]) for x in pages]
    want_kinds = [(x["rg"], x["col"], x["kind"]) for x in want]
    if got_kinds != want_kinds:
        i = next((j for j, (a, b) in enumerate(zip(got_kinds, want_kinds)) if a != b), min(len(got_kinds), len(want_kinds)))
        raise PageError(f"{file_name}: {len(pages)} pages, expected {len(want)}; from page {i} on the file holds "
                        f"{got_kinds[i:i + 3]}, expected {want_kinds[i:i + 3]}")
    order = ["k"] + c.included
    for got, w in zip(pages, want):
        where = got["where"]
        if (got["rg"], got["col"], got["kind"]) != (w["rg"], w["col"], w["kind"]):
            raise PageError(f"{where}: a {got['kind']} page where a {w['kind']} page of column {w['col']} belongs")
        h = got["hdr"]
        if codec == S.UNCOMPRESSED and h[2] != h[3]:
            raise PageError(f"{where}: compressed size {h[3]} in an uncompressed file")
        if w["kind"] == "dict":
            if (h[7][1], h[7][2]) != (w["n"], S.PLAIN_DICTIONARY):
                raise PageError(f"{where}: dictionary header {h[7]}, expected {w['n']} entries, PLAIN_DICTIONARY")
            _first_diff(got["body"], w["body"], where)
            continue
        dh = h[5]
        if (dh[1], dh[2], dh.get(3), dh.get(4)) != (w["n"], w["enc"], S.RLE, S.RLE):
            raise PageError(f"{where}: data page header {dh}, expected {w['n']} values, encoding {w['enc']}")
        if w["body"] is not None:
            _first_diff(got["body"], w["body"], where)
            continue
        # PLAIN non-null page: the run split is free; the runs must decode to n ones and the values follow them
        if not got["valid"].all() or any(r[0] != "rle" for r in got["def_runs"]) or sum(r[1] for r in got["def_runs"]) != w["n"]:
            raise PageError(f"{where}: definition levels are not runs of ones covering {w['n']} rows")
        _first_diff(got["values"], w["values"], where + " (values)")
        values_at = got["body_offset"] + got["values_at"]
        got["aligned"] = values_at % 8 == 0
        got["can_align"] = plain_alignment_possible(got["offset"] % 8, w["n"], w["plain_width"])
        if codec == S.UNCOMPRESSED and got["can_align"] and not got["aligned"]:
            raise PageError(f"{where}: values start at file offset {values_at}, not 8-byte aligned, though a run split "
                            f"aligns them")
    _check_metadata(fm, pages, c, order, len(bucket_rows), file_name, codec)
    return pages


def _check_metadata(fm, pages, c, order, nrows, file_name, codec):
    leaves = fm[2][1:]
    if [x[4].decode() for x in leaves] != order or fm[3] != nrows:
        raise PageError(f"{file_name}: schema {[x[4] for x in leaves]} / {fm[3]} rows, expected {order} / {nrows}")
    P, RG = layout_sizes(c.kw)
    want_rgs = [min(RG, nrows - r0) for r0 in range(0, nrows, RG)]
    if [rg[3] for rg in fm[4]] != want_rgs:
        raise PageError(f"{file_name}: row groups of {[rg[3] for rg in fm[4]]} rows, expected {want_rgs}")
    for g, rg in enumerate(fm[4]):
        tot_u = tot_c = 0
        for ci, cc in enumerate(rg[1]):
            md, col = cc[3], order[ci]
            where = f"{file_name}: row group {g}, column {col}"
            ptype = S.BYTE_ARRAY if c.cols[col].dtype == object else PTYPE[c.cols[col].dtype]
            mine = [p for p in pages if p["rg"] == g and p["col"] == col]
            data = [p for p in mine if p["kind"] == "data"]
            has_dict = mine[0]["kind"] == "dict"
            checks = {
                "type": (md[1], ptype, leaves[ci][1]),
                "encodings": (md[2], [S.PLAIN_DICTIONARY, S.PLAIN, S.RLE] if has_dict else [S.PLAIN, S.RLE]),
                "path": (md[3], [col.encode()]),
                "codec": (md[4], codec),
                "num_values": (md[5], rg[3], sum(p["n"] for p in data)),
                "total_uncompressed_size": (md[6], sum(p["hdr_len"] + p["hdr"][2] for p in mine)),
                "total_compressed_size": (md[7], sum(p["hdr_len"] + p["stored"] for p in mine)),
                "data_page_offset": (md[9], data[0]["offset"]),
                "dictionary_page_offset": (md.get(11), mine[0]["offset"] if has_dict else None),
                "file_offset": (cc[2], mine[0]["offset"]),
                "null_count": (md.get(12, {}).get(3), sum(int((~p["valid"]).sum()) for p in data)),
                "repetition": (leaves[ci].get(3), 1),
            }
            for what, vals in checks.items():
                if any(x != vals[0] for x in vals[1:]):
                    raise PageError(f"{where}: {what} is {vals[0]}, expected {vals[1:]}")
            tot_u += md[6]
            tot_c += md[7]
        first = rg[1][0][2]
        if (rg[2], rg.get(6, rg[2]), rg.get(5)) != (tot_u, tot_c, first):
            raise PageError(f"{file_name}: row group {g}: sizes / offset {(rg[2], rg.get(6), rg.get(5))}, "
                            f"expected {(tot_u, tot_c, first)}")
