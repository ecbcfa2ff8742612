"""Hash-partition inputs placed exactly on either side of the limits at which the partition (hash_rows / move_rows in
hyperspace_b200/csrc/hash_partition.cu) changes path, and a numpy restatement of what it must produce.

Every limit the partition turns on is restated once below, with the line it mirrors.  tests/test_partition_host.py checks
the constants against the source and that every case really has the shape it claims (CLAIMS), without a GPU;
tests/test_gpu_partition.py runs each case through hs_k_partition and compares every output byte with expected().

A case is a Case: key columns (with validity and decimal flags), the bucket count, the mode -- "local" (rows to
bucket-major order, as on one GPU), "owner" (to owner-major order, owner = bucket % world) or "peer" (every bucket's run
to its owner's buffer at a base the case lays out, with gaps standing in for the other ranks' rows) -- and the columns
that move: payload of 8, 4 and 1 bytes per row, and 0..4 uint16 code columns that leave as one 8-byte record per row.

The expected result does not come from the GPU code: bucket = the C oracle's bucket_ids (pinned to Spark's vectors in
tests/golden/spark_hash_vectors.json); the moved columns are col[argsort(bin, stable)]; key_or_and is the OR / AND of the
last key's sort encoding, a null counted as 0.  Rows are placed in chosen buckets by drawing keys from a pool hashed once.
"""
import functools
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

import sort_edge_cases as E
from oracle import oracle as O

# ---- the limits ------------------------------------------------------------------------------------------------------
FUSED_MAX_BINS = 1024  # kFusedMaxBins (hash_partition.cu:23): k_partition_rows up to here, k_partition_dest + k_scatter above
TILE_LOCAL = 4096      # kFusedTileLocal (kernels.h:171): rows per tile when the partition writes local memory
TILE_PEER = 8192       # kFusedTilePeer (kernels.h:172): rows per tile when the runs go to the owners' buffers
CHUNK = 256            # kChunk (hash_partition.cu:60): tiles per chunk of the column scan (k_chunk_sums / scan / apply)
MAX_BUCKETS = 4096     # kMaxBuckets (kernels.h:161)
WARP_ROWS = 512        # kWarpRows (hash_partition.cu:28, FusedCfg::kWarpRows): consecutive rows ranked by one warp
BITS_BANDS = ((16, 4), (256, 8), (FUSED_MAX_BINS, 10))  # launch_partition_rows (hash_partition.cu:790-792): vote bits
SENTINEL = 0xA5        # every output byte before the partition runs


def vote_bits(nbins: int) -> Optional[int]:
    """Bits match_any_bits votes on in k_partition_rows; None: the unfused partition (more than FUSED_MAX_BINS bins)."""
    for limit, bits in BITS_BANDS:
        if nbins <= limit:
            return bits
    return None


def tile_rows(mode: str) -> int:
    """hash_rows' tile (hash_partition.cu:816): the peer tile when the runs go to the owners' buffers, else the local one
    (partition_tile_rows, hash_partition.cu:797-800, says the same for a build)."""
    return TILE_PEER if mode == "peer" else TILE_LOCAL


def single_key_type(c) -> Optional[str]:
    """single_key_type_of (hash_partition.cu:724-728): one int32 / int64 key without a validity array selects the
    kernels with that key's hash inlined (a decimal int32 among them); anything else the general row hash."""
    if len(c.keys) == 1 and c.valids[0] is None and c.keys[0].dtype in (np.int32, np.int64):
        return str(c.keys[0].dtype)
    return None


# ---- cases -----------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    keys: List[np.ndarray]
    nb: int
    valids: List[Optional[np.ndarray]] = None
    decimal: List[bool] = None
    mode: str = "local"
    world: int = 1
    ncodes: int = 0
    shifted: tuple = ()      # peer: owners whose buffer starts 8 bytes past a 16-byte boundary
    payload: List[np.ndarray] = field(default=None)
    codes: List[np.ndarray] = field(default=None)

    def __post_init__(self):
        n = len(self.keys[0])
        self.valids = self.valids or [None] * len(self.keys)
        self.decimal = self.decimal or [False] * len(self.keys)
        rng = np.random.default_rng(n * 7 + self.nb)
        if self.payload is None:  # every row distinguishable in every column but the 1-byte one
            i = np.arange(n, dtype=np.uint64)
            self.payload = [O.splitmix64(5, i).view(np.int64), (O.splitmix64(6, i) >> np.uint64(32)).astype(np.uint32).view(np.int32),
                            rng.integers(0, 256, size=n, dtype=np.uint8)]
        if self.codes is None:
            self.codes = [rng.integers(0, 1 << 16, size=n, dtype=np.uint16) for _ in range(self.ncodes)]

    @property
    def nbins(self):
        return self.world if self.mode == "owner" else self.nb


CASES = {}
CLAIMS = {}


def case(name, **claims):
    def reg(fn):
        CASES[name] = fn
        CLAIMS[name] = claims
        return fn
    return reg


POOL = 1 << 17


@functools.lru_cache(maxsize=None)
def _pool(kind: str, nb: int):
    """POOL keys of `kind` ("int64", "int32" or "decimal", an int32 holding a decimal's unscaled value), their buckets
    for nb buckets, and per bucket the keys that land there: (keys, order by bucket, start of every bucket in it)."""
    rng = np.random.default_rng({"int64": 1, "int32": 2, "decimal": 3}[kind])
    if kind == "int64":
        vals = rng.integers(-2**63, 2**63 - 1, size=POOL, dtype=np.int64)
    else:
        vals = rng.integers(-2**31, 2**31 - 1, size=POOL, dtype=np.int32)
    b = bucket_ids([vals], [None], [kind == "decimal"], nb)
    order = np.argsort(b, kind="stable")
    starts = np.searchsorted(b[order], np.arange(nb + 1))
    assert (np.diff(starts) > 0).all(), f"the {kind} pool misses a bucket of {nb}"
    return vals, order, starts


def keys_in(kind: str, nb: int, buckets, seed: int = 0) -> np.ndarray:
    """A key from the pool for every entry of `buckets` (its bucket among nb), drawn at random within the bucket."""
    vals, order, starts = _pool(kind, nb)
    buckets = np.asarray(buckets, dtype=np.int64)
    rng = np.random.default_rng(seed)
    size = starts[buckets + 1] - starts[buckets]
    pick = starts[buckets] + (rng.random(len(buckets)) * size).astype(np.int64)
    return vals[order[pick]]


def bucket_ids(keys, valids, decimal, nb) -> np.ndarray:
    """The oracle's bucket: Spark hashes a decimal(p <= 9) as hashLong of its unscaled value, i.e. the int64 widening."""
    cols = [k.astype(np.int64) if d else k for k, d in zip(keys, decimal)]
    return O.bucket_ids(cols, nb, valids if any(v is not None for v in valids) else None)


def _random_keys(n, nb, kind="int64", seed=0):
    rng = np.random.default_rng(seed)
    return keys_in(kind, nb, rng.integers(0, nb, size=n), seed)


def _nulls(n, seed, frac=0.1):
    return (np.random.default_rng(seed).random(n) >= frac).astype(np.uint8)


def _floats(dtype, n, seed):
    """Keys with -0.0, +0.0 and NaNs of several payloads and both signs among ordinary values."""
    rng = np.random.default_rng(seed)
    special = E._F64_SPECIAL if dtype == np.float64 else E._F32_SPECIAL
    v = (rng.standard_normal(n) * 1000).astype(dtype)
    at = rng.choice(n, min(n, 50 * len(special)), replace=False)
    v[at] = np.resize(special, len(at))
    return v


# bucket counts on both sides of every vote width and of the fused limit
BUCKET_COUNTS = (1, 2, 15, 16, 17, 255, 256, 257, 1023, 1024, 1025, 4095, 4096)
for _nb in BUCKET_COUNTS:
    def _fn(nb=_nb):
        n = 3 * TILE_LOCAL + 1000 if nb <= 256 else 6 * TILE_LOCAL + 123
        return Case([_random_keys(n, nb, seed=nb)], nb, ncodes=2 if nb <= FUSED_MAX_BINS else 0)
    case(f"buckets_{_nb}", bits=vote_bits(_nb))(_fn)

for _nb in (16, 17, 256, 257, 1024):
    def _fn(nb=_nb):
        n = 2 * TILE_PEER + 777
        return Case([_random_keys(n, nb, seed=nb + 1)], nb, mode="peer", world=2, ncodes=2)
    case(f"peer_buckets_{_nb}", bits=vote_bits(_nb))(_fn)



def _vote_round(mode, world):
    """One warp round (rows 0..31) split between bins 0 and 16, which only the vote's fifth bit tells apart; the rest of
    the warp's 512 rows in bin 5.  At 17 bins a 4-bit vote would rank the two bins as one."""
    b = np.full(512, 5)
    b[:16], b[16:32] = 0, 16
    return Case([keys_in("int64", 17, b, 7)], 17, mode=mode, world=world, ncodes=2)


case("vote_bit_4_local", bits=8, split_round=(0, 16))(lambda: _vote_round("local", 1))
case("vote_bit_4_peer", bits=8, split_round=(0, 16))(lambda: _vote_round("peer", 2))

# row counts: a warp's rows, both tile sizes, and one row past a whole chunk of tiles (the chunk carry)
ROW_COUNTS = (0, 1, 31, 32, 33, 511, 512, 513, 4095, 4096, 4097, 8191, 8192, 8193, CHUNK * TILE_LOCAL - 1,
              CHUNK * TILE_LOCAL + 1)
for _n in ROW_COUNTS:
    def _fn(n=_n):
        return Case([_random_keys(n, 61, seed=n + 3)], 61, ncodes=1)
    case(f"rows_{_n}", n=_n)(_fn)

PEER_ROW_COUNTS = (1, 33, 513, 4097, 8191, 8192, 8193, CHUNK * TILE_PEER - 1, CHUNK * TILE_PEER + 1)
for _n in PEER_ROW_COUNTS:
    def _fn(n=_n):
        return Case([_random_keys(n, 61, seed=n + 4)], 61, mode="peer", world=3, ncodes=1)
    case(f"peer_rows_{_n}", n=_n)(_fn)


@case("owner_rows_chunk_carry", n=CHUNK * TILE_LOCAL + 1)
def _owner_chunk():
    n = CHUNK * TILE_LOCAL + 1
    return Case([_random_keys(n, 2000, seed=8)], 2000, mode="owner", world=4)


# ---- skew ------------------------------------------------------------------------------------------------------------
def _one_bin_tile(mode, world):
    t = tile_rows(mode)
    n, nb = 3 * t + 100, 64
    b = np.random.default_rng(9).integers(0, nb, size=n)
    b[t:2 * t] = 37  # the whole second tile, so every warp's 512 rows, in one bucket
    return Case([keys_in("int64", nb, b, 9)], nb, mode=mode, world=world, ncodes=2)


case("one_bin_tile_local", max_run=TILE_LOCAL)(lambda: _one_bin_tile("local", 1))
case("one_bin_tile_peer", max_run=TILE_PEER)(lambda: _one_bin_tile("peer", 2))


def _all_last_bin(mode, world):
    t = tile_rows(mode)
    n, nb = 2 * t + 1, 64
    return Case([keys_in("int64", nb, np.full(n, nb - 1), 10)], nb, mode=mode, world=world, ncodes=3)


case("all_last_bin_tail_1_local", last_bin_only=True, tail=1)(lambda: _all_last_bin("local", 1))
case("all_last_bin_tail_1_peer", last_bin_only=True, tail=1)(lambda: _all_last_bin("peer", 4))


def _empty_between(mode, world):
    n, nb = 20_000, 256
    used = np.array([0, 3, 100, 101, 254, 255])
    b = used[np.random.default_rng(11).integers(0, len(used), size=n)]
    return Case([keys_in("int32", nb, b, 11)], nb, mode=mode, world=world, ncodes=1)


case("empty_bins_between_local", empty_between=True)(lambda: _empty_between("local", 1))
case("empty_bins_between_peer", empty_between=True)(lambda: _empty_between("peer", 3))


def _tail_in_last_bin(mode, world, tail):
    t = tile_rows(mode)
    n, nb = 2 * t + tail, 64
    b = np.random.default_rng(12).integers(0, nb - 1, size=n)
    b[2 * t:] = nb - 1  # the real rows of the partial last tile all land in the last bin, beside its phantom slots
    return Case([keys_in("int64", nb, b, 12)], nb, mode=mode, world=world, ncodes=2)


for _mode, _world in (("local", 1), ("peer", 2)):
    for _tail in (1, tile_rows(_mode) - 1):
        case(f"tail_in_last_bin_{_tail}_{_mode}", tail=_tail, tail_in_last_bin=True)(
            lambda m=_mode, w=_world, tl=_tail: _tail_in_last_bin(m, w, tl))


def _one_per_bin(mode, world):
    nb = 1024
    b = np.random.default_rng(13).permutation(nb)
    return Case([keys_in("int64", nb, b, 13)], nb, mode=mode, world=world, ncodes=4)


case("one_row_per_bin_1024_local", one_per_bin=True, bits=10)(lambda: _one_per_bin("local", 1))
case("one_row_per_bin_1024_peer", one_per_bin=True, bits=10)(lambda: _one_per_bin("peer", 4))


# ---- keys ------------------------------------------------------------------------------------------------------------
_MODES = {"local": dict(mode="local"), "owner": dict(mode="owner", world=3), "peer": dict(mode="peer", world=2)}


def _key_case(kind, mode, nulls):
    n = 20_000
    nb = 4096 if mode == "owner" else 200  # the owner pass is what several GPUs run above 1024 buckets
    k = _random_keys(n, nb, "int32" if kind == "decimal" else kind, seed=14)
    return Case([k], nb, valids=[_nulls(n, 15) if nulls else None], decimal=[kind == "decimal"], ncodes=1, **_MODES[mode])


for _kind in ("int32", "int64", "decimal"):
    for _mode in ("local", "owner", "peer"):
        case(f"key_{_kind}_{_mode}", kt=("int64" if _kind == "int64" else "int32"))(
            lambda k=_kind, m=_mode: _key_case(k, m, False))
    for _mode in ("local", "owner"):
        case(f"key_{_kind}_nulls_{_mode}", kt=None)(lambda k=_kind, m=_mode: _key_case(k, m, True))

for _dt in (np.float32, np.float64):
    for _mode in ("local", "owner", "peer"):
        def _fn(dt=_dt, mode=_mode):
            n = 12_000
            return Case([_floats(dt, n, 16)], 200, valids=[_nulls(n, 17) if mode == "owner" else None], ncodes=1,
                        **_MODES[mode])
        case(f"key_{np.dtype(_dt).name}_specials_{_mode}", kt=None, specials=True)(_fn)


def _multi_key(nkeys, mode):
    n = 15_000
    rng = np.random.default_rng(18)
    keys = [rng.integers(-50, 50, size=n, dtype=np.int32), _floats(np.float64, n, 19),
            rng.integers(-2**31, 2**31 - 1, size=n, dtype=np.int32)][:nkeys]
    valids = [_nulls(n, 20), None, _nulls(n, 21, 0.3)][:nkeys]
    decimal = [False, False, True][:nkeys]
    return Case(keys, 300, valids=valids, decimal=decimal, ncodes=2, **_MODES[mode])


for _nk in (2, 3):
    for _mode in ("local", "owner", "peer"):
        case(f"keys_{_nk}_{_mode}", kt=None)(lambda k=_nk, m=_mode: _multi_key(k, m))


# ---- code records ----------------------------------------------------------------------------------------------------
for _nc in (1, 2, 3, 4):
    for _mode in ("local", "peer"):
        def _fn(nc=_nc, mode=_mode):
            n = 2 * TILE_PEER + 99
            return Case([_random_keys(n, 100, seed=22 + nc)], 100, ncodes=nc, **_MODES[mode])
        case(f"codes_{_nc}_{_mode}", ncodes=_nc)(_fn)


# ---- owners' buffers -------------------------------------------------------------------------------------------------
for _w in (2, 3, 4):
    def _fn(w=_w):
        n = 3 * TILE_PEER + 1234
        return Case([_random_keys(n, 300, seed=30 + w)], 300, mode="peer", world=w, ncodes=3)
    case(f"peer_world_{_w}", parity=True)(_fn)


@case("peer_owner_shifted_8_bytes", shifted=(1,))
def _shifted():
    n = 3 * TILE_PEER + 1234
    return Case([_random_keys(n, 300, seed=40)], 300, mode="peer", world=3, ncodes=4, shifted=(1,))


@functools.lru_cache(maxsize=None)
def case_data(name: str) -> Case:
    return CASES[name]()


# ---- the restatement -------------------------------------------------------------------------------------------------
def encode_last_key(c: Case) -> np.ndarray:
    """row_hash's last_encoded: the sort encoding of the last key column, 0 for a null."""
    enc = E.encode(c.keys[-1])
    if c.valids[-1] is not None:
        enc = np.where(c.valids[-1] != 0, enc, np.uint64(0))
    return enc


def _layout(c: Case, counts: np.ndarray):
    """The owners' buffers of a peer case: owner o lays its buckets out in increasing order, with a gap of 0..3 rows
    before every run (another rank's rows) and after the last; returns (base per bucket, rows per owner)."""
    rng = np.random.default_rng(c.nb * 31 + c.world)
    gaps = rng.integers(0, 4, size=c.nb + c.world)
    cursor = gaps[c.nb:].astype(np.int64)  # leading gap of every owner
    base = np.zeros(c.nb, dtype=np.uint64)
    for b in range(c.nb):
        o = b % c.world
        base[b] = cursor[o]
        cursor[o] += int(counts[b]) + int(gaps[b])
    return base, cursor.astype(np.uint64)


@functools.lru_cache(maxsize=None)
def analyse(name: str) -> dict:
    """Where case `name` puts every row (bucket, bin, tile, destination) and what the partition must produce."""
    c = case_data(name)
    n = len(c.keys[0])
    bucket = bucket_ids(c.keys, c.valids, c.decimal, c.nb).astype(np.int64)
    bins = bucket % c.world if c.mode == "owner" else bucket
    nbins = c.nbins
    order = np.argsort(bins, kind="stable")
    counts = np.bincount(bins, minlength=nbins)
    t = tile_rows(c.mode)
    ntiles = -(-n // t)
    tile_of = np.arange(n) // t
    tile_bin = np.bincount(tile_of * nbins + bins, minlength=ntiles * nbins).reshape(ntiles, nbins)
    enc = encode_last_key(c)
    or_and = (int(np.bitwise_or.reduce(enc)), int(np.bitwise_and.reduce(enc))) if n else (0, 2**64 - 1)
    a = dict(n=n, bucket=bucket, bins=bins, nbins=nbins, order=order, counts=counts, ntiles=ntiles, tile_bin=tile_bin,
             offsets=np.concatenate([[0], np.cumsum(counts)]).astype(np.uint64), key_or_and=or_and,
             tail=n - (ntiles - 1) * t if n else 0, kt=single_key_type(c))
    if c.mode == "peer":
        base, owner_rows = _layout(c, counts)
        a["base"], a["owner_rows"] = base, owner_rows
        a["shift"] = [8 if o in c.shifted else 0 for o in range(c.world)]
        # destination row of every row inside its owner's buffer: the bucket's base + its rank within the bucket
        rank = np.empty(n, dtype=np.int64)
        rank[order] = np.arange(n) - np.repeat(a["offsets"][:-1].astype(np.int64), counts)
        a["dest"] = base[bucket].astype(np.int64) + rank
    return a


def runs(name: str):
    """Peer cases: one (P, dst, rows, owner) per non-empty (tile, bucket) run -- P: rows of the tile's earlier buckets,
    dst: the run's first destination row (the parity pair the padded exchange layout matches)."""
    c, a = case_data(name), analyse(name)
    tb = a["tile_bin"]
    before = np.cumsum(tb, axis=1) - tb            # P per (tile, bin)
    earlier = np.cumsum(tb, axis=0) - tb           # rows of the bucket in earlier tiles
    out = []
    for t, b in zip(*np.nonzero(tb)):
        out.append((int(before[t, b]), int(a["base"][b]) + int(earlier[t, b]), int(tb[t, b]), b % c.world))
    return out


def records(c: Case) -> np.ndarray:
    """The 8-byte code record of every row: code j in bits [16 j, 16 j + 16)."""
    rec = np.zeros(len(c.keys[0]), dtype=np.uint64)
    for j, col in enumerate(c.codes):
        rec |= col.astype(np.uint64) << np.uint64(16 * j)
    return rec


def moved_columns(c: Case):
    """(name, values) of every column the partition moves, the records last."""
    cols = [(f"payload{i}_w{p.dtype.itemsize}", p) for i, p in enumerate(c.payload)]
    if c.codes:
        cols.append(("records", records(c)))
    return cols


def expected(name: str):
    """Per moved column: the expected output buffers as bytes, slack included -- one, or one per owner -- and a mask of
    the bytes inside the runs."""
    c, a = case_data(name), analyse(name)
    out = {}
    for cname, col in moved_columns(c):
        w = col.dtype.itemsize
        if c.mode != "peer":
            buf = np.full(a["n"] * w + 16, SENTINEL, dtype=np.uint8)
            buf[:a["n"] * w].view(col.dtype)[:] = col[a["order"]]
            mask = np.zeros(len(buf), dtype=bool)
            mask[:a["n"] * w] = True
            out[cname] = [(buf, mask)]
            continue
        bufs = []
        for o in range(c.world):
            s, rows = a["shift"][o], int(a["owner_rows"][o])
            buf = np.full(s + rows * w + 16, SENTINEL, dtype=np.uint8)
            mask = np.zeros(len(buf), dtype=bool)
            mine = np.flatnonzero(a["bucket"] % c.world == o)
            buf[s:s + rows * w].view(col.dtype)[a["dest"][mine]] = col[mine]
            mask[s:s + rows * w].reshape(rows, w)[a["dest"][mine]] = True
            bufs.append((buf, mask))
        out[cname] = bufs
    return out
