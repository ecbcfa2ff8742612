"""GPU tests of Spark timestamp and decimal columns: INT96 / MILLIS / MICROS timestamps and INT32 / INT64 /
FIXED_LEN_BYTE_ARRAY decimals as indexed and included columns, bucketed and sorted as Spark does (hashLong of the micros
or of the unscaled value), written back as INT64 TIMESTAMP_MICROS and INT32 / INT64 DECIMAL; the refusals Spark 3.1
makes; filter scans with timestamp and decimal literals; joins on timestamp and decimal keys; the Hyperspace API."""
import datetime
import decimal
import io
import json

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import join_oracle as J
import spark_types_oracle as S
from oracle import oracle as O

pytestmark = pytest.mark.gpu

NB = 16
N_ROWS = 6000


@pytest.fixture(scope="module")
def ctx():
    from hyperspace_b200 import _native

    c = _native.Context(0)
    yield c
    c.close()


def _image(table, **kw):
    sink = io.BytesIO()
    pq.write_table(table, sink, **kw)
    return sink.getvalue()


def _values(kind, n, rng, nulls):
    """A pyarrow array of `kind` with heavy ties, and the pyarrow type it is written from."""
    mask = (rng.random(n) < 0.1) if nulls else None
    if kind in ("int96", "micros", "millis"):
        lo, hi = S.MICROS_1900 // 1000, 4_102_444_800_000  # 1900 .. 2100 in millis
        ms = rng.integers(lo, hi, n // 8)[rng.integers(0, n // 8, n)]
        unit = "ms" if kind == "millis" else ("ns" if kind == "int96" else "us")
        mult = {"ms": 1, "us": 1000, "ns": 1_000_000}[unit]
        sub = rng.integers(0, mult, n) if mult > 1 else 0
        vals = ms * mult + sub
        return pa.array(vals, pa.timestamp(unit), mask=mask)
    p, s = {"dec9": (9, 2), "dec12": (12, 2), "dec18": (18, 2)}[kind.split("_")[0]]
    bound = 10 ** p - 1
    u = rng.integers(-bound, bound + 1, n // 8, dtype=np.int64)[rng.integers(0, n // 8, n)]
    u[:4] = [bound, -bound, 0, -1]
    return pa.array([None if (mask is not None and mask[i]) else decimal.Decimal(int(x)).scaleb(-s) for i, x in enumerate(u)],
                    pa.decimal128(p, s))


def _write_kw(kind):
    kw = dict(compression="NONE")
    if kind == "int96":
        kw["use_deprecated_int96_timestamps"] = True
    if kind == "millis":
        kw["coerce_timestamps"] = "ms"
    if kind.endswith("_int"):
        kw["store_decimal_as_integer"] = True
    return kw


# (source kind, nullable, extra writer options); decimals "_int" are stored as INT32 / INT64, the others as FLBA
SOURCES = [("int96", False, {}), ("int96", True, {"use_dictionary": False}), ("int96", False, {"use_dictionary": False}),
           ("micros", True, {}), ("millis", False, {}), ("dec9_int", False, {}), ("dec9_flba", True, {}),
           ("dec9_flba", False, {"use_dictionary": False}), ("dec12_int", True, {"data_page_version": "2.0"}),
           ("dec12_flba", False, {"compression": "SNAPPY"}), ("dec18_flba", False, {"data_page_version": "2.0"}),
           ("dec18_flba", False, {"use_dictionary": False})]


def _source(kind, nullable, extra, seed=1, n=N_ROWS):
    rng = np.random.default_rng(seed)
    t = pa.table({"c": _values(kind, n, rng, nullable), "v": pa.array(np.arange(n, dtype=np.int64))})
    kw = _write_kw(kind)
    kw.update(extra)
    return t, _image(t, row_group_size=n // 2, **kw)


def _expected_type(kind):
    if kind in ("int96", "micros", "millis"):
        return "INT64", "TIMESTAMP_MICROS", "timestamp"
    p = int(kind.split("_")[0][3:])
    return ("INT32" if p <= 9 else "INT64"), "DECIMAL", f"decimal({p},2)"


@pytest.mark.parametrize("role", ["key", "included"])
def test_parquet_mr_int96(ctx, role):
    """INT96 in parquet-mr's shape: PLAIN_DICTIONARY v1 pages with statistics, a PLAIN fallback page, a PLAIN row group."""
    from hyperspace_b200 import _native as N

    image, micros, v = S.parquet_mr_int96()
    indexed, included = (["ts"], ["v"]) if role == "key" else (["v"], ["ts"])
    res, _ = ctx.create_index([N.FileImage(data=image)], indexed, included, NB, output=N.HS_OUT_HOST)
    try:
        _check_index(ctx, res, None, "int96", indexed, included, expected=({"ts": micros, "v": v}, {}), col="ts")
    finally:
        res.free()


# hand-built decimals pyarrow does not write: (physical type, FLBA length, precision), several PLAIN pages
HAND_DECIMALS = [(2, None, 9), (S.FIXED_LEN_BYTE_ARRAY, 5, 9), (S.FIXED_LEN_BYTE_ARRAY, 16, 18), (S.FIXED_LEN_BYTE_ARRAY, 3, 6)]


@pytest.mark.parametrize("ptype,length,precision", HAND_DECIMALS)
@pytest.mark.parametrize("role", ["key", "included"])
def test_hand_built_decimals(ctx, ptype, length, precision, role):
    """INT64-stored decimal(9,2) (narrowed to int32) and FIXED_LEN_BYTE_ARRAY decimals of 5, 16 and 3 bytes."""
    from hyperspace_b200 import _native as N

    rng = np.random.default_rng(precision + (length or 0))
    bound = 10 ** precision - 1
    u = rng.integers(-bound, bound + 1, 5000, dtype=np.int64)
    u[:4] = [bound, -bound, 0, -1]
    image = S.decimal_file(ptype, u, precision, 2, length=length, rows_per_page=1300)
    indexed, included = (["d"], ["v"]) if role == "key" else (["v"], ["d"])
    res, _ = ctx.create_index([N.FileImage(data=image)], indexed, included, NB, output=N.HS_OUT_HOST)
    try:
        exp = ({"d": u, "v": np.arange(len(u), dtype=np.int64)}, {})
        _check_index(ctx, res, None, f"dec{precision}", indexed, included, expected=exp, col="d")
    finally:
        res.free()


@pytest.mark.parametrize("ptype,length", [(2, None), (S.FIXED_LEN_BYTE_ARRAY, 5), (S.FIXED_LEN_BYTE_ARRAY, 16)])
def test_decimal_wider_than_its_width_is_a_format_error(ctx, ptype, length):
    """A decimal(9,2) value that does not fit an int32, or a decimal(18,2) in 16 bytes that does not fit an int64:
    HS_EFORMAT naming the column."""
    from hyperspace_b200 import _native as N

    precision = 18 if length == 16 else 9
    too_wide = 2**31 if precision == 9 else 2**63
    u = [1, -2, too_wide, 3]
    if precision == 18:
        import parquet_shapes as P
        d = P.Col("d", S.FIXED_LEN_BYTE_ARRAY, False,
                  [P.Chunk([P.Page(rows=4, values=np.array([int(x).to_bytes(16, "big", signed=True) for x in u], "V16"))])])
        vcol, _ = S._v_column(4, [4])
        image = S.annotate_leaf(S.write_shapes_file(P.FileSpec([d, vcol]), {S.FIXED_LEN_BYTE_ARRAY: 16}), "d",
                                S.FIXED_LEN_BYTE_ARRAY, False, type_length=16, converted=S.CT_DECIMAL, precision=18, scale=2)
    else:
        image = S.decimal_file(ptype, u, precision, 2, length=length)
    with pytest.raises(N.HyperspaceGpuError) as e:
        ctx.create_index([N.FileImage(data=image)], ["d"], ["v"], NB, output=N.HS_OUT_HOST)
    assert e.value.code == -4 and "'d'" in str(e.value)


def _expected(src, names):
    """{name: Spark int64 values} and {name: validity} of the columns of a pyarrow table."""
    back = pq.read_table(io.BytesIO(_image(src, use_deprecated_int96_timestamps=True)), coerce_int96_timestamp_unit="us")
    cols, valids = {}, {}
    for name in names:
        vals, valid = S.spark_int64(back.column(name))
        cols[name] = vals
        if valid is not None:
            valids[name] = valid
    return cols, valids


def _check_index(ctx, res, src, kind, indexed, included, expected=None, col="c"):
    """Every file: the oracle's rows on the Spark values (bucket and order), the table's physical / converted types and
    Spark schema, key min / max; and hs_verify_index is clean.  expected: (columns, validities) instead of `src`'s."""
    from hyperspace_b200 import _native as N

    cols, valids = expected if expected is not None else _expected(src, indexed + included)
    nrows = len(cols[indexed[0]])
    perm, offs, _ = O.index_rows(cols, indexed, included, NB, {k: v.astype(np.uint8) for k, v in valids.items()} or None)
    phys, conv, spark = _expected_type(kind)
    images = []
    for i, f in enumerate(res.files):
        image = res.host_bytes(i)
        images.append(N.FileImage(data=image))
        lo, hi = int(offs[f.bucket]), int(offs[f.bucket + 1])
        assert f.rows == hi - lo
        pf = pq.ParquetFile(io.BytesIO(image))
        got = pf.read()
        for name in indexed + included:
            vals, valid = S.spark_int64(got.column(name))
            want = cols[name][perm[lo:hi]]
            if name in valids:
                wv = valids[name][perm[lo:hi]]
                assert np.array_equal(np.ones(len(vals), bool) if valid is None else valid, wv)
                want = np.where(wv, want, 0)
            assert np.array_equal(vals, want), (name, f.bucket)
        c = pf.metadata.schema.column(pf.schema_arrow.get_field_index(col))
        assert (c.physical_type, c.converted_type) == (phys, conv)
        if conv == "DECIMAL":
            assert (c.precision, c.scale) == (int(spark[8:-1].split(",")[0]), 2)
        fields = {x["name"]: x["type"] for x in json.loads(pf.metadata.metadata[b"org.apache.spark.sql.parquet.row.metadata"])["fields"]}
        assert fields[col] == spark
        if indexed == [col] and col not in valids:
            for g in range(pf.metadata.num_row_groups):
                st = pf.metadata.row_group(g).column(0).statistics
                assert st is not None and st.has_min_max
    rep = ctx.verify_index(images, [f.bucket for f in res.files], indexed, included, NB)
    assert rep["bucket_mismatches"] == 0 and rep["order_violations"] == 0 and rep["rows"] == nrows


@pytest.mark.parametrize("kind,nullable,extra", SOURCES)
@pytest.mark.parametrize("role", ["key", "included"])
def test_create_index(ctx, kind, nullable, extra, role):
    from hyperspace_b200 import _native as N

    src, image = _source(kind, nullable, extra)
    indexed, included = (["c"], ["v"]) if role == "key" else (["v"], ["c"])
    res, _ = ctx.create_index([N.FileImage(data=image)], indexed, included, NB, output=N.HS_OUT_HOST, job_uuid="st")
    try:
        _check_index(ctx, res, src, kind, indexed, included)
    finally:
        res.free()


def test_decimal9_key_hashes_as_long(ctx):
    """A decimal(9,2) key lands in hashLong's bucket, which differs from hashInt's for this value."""
    from hyperspace_b200 import _native as N

    u = next(x for x in range(12345, 13000)
             if O.np_pmod(O.np_hash_long(np.array([x], np.int64)), NB)[0] != O.np_pmod(O.np_hash_int(np.array([x], np.int32)), NB)[0])
    t = pa.table({"c": pa.array([decimal.Decimal(u).scaleb(-2)], pa.decimal128(9, 2))})
    res, _ = ctx.create_index([N.FileImage(data=_image(t, store_decimal_as_integer=True))], ["c"], [], NB, output=N.HS_OUT_HOST)
    try:
        assert [f.bucket for f in res.files] == [int(O.np_pmod(O.np_hash_long(np.array([u], np.int64)), NB)[0])]
    finally:
        res.free()


def test_two_column_key(ctx):
    from hyperspace_b200 import _native as N

    rng = np.random.default_rng(5)
    t = pa.table({"ts": _values("int96", N_ROWS, rng, True), "d": _values("dec12", N_ROWS, rng, True),
                  "v": pa.array(np.arange(N_ROWS, dtype=np.int64))})
    image = _image(t, use_deprecated_int96_timestamps=True)
    res, _ = ctx.create_index([N.FileImage(data=image)], ["ts", "d"], ["v"], NB, output=N.HS_OUT_HOST)
    try:
        cols = {n: S.spark_int64(pq.read_table(io.BytesIO(image), coerce_int96_timestamp_unit="us").column(n)) for n in ("ts", "d", "v")}
        perm, offs, _ = O.index_rows({n: c[0] for n, c in cols.items()}, ["ts", "d"], ["v"], NB,
                                     {n: c[1].astype(np.uint8) for n, c in cols.items() if c[1] is not None})
        for i, f in enumerate(res.files):
            got = pq.read_table(io.BytesIO(res.host_bytes(i))).column("v").to_numpy()
            assert np.array_equal(got, cols["v"][0][perm[offs[f.bucket]:offs[f.bucket + 1]]])
        rep = ctx.verify_index([N.FileImage(data=res.host_bytes(i)) for i in range(len(res.files))],
                               [f.bucket for f in res.files], ["ts", "d"], ["v"], NB)
        assert rep["bucket_mismatches"] == 0 and rep["order_violations"] == 0
    finally:
        res.free()


def _refused(ctx, image, column, indexed=None):
    from hyperspace_b200 import _native as N

    with pytest.raises(N.HyperspaceGpuError) as e:
        ctx.create_index([N.FileImage(data=image)], indexed or [column], [], NB, output=N.HS_OUT_HOST)
    assert e.value.code == -6  # HS_EUNSUPPORTED
    assert column in str(e.value)


def test_refusals(ctx):
    from hyperspace_b200 import _native as N

    first = S.MICROS_1900 * 1000  # 1900-01-01T00:00:00Z in nanos
    ok = pa.table({"ts": pa.array([first, first + 5], pa.timestamp("ns"))})
    res, _ = ctx.create_index([N.FileImage(data=_image(ok, use_deprecated_int96_timestamps=True))], ["ts"], [], NB, output=N.HS_OUT_HOST)
    res.free()
    early = pa.table({"ts": pa.array([first, first - 1000], pa.timestamp("ns"))})  # 1899-12-31T23:59:59.999999Z
    _refused(ctx, _image(early, use_deprecated_int96_timestamps=True), "ts")
    nanos = pa.table({"tn": pa.array([1, 2], pa.timestamp("ns"))})
    _refused(ctx, _image(nanos, version="2.6", coerce_timestamps=None), "tn")
    wide = pa.table({"d19": pa.array([decimal.Decimal(1)], pa.decimal128(19, 0))})
    _refused(ctx, _image(wide), "d19")
    big = pa.table({"ms": pa.array([2**62], pa.timestamp("ms"))})
    _refused(ctx, _image(big, coerce_timestamps="ms"), "ms")


def _files_of(res):
    from hyperspace_b200 import _native as N

    return [N.FileImage(data=res.host_bytes(i)) for i in range(len(res.files))], [f.bucket for f in res.files]


def test_filters(ctx):
    from hyperspace_b200 import _native as N

    rng = np.random.default_rng(9)
    n = N_ROWS
    t = pa.table({"d": _values("dec9", n, rng, True), "ts": _values("int96", n, rng, False), "v": pa.array(np.arange(n, dtype=np.int64))})
    image = _image(t, use_deprecated_int96_timestamps=True)
    back = pq.read_table(io.BytesIO(image), coerce_int96_timestamp_unit="us")
    d, dvalid = S.spark_int64(back.column("d"))
    ts, _ = S.spark_int64(back.column("ts"))
    v = back.column("v").to_numpy()
    dv = np.ones(n, bool) if dvalid is None else dvalid
    for key, inc in ((["d"], ["ts", "v"]), (["ts"], ["d", "v"])):
        res, _ = ctx.create_index([N.FileImage(data=image)], key, inc, NB, output=N.HS_OUT_HOST)
        files, _ = _files_of(res)
        mid = int(np.median(ts))
        cases = [  # (predicates, numpy mask)
            ([("d", decimal.Decimal("12.345"), False, None, False)], dv & (d * 10 >= 12345)),      # more digits than the column
            ([("d", decimal.Decimal("12.345"), True, None, False)], dv & (d * 10 > 12345)),
            ([("d", None, False, decimal.Decimal("-7.1"), True)], dv & (d < -710)),               # fewer digits
            ([("d", 10, True, 10_000, False)], dv & (d > 1000) & (d <= 1_000_000)),               # integers on a decimal
            ([("d", decimal.Decimal("0.50"), False, decimal.Decimal("0.50"), False)], dv & (d == 50)),
            ([("d", decimal.Decimal("99999999999999"), False, None, False)], np.zeros(n, bool)),  # above every value
            ([("ts", mid, False, None, False)], ts >= mid),
            ([("ts", datetime.datetime(1990, 1, 1), True, datetime.datetime(2000, 1, 1), False)],
             (ts > N.timestamp_micros(datetime.datetime(1990, 1, 1))) & (ts <= N.timestamp_micros(datetime.datetime(2000, 1, 1)))),
            ([("ts", mid, True, None, False), ("d", decimal.Decimal("-100.005"), False, decimal.Decimal("100.005"), True)],
             (ts > mid) & dv & (d >= -10000) & (d <= 10000)),
        ]
        try:
            for preds, mask in cases:
                b, _ = ctx.filter_scan_where(files, key[0], ["v"], preds, sorted_on_key=True)
                got = np.sort(b.column("v").copy())
                b.free()
                assert np.array_equal(got, np.sort(v[mask])), (key, preds)
            for col_, lit in (("d", 1.5), ("ts", 1.5), ("ts", decimal.Decimal("1.5"))):
                with pytest.raises(N.HyperspaceGpuError) as e:
                    ctx.filter_scan_where(files, key[0], ["v"], [(col_, lit, False, None, False)], sorted_on_key=True)
                assert e.value.code == -6 and col_ in str(e.value)
        finally:
            res.free()


def test_joins(ctx):
    """Joins on a timestamp key and on (timestamp, decimal) keys, with null keys, a filter below one side and two files per
    bucket on the left; rows equal the oracle's merge join."""
    from hyperspace_b200 import _native as N

    rng = np.random.default_rng(3)

    def table(n, seed_shift):
        r = np.random.default_rng(seed_shift)
        ts = (r.integers(0, 300, n) * 1_000_000_000).astype(np.int64)  # few distinct instants: many matches
        mask = r.random(n) < 0.05
        d = r.integers(-3, 4, n)
        return pa.table({"ts": pa.array(ts, pa.timestamp("ns"), mask=mask),
                         "d": pa.array([decimal.Decimal(int(x)).scaleb(-2) for x in d], pa.decimal128(12, 2)),
                         "v": pa.array(np.arange(n, dtype=np.int64) + seed_shift * 100000)})

    left_parts = [table(3000, 1), table(2000, 2)]
    right = table(2500, 3)
    for keys in (["ts"], ["ts", "d"]):
        lres = [ctx.create_index([N.FileImage(data=_image(p, use_deprecated_int96_timestamps=True))], keys, ["v"], NB,
                                 output=N.HS_OUT_HOST)[0] for p in left_parts]
        rres = ctx.create_index([N.FileImage(data=_image(right, use_deprecated_int96_timestamps=True))], keys, ["v"], NB, output=N.HS_OUT_HOST)[0]
        try:
            lf, lb = [], []
            for r in lres:
                f, b = _files_of(r)
                lf += f
                lb += b
            rf, rb = _files_of(rres)
            preds = [("v", 300, False, None, False)]
            batch, _ = ctx.bucket_join_where(lf, lb, rf, rb, NB, keys, keys, ["v"], ["v"], right_predicates=preds)
            got = sorted(zip(batch.columns[0][1].tolist(), batch.columns[1][1].tolist()))
            batch.free()

            def cols(tab):
                out, val = {}, {}
                for nm in keys + ["v"]:
                    x, m = S.spark_int64(pq.read_table(io.BytesIO(_image(tab))).column(nm))
                    out[nm] = x
                    if m is not None:
                        val[nm] = m
                return out, val

            L = [cols(p) for p in left_parts]
            lcols = {k: np.concatenate([c[0][k] for c in L]) for k in keys + ["v"]}
            lval = {k: np.concatenate([c[1].get(k, np.ones(len(c[0][k]), bool)) for c in L]) for k in keys}
            rcols, rval = cols(right)
            li, ri = J.bucket_join(lcols, rcols, NB, keys, keys, right_predicates=preds, left_valids=lval, right_valids=rval)
            want = sorted(zip(lcols["v"][li].tolist(), rcols["v"][ri].tolist()))
            assert got == want and len(got) > 0
        finally:
            for r in lres + [rres]:
                r.free()
    # a decimal(12,2) key never pairs with an int64 key, nor a decimal(9,2) with an int32
    a = pa.table({"k": pa.array([decimal.Decimal("1.00")], pa.decimal128(9, 2))})
    b = pa.table({"k": pa.array([100], pa.int32())})
    ra = ctx.create_index([N.FileImage(data=_image(a, store_decimal_as_integer=True))], ["k"], [], NB, output=N.HS_OUT_HOST)[0]
    rb_ = ctx.create_index([N.FileImage(data=_image(b))], ["k"], [], NB, output=N.HS_OUT_HOST)[0]
    try:
        (fa, ba), (fb, bb) = _files_of(ra), _files_of(rb_)
        with pytest.raises(N.HyperspaceGpuError) as e:
            ctx.bucket_join_where(fa, ba, fb, bb, NB, ["k"], ["k"], ["k"], ["k"])
        assert e.value.code == -6
    finally:
        ra.free()
        rb_.free()


def test_hyperspace_api_int96(tmp_path):
    """The reference README flow over a table with an INT96 column: answers equal with and without the index."""
    from hyperspace_b200.hyperspace import Hyperspace
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import HyperspaceSession, col

    src = tmp_path / "events"
    src.mkdir()
    rng = np.random.default_rng(11)
    for i in range(2):
        t = pa.table({"ts": _values("int96", 4000, rng, False), "amount": _values("dec12", 4000, rng, False),
                      "id": pa.array(np.arange(4000, dtype=np.int64) + i * 4000)})
        pq.write_table(t, src / f"part-{i}.parquet", use_deprecated_int96_timestamps=True)
    s = HyperspaceSession({"spark.hyperspace.system.path": str(tmp_path / "indexes"), "spark.hyperspace.index.numBuckets": "8"})
    hs = Hyperspace(s)
    df = s.read.parquet(str(src))
    assert dict(df.plan.schema)["ts"] == "timestamp" and dict(df.plan.schema)["amount"] == "decimal(12,2)"
    hs.createIndex(df, IndexConfig("ev", ["ts"], ["amount", "id"]))
    q = lambda: df.filter((col("ts") >= datetime.datetime(1980, 1, 1)) & (col("ts") < datetime.datetime(2050, 6, 1))) \
        .select("ts", "amount", "id").collect()
    s.disableHyperspace()
    plain = q()
    s.enableHyperspace()
    assert "Hyperspace" in df.filter(col("ts") >= datetime.datetime(1980, 1, 1)).select("ts", "id").explain()
    indexed = q()
    o1, o2 = np.argsort(plain["id"]), np.argsort(indexed["id"])
    for c in ("ts", "amount", "id"):
        assert plain[c][o1].tolist() == indexed[c][o2].tolist()
    assert plain["ts"].dtype == np.dtype("datetime64[us]") and isinstance(plain["amount"][0], decimal.Decimal)
    assert len(plain["id"]) > 0
    s.stop()
