"""Boolean included columns without a GPU: the page restatement of bool_pages.py against pages pyarrow writes (PLAIN and
RLE, v1 and v2), and the Python layer (schema JSON, the refusal of a boolean indexed column, refresh and Hybrid Scan
planning with boolean columns)."""
import os

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import bool_pages as B
import parquet_shapes as S


def _bools(n, seed, null_frac=0.0):
    rng = np.random.default_rng(seed)
    v = rng.random(n) < 0.5
    valid = rng.random(n) >= null_frac if null_frac else None
    return v, valid


@pytest.mark.parametrize("n", [0, 1, 7, 8, 9, 63, 64, 65, 4097])
def test_null_free_body(n):
    v, _ = _bools(n, n)
    body = B.page_body(v)
    defs = S.varint(n << 1) + b"\x01"
    assert body[:4] == len(defs).to_bytes(4, "little") and body[4:4 + len(defs)] == defs
    vals = body[4 + len(defs):]
    assert len(vals) == (n + 7) // 8
    assert np.array_equal(np.unpackbits(np.frombuffer(vals, np.uint8), bitorder="little")[:n].astype(bool), v)
    if n % 8:
        assert vals[-1] >> (n % 8) == 0  # padding bits zero


@pytest.mark.parametrize("n", [1, 9, 100, 4097])
def test_nullable_body(n):
    v, valid = _bools(n, n + 1, 0.3)
    body = B.page_body(v, valid)
    dl = int.from_bytes(body[:4], "little")
    groups = (n + 7) // 8
    got_valid = B.read_hybrid(body, 4, 4 + dl, 1, n)[0].astype(bool)
    assert np.array_equal(got_valid, valid)
    assert dl == len(S.varint((groups << 1) | 1)) + groups
    vals = body[4 + dl:]
    m = int(valid.sum())
    assert len(vals) == (m + 7) // 8
    assert np.array_equal(np.unpackbits(np.frombuffer(vals, np.uint8), bitorder="little")[:m].astype(bool), v[valid])


def test_all_null_body():
    body = B.page_body(np.zeros(10, bool), np.zeros(10, bool))
    assert body == (3).to_bytes(4, "little") + S.varint(5) + b"\x00\x00"  # no value bytes


@pytest.mark.parametrize("encoding", ["PLAIN", "RLE"])
@pytest.mark.parametrize("version", ["1.0", "2.0"])
@pytest.mark.parametrize("null_frac", [0.0, 0.2])
@pytest.mark.parametrize("codec", ["NONE", "SNAPPY"])
def test_restatement_against_pyarrow_pages(tmp_path, encoding, version, null_frac, codec):
    n = 30_000
    v, valid = _bools(n, 7, null_frac)
    arr = pa.array(v, mask=None if valid is None else ~valid)
    path = str(tmp_path / "b.parquet")
    pq.write_table(pa.table({"b": arr}), path, use_dictionary=False, column_encoding={"b": encoding}, compression=codec,
                   data_page_version=version, data_page_size=1 << 12)
    pages = B.data_pages(open(path, "rb").read(), "b")
    assert len(pages) > 1 and {p["enc"] for p in pages} == {S.PLAIN if encoding == "PLAIN" else S.RLE}
    assert all(p["v2"] == (version == "2.0") for p in pages)
    want = pq.read_table(path).column("b").combine_chunks()
    got_valid = np.concatenate([p["valid"] for p in pages])
    got_vals = np.concatenate([p["values"] for p in pages])
    assert np.array_equal(got_valid, np.asarray(want.is_valid()))
    assert np.array_equal(got_vals, np.asarray(want.drop_null()).astype(bool))
    for p in pages:
        if encoding == "PLAIN":  # the value bytes are exactly the restatement's (pyarrow pads with zero bits too)
            assert p["body"][p["values_at"]:] == B.packbits(p["values"])


def test_read_hybrid_refuses_runs_past_the_stream():
    with pytest.raises(ValueError):
        B.read_hybrid(bytes([(10 << 1) | 1, 0xff, 0xff]), 0, 3, 1, 16)
    with pytest.raises(ValueError):
        B.read_hybrid(bytes([32 << 1]), 0, 1, 1, 32)
    v, _ = B.read_hybrid(bytes([0x80, 0x01, 0x01]), 0, 3, 1, 64)
    assert v.tolist() == [1] * 64


# ---- Python layer ----------------------------------------------------------------------------------------------------
@pytest.fixture()
def env(tmp_path):
    from hyperspace_b200.hyperspace import Hyperspace
    from hyperspace_b200.session import HyperspaceSession

    s = HyperspaceSession({"spark.hyperspace.system.path": str(tmp_path / "indexes"), "spark.hyperspace.index.numBuckets": "4"})
    yield s, Hyperspace(s), tmp_path
    s.stop()


def _write(tmp_path, name, n, seed):
    os.makedirs(tmp_path / "t", exist_ok=True)
    v, valid = _bools(n, seed, 0.1)
    pq.write_table(pa.table({"k": pa.array(np.arange(n, dtype=np.int64)), "flag": pa.array(v, mask=~valid)}),
                   str(tmp_path / "t" / name))


def test_schema_reads_boolean(tmp_path):
    from hyperspace_b200.session import read_parquet_schema

    _write(tmp_path, "a.parquet", 10, 1)
    assert dict(read_parquet_schema(str(tmp_path / "t" / "a.parquet")))["flag"] == "boolean"


@pytest.mark.parametrize("indexed", [["flag"], ["k", "flag"], ["FLAG"]])
def test_boolean_indexed_column_refused_before_anything_is_written(env, indexed):
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.log_entry import HyperspaceException

    s, hs, tmp = env
    _write(tmp, "a.parquet", 10, 1)
    with pytest.raises(HyperspaceException, match="'%s' is boolean" % indexed[-1]):
        hs.createIndex(s.read.parquet(str(tmp / "t")), IndexConfig("idx", indexed, []))
    assert not os.path.exists(tmp / "indexes" / "idx")


def test_log_entry_schema_carries_boolean(env):
    from hyperspace_b200.hyperspace import CreateAction
    from hyperspace_b200.index_config import IndexConfig

    s, hs, tmp = env
    _write(tmp, "a.parquet", 10, 1)
    lm, dm = hs._paths("idx")
    act = CreateAction(s, s.read.parquet(str(tmp / "t")), IndexConfig("idx", ["k"], ["flag"]), lm, dm)
    act.validate()
    fields = act.log_entry().schema["fields"]
    assert [(f["name"], f["type"]) for f in fields] == [("k", "long"), ("flag", "boolean")]


def test_refresh_and_hybrid_scan_planning_with_booleans(env):
    """An index over a boolean included column serves a query projecting it; an appended file makes a Hybrid Scan."""
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import col
    import hyperspace_b200.hyperspace as H
    from hyperspace_b200 import log_entry as LE

    s, hs, tmp = env
    _write(tmp, "a.parquet", 100, 1)
    calls = []
    # the build itself needs the GPU: the files it would write are left out, the log is written as for any build
    orig = H._DataAction._write
    H._DataAction._write = lambda self, files, indexed, included, *a, **k: calls.append((list(indexed), list(included)))
    try:
        hs.createIndex(s.read.parquet(str(tmp / "t")), IndexConfig("idx", ["k"], ["flag"]))
        assert calls == [(["k"], ["flag"])]
        _write(tmp, "b.parquet", 50, 2)
        hs.refreshIndex("idx", "incremental")
        assert calls[-1] == (["k"], ["flag"])
    finally:
        H._DataAction._write = orig
    e = LE.IndexLogManager(str(tmp / "indexes" / "idx")).get_latest_stable_log()
    assert [f["type"] for f in e.schema["fields"]] == ["long", "boolean"]
    _write(tmp, "c.parquet", 20, 3)
    s.enableHyperspace()
    s.conf.set("spark.hyperspace.index.hybridscan.enabled", True)
    q = s.read.parquet(str(tmp / "t")).filter(col("k") <= 5).select("k", "flag")
    plan = q.explain()
    assert "Name: idx" in plan and "hybridScan(appended=1" in plan
