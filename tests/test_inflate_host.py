"""The GZIP page decoder's per-stream code (hyperspace_b200/csrc/inflate.h) built as host code and compared bit for bit
with Python's zlib: every stream of tests/gzip_corpus.py must decode to its input, and every damaged one must fail the
check it was built to hit.  The driver is built with AddressSanitizer when the host compiler supports it, so a read or
write outside a stream or its output buffer fails the test."""
import os
import shutil
import struct
import subprocess
import zlib

import pytest

import gzip_corpus as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def native(tmp_path_factory):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not on PATH")
    d = tmp_path_factory.mktemp("inflate")
    src = os.path.join(ROOT, "tests", "native", "inflate.cu")
    base = ["nvcc", "-std=c++17", "-O1", "-g", "-Wno-deprecated-gpu-targets", "-o", str(d / "inflate"), src]
    try:  # AddressSanitizer: any access outside a stream or its output is an error
        subprocess.check_call(base + ["-Xcompiler", "-fsanitize=address,-fno-omit-frame-pointer"],
                              stderr=subprocess.DEVNULL)
        asan = subprocess.run([str(d / "inflate")], capture_output=True).returncode == 2  # usage error, sanitizer runtime loaded
    except subprocess.CalledProcessError:
        asan = False
    if not asan:
        subprocess.check_call(base)
    return str(d / "inflate")


def run(native, tmp_path, cases):
    """[(stream, uncompressed length)] -> [(error, output)]"""
    (tmp_path / "in").write_bytes(G.records(cases))
    subprocess.check_call([native, str(tmp_path / "in"), str(tmp_path / "out")])
    raw, p, out = (tmp_path / "out").read_bytes(), 0, []
    for _ in cases:
        e, n = struct.unpack_from("<II", raw, p)
        p += 8
        out.append((e, raw[p:p + n]))
        p += n
    assert p == len(raw)
    return out


def test_valid_streams_match_zlib(native, tmp_path):
    cases = G.valid()
    names = {c[0] for c in cases}
    assert {"run258_d32768", "dist_single_code", "dist_empty", "members3", "flags31", "skewed15/l9"} <= names
    for name, stream, data in cases:  # the corpus itself: what zlib (or gzip's multi-member rule) makes of each stream
        d = zlib.decompressobj(31)
        got, rest = d.decompress(stream), d.unused_data
        while rest:
            d = zlib.decompressobj(31)
            got += d.decompress(rest)
            rest = d.unused_data
        assert got == data, name
    res = run(native, tmp_path, [(s, len(d)) for _, s, d in cases])
    bad = [(name, e) for (name, _, data), (e, out) in zip(cases, res) if e != 0 or out != data]
    assert not bad, bad[:10]


def test_sync_and_full_flush_write_empty_stored_blocks():
    s = G._flushed(b"abc" * 1000, zlib.Z_SYNC_FLUSH)
    assert b"\x00\x00\xff\xff" in s  # the empty stored block a flush ends with


def test_damaged_streams_fail_their_check(native, tmp_path):
    cases = G.damaged()
    res = run(native, tmp_path, [(s, n) for _, s, n, _ in cases])
    wrong = [(name, want, e) for (name, _, _, want), (e, _) in zip(cases, res) if e != want]
    assert not wrong, wrong
