"""The LZ4 page decoder's per-stream code (hyperspace_b200/csrc/lz4_block.h) built as host code and compared with pyarrow:
every stream of tests/lz4_corpus.py must decode to its data, every damaged one must fail the check it was built to hit,
and on every seeded mutation of a valid stream the decoder must accept exactly when pyarrow accepts with the exact
length, with the same output.  The one intended difference: pyarrow's LZ4 accepts a match offset of 0 (which the block
format declares invalid, and which it decodes as zeros); the decoder refuses it.  The driver is built with
AddressSanitizer when the host compiler supports it, so a read or write outside a stream or its output buffer fails the
test."""
import os
import shutil
import struct
import subprocess

import pytest

import lz4_corpus as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def native(tmp_path_factory):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not on PATH")
    d = tmp_path_factory.mktemp("lz4")
    src = os.path.join(ROOT, "tests", "native", "lz4.cu")
    base = ["nvcc", "-std=c++17", "-O1", "-g", "-Wno-deprecated-gpu-targets", "-o", str(d / "lz4"), src]
    try:  # AddressSanitizer: any access outside a stream or its output is an error
        subprocess.check_call(base + ["-Xcompiler", "-fsanitize=address,-fno-omit-frame-pointer"],
                              stderr=subprocess.DEVNULL)
        asan = subprocess.run([str(d / "lz4")], capture_output=True).returncode == 2  # usage error, sanitizer runtime loaded
    except subprocess.CalledProcessError:
        asan = False
    if not asan:
        subprocess.check_call(base)
    return str(d / "lz4")


def run(native, tmp_path, cases):
    """[(codec, stream, uncompressed length)] -> [(error, output)]"""
    (tmp_path / "in").write_bytes(L.records(cases))
    subprocess.check_call([native, str(tmp_path / "in"), str(tmp_path / "out")])
    raw, p, out = (tmp_path / "out").read_bytes(), 0, []
    for _ in cases:
        e, n = struct.unpack_from("<II", raw, p)
        p += 8
        out.append((e, raw[p:p + n]))
        p += n
    assert p == len(raw)
    return out


def test_valid_streams_decode_bit_identically(native, tmp_path):
    cases = L.valid()
    names = {c[0] for c in cases}
    assert {"offset65535", "literals525", "match529", "match_from_first_byte", "short_path_lit14_match18_last0",
            "hadoop_one_group_several_chunks", "hadoop_raw_fallback_plausible_header", "size0_random", "big1.5MB/l12"} <= names
    for name, codec, stream, data in cases:  # the corpus itself: pyarrow takes every raw block at its exact length
        if codec == L.LZ4_RAW:
            assert L.pyarrow_accepts(stream, len(data)) and L.pyarrow_decode(stream, len(data)) == data, name
    res = run(native, tmp_path, [(c, s, len(d)) for _, c, s, d in cases])
    bad = [(name, e) for (name, _, _, data), (e, out) in zip(cases, res) if e != 0 or out != data]
    assert not bad, bad[:10]


def test_pyarrow_levels_differ():
    data = L.inputs()["T_v1"]
    assert len({len(L.compress(data, lv)) for lv in (1, 3, 9, 12)}) > 1


def test_damaged_streams_fail_their_check(native, tmp_path):
    cases = L.damaged()
    assert {c[4] for c in cases} == set(range(1, 7))  # every named check
    res = run(native, tmp_path, [(c, s, n) for _, c, s, n, _ in cases])
    wrong = [(name, want, e) for (name, _, _, _, want), (e, _) in zip(cases, res) if e != want]
    assert not wrong, wrong
    for name, codec, stream, n, check in cases:  # pyarrow refuses them too, but for offset 0
        if codec == L.LZ4_RAW:
            assert L.pyarrow_accepts(stream, n) == (check == L.OFFSET_ZERO), name


def test_mutations_agree_with_pyarrow(native, tmp_path):
    cases = L.mutations()
    assert len(cases) == 2000
    res = run(native, tmp_path, [(L.LZ4_RAW, s, n) for _, s, n in cases])
    disagree, accepted = [], 0
    for (name, stream, n), (e, out) in zip(cases, res):
        theirs = L.pyarrow_accepts(stream, n)
        if theirs and e == L.OFFSET_ZERO:
            continue
        if (e == 0) != theirs or (theirs and out != L.pyarrow_decode(stream, n)):
            disagree.append((name, e, theirs))
        accepted += theirs
    assert not disagree, disagree[:10]
    assert 200 < accepted < 1800  # both verdicts are well represented
