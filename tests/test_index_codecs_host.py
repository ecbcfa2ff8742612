"""The index page compressors' per-stream code (hyperspace_b200/csrc/deflate.h and the encoder half of lz4_block.h) built
as host code, under AddressSanitizer when the host compiler supports it: the length-limited Huffman builder, the gzip
member's header, sync flush and trailer, the worst-case sizes, and the LZ4 sequence encoder under the end-of-block rules."""
import os
import random
import shutil
import struct
import subprocess
import zlib

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [0, 1, 4, 5, 12, 13, 65535, 65536, 65537, 1 << 20 | 4321]


@pytest.fixture(scope="module")
def native(tmp_path_factory):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not on PATH")
    d = tmp_path_factory.mktemp("index_codecs")
    src = os.path.join(ROOT, "tests", "native", "index_codecs.cu")
    exe = str(d / "index_codecs")
    base = ["nvcc", "-std=c++17", "-O1", "-g", "-Wno-deprecated-gpu-targets", "-o", exe, src]
    try:
        subprocess.check_call(base + ["-Xcompiler", "-fsanitize=address,-fno-omit-frame-pointer"], stderr=subprocess.DEVNULL)
        asan = subprocess.run([exe], capture_output=True).returncode == 2
    except subprocess.CalledProcessError:
        asan = False
    if not asan:
        subprocess.check_call(base)
    return exe


def run(native, tmp_path, cmd, data: bytes) -> bytes:
    (tmp_path / "in").write_bytes(data)
    subprocess.check_call([native, cmd, str(tmp_path / "in"), str(tmp_path / "out")])
    return (tmp_path / "out").read_bytes()


def lengths(native, tmp_path, cases):
    """[(frequencies, limit)] -> [code lengths]"""
    rec = b"".join(struct.pack(f"<II{len(f)}I", len(f), limit, *f) for f, limit in cases)
    raw, out, p = run(native, tmp_path, "lengths", rec), [], 0
    for f, _ in cases:
        out.append(list(raw[p:p + len(f)]))
        p += len(f)
    assert p == len(raw)
    return out


def fib(n):
    a, b, out = 1, 1, []
    for _ in range(n):
        out.append(a)
        a, b = b, a + b
    return out


def histograms():
    rng = random.Random(7)
    return [
        ("fibonacci30/286", fib(30) + [0] * 256, 15),
        ("fibonacci25/all286", fib(25) + [1] * 261, 15),
        ("fibonacci19/cl", fib(19), 7),
        ("one symbol", [0] * 100 + [5] + [0] * 185, 15),
        ("one symbol/dist", [0] * 29 + [9], 15),
        ("none/dist", [0] * 30, 15),
        ("two symbols", [0] * 7 + [1000, 1] + [0] * 277, 15),
        ("all 286 equal", [3] * 286, 15),
        ("random", [rng.randrange(0, 65537) for _ in range(286)], 15),
        ("geometric/cl", [1 << i for i in range(19)], 7),
    ]


def test_huffman_lengths_limited_complete_deterministic(native, tmp_path):
    cases = histograms()
    got = lengths(native, tmp_path, [(f, limit) for _, f, limit in cases])
    again = lengths(native, tmp_path, [(f, limit) for _, f, limit in cases])
    assert got == again
    for (name, freq, limit), lens in zip(cases, got):
        assert max(lens) <= limit, name
        used = [l for l in lens if l]
        assert len(used) >= 2, name
        assert sum(2.0 ** -l for l in used) == 1.0, name  # complete: Kraft sum 1
        for s, f in enumerate(freq):  # every symbol that occurs has a code; more frequent never longer
            if f:
                assert lens[s] > 0, (name, s)
        occurring = sorted((f, s) for s, f in enumerate(freq) if f)
        for (f1, s1), (f2, s2) in zip(occurring, occurring[1:]):
            if f1 < f2:
                assert lens[s1] >= lens[s2], (name, s1, s2)
    fib_lens = got[0]
    assert max(fib_lens) == 15  # the unlimited code would be 29 deep


def test_huffman_lengths_are_optimal_when_not_limited(native, tmp_path):
    """Without the cap the builder is Huffman's: its cost equals a reference Huffman construction's."""
    import heapq
    rng = random.Random(11)
    cases = [[rng.randrange(100, 1000) for _ in range(n)] for n in (2, 3, 19, 30, 286)]  # no code deeper than 15
    got = lengths(native, tmp_path, [(f, 15) for f in cases])
    for freq, lens in zip(cases, got):
        h = list(freq)
        heapq.heapify(h)
        cost = 0
        while len(h) > 1:
            a, b = heapq.heappop(h), heapq.heappop(h)
            cost += a + b
            heapq.heappush(h, a + b)
        assert sum(f * l for f, l in zip(freq, lens)) == cost


@pytest.mark.parametrize("size", SIZES)
def test_gzip_member_of_stored_fragments(native, tmp_path, size):
    data = random.Random(size).randbytes(size // 2) + bytes(size - size // 2)
    raw = run(native, tmp_path, "gzip", data)
    bound, err = struct.unpack_from("<QI", raw)
    member = raw[12:]
    assert err == 0  # inflate.h gives the input back, CRC-32 and ISIZE checked
    assert zlib.decompress(member, wbits=31) == data
    assert member[:10] == bytes([0x1F, 0x8B, 8, 0, 0, 0, 0, 0, 0, 0xFF])
    assert member[-10:-8] == b"\x03\x00"
    assert len(member) == bound  # the stored form is the worst case, and the bound is exact for it


@pytest.mark.parametrize("size", SIZES)
def test_lz4_sequence_encoder(native, tmp_path, size):
    pa = pytest.importorskip("pyarrow")
    rng = random.Random(size)
    data = bytearray()
    while len(data) < size:  # runs, repeats at near and far offsets, and noise
        k = rng.randrange(4)
        if k == 0 or not data:
            data += rng.randbytes(rng.randrange(1, 40))
        elif k == 1:
            data += bytes([rng.randrange(256)]) * rng.randrange(1, 300)
        else:
            off = rng.randrange(1, min(len(data), 70000) + 1)
            start = len(data) - off
            data += bytes(data[start:start + rng.randrange(4, 200)])
    data = bytes(data[:size])
    raw = run(native, tmp_path, "lz4", data)
    bound, err = struct.unpack_from("<QI", raw)
    stream = raw[12:]
    assert err == 0  # lz4_block.h decodes it, Hadoop framing, at exact capacities
    assert len(stream) <= bound
    codec = pa.Codec("lz4_raw")
    p, back = 0, b""
    while p < len(stream):  # one group of one chunk per 64 KB; every block is a complete LZ4 block
        u, c = struct.unpack_from(">II", stream, p)
        blk = stream[p + 8:p + 8 + c]
        assert u <= 65536
        if u >= 13:
            # the end-of-block rules: the last sequence carries at least the last 5 bytes as literals
            assert blk[-5:] == data[len(back) + u - 5:len(back) + u]
        back += codec.decompress(blk, decompressed_size=u).to_pybytes()
        p += 8 + c
    assert back == data
