"""ClickHouse INSERT-body compressor, CPU side:
* the restatement's strict LZ4 decoder (tests/clickhouse_lz4_ref.py) pinned against pyarrow's lz4_raw codec (liblz4, an
  independent implementation): pyarrow-compressed random, structured and run-heavy inputs decode to the input, and
  hand-built edge blocks (length extensions at 15 and 15 + 255, overlapping offset-1 matches, offset 65535, blocks of
  0-13 bytes) decode the same through both; blocks that break the end-of-block rules are rejected;
* the device helpers (etl_b200/csrc/clickhouse_lz4.cuh) compiled for the host (tests/emul/host_ch_lz4.cpp): CityHash128
  v1.0.2 against the restatement over every length 0-1024, 128 KiB +- 3 and seeded lengths up to 64 KiB + 25, the
  sequence writer over seeded literal and match lengths, the block framing and the block size;
* the greedy INSERT split on hand-worked offsets.
No CityHash128 v1.0.2 known-answer vector is available offline: the checksum rests on the restatement and the
host-compiled device code agreeing (DESIGN.md §5, unpinned)."""
import ctypes as C
import os
import random
import subprocess
import sys
import tempfile

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.normpath(os.path.join(HERE, ".."))
sys.path.insert(0, HERE)
import clickhouse_lz4_ref as R  # noqa: E402

pa = pytest.importorskip("pyarrow")
if not pa.Codec.is_available("lz4_raw"):
    pytest.skip("pyarrow without lz4_raw", allow_module_level=True)
CODEC = pa.Codec("lz4_raw")


def pa_compress(b):
    return CODEC.compress(b, asbytes=True)


def pa_decompress(b, n):
    return CODEC.decompress(b, decompressed_size=n, asbytes=True)


def rowbinary_like(rng, n):
    """rows of a RowBinary-ish table: small ints, repeated status text, a counter, an LSN"""
    out = bytearray()
    i = 0
    while len(out) < n:
        out += i.to_bytes(8, "little") + bytes([0, 6]) + rng.choice([b"INSERT", b"UPDATE", b"DELETE"])
        t = rng.choice([b"active", b"inactive", b"pending review", b"x" * rng.randrange(40)])
        out += bytes([len(t)]) + t + rng.randrange(1 << 20).to_bytes(4, "little") + (1000 + i // 7).to_bytes(8, "little")
        i += 1
    return bytes(out[:n])


def inputs():
    rng = random.Random(11)
    yield "random", bytes(rng.randrange(256) for _ in range(70000))
    yield "structured", rowbinary_like(rng, 100000)
    yield "zeros", bytes(65536)
    yield "runs", b"".join(bytes([rng.randrange(4)]) * rng.randrange(1, 600) for _ in range(400))
    yield "period3", b"abc" * 20000
    for n in range(0, 40):
        yield f"short{n}", bytes(rng.randrange(3) for _ in range(n))


# ------------------------------------------------------------------------------------------------ decoder vs liblz4
@pytest.mark.parametrize("name,data", list(inputs()), ids=lambda x: x if isinstance(x, str) else "")
def test_decoder_reads_liblz4_blocks(name, data):
    z = pa_compress(data)
    assert R.lz4_decode(z, len(data)) == data


TAIL = b"twelve bytes"                  # closes a block after a match: 12 literals satisfy both end-of-block rules


def edge_blocks():
    """(name, block, expected bytes)"""
    rng = random.Random(12)
    lit = lambda n: bytes(rng.randrange(256) for _ in range(n))  # noqa: E731
    out = []
    for n in (14, 15, 16, 269, 270, 271, 524, 525):                            # literal-length extensions
        a = lit(n)
        out.append((f"literals{n}", R.sequence(a), a))
    for ml in (4, 18, 19, 20, 273, 274, 275, 529, 1000):                     # match-length extensions
        a = lit(8)
        want = a + (a * (ml // 8 + 1))[:ml] + TAIL
        out.append((f"match{ml}", R.sequence(a, 8, ml) + R.sequence(TAIL), want))
    for ml in (4, 5, 15, 19, 300):                                           # offset 1: an overlapping run
        want = b"z" * (1 + ml) + TAIL
        out.append((f"offset1_{ml}", R.sequence(b"z", 1, ml) + R.sequence(TAIL), want))
    a = lit(65535)                                                            # offset 65535
    want = a + a[:40] + TAIL
    out.append(("offset65535", R.sequence(a, 65535, 40) + R.sequence(TAIL), want))
    for n in range(0, 14):                                                    # short blocks: literals only
        a = lit(n)
        out.append((f"short{n}", R.sequence(a), a))
    return out


@pytest.mark.parametrize("name,block,want", edge_blocks(), ids=lambda x: x if isinstance(x, str) else "")
def test_edge_blocks_agree_with_liblz4(name, block, want):
    assert pa_decompress(block, len(want)) == want
    assert R.lz4_decode(block, len(want)) == want
    assert R.lz4_decode(pa_compress(want), len(want)) == want


@pytest.mark.parametrize("name,block,size", [   # size: the output the block claims; 0: liblz4 accepts it
    ("offset0", bytes([0x80]) + b"abcdefgh" + b"\x00\x00" + R.sequence(b"0123456789abc"), 0),
    ("offset_past_output", R.sequence(b"abcd", 5, 4) + R.sequence(b"0123456789abc"), 21),
    ("last_sequence_match", R.sequence(b"abcd", 4, 20), 24),
    ("match_in_last_12", R.sequence(b"abcdefgh", 4, 4) + R.sequence(b"012345"), 18),
    ("match_ends_in_last_5", R.sequence(b"abcdefghijklmnop", 4, 12) + R.sequence(b"0123"), 32),
    ("truncated_literals", R.sequence(b"abcdefgh")[:-1], 8),
    ("truncated_offset", R.sequence(b"abcdefgh", 4, 4)[:-1], 16),
    ("empty_input", b"", 0),
], ids=lambda x: x if isinstance(x, str) else "")
def test_decoder_rejects_broken_blocks(name, block, size):
    with pytest.raises(R.Lz4Error):
        R.lz4_decode(block)
    if size:                                           # liblz4's safe decoder, given the exact size, rejects it too
        with pytest.raises(OSError):
            pa_decompress(block, size)


def test_decoder_accepts_the_limits():
    """a match starting exactly 12 bytes before the end and ending exactly 5 before it is valid"""
    blk = R.sequence(b"abcd", 4, 7) + R.sequence(b"01234")
    assert R.lz4_decode(blk) == b"abcd" + b"abcdabc" + b"01234"
    assert pa_decompress(blk, 16) == b"abcdabcdabc01234"


def test_decoder_checks_the_declared_size():
    with pytest.raises(R.Lz4Error):
        R.lz4_decode(R.sequence(b"abc"), 4)


# ------------------------------------------------------------------------------------------------ split
def test_split_known_answers():
    off = [0, 10, 20, 30, 40, 50]                    # five rows of 10 bytes
    assert R.split(off, 0, 5, 1) == [0, 1, 2, 3, 4, 5]
    assert R.split(off, 0, 5, 10) == [0, 1, 2, 3, 4, 5]
    assert R.split(off, 0, 5, 11) == [0, 2, 4, 5]    # the row that crosses the limit stays in the INSERT
    assert R.split(off, 0, 5, 20) == [0, 2, 4, 5]
    assert R.split(off, 0, 5, 21) == [0, 3, 5]
    assert R.split(off, 0, 5, 1 << 64) == [0, 5]
    assert R.split(off, 1, 4, 15) == [1, 3, 4]       # a range restarts the rule at its first row
    assert R.split(off, 2, 2, 15) == [2]
    with pytest.raises(AssertionError):
        R.split(off, 0, 5, 0)


# ------------------------------------------------------------------------------------------------ host build of the device helpers
@pytest.fixture(scope="module")
def emu():
    src = os.path.join(HERE, "emul", "host_ch_lz4.cpp")
    out_dir = tempfile.mkdtemp(prefix="etl_host_ch_lz4_")
    so = os.path.join(out_dir, "libhost_ch_lz4.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           "-I", os.path.join(ROOT, "etl_b200", "csrc"), "-o", so, src])
    L = C.CDLL(so)
    L.emu_block_size.restype = C.c_uint32
    L.emu_city128.argtypes = [C.c_char_p, C.c_uint64, C.POINTER(C.c_uint64)]
    L.emu_sequence.restype = C.c_uint32
    L.emu_sequence.argtypes = [C.c_char_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_char_p]
    L.emu_frame.argtypes = [C.c_char_p, C.c_uint32, C.c_uint32]
    L.emu_lit_header_len.restype = C.c_uint32
    L.emu_lit_header_len.argtypes = [C.c_uint32]
    return L


def host_city(emu, b):
    out = (C.c_uint64 * 2)()
    emu.emu_city128(b, len(b), out)
    return out[0], out[1]


def test_block_size(emu):
    assert emu.emu_block_size() == R.KBLOCK


def test_city128_every_short_length(emu):
    rng = random.Random(21)
    data = bytes(rng.randrange(256) for _ in range(1024))
    for n in range(0, 1025):
        assert host_city(emu, data[:n]) == R.city128(data[:n]), n


def test_city128_long_and_seeded_lengths(emu):
    rng = random.Random(22)
    big = bytes(rng.randrange(256) for _ in range(128 * 1024 + 3))
    for n in range(128 * 1024 - 3, 128 * 1024 + 4):
        assert host_city(emu, big[:n]) == R.city128(big[:n]), n
    for _ in range(60):
        n = rng.randrange(65536 + 26)
        off = rng.randrange(8)                                  # unaligned starts too
        b = big[off:off + n]
        assert host_city(emu, b) == R.city128(b), (n, off)


def test_sequence_writer(emu):
    rng = random.Random(23)
    out = C.create_string_buffer(140000)
    for i in range(3000):
        lit_len = rng.choice([0, 1, 14, 15, 16, 269, 270, 271, rng.randrange(600), rng.randrange(70000)])
        ml = 0 if i % 5 == 0 else rng.choice([4, 18, 19, 20, 273, 274, 275, rng.randrange(4, 2000)])
        lit = bytes(rng.randrange(256) for _ in range(lit_len)) if lit_len < 2000 else bytes(lit_len)
        offset = rng.randrange(1, 65536) if ml else 0
        n = emu.emu_sequence(lit, lit_len, offset, ml, out)
        want = R.sequence(lit, offset, ml)
        assert out.raw[:n] == want, (lit_len, offset, ml)
        assert emu.emu_lit_header_len(lit_len) == len(R.sequence(lit)) - lit_len
        if ml and lit_len:                              # a valid block: the match repeats the literals' tail
            off = min(offset, lit_len)
            blk = R.sequence(lit, off, ml) + R.sequence(b"12345" + bytes(7))
            want_bytes = R.lz4_decode(blk)
            assert pa_decompress(blk, len(want_bytes)) == want_bytes


def test_frame(emu):
    rng = random.Random(24)
    for n in (0, 1, 13, 100, 5000, R.KBLOCK):
        raw = bytes(rng.randrange(4) for _ in range(n))
        payload = pa_compress(raw)
        buf = C.create_string_buffer(R.HEADER + len(payload))
        C.memmove(C.addressof(buf) + R.HEADER, payload, len(payload))
        emu.emu_frame(buf, len(payload), n)
        want = R.frame(payload, n)
        assert buf.raw[:R.HEADER + len(payload)] == want, n
        (csum, method, csize, rawlen, pl, hp), = R.parse_blocks(want)
        assert (method, csize, rawlen, pl) == (0x82, 9 + len(payload), n, payload)
        if n:
            assert R.body_bytes(want) == raw
