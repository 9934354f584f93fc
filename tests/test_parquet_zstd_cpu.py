"""CPU checks of the Parquet writer's Zstandard pages (ETL_PQ_ZSTD): the device's block compressor
(etl_b200/csrc/zstd_format.cuh) compiled for the host (tests/emul/host_parquet_zstd.cpp) writes frames that pyarrow's
libzstd decodes to their input; every block re-framed alone decodes to its fragment (so fragments compress
independently); a structural walk of every frame checks the header, the blocks' Last_Block flags and sizes, and that no
block uses Treeless literals or a Repeat sequence mode; and the pages of the Python writer's files are smaller in ZSTD
than in Snappy."""
import ctypes as C
import os
import struct
import subprocess
import tempfile

import numpy as np
import pyarrow as pa
import pytest

import parquet_ref as R
from test_parquet_cpu import sample_columns

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FRAG = 65536
CODEC = pa.Codec("zstd")


def _build(name, src):
    out_dir = tempfile.mkdtemp(prefix="etl_host_zstd_")
    so = os.path.join(out_dir, name)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           "-I", os.path.join(ROOT, "etl_b200", "csrc"), "-o", so, os.path.join(HERE, "emul", src)])
    return C.CDLL(so)


@pytest.fixture(scope="module")
def host():
    lib = _build("libhost_parquet_zstd.so", "host_parquet_zstd.cpp")
    lib.emu_zstd.argtypes = [C.c_char_p, C.c_uint64, C.c_void_p]
    lib.emu_zstd.restype = C.c_uint64
    lib.emu_zstd_bound.argtypes = [C.c_uint64]
    lib.emu_zstd_bound.restype = C.c_uint64
    return lib


@pytest.fixture(scope="module")
def snappy_host():
    lib = _build("libhost_parquet.so", "host_parquet.cpp")
    lib.emu_snappy.argtypes = [C.c_char_p, C.c_uint64, C.c_void_p]
    lib.emu_snappy.restype = C.c_uint64
    return lib


def zstd(lib, data):
    out = C.create_string_buffer(lib.emu_zstd_bound(len(data)))
    n = lib.emu_zstd(data, len(data), out)
    return out.raw[:n]


def snappy(lib, data):
    out = C.create_string_buffer(10 + len(data) + len(data) // 6 + 32 * (len(data) // FRAG + 1))
    n = lib.emu_snappy(data, len(data), out)
    return out.raw[:n]


def walk(frame, n):
    """the structural rules of include/etl_decode.h: [(block type, block bytes incl. header, literal type, modes)]"""
    assert frame[:5] == b"\x28\xb5\x2f\xfd\xa0" and struct.unpack_from("<I", frame, 5)[0] == n
    pos, blocks, nb = 9, [], max(1, (n + FRAG - 1) // FRAG)
    for k in range(nb):
        h = int.from_bytes(frame[pos:pos + 3], "little")
        last, btype, size = h & 1, (h >> 1) & 3, h >> 3
        frag = min(FRAG, n - k * FRAG)
        assert last == (k == nb - 1) and btype != 3
        lit_type = modes = None
        if btype == 0:
            assert size == frag
            body = 3 + size
        elif btype == 1:
            assert size == frag
            body = 4
        else:
            assert size < frag                           # Compressed only when strictly smaller
            b = frame[pos + 3:pos + 3 + size]
            lit_type, sf = b[0] & 3, (b[0] >> 2) & 3
            assert lit_type != 3                         # never Treeless
            if lit_type < 2:
                hl = 1 if sf in (0, 2) else 2 if sf == 1 else 3
                v = int.from_bytes(b[:hl], "little")
                regen = v >> 3 if hl == 1 else v >> 4
                q = hl + (regen if lit_type == 0 else 1)
            else:
                hl = {0: 3, 1: 3, 2: 4, 3: 5}[sf]
                v = int.from_bytes(b[:hl], "little")
                bits = {3: 10, 4: 14, 5: 18}[hl]
                q = hl + ((v >> (4 + bits)) & ((1 << bits) - 1))
            ns = b[q]
            if ns:
                ms = b[q + (1 if ns < 128 else 2 if ns < 255 else 3)]
                modes = (ms >> 6, (ms >> 4) & 3, (ms >> 2) & 3)
                assert 3 not in modes and ms & 3 == 0    # never Repeat
            body = 3 + size
        blocks.append((btype, frame[pos:pos + body], lit_type, modes))
        pos += body
    assert pos == len(frame)
    return blocks


def check(lib, data):
    f = zstd(lib, data)
    assert CODEC.decompress(f, decompressed_size=len(data)).to_pybytes() == data
    blocks = walk(f, len(data))
    if len(blocks) > 1:                                  # every block alone, as the last block of a one-fragment frame
        for k, (_, blk, _, _) in enumerate(blocks):
            frag = data[k * FRAG:(k + 1) * FRAG]
            h = int.from_bytes(blk[:3], "little") | 1
            alone = b"\x28\xb5\x2f\xfd\xa0" + struct.pack("<I", len(frag)) + h.to_bytes(3, "little") + blk[3:]
            assert CODEC.decompress(alone, decompressed_size=len(frag)).to_pybytes() == frag, k
    return f, blocks


# ------------------------------------------------------------------------------------------------ frames decode
def test_every_small_length(host):
    rng = np.random.default_rng(1)
    text = np.frombuffer(b"etaoin shrdlu ETAOIN,.;0123456789", np.uint8)
    for n in range(1025):
        check(host, rng.integers(0, 256, n, dtype=np.uint8).tobytes())
        check(host, bytes(rng.choice(text, n)))
        check(host, bytes(np.repeat(rng.integers(0, 5, n // 6 + 1, dtype=np.uint8), 6)[:n]))


def test_fragment_edges_and_block_types(host):
    rng = np.random.default_rng(2)
    seq = np.arange(3 * FRAG, dtype=np.int64).tobytes()
    for n in (FRAG - 1, FRAG, FRAG + 1, 3 * FRAG + 5):
        _, blocks = check(host, seq[:n])
        assert all(b[0] == 2 for b in blocks if len(b[1]) > 16)   # a 1-byte tail fragment is an RLE block
    _, blocks = check(host, rng.integers(0, 256, 3 * FRAG + 5, dtype=np.uint8).tobytes())
    assert [b[0] for b in blocks] == [0, 0, 0, 0]        # incompressible: Raw
    _, blocks = check(host, b"\x07" * (2 * FRAG + 9))
    assert [b[0] for b in blocks] == [1, 1, 1] and all(len(b[1]) == 4 for b in blocks)   # one byte value: RLE
    f, blocks = check(host, b"")
    assert f == b"\x28\xb5\x2f\xfd\xa0" + bytes(4) + b"\x01\x00\x00"
    _, blocks = check(host, b"x" + b"a" * FRAG)            # an offset-1 match over a whole fragment
    assert blocks[0][0] == 2


def _skewed(n, top, rng):
    """n bytes, mostly below 16 (so Huffman pays), the rest spread up to and including top"""
    a = np.where(rng.random(n) < 0.9, rng.integers(0, 16, n), rng.integers(0, top + 1, n)).astype(np.uint8)
    a[rng.integers(0, n)] = top
    return a.tobytes()


def _literals(blk):
    """(literal type, header bytes, regenerated size) of a Compressed block"""
    b = blk[3:]
    t, sf = b[0] & 3, (b[0] >> 2) & 3
    if t < 2:
        hl = 1 if sf in (0, 2) else 2 if sf == 1 else 3
        v = int.from_bytes(b[:hl], "little")
        return t, hl, v >> 3 if hl == 1 else v >> 4
    hl = {0: 3, 1: 3, 2: 4, 3: 5}[sf]
    bits = {3: 10, 4: 14, 5: 18}[hl]
    return t, hl, (int.from_bytes(b[:hl], "little") >> 4) & ((1 << bits) - 1)


@pytest.mark.parametrize("top", [127, 128, 129, 255])
def test_direct_and_fse_weights(host, top):
    rng = np.random.default_rng(top)
    _, blocks = check(host, _skewed(4000, top, rng))
    t, hl, _ = _literals(blocks[0][1])
    assert t == 2                                        # Huffman literals
    desc = blocks[0][1][3 + hl]                          # the tree description's header byte
    assert (desc >= 128) == (top <= 128), desc            # direct weights up to 128 of them, else FSE


def test_length_limit(host):
    """a geometric histogram whose optimal code is far deeper than 11 bits"""
    rng = np.random.default_rng(5)
    p = 0.5 ** np.arange(1, 41)
    p /= p.sum()
    sym = rng.choice(40, 60000, p=p).astype(np.uint8) * 5
    check(host, sym.tobytes())
    check(host, bytes(sorted(range(256))) + bytes(rng.choice(3, 20000).astype(np.uint8)))


def test_literal_and_sequence_counts(host):
    """literal sections on both sides of 1 024 (one stream / four) and 16 384 (14- / 18-bit sizes), sequence counts
    127 and 128 (one / two header bytes)"""
    rng = np.random.default_rng(6)
    seen = set()
    for nl in list(range(1000, 1060, 3)) + list(range(16300, 16600, 20)) + [40000]:
        _, blocks = check(host, _skewed(nl, 40, rng))
        t, hl, regen = _literals(blocks[0][1])
        if t == 2:
            assert hl == (3 if regen < 1024 else 4 if regen < 16384 else 5), (nl, regen, hl)
            seen.add(hl)
    assert seen == {3, 4, 5}
    unit = [bytes(rng.integers(0, 256, 24, dtype=np.uint8)) for _ in range(200)]
    for ns in (127, 128):
        data = b"".join(unit[i] + unit[i][:8] for i in range(ns))   # one 8-byte match per unit
        _, blocks = check(host, data)
        b = blocks[0][1][3:]
        t, hl, regen = _literals(blocks[0][1])
        q = hl + (regen if t == 0 else 1) if t < 2 else hl + ((int.from_bytes(b[:hl], "little") >> (4 + {3: 10, 4: 14, 5: 18}[hl])) & ((1 << {3: 10, 4: 14, 5: 18}[hl]) - 1))
        got = b[q] if b[q] < 128 else ((b[q] - 128) << 8) + b[q + 1]
        assert got == ns


def test_fuzz(host):
    rng = np.random.default_rng(7)
    for i in range(10000):
        n = int(rng.integers(0, 150000)) if i % 50 == 0 else int(rng.integers(0, 3000))
        k = i % 5
        if k == 0:
            data = rng.integers(0, int(rng.integers(1, 257)), n, dtype=np.uint8).tobytes()
        elif k == 1:
            data = np.cumsum(rng.integers(0, 3, n // 8 + 1)).astype(np.int64).tobytes()[:n]
        elif k == 2:
            data = bytes(rng.geometric(float(rng.uniform(0.01, 0.9)), n).clip(0, 255).astype(np.uint8))
        elif k == 3:
            data = (bytes(rng.integers(0, 256, int(rng.integers(1, 60)), dtype=np.uint8)) * (n // 10 + 1))[:n]
        else:
            words = [bytes(rng.integers(97, 123, int(rng.integers(1, 9)), dtype=np.uint8)) for _ in range(50)]
            data = b" ".join(words[j] for j in rng.integers(0, 50, n // 4 + 1))[:n]
        check(host, data)


# ------------------------------------------------------------------------------------------------ ZSTD < Snappy
def _copy_like(n, seed=41):
    """a COPY-shaped table: int key, text, float, timestamps, bytea, a nullable int"""
    rng = np.random.default_rng(seed)
    valid = rng.random(n) > 0.1
    words = [b"alpha", b"beta", b"gamma", b"delta", b"eps"]
    texts = [b"%s-%d" % (words[i % 5], i % 977) for i in range(n)]
    offs = np.concatenate([[0], np.cumsum([len(t) for t in texts])]).astype(np.int64)
    cols = [
        {"type": R.INT32, "valid": np.ones(n, bool), "values": np.arange(n, dtype=np.int32)},
        {"type": R.UTF8, "valid": np.ones(n, bool), "offsets": offs, "data": b"".join(texts)},
        {"type": R.FLOAT64, "valid": valid, "values": np.round(rng.normal(100, 15, n), 2)},
        {"type": R.TIMESTAMPTZ_US, "valid": np.ones(n, bool), "values": 1_700_000_000_000_000 + np.arange(n, dtype=np.int64) * 1000},
        {"type": R.INT64, "valid": valid, "values": rng.integers(0, 1000, n)},
    ]
    fields = [(f"c{i}", i + 1, 100 + i, 1 if i == 0 else 0) for i in range(len(cols))]
    return cols, fields


@pytest.mark.parametrize("table", ["sample", "copy"])
def test_zstd_smaller_than_snappy(host, snappy_host, table):
    cols, fields = sample_columns(30000) if table == "sample" else _copy_like(200000)
    _, _, pages = R.write(cols, fields, 0, len(cols[0]["valid"]))
    z = s = raw = 0
    for _, _, payload in pages:
        f = zstd(host, payload)
        assert CODEC.decompress(f, decompressed_size=len(payload)).to_pybytes() == payload
        z += len(f)
        s += len(snappy(snappy_host, payload))
        raw += len(payload)
    print(f"{table}: {len(pages)} pages, uncompressed {raw} B, Snappy {s} B, ZSTD {z} B")
    assert z < s
