"""CPU checks of the bloom filters of etl_dec_parquet_write_bloom: the Python restatement (tests/parquet_bloom_ref.py)
against the split-block filters pyarrow 24 (Arrow C++) writes for the same columns, ndv and fpp, byte for byte; its
placement of the filters in a file; XXH64 known answers; the etl_parquet_bloom layout against its ctypes mirror; and
the device's hash, insert, header and sizing compiled for the host (tests/emul/host_parquet_bloom.cpp) against the
restatement."""
import ctypes as C
import io
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest

import parquet_bloom_ref as B
import parquet_index_ref as X
import parquet_ref as R
from etl_b200 import abi

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


# ------------------------------------------------------------------------------------------------ pinned by pyarrow
def _table(n, seed):
    """every flat physical type as a pyarrow table and as parquet_ref columns, with their fields"""
    pa = pytest.importorskip("pyarrow")
    rng = np.random.default_rng(seed)
    valid = lambda p: rng.random(n) >= p                                  # noqa: E731
    cols, arrays, names = [], [], []

    def fixed(name, t, values, v, pa_type):
        cols.append({"type": t, "valid": v, "values": values})
        arrays.append(pa.array(values, type=pa_type, mask=~v))
        names.append(name)

    def byte_array(name, t, vals, v, pa_type):
        off = np.concatenate([[0], np.cumsum([len(e) if ok else 0 for e, ok in zip(vals, v)])]).astype(np.int64)
        cols.append({"type": t, "valid": v, "offsets": off, "data": b"".join(e for e, ok in zip(vals, v) if ok)})
        arrays.append(pa.array([e if ok else None for e, ok in zip(vals, v)], type=pa_type))
        names.append(name)

    fixed("i32", R.INT32, rng.integers(-2**31, 2**31, n).astype(np.int32), valid(0.1), pa.int32())
    fixed("i64", R.INT64, rng.integers(-2**63, 2**63 - 1, n).astype(np.int64), valid(0.1), pa.int64())
    f = rng.normal(size=n)
    f[rng.random(n) < 0.1] = 0.0
    f[rng.random(n) < 0.1] = -0.0
    f[rng.random(n) < 0.05] = np.nan
    fixed("f64", R.FLOAT64, f, valid(0.1), pa.float64())
    fixed("f32", R.FLOAT32, np.where(rng.random(n) < 0.2, -0.0, f).astype(np.float32), valid(0.1), pa.float32())
    fixed("ts", R.TIMESTAMP_US, 1_700_000_000_000_000 + rng.integers(0, 10**12, n).astype(np.int64), valid(0.1), pa.timestamp("us"))
    fixed("date", R.DATE32, rng.integers(-10000, 30000, n).astype(np.int32), valid(0.1), pa.date32())
    fixed("all_null", R.INT64, np.zeros(n, np.int64), np.zeros(n, bool), pa.int64())
    u = rng.integers(0, 256, (n, 16), dtype=np.uint8)
    uv = valid(0.1)
    cols.append({"type": R.UUID, "valid": uv, "values": u})
    arrays.append(pa.array([bytes(u[i]) if uv[i] else None for i in range(n)], type=pa.binary(16)))
    names.append("uuid")
    lens = [0, 1, 7, 31, 32, 33, 100, 1024, 1500]
    strs = [("é" * int(rng.integers(0, 4)) + "x" * lens[int(rng.integers(0, len(lens)))]).encode() for _ in range(n)]
    byte_array("text", R.UTF8, strs, valid(0.1), pa.string())
    blobs = [bytes(rng.integers(0, 256, int(rng.integers(0, 80)), dtype=np.uint8)) for _ in range(n)]
    byte_array("bin", R.LARGE_BINARY, blobs, valid(0.1), pa.large_binary())
    fields = [(nm, i + 1, 1000 + i, 0) for i, nm in enumerate(names)]
    return pa.Table.from_arrays(arrays, names=names), cols, fields


def _pyarrow_file(table, opts, row_group_size=None, **kw):
    pq = pytest.importorskip("pyarrow.parquet")
    buf = io.BytesIO()
    pq.write_table(table, buf, bloom_filter_options=opts, use_dictionary=False, compression="none", store_schema=False,
                   row_group_size=row_group_size, **kw)
    return buf.getvalue()


def _chunk_ranges(fm):
    out, r0 = [], 0
    for rg in fm[4]:
        out.append((r0, r0 + rg[3]))
        r0 += rg[3]
    return out


@pytest.mark.parametrize("ndv_fpp", [(0, 0.01), (100, 0.05), (5000, 0.01), (10, 0.1)])
def test_filters_match_pyarrow(ndv_fpp):
    """header and bitset of every chunk of every flat type, two row groups; ndv 0 stands for the chunk's non-null count
    (pyarrow needs an explicit ndv, so it is given that count).  pyarrow's filters sit behind all the data, row-group
    major and contiguous, where the restatement puts them."""
    n = 3000
    table, cols, fields = _table(n, 5 + ndv_fpp[0])
    ndv, fpp = ndv_fpp
    leaves = [R.Leaf(c, f) for c, f in zip(cols, fields)]
    rgs = [(0, 1700), (1700, n)]
    # pyarrow writes one ndv per column for the whole file: with ndv 0 compare per row group with its own count
    for gi, (g0, g1) in enumerate(rgs):
        sub = table.slice(g0, g1 - g0)
        opts = {}
        for nm, leaf in zip(table.column_names, leaves):
            nn = int(np.count_nonzero(leaf.vcol["valid"][g0:g1]))
            opts[nm] = {"ndv": ndv or max(1, nn), "fpp": fpp}
        data = _pyarrow_file(sub, opts, row_group_size=g1 - g0)
        got = B.read_filters(data)
        for li, leaf in enumerate(leaves):
            want = B.chunk_filter(leaf, g0, g1, (fpp, ndv, B.MAX_BYTES))
            off, length, hdr, hb, bits = got[li]
            assert hb + bits == want, (fields[li][0], gi)
            assert length in (None, len(want))
    # placement in pyarrow's own two-row-group file
    data = _pyarrow_file(table, {nm: {"ndv": ndv or 1000, "fpp": fpp} for nm in table.column_names}, row_group_size=1700)
    fm, foot_at, _ = X.file_footer(data)
    got = B.read_filters(data)
    assert len(fm[4]) == 2 and all(g is not None for g in got)
    end = B.data_end(data)
    at = end
    for off, length, hdr, hb, bits in got:
        assert off == at                                  # contiguous, row-group major, from the end of the data
        at += len(hb) + len(bits)
    for (g0, g1), rg in zip(_chunk_ranges(fm), fm[4]):
        assert rg[3] == g1 - g0


def test_header_lengths():
    assert [len(B.header(b)) for b in (32, 128, 8192)] == [15, 16, 17]


# (ndv, fpp) -> bytes measured with pyarrow 24
SIZES = [((100, .05), 128), ((5000, .01), 8192), ((10, .1), 32), ((3, .05), 32), ((1, .5), 32), ((10**6, .05), 1 << 20),
         ((10**6, .01), 2 << 20)]


def _edges():
    """(ndv, fpp) pairs whose bit count lands on, just below and just above 8 × a power of two, at 32 B, and at
    128 MiB"""
    out = [(1, 0.999), (1, 1e-9), (2, 0.5), (10**8, 0.01), (2 * 10**8, 0.001), (2**31 - 1, 0.2)]
    for fpp in (0.01, 0.05, 0.1, 0.3):
        c = -8.0 / math.log(1 - math.pow(fpp, 1.0 / 8))
        for k in (8, 9, 12, 17, 20):
            t = int(8 * (1 << k) / c)
            out += [(t - 1, fpp), (t, fpp), (t + 1, fpp), (t + 2, fpp)]
    return out


@pytest.mark.parametrize("ndv,fpp", [p for p, _ in SIZES] + _edges())
def test_sizes_match_pyarrow(ndv, fpp):
    """the bitset size, including the power-of-two rounding (Arrow C++ rounds the bit count up, so a bit count just
    past 8 × 2^k gives 2^(k+1) bytes) and both clamps; the header of pyarrow's filter is the restatement's"""
    pa = pytest.importorskip("pyarrow")
    want = B.bloom_bytes(ndv, fpp, B.MAX_BYTES)
    data = _pyarrow_file(pa.table({"a": pa.array([7], pa.int64())}), {"a": {"ndv": ndv, "fpp": fpp}})
    off, length, hdr, hb, bits = B.read_filters(data)[0]
    assert hdr[1] == want and hb == B.header(want), (ndv, fpp, hdr[1], want)
    for (nd, fp), size in SIZES:
        if (nd, fp) == (ndv, fpp):
            assert want == size
    assert 32 <= want <= B.MAX_BYTES and want & (want - 1) == 0


def test_size_cap_and_default():
    assert B.bloom_bytes(10**6, 0.01, 0) == 1 << 20          # max_bytes 0: 1 MiB
    assert B.bloom_bytes(10**6, 0.01, 1 << 27) == 2 << 20
    assert B.bloom_bytes(10**6, 0.01, 4096) == 4096
    assert B.bloom_bytes(1, 0.5, 4096) == 32
    assert B.bloom_bytes(10**12, 0.01, 1 << 27) == 1 << 27


# ------------------------------------------------------------------------------------------------ XXH64
def _seeded(n=1200):
    return bytes(np.random.default_rng(77).integers(0, 256, n, dtype=np.uint8))


def test_xxh64_known_answers():
    """lengths 0-100 over a seeded buffer (across the 4 / 8 / 32-byte tails and the stripe loop): the reference form,
    the vectorised form and pyarrow's filters agree"""
    pa = pytest.importorskip("pyarrow")
    assert B.xxh64(b"") == 0xEF46DB3751D8E999
    buf = _seeded()
    vals = [buf[k:k + k + 3][:k] for k in range(101)]
    ref = [B.xxh64(v) for v in vals]
    assert list(B.hash_values(vals)) == ref
    for k, v in enumerate(vals):                          # one filter per value: its 8 bits are exactly its hash's
        data = _pyarrow_file(pa.table({"b": pa.array([v], pa.binary())}), {"b": {"ndv": 1, "fpp": 0.5}})
        _, _, _, _, bits = B.read_filters(data)[0]
        assert bits == B.bitset(np.array([ref[k]], np.uint64), 32), k


# ------------------------------------------------------------------------------------------------ placement
def _norm(col):
    """a column's values, comparable with NaN (by repr) and with the UUID logical type read back as bytes"""
    return [repr(getattr(x, "bytes", x)) for x in col.to_pylist()]


def test_placement_restatement():
    """with_bloom on a file written by parquet_ref (with and without a page index): bytes before the data end kept,
    the filters behind it in chunk order, the page index moved behind them and still parsed at its new offsets, and
    pyarrow reads the values back"""
    pq = pytest.importorskip("pyarrow.parquet")
    n = 25000
    table, cols, fields = _table(n, 3)
    bloom = [(0.01, 0, 0), (0.05, 100, 0), (0.1, 0, 64), (0.01, 0, 0), (0.2, 7, 0), (0.01, 0, 0), (0.01, 0, 0),
             (0.01, 0, 0), (0, 0, 0), (0.3, 0, 32)]
    assert len(bloom) == len(cols)
    for rb, re in ((0, n), (11, 20050), (5, 5)):
        plain, _, _ = R.write(cols, fields, rb, re)
        for base in (plain, X.with_index(plain, cols, fields, rb, re)):
            f = B.with_bloom(base, cols, fields, rb, re, bloom)
            if rb == re:
                assert f == base
                continue
            end = B.data_end(base)
            assert f[:end] == base[:end] and B.data_end(f) == end
            got = B.read_filters(f)
            want = B.chunk_filters(cols, fields, rb, re, bloom)
            at = end
            for g, w in zip(got, want):
                assert (g is None) == (w is None)
                if g is not None:
                    assert g[0] == at and g[1] == len(w) and g[3] + g[4] == w
                    at += len(w)
            assert B.with_bloom(base, cols, fields, rb, re, None) == base
            assert B.with_bloom(base, cols, fields, rb, re, [(0, 0, 0)] * len(cols)) == base
            old, new = X.read_indexes(base), X.read_indexes(f)    # parsed at their stated offsets and lengths
            assert old == new
            got_t = pq.ParquetFile(io.BytesIO(f)).read()
            for nm in table.column_names:
                assert _norm(got_t.column(nm)) == _norm(table.column(nm).slice(rb, re - rb)), nm


# ------------------------------------------------------------------------------------------------ ABI
def test_struct_layout(tmp_path):
    ct = abi.ParquetBloom
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "etl_decode.h"', 'int main(void) {',
             '  printf("size %zu\\n", sizeof(etl_parquet_bloom));']
    for fname, _ in ct._fields_:
        lines.append(f'  printf("{fname} %zu\\n", offsetof(etl_parquet_bloom, {fname}));')
    lines += ['  return 0;', '}']
    src = tmp_path / "bloom_sizes.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "bloom_sizes"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    assert int(got["size"]) == C.sizeof(ct) == 24
    for fname, _ in ct._fields_:
        assert int(got[fname]) == getattr(ct, fname).offset, fname


# ------------------------------------------------------------------------------------------------ host-compiled pieces
@pytest.fixture(scope="module")
def host():
    out_dir = tempfile.mkdtemp(prefix="etl_host_parquet_bloom_")
    so = os.path.join(out_dir, "libhost_parquet_bloom.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           "-I", os.path.join(ROOT, "etl_b200", "csrc"), "-o", so, os.path.join(HERE, "emul", "host_parquet_bloom.cpp")])
    lib = C.CDLL(so)
    lib.emu_xxh64.argtypes = [C.c_char_p, C.c_uint64]
    lib.emu_xxh64_u32.argtypes = [C.c_uint32]
    lib.emu_xxh64_u64.argtypes = [C.c_uint64]
    for f in (lib.emu_xxh64, lib.emu_xxh64_u32, lib.emu_xxh64_u64, lib.emu_bloom_bytes):
        f.restype = C.c_uint64
    lib.emu_bloom_insert.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64]
    lib.emu_bloom_insert.restype = None
    lib.emu_bloom_header.argtypes = [C.c_void_p, C.c_uint32]
    lib.emu_bloom_header.restype = C.c_uint32
    lib.emu_bloom_bytes.argtypes = [C.c_uint64, C.c_double, C.c_uint64]
    return lib


def test_host_hash_fuzz(host):
    """100 000 values: every length 0-1024, then random lengths; the fixed-width fast paths against the generic hash"""
    rng = np.random.default_rng(2025)
    buf = bytes(rng.integers(0, 256, 4096, dtype=np.uint8))
    vals = []
    for i in range(100000):
        k = i if i <= 1024 else int(rng.integers(0, 1025))
        s = int(rng.integers(0, 4096 - k + 1))
        vals.append(buf[s:s + k])
    got = np.array([host.emu_xxh64(v, len(v)) for v in vals], np.uint64)
    assert np.array_equal(got, B.hash_values(vals))
    for v in vals[:3000]:
        if len(v) >= 8:
            assert host.emu_xxh64_u32(int.from_bytes(v[:4], "little")) == B.xxh64(v[:4])
            assert host.emu_xxh64_u64(int.from_bytes(v[:8], "little")) == B.xxh64(v[:8])


def test_host_insert_fuzz(host):
    """bitsets of 32 B to 1 MiB against the restatement's, and the header"""
    rng = np.random.default_rng(31)
    for nbytes in [32 << k for k in range(16)]:
        h = rng.integers(0, 2**64 - 1, int(rng.integers(1, 20000)), dtype=np.uint64)
        words = np.zeros(nbytes // 4, np.uint32)
        host.emu_bloom_insert(words.ctypes.data, nbytes, h.ctypes.data, len(h))
        assert words.tobytes() == B.bitset(h, nbytes), nbytes
        assert all(B.contains(words.tobytes(), int(x)) for x in h[:200])
        out = C.create_string_buffer(32)
        k = host.emu_bloom_header(out, nbytes)
        assert out.raw[:k] == B.header(nbytes) and host.emu_bloom_header(None, nbytes) == k


def test_host_sizes(host):
    for ndv, fpp in [p for p, _ in SIZES] + _edges():
        for mb in (0, 32, 4096, 1 << 20, 1 << 27):
            assert host.emu_bloom_bytes(ndv, fpp, mb or B.DEFAULT_MAX_BYTES) == B.bloom_bytes(ndv, fpp, mb), (ndv, fpp, mb)
