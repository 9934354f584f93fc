"""CPU checks of the Parquet page index (ETL_PQ_PAGE_INDEX): the Python restatement (tests/parquet_index_ref.py) against
the ColumnIndex and OffsetIndex pyarrow writes for the same columns and page cuts, the 64-byte truncation of byte-array
bounds by its properties and at its exact edges, and the device's truncation and PageLocation compiled for the host
(tests/emul/host_parquet_index.cpp) against the restatement."""
import ctypes as C
import io
import os
import subprocess
import tempfile

import numpy as np
import pytest

import parquet_index_ref as X
import parquet_ref as R
from etl_b200 import abi

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


# ------------------------------------------------------------------------------------------------ pinned by pyarrow
def _table(n, seed):
    """the same columns as a pyarrow table and as parquet_ref columns, with their fields"""
    pa = pytest.importorskip("pyarrow")
    rng = np.random.default_rng(seed)
    valid = lambda p: rng.random(n) >= p                                  # noqa: E731
    cols, arrays, names = [], [], []

    def fixed(name, t, values, v, pa_type):
        cols.append({"type": t, "valid": v, "values": values})
        arrays.append(pa.array(values, type=pa_type, mask=~v))
        names.append(name)

    fixed("i32", R.INT32, rng.integers(-2**31, 2**31, n).astype(np.int32), valid(0.1), pa.int32())
    fixed("i64_asc", R.INT64, np.arange(n, dtype=np.int64) * 3 - 1000, valid(0.05), pa.int64())
    fixed("i64_desc", R.INT64, (n - np.arange(n, dtype=np.int64)) * 7, np.ones(n, bool), pa.int64())
    fixed("const", R.INT32, np.full(n, 42, np.int32), valid(0.2), pa.int32())
    f = rng.normal(size=n)
    f[rng.random(n) < 0.1] = 0.0
    f[rng.random(n) < 0.1] = -0.0
    fixed("f64", R.FLOAT64, f, valid(0.1), pa.float64())
    z = np.where(np.arange(n) % 2 == 0, 0.0, -0.0)                        # pages of ±0 only
    fixed("f64_zero", R.FLOAT64, z, valid(0.3), pa.float64())
    fixed("ts", R.TIMESTAMP_US, 1_700_000_000_000_000 + np.arange(n, dtype=np.int64) * 1_000_003, valid(0.1), pa.timestamp("us"))
    fixed("boolean", R.BOOLEAN, rng.random(n) < 0.5, valid(0.1), pa.bool_())
    vb = valid(0.1)
    vb[n // 3:n // 3 + 4000] = False                                      # null pages in the middle
    fixed("sparse", R.INT64, rng.integers(0, 100, n).astype(np.int64), vb, pa.int64())
    alphabet = ["a", "z", "é", "ж", "€", "中", "😀", "\U0010ffff"]
    strs = ["".join(alphabet[int(k)] for k in rng.integers(0, len(alphabet), int(rng.integers(0, 16)))) for _ in range(n)]
    sv = valid(0.1)
    enc = [s.encode() for s in strs]
    assert max(len(e) for e in enc) <= 64
    off = np.concatenate([[0], np.cumsum([len(e) if ok else 0 for e, ok in zip(enc, sv)])]).astype(np.int64)
    cols.append({"type": R.UTF8, "valid": sv, "offsets": off, "data": b"".join(e for e, ok in zip(enc, sv) if ok)})
    arrays.append(pa.array([s if ok else None for s, ok in zip(strs, sv)], type=pa.string()))
    names.append("text")
    # list<int32> with null lists, empty lists and null elements
    lens = rng.integers(0, 6, n)
    lv = valid(0.1)
    lens = np.where(lv, lens, 0)
    loff = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    kid_vals = rng.integers(-1000, 1000, int(loff[-1])).astype(np.int32)
    kid_valid = rng.random(int(loff[-1])) >= 0.1
    cols.append({"type": R.LIST, "valid": lv, "offsets": loff,
                 "child": {"type": R.INT32, "valid": kid_valid, "values": kid_vals}})
    py = [None if not lv[r] else [int(kid_vals[k]) if kid_valid[k] else None for k in range(loff[r], loff[r + 1])] for r in range(n)]
    arrays.append(pa.array(py, type=pa.list_(pa.field("element", pa.int32()))))
    names.append("ints")
    fields = [(nm, i + 1, 1000 + i, 0) for i, nm in enumerate(names)]
    return pa.Table.from_arrays(arrays, names=names), cols, fields


def _pyarrow_file(table):
    pq = pytest.importorskip("pyarrow.parquet")
    buf = io.BytesIO()
    pq.write_table(table, buf, write_page_index=True, use_dictionary=False, compression="none", data_page_version="1.0",
                   data_page_size=4096, row_group_size=30000, write_statistics=True, store_schema=False)
    return buf.getvalue()


def test_restatement_matches_pyarrow_page_index():
    """ColumnIndex fields 1-5 and the OffsetIndex against pyarrow's, on pyarrow's own page cuts.  Not compared:
    the boundary order of an all-null chunk (Arrow C++ writes UNORDERED, arrow-rs and this writer ASCENDING), truncation
    (Arrow C++ does not truncate by default, so every string here is at most 64 bytes), and the fields pyarrow writes
    that this writer does not (ColumnIndex 6/7 level histograms, OffsetIndex 2 unencoded byte-array sizes)."""
    n = 70000
    table, cols, fields = _table(n, 3)
    data = _pyarrow_file(table)
    fm, _, _ = X.file_footer(data)
    leaves = [R.Leaf(c, f) for c, f in zip(cols, fields)]
    walk = X.page_walk(data)
    got_idx = X.read_indexes(data)
    orders = set()
    r0 = 0
    ci = 0
    for rg in fm[4]:
        rows = rg[3]
        for li, cc in enumerate(rg[1]):
            cidx, oidx = got_idx[ci]
            assert cidx is not None and oidx is not None, fields[li][0]
            locs = oidx[1]
            firsts = [loc[3] for loc in locs] + [rows]
            page_rows = [(r0 + a, r0 + b) for a, b in zip(firsts[:-1], firsts[1:])]
            want = X.column_index_fields(leaves[li], page_rows)
            what = (fields[li][0], ci)
            for k in (1, 2, 3, 5):
                assert cidx[k] == want[k], (what, k)
            if not all(want[1]):
                assert cidx[4] == want[4], what
                orders.add((fields[li][0], want[4]))
            data_pages = [(off, size) for typ, off, size in walk[ci] if typ == 0]
            assert [(loc[1], loc[2]) for loc in locs] == data_pages, what
            ours = X.offset_index_bytes([(o, sz, f) for (o, sz), f in zip(data_pages, firsts)])
            assert X.parse(ours, 0, len(ours))[1] == [{1: loc[1], 2: loc[2], 3: loc[3]} for loc in locs], what
            ci += 1
        r0 += rows
    assert ("i64_asc", X.ASCENDING) in orders and ("i64_desc", X.DESCENDING) in orders and ("i32", X.UNORDERED) in orders
    assert ("const", X.ASCENDING) in orders


def test_restatement_file_reads_back():
    """the restatement's file with the index: pyarrow reads the values and sees both indexes on every chunk"""
    pq = pytest.importorskip("pyarrow.parquet")
    n = 45000
    table, cols, fields = _table(n, 9)
    for rb, re in ((0, n), (123, 40000), (7, 7)):
        plain, _, _ = R.write(cols, fields, rb, re)
        f = X.with_index(plain, cols, fields, rb, re)
        _, foot_at, _ = X.file_footer(plain)
        assert f[:foot_at] == plain[:foot_at]
        if rb == re:
            assert f == plain
            continue
        pf = pq.ParquetFile(io.BytesIO(f))
        got = pf.read()
        for nm in table.column_names:
            assert got.column(nm).to_pylist() == table.column(nm).slice(rb, re - rb).to_pylist(), nm
        for g in range(pf.metadata.num_row_groups):
            for c in range(pf.metadata.num_columns):
                col = pf.metadata.row_group(g).column(c)
                assert col.has_offset_index and col.has_column_index


def test_nan_page_has_no_column_index():
    n = 30000
    v = np.arange(n, dtype=np.float64)
    v[:20000] = np.nan                                                   # the first page is all NaN
    cols = [{"type": R.FLOAT64, "valid": np.ones(n, bool), "values": v}]
    fields = [("f", 1, 1000, 0)]
    plain, _, _ = R.write(cols, fields, 0, n)
    idx = X.read_indexes(X.with_index(plain, cols, fields, 0, n))
    assert idx[0][0] is None and len(idx[0][1][1]) == 2


# ------------------------------------------------------------------------------------------------ truncation
EDGE_CHARS = ["a", "\x7f", "é", "߿", "ࠀ", "€", "퟿", "", "￿", "😀", "\U0010ffff"]


def _rand_str(rng, lo, hi):
    s = "".join(EDGE_CHARS[int(k)] for k in rng.integers(0, len(EDGE_CHARS), int(rng.integers(lo, hi))))
    return s.encode()


def test_truncation_properties():
    rng = np.random.default_rng(11)
    for _ in range(20000):
        b = _rand_str(rng, 10, 60)
        mn, mx = X.truncate_min(b, True), X.truncate_max(b, True)
        assert mn <= b <= mx and len(mn) <= 64
        mn.decode(); mx.decode()
        assert len(mx) <= 64 or mx == b
        if len(b) <= 64:
            assert mn == b == mx
        r = bytes(rng.integers(0, 256, int(rng.integers(0, 140)), dtype=np.uint8))
        if rng.random() < 0.3:
            r = r[:int(rng.integers(0, 70))] + b"\xff" * int(rng.integers(0, 80))
        mn, mx = X.truncate_min(r, False), X.truncate_max(r, False)
        assert mn <= r <= mx and len(mn) <= 64 and (len(mx) <= 64 or mx == r)


def test_truncation_exact_cases():
    t = X.TRUNCATE
    assert X.truncate_min(b"a" * 65, True) == b"a" * 64
    assert X.truncate_max(b"a" * 65, True) == b"a" * 63 + b"b"
    assert X.truncate_min(b"a" * 63 + "é".encode(), True) == b"a" * 63             # 65 bytes, é straddles byte 64
    assert X.truncate_max(b"a" * 63 + "é".encode(), True) == b"a" * 62 + b"b"
    s = b"a" * 62 + "€".encode() + b"zz"                                         # € at bytes 62..64
    assert X.truncate_min(s, True) == b"a" * 62 and X.truncate_max(s, True) == b"a" * 61 + b"b"
    s = b"a" * 61 + "😀".encode() + b"z"                                         # 4 bytes at 61..64
    assert X.truncate_max(s, True) == b"a" * 60 + b"b"
    s = b"a" * 60 + "😀".encode() + b"z"                                         # ends exactly at 64
    assert X.truncate_max(s, True) == b"a" * 60 + "😁".encode()
    for ch in ("\U0010ffff", "￿", "퟿"):                               # cannot be incremented: the one before is
        e = ch.encode()
        s = b"q" * (t - len(e)) + e + b"tail"
        assert X.truncate_max(s, True) == b"q" * (t - len(e) - 1) + b"r", ch
        only = e * (t // len(e) + 2)                                             # nothing can be incremented
        assert X.truncate_max(only, True) == only
    assert X.truncate_max(b"\x7f" * 70, True) == b"\x7f" * 70
    assert X.truncate_max(b"\xff" * 70, False) == b"\xff" * 70                  # all 0xFF: untruncated
    assert X.truncate_max(b"\x01" + b"\xff" * 69, False) == b"\x02" + b"\x00" * 63
    assert X.truncate_max(b"\x00" * 63 + b"\xfe\xff", False) == b"\x00" * 63 + b"\xff"
    assert X.truncate_min(bytes(range(100)), False) == bytes(range(64))


# ------------------------------------------------------------------------------------------------ host-compiled pieces
@pytest.fixture(scope="module")
def host():
    out_dir = tempfile.mkdtemp(prefix="etl_host_parquet_index_")
    so = os.path.join(out_dir, "libhost_parquet_index.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           "-I", os.path.join(ROOT, "etl_b200", "csrc"), "-o", so, os.path.join(HERE, "emul", "host_parquet_index.cpp")])
    lib = C.CDLL(so)
    for f in (lib.emu_index_min, lib.emu_index_max):
        f.argtypes = [C.c_char_p, C.c_uint64, C.c_int, C.c_void_p]
        f.restype = C.c_uint64
    lib.emu_page_location.argtypes = [C.c_uint64, C.c_uint32, C.c_uint64, C.c_void_p]
    lib.emu_page_location.restype = C.c_uint32
    return lib


def test_host_formatters_fuzz(host):
    rng = np.random.default_rng(2024)
    out = C.create_string_buffer(4096)
    for i in range(100000):
        if i % 2:
            v = _rand_str(rng, 0, 70) if i % 4 == 1 else _rand_str(rng, 14, 24) + (EDGE_CHARS[int(rng.integers(0, len(EDGE_CHARS)))] * 20).encode()
            utf8 = True
        else:
            n = int(rng.integers(0, 130))
            v = bytes(rng.integers(0, 256, n, dtype=np.uint8))
            if i % 6 == 0:
                v = v[:int(rng.integers(0, 66))] + b"\xff" * int(rng.integers(0, 70))
            utf8 = False
        for f, ref in ((host.emu_index_min, X.truncate_min), (host.emu_index_max, X.truncate_max)):
            k = f(v, len(v), int(utf8), out)
            assert out.raw[:k] == ref(v, utf8), (v, utf8, ref.__name__)
            assert f(v, len(v), int(utf8), None) == k


def test_host_page_location(host):
    out = C.create_string_buffer(64)
    for off, size, first in ((4, 100, 0), (2**40 + 3, 2**31 - 1, 2**20 - 1), (2**62, 1, 12345)):
        k = host.emu_page_location(off, size, first, out)
        assert k <= 29
        assert out.raw[:k] == X.offset_index_bytes([(off, size, first)])[2:-1]


def test_flag_constant():
    src = os.path.join(tempfile.mkdtemp(prefix="pq_pidx_"), "f.c")
    with open(src, "w") as fh:
        fh.write('#include <stdio.h>\n#include "etl_decode.h"\nint main(void) { printf("%u", (unsigned)ETL_PQ_PAGE_INDEX); return 0; }\n')
    exe = src[:-2]
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", exe, src])
    assert int(subprocess.check_output([exe], text=True)) == abi.PQ_PAGE_INDEX == X.PAGE_INDEX == 0x400
