"""The host-side pieces of etl_dec_parquet_write_files, compiled from the device's own source for the host
(tests/emul/host_parquet_files.cpp): the row-group table built from the files' row offsets against a Python restatement
(empty files, files of exactly 1 048 576 and 1 048 577 rows, a slice starting above 0), and the footer every file
gets on the device — the host's schema prefix, then the __host__ __device__ footer tail over flat chunk records —
byte for byte against footer() and against a Python restatement of the whole footer (parquet_dict_ref's, with the
bloom-filter and page-index fields added) on randomised records: several row groups, dictionary, page-index and bloom
fields, statistics of 0 and 64 bytes, and offsets at varint-width boundaries; plain records also against
parquet_ref.footer."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import parquet_dict_ref as D
import parquet_ref as R

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
RG_ROWS = 1 << 20


class EmuLeaf(C.Structure):
    _fields_ = [("name", C.c_char_p), ("field_id", C.c_int32), ("element_field_id", C.c_int32), ("ptype", C.c_uint32),
                ("converted", C.c_int32), ("logical", C.c_uint32), ("flags", C.c_uint32)]


class EmuRec(C.Structure):
    _fields_ = [(f, C.c_uint64) for f in ("offset", "num_values", "usize", "csize", "null_count", "data_offset", "data_pages",
                                          "ci_offset", "oi_offset", "bloom_offset")] + \
               [(f, C.c_uint32) for f in ("ci_len", "oi_len", "bloom_len", "min_len", "max_len", "has", "dict", "page_index")] + \
               [("min", C.c_uint8 * 64), ("max", C.c_uint8 * 64)]


@pytest.fixture(scope="module")
def host():
    out_dir = tempfile.mkdtemp(prefix="etl_host_parquet_files_")
    so = os.path.join(out_dir, "libhost_parquet_files.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           "-I", os.path.join(ROOT, "etl_b200", "csrc"), "-o", so, os.path.join(HERE, "emul", "host_parquet_files.cpp")])
    lib = C.CDLL(so)
    lib.emu_row_groups.argtypes = [C.c_void_p, C.c_uint64] + [C.c_void_p] * 3 + [C.c_uint64, C.c_void_p]
    lib.emu_row_groups.restype = C.c_uint64
    lib.emu_footer_host.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64]
    lib.emu_footer_host.restype = C.c_uint64
    lib.emu_footer_split.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p, C.c_uint32,
                                     C.c_void_p, C.c_uint64]
    lib.emu_footer_split.restype = C.c_uint64
    return lib


# ------------------------------------------------------------------------------------------------ row-group table
def row_groups(ro):
    """(row0 relative to ro[0], rows, file) per row group, and each file's first row group (K + 1 entries)"""
    t, first = [], []
    for k in range(len(ro) - 1):
        first.append(len(t))
        r = ro[k]
        while r < ro[k + 1]:
            t.append((r - ro[0], min(RG_ROWS, ro[k + 1] - r), k))
            r += RG_ROWS
    first.append(len(t))
    return t, first


def _emu_row_groups(host, ro):
    K = len(ro) - 1
    cap = sum((ro[k + 1] - ro[k] + RG_ROWS - 1) // RG_ROWS for k in range(K)) + 1
    a = (C.c_uint64 * len(ro))(*ro)
    row0, rows, file, first = (C.c_uint64 * cap)(), (C.c_uint64 * cap)(), (C.c_uint64 * cap)(), (C.c_uint64 * (K + 1))()
    n = host.emu_row_groups(a, K, row0, rows, file, cap, first)
    return [(row0[g], rows[g], file[g]) for g in range(n)], list(first)


@pytest.mark.parametrize("ro", [
    [0], [5], [0, 0], [7, 7, 7], [0, 1], [0, RG_ROWS], [0, RG_ROWS + 1], [3, 3 + RG_ROWS, 3 + 2 * RG_ROWS + 1],
    [10, 10, 15, 15, 15 + RG_ROWS + 1, 15 + RG_ROWS + 1, 20 + 3 * RG_ROWS],
    [100] + [100 + RG_ROWS * k + k for k in range(1, 5)],
], ids=lambda ro: "-".join(map(str, ro[:4])) + ("…" if len(ro) > 4 else ""))
def test_row_group_table(host, ro):
    got = _emu_row_groups(host, ro)
    assert got == row_groups(ro)
    t, first = got
    # the row groups tile [0, ro[K] - ro[0]) in order, and each file's row groups add up to its rows
    assert sum(r for _, r, _ in t) == ro[-1] - ro[0]
    assert all(t[g][0] + t[g][1] == t[g + 1][0] for g in range(len(t) - 1))
    for k in range(len(ro) - 1):
        assert sum(t[g][1] for g in range(first[k], first[k + 1])) == ro[k + 1] - ro[k]


def test_row_group_table_random(host):
    rng = np.random.default_rng(11)
    for _ in range(50):
        K = int(rng.integers(0, 40))
        lens = rng.choice([0, 1, 5, RG_ROWS - 1, RG_ROWS, RG_ROWS + 1, 3 * RG_ROWS], size=K)
        ro = [int(rng.integers(0, 1000))]
        for x in lens:
            ro.append(ro[-1] + int(x))
        assert _emu_row_groups(host, ro) == row_groups(ro)


# ------------------------------------------------------------------------------------------------ footer tail
TYPES = [R.BOOLEAN, R.INT32, R.INT64, R.FLOAT32, R.FLOAT64, R.UTF8, R.LARGE_BINARY, R.DATE32, R.TIME64_US, R.TIMESTAMP_US,
         R.TIMESTAMPTZ_US, R.UUID]
# offsets and sizes at varint-width boundaries (7-bit groups of the zigzag value)
EDGES = [0, 1, 63, 64, 127, 128, 8191, 8192, 2**20 - 1, 2**20, 2**27 - 1, 2**27, 2**31 - 1, 2**34 - 1, 2**34, 2**41, 2**48 + 3,
         2**55 - 1, 2**55, 2**62 - 1]


def _leaves():
    cols, fields = [], []
    for i, t in enumerate(TYPES + TYPES[:6]):
        is_list = i >= len(TYPES)
        cols.append({"type": R.LIST, "child": {"type": t}} if is_list else {"type": t})
        fields.append((f"f{i}" * (1 + i % 3), 10 + i, 500 + i, int(i % 4 == 0)))
    leaves = [R.Leaf(c, f) for c, f in zip(cols, fields)]
    emu = (EmuLeaf * len(leaves))()
    for e, L in zip(emu, leaves):
        e.name, e.field_id, e.element_field_id, e.ptype = L.name.encode(), L.field_id, L.element_field_id, R.PT[L.atype]
        e.converted, e.logical = R.CONVERTED.get(L.atype, -1), R.LOGICAL.get(L.atype, 0)
        e.flags = int(L.required) | (2 if L.is_list else 0) | (4 if L.atype == R.TIMESTAMPTZ_US else 0)
    return leaves, emu


def _records(rng, n, plain, page_index):
    recs = (EmuRec * max(1, n))()
    chunks = []
    # the restatements' row-group totals are unbounded integers: the sizes stay below 2^42, so their sums fit 63 bits
    small = [x for x in EDGES if x < 2**42]
    v = lambda: int(rng.choice(EDGES)) if rng.random() < 0.5 else int(rng.integers(0, 2**40))  # noqa: E731
    sz = lambda: int(rng.choice(small)) if rng.random() < 0.5 else int(rng.integers(0, 2**40))  # noqa: E731
    for k in range(n):
        e = recs[k]
        e.offset, e.num_values, e.usize, e.csize, e.null_count = v(), v(), sz(), sz(), v()
        e.has = int(rng.random() > 0.3)
        mn = bytes(rng.integers(0, 256, int(rng.choice([0, 1, 8, 63, 64]))).astype(np.uint8))
        mx = bytes(rng.integers(0, 256, int(rng.choice([0, 4, 16, 64]))).astype(np.uint8))
        e.min_len, e.max_len = (len(mn), len(mx)) if e.has else (0, 0)
        C.memmove(e.min, mn, len(mn))
        C.memmove(e.max, mx, len(mx))
        if not plain:
            e.dict = int(rng.random() < 0.5)
            e.data_offset, e.data_pages = v(), int(rng.choice([1, 14, 15, 2**31 - 1]))
            e.page_index = page_index
            e.ci_len = int(rng.choice([0, 1, 127, 128, 2**31 - 1])) if page_index else 0
            e.oi_len = int(rng.choice([1, 127, 128, 2**31 - 1])) if page_index else 0
            e.ci_offset, e.oi_offset = v(), v()
            if rng.random() < 0.5:
                e.bloom_offset, e.bloom_len = v(), int(rng.choice([47, 128 + 16, 2**27 + 19]))
        chunks.append(dict(offset=e.offset, num_values=e.num_values, usize=e.usize, csize=e.csize, null_count=e.null_count,
                           min=mn if e.has else None, max=mx if e.has else None, dict=bool(e.dict), data_offset=e.data_offset,
                           data_pages=e.data_pages, page_index=e.page_index, ci_offset=e.ci_offset, ci_len=e.ci_len,
                           oi_offset=e.oi_offset, oi_len=e.oi_len, bloom_offset=e.bloom_offset, bloom_len=e.bloom_len))
    return recs, chunks


def ref_footer(leaves, rg_rows, chunks, codec):
    """parquet_dict_ref.footer's restatement (tests/parquet_dict_ref.py) with the ColumnMetaData's bloom_filter_offset /
    _length (14, 15) and the ColumnChunk's offset_index_* / column_index_* (4–7), as include/etl_decode.h states them"""
    w = D.TWriter()
    w.i32(1, 1)
    w.list(2, 12, 1 + sum(3 if L.is_list else 1 for L in leaves))
    w.elem(); w.binary(4, b"schema"); w.i32(5, len(leaves)); w.end()
    for L in leaves:
        if not L.is_list:
            D._schema_leaf(w, L, False)
            continue
        w.elem(); w.i32(3, 0 if L.required else 1); w.binary(4, L.name.encode()); w.i32(5, 1); w.i32(6, 3); w.i32(9, L.field_id)
        w.begin(10); w.begin(3); w.end(); w.end(); w.end()
        w.elem(); w.i32(3, 2); w.binary(4, b"list"); w.i32(5, 1); w.end()
        D._schema_leaf(w, L, True)
    w.i64(3, sum(rg_rows))
    w.list(4, 12, len(rg_rows))
    nl = len(leaves)
    for g, rows in enumerate(rg_rows):
        cs = chunks[g * nl:(g + 1) * nl]
        w.elem()
        w.list(1, 12, nl)
        for L, c in zip(leaves, cs):
            w.elem()
            w.i64(2, c["offset"])
            w.begin(3)
            w.i32(1, R.PT[L.atype])
            levels = L.is_list or not L.required
            dic = c["dict"]
            w.list(2, 5, (2 if levels else 1) + dic)
            w.var(0)
            if levels:
                w.var(6)
            if dic:
                w.var(D.RLE_DICTIONARY << 1)
            path = [L.name.encode()] + ([b"list", b"element"] if L.is_list else [])
            w.list(3, 8, len(path))
            for p in path:
                w.var(len(p)); w.out += p
            w.i32(4, codec & 0xFF)
            w.i64(5, c["num_values"])
            w.i64(6, c["usize"])
            w.i64(7, c["csize"])
            w.i64(9, c["data_offset"] if dic else c["offset"])
            if dic:
                w.i64(11, c["offset"])
            w.begin(12)
            w.i64(3, c["null_count"])
            if c["min"] is not None:
                w.binary(5, c["max"])
                w.binary(6, c["min"])
            w.end()
            if dic:
                w.list(13, 12, 2)
                w.elem(); w.i32(1, 2); w.i32(2, 0); w.i32(3, 1); w.end()
                w.elem(); w.i32(1, 0); w.i32(2, D.RLE_DICTIONARY); w.i32(3, c["data_pages"]); w.end()
            if c["bloom_len"]:
                w.i64(14, c["bloom_offset"])
                w.i32(15, c["bloom_len"])
            w.end()
            if c["page_index"]:
                w.i64(4, c["oi_offset"])
                w.i32(5, c["oi_len"])
                if c["ci_len"]:
                    w.i64(6, c["ci_offset"])
                    w.i32(7, c["ci_len"])
            w.end()
        w.i64(2, sum(c["usize"] for c in cs))
        w.i64(3, rows)
        w.i64(5, cs[0]["offset"])
        w.i64(6, sum(c["csize"] for c in cs))
        w.i16(7, g)
        w.end()
    w.binary(6, D.CREATED_BY)
    w.list(7, 12, nl)
    for _ in leaves:
        w.elem(); w.begin(1); w.end(); w.end()
    w.end()
    return bytes(w.out)


@pytest.mark.parametrize("n_rg", [0, 1, 2, 3, 15, 16])
@pytest.mark.parametrize("kind", ["plain", "dict-bloom", "dict-bloom-index"])
def test_footer_tail_equals_footer(host, n_rg, kind):
    rng = np.random.default_rng(100 * n_rg + len(kind))
    leaves, emu = _leaves()
    recs, chunks = _records(rng, n_rg * len(leaves), kind == "plain", int(kind.endswith("index")))
    rows = [int(rng.choice([1, 127, 128, RG_ROWS - 1, RG_ROWS])) for _ in range(n_rg)]
    rg = (C.c_uint64 * max(1, n_rg))(*rows)
    for codec in (0, 1, 6):
        want = C.create_string_buffer(1 << 20)
        kw = host.emu_footer_host(emu, len(leaves), rg, n_rg, recs, codec, want, 1 << 20)
        assert kw
        # the tail's row-group starts may have any origin (a file's row groups inside the call's table)
        for rg0 in (0, 12345, 2**33):
            got = C.create_string_buffer(1 << 20)
            kg = host.emu_footer_split(emu, len(leaves), rg, n_rg, rg0, recs, codec, got, 1 << 20)
            assert got.raw[:kg] == want.raw[:kw], (n_rg, kind, codec, rg0)
        # against the independent restatements: parquet_ref for plain records, the one above for every field
        assert want.raw[:kw] == ref_footer(leaves, rows, chunks, codec), (n_rg, kind, codec)
        if kind == "plain":
            assert want.raw[:kw] == R.footer(leaves, rows, chunks, codec), (n_rg, codec)
