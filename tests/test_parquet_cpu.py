"""CPU checks of the Parquet writer's contract: the Python restatement (tests/parquet_ref.py) read back by pyarrow as an
independent reader (values, field ids, physical / logical types, repetitions, statistics, column orders), the RLE
hybrid against the Parquet spec's bit-packing example, the device's Snappy fragment compressor compiled for the host
(tests/emul/host_parquet.cpp) against pyarrow's Snappy, the device's level encoder, page header and footer writer
byte for byte against the restatement, and the ctypes mirror of the new structs."""
import ctypes as C
import io
import os
import subprocess
import tempfile

import numpy as np
import pytest

import parquet_ref as R
from etl_b200 import abi

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def host():
    out_dir = tempfile.mkdtemp(prefix="etl_host_parquet_")
    so = os.path.join(out_dir, "libhost_parquet.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           "-I", os.path.join(ROOT, "etl_b200", "csrc"), "-o", so, os.path.join(HERE, "emul", "host_parquet.cpp")])
    lib = C.CDLL(so)
    lib.emu_snappy.argtypes = [C.c_char_p, C.c_uint64, C.c_void_p]
    lib.emu_snappy.restype = C.c_uint64
    lib.emu_levels.argtypes = [C.c_char_p, C.c_uint64, C.c_uint32, C.c_void_p]
    lib.emu_levels.restype = C.c_uint64
    lib.emu_page_header.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
    lib.emu_page_header.restype = C.c_uint32
    lib.emu_footer.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64]
    lib.emu_footer.restype = C.c_uint64
    return lib


# ------------------------------------------------------------------------------------------------ the restatement vs pyarrow
def _strings(rng, n, valid, long_every=0):
    vals = [(b"v%d-" % rng.integers(0, 50)) * int(rng.integers(0, 4)) for _ in range(n)]
    if long_every:
        for i in range(0, n, long_every):
            vals[i] = b"\xff" + b"z" * 80
    offs = np.concatenate([[0], np.cumsum([len(v) if ok else 0 for v, ok in zip(vals, valid)])]).astype(np.int64)
    return offs, b"".join(v for v, ok in zip(vals, valid) if ok), vals


def sample_columns(n, seed=3):
    rng = np.random.default_rng(seed)
    valid = rng.random(n) > 0.2
    s_offs, s_data, _ = _strings(rng, n, valid)
    b_offs, b_data, _ = _strings(rng, n, valid, long_every=7)
    lvalid = rng.random(n) > 0.2
    lens = np.where(lvalid, rng.integers(0, 4, n), 0)
    loffs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    ne = int(loffs[-1])
    f = rng.normal(size=n)
    f[::9] = np.nan
    f[1::9] = 0.0
    f[2::9] = -np.inf
    cols = [
        {"type": R.INT64, "valid": np.ones(n, bool), "values": np.arange(n, dtype=np.int64) * 3 - 7},
        {"type": R.INT32, "valid": valid, "values": rng.integers(-2**31, 2**31, n).astype(np.int32)},
        {"type": R.BOOLEAN, "valid": valid, "values": rng.random(n) > 0.5},
        {"type": R.FLOAT32, "valid": valid, "values": f.astype(np.float32)},
        {"type": R.FLOAT64, "valid": valid, "values": f},
        {"type": R.UTF8, "valid": valid, "offsets": s_offs, "data": s_data},
        {"type": R.LARGE_BINARY, "valid": valid, "offsets": b_offs, "data": b_data},
        {"type": R.DATE32, "valid": valid, "values": rng.integers(-10**5, 10**5, n).astype(np.int32)},
        {"type": R.TIME64_US, "valid": valid, "values": rng.integers(0, 86400 * 10**6, n)},
        {"type": R.TIMESTAMP_US, "valid": valid, "values": rng.integers(-10**16, 10**16, n)},
        {"type": R.TIMESTAMPTZ_US, "valid": valid, "values": rng.integers(-10**16, 10**16, n)},
        {"type": R.UUID, "valid": valid, "values": rng.integers(0, 256, (n, 16)).astype(np.uint8)},
        {"type": R.LIST, "valid": lvalid, "offsets": loffs,
         "child": {"type": R.INT32, "valid": rng.random(ne) > 0.3, "values": rng.integers(-5, 5, ne).astype(np.int32)}},
    ]
    fields = [(f"col_{i}", i + 1, 100 + i, 1 if i == 0 else 0) for i in range(len(cols))]
    return cols, fields


def _py(col, i):
    t = col["type"]
    if not col["valid"][i]:
        return None
    if t in (R.UTF8, R.LARGE_BINARY):
        b = col["data"][col["offsets"][i]:col["offsets"][i + 1]]
        return b.decode() if t == R.UTF8 else b
    if t == R.UUID:
        return bytes(col["values"][i])
    if t == R.LIST:
        kid = col["child"]
        return [_py(kid, k) for k in range(col["offsets"][i], col["offsets"][i + 1])]
    if t == R.BOOLEAN:
        return bool(col["values"][i])
    if t in (R.FLOAT32, R.FLOAT64):
        return float(col["values"][i])
    return int(col["values"][i])


def _same(a, b):
    if isinstance(a, float) and isinstance(b, float) and np.isnan(a) and np.isnan(b):
        return True
    if isinstance(a, float) and isinstance(b, float):
        return a == b and np.signbit(a) == np.signbit(b)
    return a == b


@pytest.mark.parametrize("n,rb,re", [(300, 0, 300), (45000, 123, 44000), (10, 4, 4)])
def test_restatement_reads_back_in_pyarrow(n, rb, re):
    import pyarrow as pa
    import pyarrow.parquet as pq
    cols, fields = sample_columns(n)
    data, metrics, _ = R.write(cols, fields, rb, re)
    pf = pq.ParquetFile(io.BytesIO(data))
    tab = pf.read()
    assert tab.num_rows == re - rb
    for i, (col, f) in enumerate(zip(cols, fields)):
        got = tab.column(i).combine_chunks()
        if isinstance(got.type, pa.BaseExtensionType):
            got = got.storage
        if pa.types.is_timestamp(got.type) or pa.types.is_time64(got.type):
            got = got.view(pa.int64())
        elif pa.types.is_date32(got.type):
            got = got.view(pa.int32())
        got = got.to_pylist()
        want = [_py(col, r) for r in range(rb, re)]
        assert len(got) == len(want)
        assert all((_same(x, y) if not isinstance(x, list) else x == y) for x, y in zip(got, want)), f[0]
        assert tab.schema.field(i).metadata[b"PARQUET:field_id"] == str(f[1]).encode()
    # types and repetitions as the contract states
    sch = pf.schema
    phys = [sch.column(i).physical_type for i in range(len(cols))]
    assert phys == ["INT64", "INT32", "BOOLEAN", "FLOAT", "DOUBLE", "BYTE_ARRAY", "BYTE_ARRAY", "INT32", "INT64", "INT64",
                    "INT64", "FIXED_LEN_BYTE_ARRAY", "INT32"]
    logical = [str(sch.column(i).logical_type) for i in range(len(cols))]
    assert logical[5] == "String" and logical[6] == "None" and logical[7] == "Date" and logical[11] == "UUID"
    assert "isAdjustedToUTC=false" in logical[8] and "isAdjustedToUTC=false" in logical[9] and "isAdjustedToUTC=true" in logical[10]
    assert [sch.column(i).max_definition_level for i in range(len(cols))] == [0] + [1] * 11 + [3]
    assert sch.column(12).max_repetition_level == 1
    el = tab.schema.field(12).type.value_field
    assert el.metadata[b"PARQUET:field_id"] == b"112" and el.nullable
    assert not tab.schema.field(0).nullable
    # statistics: null counts and min / max per row group, trusted for byte arrays thanks to column_orders
    md = pf.metadata
    assert md.num_row_groups == (1 if re > rb else 0)
    for g in range(md.num_row_groups):
        for i, col in enumerate(cols):
            st = md.row_group(g).column(i).statistics
            leaf = R.Leaf(col, fields[i])
            it0, it1 = leaf.items(rb, re)
            mn, mx, _ = leaf.stats(it0, it1)
            rep, dfn = leaf.levels(rb, re)
            assert st.null_count == int(np.count_nonzero(dfn < leaf.max_def)) if leaf.max_def else st.null_count == 0
            assert st.has_min_max == (mn is not None), fields[i][0]
    if re > rb:
        st = md.row_group(0).column(5).statistics
        assert st.has_min_max and st.min == min(x for x in (_py(cols[5], r) for r in range(rb, re)) if x is not None)
        st = md.row_group(0).column(4).statistics
        fin = [x for x in (_py(cols[4], r) for r in range(rb, re)) if x is not None and not np.isnan(x)]
        assert st.min == min(fin) and st.max == max(fin)
    # metrics are the file's: the long (> 64 byte) LargeBinary values leave no bounds; NaN counted
    assert metrics[6]["min"] is None or re - rb < 7
    assert metrics[4]["nan_count"] == sum(1 for r in range(rb, re) if cols[4]["valid"][r] and np.isnan(cols[4]["values"][r]))


def test_two_row_groups_and_pages():
    import pyarrow.parquet as pq
    n = (1 << 20) + 5
    cols = [{"type": R.INT32, "valid": np.arange(n) % 5 != 0, "values": (np.arange(n) % 1000).astype(np.int32)}]
    data, _, pages = R.write(cols, [("x", 7, 0, 0)], 0, n)
    md = pq.ParquetFile(io.BytesIO(data)).metadata
    assert md.num_row_groups == 2 and md.row_group(1).num_rows == 5
    assert len(pages) == -(-(1 << 20) // R.PAGE_ROWS) + 1
    assert pq.read_table(io.BytesIO(data)).column(0).null_count == n // 5 + 1


def test_rle_hybrid_known_answer():
    """the bit-packing example of the Parquet encoding spec: 0..7 at bit width 3 packs to 10001000 11000110 11111010"""
    assert R.levels_encode(list(range(8)), 3) == bytes([0x03, 0x88, 0xC6, 0xFA])
    assert R.levels_encode([1] * 100, 1) == bytes([0xC8, 0x01, 1])          # varint(100 << 1), value
    assert R.levels_encode([1, 1, 1], 1) == bytes([6, 1])
    assert R.levels_encode([1, 0, 1], 1) == bytes([3, 0b101])


def test_level_encoder_matches_restatement(host):
    rng = np.random.default_rng(11)
    cases = [np.zeros(0, np.uint8), np.ones(1, np.uint8), np.array([0, 1, 2, 3] * 3, np.uint8)]
    for n in (7, 8, 9, 63 * 8, 63 * 8 + 1, 64 * 8 + 3, 5000):
        for w in (1, 2):
            hi = (1 << w)
            cases.append(rng.integers(0, hi, n).astype(np.uint8))                     # mostly bit-packed
            runs = np.repeat(rng.integers(0, hi, n // 7 + 1), rng.integers(1, 40, n // 7 + 1))[:n].astype(np.uint8)
            cases.append(runs)                                                         # runs of every length
    out = C.create_string_buffer(1 << 16)
    for lv in cases:
        w = 2 if lv.size and lv.max() > 1 else 1
        k = host.emu_levels(lv.tobytes(), lv.size, w, out)
        assert out.raw[:k] == R.levels_encode(lv, w), (lv.size, w)
        assert k + 4 <= 14 + ((lv.size + 7) // 8) * (w + 2)                          # levels_bound


def test_page_header_matches_restatement(host):
    out = C.create_string_buffer(64)
    for u, c, nv in [(0, 0, 0), (1, 1, 1), (127, 128, 20000), (1 << 20, 12345, 1 << 21), (2**31 - 1, 2**31 - 1, 2**31 - 1)]:
        k = host.emu_page_header(u, c, nv, out)
        assert out.raw[:k] == R.page_header(u, c, nv) and k <= 48
        h, end = R.read_struct(out.raw[:k])
        assert end == k and h[2] == u and h[3] == c and h[5][1] == nv


def test_footer_matches_restatement(host):
    rng = np.random.default_rng(2)
    types = [R.BOOLEAN, R.INT32, R.INT64, R.FLOAT32, R.FLOAT64, R.UTF8, R.LARGE_BINARY, R.DATE32, R.TIME64_US, R.TIMESTAMP_US,
             R.TIMESTAMPTZ_US, R.UUID]
    for n_rg in (0, 1, 3):
        cols, fields = [], []
        for i, t in enumerate(types + types[:6]):
            is_list = i >= len(types)
            col = {"type": R.LIST, "child": {"type": t}} if is_list else {"type": t}
            cols.append(col)
            fields.append((f"f{i}" * (1 + i % 3), 10 + i, 500 + i, int(i % 4 == 0)))
        leaves = [R.Leaf(c, f) for c, f in zip(cols, fields)]
        emu = (C.c_byte * (40 * len(leaves)))()
        EmuLeaf = type("EmuLeaf", (C.Structure,), {"_fields_": [("name", C.c_char_p), ("field_id", C.c_int32), ("element_field_id", C.c_int32),
                                                                ("ptype", C.c_uint32), ("converted", C.c_int32), ("logical", C.c_uint32),
                                                                ("flags", C.c_uint32)]})
        EmuChunk = type("EmuChunk", (C.Structure,), {"_fields_": [("offset", C.c_uint64), ("num_values", C.c_uint64), ("usize", C.c_uint64),
                                                                  ("csize", C.c_uint64), ("null_count", C.c_uint64), ("min", C.c_char_p),
                                                                  ("max", C.c_char_p), ("min_len", C.c_uint32), ("max_len", C.c_uint32)]})
        emu = (EmuLeaf * len(leaves))()
        for e, L in zip(emu, leaves):
            e.name, e.field_id, e.element_field_id, e.ptype = L.name.encode(), L.field_id, L.element_field_id, R.PT[L.atype]
            e.converted, e.logical = R.CONVERTED.get(L.atype, -1), R.LOGICAL.get(L.atype, 0)
            e.flags = int(L.required) | (2 if L.is_list else 0) | (4 if L.atype == R.TIMESTAMPTZ_US else 0)
        chunks, rows = [], [int(rng.integers(1, 1 << 20)) for _ in range(n_rg)]
        ech = (EmuChunk * max(1, n_rg * len(leaves)))()
        for k in range(n_rg * len(leaves)):
            has = rng.random() > 0.3
            mn, mx = bytes(rng.integers(0, 256, int(rng.integers(0, 65))).astype(np.uint8)), bytes(rng.integers(0, 256, 8).astype(np.uint8))
            c = dict(offset=int(rng.integers(4, 2**40)), num_values=int(rng.integers(0, 2**30)), usize=int(rng.integers(0, 2**34)),
                     csize=int(rng.integers(0, 2**34)), null_count=int(rng.integers(0, 2**20)), min=mn if has else None, max=mx if has else None)
            chunks.append(c)
            e = ech[k]
            e.offset, e.num_values, e.usize, e.csize, e.null_count = c["offset"], c["num_values"], c["usize"], c["csize"], c["null_count"]
            e.min, e.max = mn, mx
            e.min_len, e.max_len = (len(mn), len(mx)) if has else (2**32 - 1, 0)
        rg = (C.c_uint64 * max(1, n_rg))(*rows)
        for codec in (0, 1):
            out = C.create_string_buffer(1 << 20)
            k = host.emu_footer(emu, len(leaves), rg, n_rg, ech, codec, out, 1 << 20)
            assert out.raw[:k] == R.footer(leaves, rows, chunks, codec), (n_rg, codec)


# ------------------------------------------------------------------------------------------------ Snappy fragments
def _snappy_cases():
    rng = np.random.default_rng(7)
    text = b"".join(b"%d\tuser-%d@example.org\t2024-01-%02d\n" % (i, i % 977, i % 28 + 1) for i in range(9000))
    arrowish = np.repeat(np.arange(40000, dtype=np.int64) // 7, 2).tobytes() + b"INSERT" * 20000 + b"0000000000000000/00000000000000%02x" % 3 * 3000
    cases = {f"zeros-{n}": bytes(n) for n in (0, 1, 2, 15, 16, 65535, 65536, 65537, 200000)}
    cases.update({f"random-{n}": rng.integers(0, 256, n).astype(np.uint8).tobytes() for n in (1, 5, 64, 4097, 65535, 65536, 65537, 300001)})
    cases["text"] = text
    cases["arrow"] = arrowish
    cases["mixed"] = text[:70000] + rng.integers(0, 256, 70000).astype(np.uint8).tobytes() + bytes(70000)
    cases["periodic"] = (b"abcdefghijklmnopqrstuvwxyz0123" * 20000)[:500000]
    for k in range(20):
        n = int(rng.integers(0, 150000))
        alpha = int(rng.integers(1, 256))
        cases[f"fuzz-{k}"] = rng.integers(0, alpha, n).astype(np.uint8).tobytes()
    return cases


def test_snappy_fragments_decompress_in_pyarrow(host):
    import pyarrow as pa
    codec = pa.Codec("snappy")
    for name, data in _snappy_cases().items():
        n = len(data)
        out = C.create_string_buffer(10 + (n // 65536 + 1) * (32 + 65536 + 65536 // 6))
        k = host.emu_snappy(data, n, out)
        comp = out.raw[:k]
        assert codec.decompress(comp, decompressed_size=n).to_pybytes() == data, name
        assert k <= 10 + sum(32 + f + f // 6 for f in [min(65536, n - o) for o in range(0, n, 65536)]), name
        if name == "periodic":
            assert k * 20 < n, (name, k)          # a literal-only encoder would be larger than the input
        if name == "arrow":
            assert k * 4 < n, (name, k)


# ------------------------------------------------------------------------------------------------ ABI mirror
def test_struct_layouts(tmp_path):
    pairs = [("etl_parquet_field", abi.ParquetField), ("etl_parquet_metrics", abi.ParquetMetrics)]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "etl_decode.h"', 'int main(void) {']
    for cname, ct in pairs:
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in ct._fields_:
            lines.append(f'  printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ['  printf("codecs %d %d %u\\n", ETL_PQ_UNCOMPRESSED, ETL_PQ_SNAPPY, ETL_PQ_HAS_MIN_MAX);', '  return 0;', '}']
    src = tmp_path / "pq_sizes.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "pq_sizes"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = dict(l.split(" ", 1) for l in subprocess.check_output([str(exe)], text=True).splitlines())
    for cname, ct in pairs:
        assert int(got[cname]) == C.sizeof(ct), cname
        for fname, _ in ct._fields_:
            assert int(got[f"{cname}.{fname}"]) == getattr(ct, fname).offset, f"{cname}.{fname}"
    assert got["codecs"] == f"{abi.PQ_UNCOMPRESSED} {abi.PQ_SNAPPY} {abi.PQ_HAS_MIN_MAX}"
