"""CPU checks of the Parquet writer's dictionary encoding (ETL_PQ_DICTIONARY): the Python restatement
(tests/parquet_dict_ref.py, dictionary=True) read back by pyarrow with its dictionary metadata, the dictionary pages against a
first-occurrence list computed here and the data pages decoded by this file's own hybrid reader, the index hybrid
against hand-worked runs, the device's byte-level pieces compiled for the host (tests/emul/host_parquet_dict.cpp) against the
restatement, and the per-chunk decision at its edges."""
import ctypes as C
import io
import os
import struct
import subprocess
import tempfile

import numpy as np
import pytest

import parquet_dict_ref as R
from etl_b200 import abi
from test_parquet_cpu import _py, _same, sample_columns

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def host():
    out_dir = tempfile.mkdtemp(prefix="etl_host_parquet_dict_")
    so = os.path.join(out_dir, "libhost_parquet.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           "-I", os.path.join(ROOT, "etl_b200", "csrc"), "-o", so, os.path.join(HERE, "emul", "host_parquet_dict.cpp")])
    lib = C.CDLL(so)
    lib.emu_indices.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p]
    lib.emu_indices.restype = C.c_uint64
    lib.emu_dict_page_header.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
    lib.emu_dict_page_header.restype = C.c_uint32
    lib.emu_page_header_enc.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
    lib.emu_page_header_enc.restype = C.c_uint32
    lib.emu_footer_dict.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_uint32, C.c_void_p, C.c_uint64]
    lib.emu_footer_dict.restype = C.c_uint64
    return lib


# ------------------------------------------------------------------------------------------------ an independent reader
def hybrid_decode(buf, w, n):
    """the first n values of an RLE / bit-packed hybrid stream at bit width w"""
    out, pos = [], 0
    while len(out) < n:
        h, s = 0, 0
        while True:
            b = buf[pos]
            pos += 1
            h |= (b & 0x7F) << s
            s += 7
            if b < 0x80:
                break
        if h & 1:
            nbytes = (h >> 1) * w
            bits = int.from_bytes(bytes(buf[pos:pos + nbytes]), "little")
            out += [(bits >> (w * k)) & ((1 << w) - 1) for k in range((h >> 1) * 8)]
            pos += nbytes
        else:
            vb = (w + 7) // 8
            out += [int.from_bytes(bytes(buf[pos:pos + vb]), "little")] * (h >> 1)
            pos += vb
    return out[:n], pos


def split_entries(payload, leaf):
    """the PLAIN entries of a dictionary page (byte arrays without their length)"""
    if leaf.atype in (R.UTF8, R.LARGE_BINARY):
        out, pos = [], 0
        while pos < len(payload):
            k = struct.unpack_from("<I", payload, pos)[0]
            out.append(payload[pos + 4:pos + 4 + k])
            pos += 4 + k
        return out
    w = R.WIDTH[leaf.atype]
    return [payload[k:k + w] for k in range(0, len(payload), w)]


def present_keys(leaf, it0, it1):
    """PLAIN bytes (byte arrays: the bytes) of the present items, in item order"""
    v = leaf.vcol
    ok = np.nonzero(v["valid"][it0:it1])[0] + it0
    if leaf.atype in (R.UTF8, R.LARGE_BINARY):
        return [bytes(v["data"][int(v["offsets"][i]):int(v["offsets"][i + 1])]) for i in ok]
    if leaf.atype == R.UUID:
        return [bytes(v["values"][i]) for i in ok]
    raw = np.asarray(v["values"], dtype=R.NP[leaf.atype])[ok]
    return [x.tobytes() for x in raw]


def first_occurrence(keys):
    """distinct keys ordered by first occurrence: numpy's unique over the bytes, its first indices in item order"""
    if not keys:
        return []
    arr = np.empty(len(keys), dtype=object)
    arr[:] = keys
    _, first = np.unique(arr, return_index=True)
    return [keys[i] for i in np.sort(first)]


def check_dictionary_file(data, cols, fields, rb, re):
    """every dictionary chunk: its page holds the first-occurrence list, its data pages decode to the values"""
    pages = R.walk_pages(data)
    fm, _ = R.file_footer(data)
    leaves = [R.Leaf(c, f) for c, f in zip(cols, fields)]
    nl = len(leaves)
    rgs = [(rb + g, min(re, rb + g + R.ROW_GROUP_ROWS)) for g in range(0, re - rb, R.ROW_GROUP_ROWS)]
    n_dict = 0
    for ci in range(len(rgs) * nl):
        L, (g0, g1) = leaves[ci % nl], rgs[ci // nl]
        md = fm[4][ci // nl][1][ci % nl][3]
        mine = [p for p in pages if p[0] == ci]
        if 11 not in md:
            assert all(h[1] == 0 and h[5][2] == 0 for _, h, _, _ in mine)
            continue
        n_dict += 1
        _, h, _, payload = mine[0]
        assert h[1] == 2 and h[7][2] == 0 and md[11] == fm[4][ci // nl][1][ci % nl][2]
        entries = split_entries(payload, L)
        keys = present_keys(L, *L.items(g0, g1))
        assert entries == first_occurrence(keys) and h[7][1] == len(entries)
        assert md[2][-1] == R.RLE_DICTIONARY and md[13] == [{1: 2, 2: 0, 3: 1}, {1: 0, 2: 8, 3: len(mine) - 1}]
        w = max(1, (len(entries) - 1).bit_length())
        got = []
        for _, hd, _, body in mine[1:]:
            assert hd[1] == 0 and hd[5][2] == R.RLE_DICTIONARY
            pos = 0
            for _ in range((L.max_rep > 0) + (L.max_def > 0)):
                pos += 4 + struct.unpack_from("<I", body, pos)[0]
            assert body[pos] == w
            nn = hd[5][1] if not L.max_def else None
            if nn is None:                                   # present values: the entries at max definition level
                lv_pos = 4 + struct.unpack_from("<I", body, 0)[0] if L.max_rep else 0
                dlen = struct.unpack_from("<I", body, lv_pos)[0]
                dfn, _ = hybrid_decode(body[lv_pos + 4:lv_pos + 4 + dlen], L.w, hd[5][1])
                nn = sum(1 for x in dfn if x == L.max_def)
            ids, used = hybrid_decode(body[pos + 1:], w, nn)
            assert pos + 1 + used == len(body)
            got += [entries[i] for i in ids]
        assert got == keys
    return n_dict


# ------------------------------------------------------------------------------------------------ the restatement vs pyarrow
def low_cardinality(n, seed=4):
    rng = np.random.default_rng(seed)
    valid = rng.random(n) > 0.1
    words = [b"active", b"pending", b"shipped", b"cancelled", b"", b"returned", b"x" * 70]
    pick = [words[k] for k in rng.integers(0, len(words), n)]
    offs = np.concatenate([[0], np.cumsum([len(v) if ok else 0 for v, ok in zip(pick, valid)])]).astype(np.int64)
    pool = rng.integers(0, 256, (5, 16)).astype(np.uint8)
    lvalid = rng.random(n) > 0.1
    lens = np.where(lvalid, rng.integers(0, 5, n), 0)          # a null list has no elements, as in an Arrow emit
    loffs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    ne = int(loffs[-1])
    tags = [b"red", b"green", b"blue"]
    tpick = [tags[k] for k in rng.integers(0, 3, ne)]
    tvalid = rng.random(ne) > 0.05
    toffs = np.concatenate([[0], np.cumsum([len(v) if ok else 0 for v, ok in zip(tpick, tvalid)])]).astype(np.int64)
    cols = [
        {"type": R.UTF8, "valid": valid, "offsets": offs, "data": b"".join(v for v, ok in zip(pick, valid) if ok)},
        {"type": R.INT32, "valid": valid, "values": rng.integers(0, 12, n).astype(np.int32)},
        {"type": R.DATE32, "valid": np.ones(n, bool), "values": (19000 + rng.integers(0, 30, n)).astype(np.int32)},
        {"type": R.UUID, "valid": valid, "values": pool[rng.integers(0, 5, n)]},
        {"type": R.LIST, "valid": lvalid, "offsets": loffs,
         "child": {"type": R.UTF8, "valid": tvalid, "offsets": toffs, "data": b"".join(v for v, ok in zip(tpick, tvalid) if ok)}},
        {"type": R.BOOLEAN, "valid": valid, "values": rng.random(n) > 0.5},
    ]
    fields = [(f"lc_{i}", 50 + i, 150 + i, 1 if i == 2 else 0) for i in range(len(cols))]
    return cols, fields


def _read_back(data, cols, fields, rb, re):
    import pyarrow as pa
    import pyarrow.parquet as pq
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
        assert all((_same(x, y) if not isinstance(x, list) else x == y) for x, y in zip(got, want)), f[0]
        assert tab.schema.field(i).metadata[b"PARQUET:field_id"] == str(f[1]).encode()
    return pf.metadata


@pytest.mark.parametrize("n,rb,re", [(300, 0, 300), (45000, 123, 44000), (10, 4, 4)])
def test_restatement_reads_back_in_pyarrow(n, rb, re):
    for cols, fields in (sample_columns(n), low_cardinality(n)):
        data, metrics, _ = R.write(cols, fields, rb, re, dictionary=True)
        md = _read_back(data, cols, fields, rb, re)
        plain, plain_m, _ = R.write(cols, fields, rb, re)
        for g in range(md.num_row_groups):
            for i, col in enumerate(cols):
                cc = md.row_group(g).column(i)
                leaf = R.Leaf(col, fields[i])
                dic = R.chunk_dictionary(leaf, rb, re) is not None
                assert cc.has_dictionary_page == dic, fields[i][0]
                levels = leaf.max_def > 0
                want = ("PLAIN",) + (("RLE",) if levels else ()) + (("RLE_DICTIONARY",) if dic else ())
                assert sorted(cc.encodings) == sorted(want), (fields[i][0], cc.encodings)
                if dic:
                    assert cc.dictionary_page_offset < cc.data_page_offset
                else:
                    assert leaf.atype == R.BOOLEAN or not leaf.vcol["valid"][slice(*leaf.items(rb, re))].any()
        # metrics: counts and bounds as without the dictionary, sizes with its page
        for m, p in zip(metrics, plain_m):
            assert {k: v for k, v in m.items() if not k.endswith("_bytes")} == {k: v for k, v in p.items() if not k.endswith("_bytes")}
        if re > rb:
            assert check_dictionary_file(data, cols, fields, rb, re) > 0


def test_without_the_flag_is_the_plain_restatement():
    import parquet_ref
    for cols, fields in (sample_columns(3000), low_cardinality(3000)):
        for rb, re in ((0, 3000), (17, 2500), (5, 5)):
            d, dm, dp = R.write(cols, fields, rb, re)
            p, pm, pp = parquet_ref.write(cols, fields, rb, re)
            assert d == p and dm == pm and dp == pp


def test_low_cardinality_shrinks():
    cols, fields = low_cardinality(50000)
    d, _, _ = R.write(cols, fields, 0, 50000, dictionary=True)
    p, _, _ = R.write(cols, fields, 0, 50000)
    assert len(d) * 3 < len(p)


def test_two_row_groups_each_their_own_dictionary():
    n = (1 << 20) + 5
    cols = [{"type": R.INT32, "valid": np.arange(n) % 5 != 0, "values": (np.arange(n) % 1000).astype(np.int32)}]
    data, _, pages = R.write(cols, [("x", 7, 0, 0)], 0, n, dictionary=True)
    md = _read_back(data, cols, [("x", 7, 0, 0)], 0, n)
    assert md.num_row_groups == 2 and all(md.row_group(g).column(0).has_dictionary_page for g in range(2))
    assert check_dictionary_file(data, cols, [("x", 7, 0, 0)], 0, n) == 2
    ents = [len(split_entries(p[2], R.Leaf(cols[0], ("x", 7, 0, 0)))) for p in pages if R.read_struct(p[1])[0][1] == 2]
    assert ents == [800, 4]          # values 0..999 but the multiples of 5 (always null); rows 2^20 .. 2^20 + 4: 576..580, 580 null


# ------------------------------------------------------------------------------------------------ the index hybrid
HAND = [
    (1, [1] * 8, "1001"),                                   # one RLE run of 8: varint(16), 1 value byte
    (1, [0, 1] * 4, "03aa"),                                # one bit-packed group: 0b10101010
    (2, [0, 1, 2, 3, 3, 2, 1, 0], "03e41b"),
    (8, [200] * 20, "28c8"),                                # 20 entries, partial last group, one run
    (9, [256] * 8 + list(range(8)), "1000010300" + "02081840a0808103"),
    (17, [65541] * 3, "06050001"),                          # value in 3 bytes
    (18, [(1 << 18) - 1] + [0] * 7 + [1], "03" + "ffff03" + "00" * 15 + "02010000"),
]


@pytest.mark.parametrize("w,idx,hexed", HAND)
def test_index_hybrid_hand_worked(w, idx, hexed, host):
    want = bytes.fromhex(hexed)
    assert R.indices_encode(idx, w) == want
    x = np.asarray(idx, dtype=np.uint32)
    out = C.create_string_buffer(4096)
    k = host.emu_indices(x.ctypes.data, len(x), w, out)
    assert out.raw[:k] == want
    assert hybrid_decode(want, w, len(idx))[0] == list(idx)


def test_index_hybrid_stretch_of_64_groups_is_two_runs():
    idx = np.tile(np.arange(8, dtype=np.uint32), 64)          # 64 non-uniform groups: 63 + 1
    enc = R.indices_encode(idx, 3)
    assert enc[0] == (63 << 1) | 1 and enc[1 + 63 * 3] == 3 and len(enc) == 2 + 64 * 3


def test_device_pieces_match_restatement(host):
    rng = np.random.default_rng(8)
    out = C.create_string_buffer(1 << 22)
    for w in (1, 2, 3, 7, 8, 9, 12, 16, 17, 18):
        hi = 1 << w
        for n in (0, 1, 7, 8, 9, 63 * 8, 63 * 8 + 1, 64 * 8 + 3, 20000):
            for runs in (False, True):
                x = (np.repeat(rng.integers(0, hi, n // 5 + 1), rng.integers(1, 60, n // 5 + 1))[:n] if runs
                     else rng.integers(0, hi, n)).astype(np.uint32)
                k = host.emu_indices(x.ctypes.data, n, w, out)
                assert out.raw[:k] == R.indices_encode(x, w), (w, n, runs)
                assert k + 1 <= 1 + ((n + 7) // 8) * 19                       # indices_bound
                assert hybrid_decode(out.raw[:k], w, n)[0] == x.tolist()
    for u, c, e in [(0, 0, 0), (1, 1, 1), (1 << 20, 12345, 262144), (2**31 - 1, 2**31 - 1, 2**31 - 1)]:
        k = host.emu_dict_page_header(u, c, e, out)
        assert out.raw[:k] == R.dict_page_header(u, c, e) and k <= 25
        h, end = R.read_struct(out.raw[:k])
        assert end == k and h == {1: 2, 2: u, 3: c, 7: {1: e, 2: 0}}
        k = host.emu_page_header_enc(u, c, e, 8, out)
        assert out.raw[:k] == R.page_header(u, c, e, 8) and k <= 48


def test_footer_with_dictionary_chunks_matches_restatement(host):
    rng = np.random.default_rng(9)
    types = [R.BOOLEAN, R.INT32, R.UTF8, R.UUID, R.FLOAT64]
    cols = [{"type": t} for t in types] + [{"type": R.LIST, "child": {"type": R.INT64}}]
    fields = [(f"d{i}", 10 + i, 500 + i, int(i % 2 == 0)) for i in range(len(cols))]
    leaves = [R.Leaf(c, f) for c, f in zip(cols, fields)]
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
        e.flags = int(L.required) | (2 if L.is_list else 0)
    for n_rg in (1, 2):
        nc = n_rg * len(leaves)
        ech = (EmuChunk * nc)()
        dic = (C.c_uint8 * nc)()
        doff, dpages = (C.c_uint64 * nc)(), (C.c_uint64 * nc)()
        chunks = []
        for k in range(nc):
            mn, mx = b"\x01\x02", b"\x09"
            c = dict(offset=int(rng.integers(4, 2**40)), num_values=int(rng.integers(0, 2**30)), usize=int(rng.integers(0, 2**34)),
                     csize=int(rng.integers(0, 2**34)), null_count=int(rng.integers(0, 2**20)), min=mn, max=mx)
            if k % len(leaves) and rng.random() > 0.3:
                c.update(dict=True, data_offset=c["offset"] + int(rng.integers(1, 2**20)), data_pages=int(rng.integers(1, 2**31)))
                dic[k], doff[k], dpages[k] = 1, c["data_offset"], c["data_pages"]
            chunks.append(c)
            e = ech[k]
            e.offset, e.num_values, e.usize, e.csize, e.null_count = c["offset"], c["num_values"], c["usize"], c["csize"], c["null_count"]
            e.min, e.max, e.min_len, e.max_len = mn, mx, len(mn), len(mx)
        rows = (C.c_uint64 * n_rg)(*[1000] * n_rg)
        for codec in (0, 1, 0x100, 0x101):
            out = C.create_string_buffer(1 << 20)
            k = host.emu_footer_dict(emu, len(leaves), rows, n_rg, ech, dic, doff, dpages, codec, out, 1 << 20)
            want = R.footer(leaves, [1000] * n_rg, chunks, codec)
            assert out.raw[:k] == want, (n_rg, codec)
            fm, _ = R.read_struct(want)
            assert all(cc[3][4] == codec & 0xFF for rg in fm[4] for cc in rg[1])


# ------------------------------------------------------------------------------------------------ the decision at its edges
def _utf8(vals, valid=None):
    valid = np.ones(len(vals), bool) if valid is None else valid
    offs = np.concatenate([[0], np.cumsum([len(v) if ok else 0 for v, ok in zip(vals, valid)])]).astype(np.int64)
    return {"type": R.UTF8, "valid": valid, "offsets": offs, "data": b"".join(v for v, ok in zip(vals, valid) if ok)}


@pytest.mark.parametrize("extra,dic", [(0, True), (1, False)])
def test_decision_at_one_mib(extra, dic):
    # 16 distinct values of 65 532 (+ extra on the last) bytes, each repeated: 16 × (4 + 65 532) = 1 048 576 (+ extra)
    distinct = [bytes([65 + k]) * (65532 + (extra if k == 15 else 0)) for k in range(16)]
    vals = [distinct[k % 16] for k in range(40)]
    cols, fields = [_utf8(vals), {"type": R.INT32, "valid": np.ones(40, bool), "values": np.zeros(40, np.int32)}], [("s", 1, 0, 0), ("z", 2, 0, 1)]
    data, _, _ = R.write(cols, fields, 0, 40, dictionary=True)
    md = _read_back(data, cols, fields, 0, 40)
    assert md.row_group(0).column(0).has_dictionary_page == dic and md.row_group(0).column(1).has_dictionary_page
    check_dictionary_file(data, cols, fields, 0, 40)
    if not dic:                                              # the fallen-back chunk is the PLAIN chunk, byte for byte
        plain, _, _ = R.write(cols, fields, 0, 40)
        fm, _ = R.file_footer(plain)
        md0 = fm[4][0][1][0][3]
        assert data[4:4 + md0[7]] == plain[4:4 + md0[7]]
        only, _, _ = R.write(cols[:1], fields[:1], 0, 40, dictionary=True)
        assert only == R.write(cols[:1], fields[:1], 0, 40)[0]


@pytest.mark.parametrize("entries", [1, 2, 256, 257, 65537])
def test_entry_counts_and_bit_widths(entries):
    n = max(3 * entries, 30000)
    vals = (np.arange(n) % entries * 7 - 3).astype(np.int32)
    cols, fields = [{"type": R.INT32, "valid": np.arange(n) % 13 != 0, "values": vals}], [("v", 1, 0, 0)]
    data, _, pages = R.write(cols, fields, 0, n, dictionary=True)
    _read_back(data, cols, fields, 0, n)
    assert check_dictionary_file(data, cols, fields, 0, n) == 1
    dh = R.read_struct(pages[0][1])[0]
    assert dh[7][1] == entries
    w = max(1, (entries - 1).bit_length())
    assert w == {1: 1, 2: 1, 256: 8, 257: 9, 65537: 17}[entries]


def test_single_value_and_all_null_page():
    n = 45000
    valid = np.arange(n) >= 20000                            # the first page (20 000 rows) has no value
    cols = [{"type": R.INT64, "valid": valid, "values": np.full(n, 42, np.int64)}]
    fields = [("one", 1, 0, 0)]
    data, _, pages = R.write(cols, fields, 0, n, dictionary=True)
    _read_back(data, cols, fields, 0, n)
    assert check_dictionary_file(data, cols, fields, 0, n) == 1
    assert pages[0][2] == struct.pack("<q", 42)
    first = pages[1][2]
    dlen = struct.unpack_from("<I", first)[0]
    assert first[4 + dlen:] == bytes([1])                    # levels, then only the bit-width byte
    assert pages[2][2].endswith(bytes([1]) + R.indices_encode([0] * 20000, 1))


def test_float_zero_signs_and_nan_payloads_bitwise():
    bits = np.array([0, 0x8000000000000000, 0x7FF8000000000001, 0x7FF8000000000001, 0x7FF8000000000002, 0, 0x3FF0000000000000],
                    dtype=np.uint64)
    f64 = bits.view(np.float64)
    f32 = np.array([0, 0x80000000, 0x7FC00001, 0x7FC00001, 0x7FC00002, 0, 0x3F800000], dtype=np.uint32).view(np.float32)
    cols = [{"type": R.FLOAT64, "valid": np.ones(7, bool), "values": f64}, {"type": R.FLOAT32, "valid": np.ones(7, bool), "values": f32}]
    fields = [("d", 1, 0, 0), ("f", 2, 0, 0)]
    data, metrics, pages = R.write(cols, fields, 0, 7, dictionary=True)
    assert check_dictionary_file(data, cols, fields, 0, 7) == 2
    assert len(split_entries(pages[0][2], R.Leaf(cols[0], fields[0]))) == 5     # +0, -0, two NaN payloads, 1.0
    assert metrics[0]["nan_count"] == 3 and metrics[1]["nan_count"] == 3
    import pyarrow.parquet as pq
    tab = pq.read_table(io.BytesIO(data))
    assert tab.column(0).to_numpy().view(np.uint64).tolist() == bits.tolist()
    assert tab.column(1).to_numpy().view(np.uint32).tolist() == f32.view(np.uint32).tolist()


def test_flag_constant():
    src = os.path.join(tempfile.mkdtemp(prefix="pq_flag_"), "f.c")
    with open(src, "w") as fh:
        fh.write('#include <stdio.h>\n#include "etl_decode.h"\nint main(void) { printf("%u", (unsigned)ETL_PQ_DICTIONARY); return 0; }\n')
    exe = src[:-2]
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", exe, src])
    assert int(subprocess.check_output([exe], text=True)) == abi.PQ_DICTIONARY == R.DICTIONARY == 0x100
