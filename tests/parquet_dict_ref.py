"""Python restatement of the Iceberg Parquet data file with ETL_PQ_DICTIONARY (include/etl_decode.h,
etl_dec_parquet_write): tests/parquet_ref.py's file, whose names it re-exports, with per-chunk dictionaries.  write(...,
dictionary=False) is parquet_ref's file; footer() and walk_pages() also take the dictionary chunk's fields."""
from __future__ import annotations

import struct

import numpy as np

from parquet_ref import *  # noqa: F401,F403  (the types, constants, Thrift writer / reader and leaves of the PLAIN file)
from parquet_ref import (BOOLEAN, LARGE_BINARY, NP, PT, ROW_GROUP_ROWS, UNCOMPRESSED, UTF8, UUID, WIDTH, CREATED_BY, Leaf,
                         TWriter, _schema_leaf, _uvar, file_footer, levels_encode, pages_of, read_struct)

DICTIONARY = 0x100                      # codec flag bit (ETL_PQ_DICTIONARY)
DICT_BYTES = 1 << 20                    # a chunk is dictionary-encoded while its entries' PLAIN size is at most this
RLE_DICTIONARY = 8


def page_header(usize, csize, num_values, encoding=0):
    """DATA_PAGE header; encoding PLAIN (0) or RLE_DICTIONARY (8)"""
    w = TWriter()
    w.i32(1, 0)
    w.i32(2, usize)
    w.i32(3, csize)
    w.begin(5)
    w.i32(1, num_values)
    w.i32(2, encoding)
    w.i32(3, 3)
    w.i32(4, 3)
    w.end()
    w.end()
    return bytes(w.out)


def dict_page_header(usize, csize, entries):
    """DICTIONARY_PAGE {type 2, sizes, dictionary_page_header (7) {num_values, encoding PLAIN}}"""
    w = TWriter()
    w.i32(1, 2)
    w.i32(2, usize)
    w.i32(3, csize)
    w.begin(7)
    w.i32(1, entries)
    w.i32(2, 0)
    w.end()
    w.end()
    return bytes(w.out)


def dict_width(entries):
    """bit width of the indices of a dictionary of this many entries"""
    return max(1, (entries - 1).bit_length())


def indices_encode(idx, w):
    """RLE / bit-packed hybrid of dictionary indices at bit width w (no bit-width byte, no length prefix), under the run
    rule of the levels; an RLE value takes ceil(w / 8) little-endian bytes"""
    x = np.asarray(idx, dtype=np.uint32)
    n = len(x)
    ng = (n + 7) // 8
    if not ng:
        return b""
    pad = np.zeros(ng * 8, dtype=np.uint32)
    pad[:n] = x
    g = pad.reshape(ng, 8)
    cls = np.where((g == g[:, :1]).all(axis=1), g[:, 0].astype(np.int64), -1)
    m = n - (ng - 1) * 8
    if m < 8:
        cls[-1] = g[-1, 0] if (g[-1, :m] == g[-1, 0]).all() else -1
    out = bytearray()
    k = 0
    while k < ng:
        c = int(cls[k])
        h = k + 1
        if c >= 0:
            while h < ng and cls[h] == c:
                h += 1
            cnt = (n if h == ng else h * 8) - k * 8
            out += _uvar(cnt << 1) + c.to_bytes((w + 7) // 8, "little")
        else:
            while h < ng and h - k < 63 and cls[h] < 0:
                h += 1
            out.append(((h - k) << 1) | 1)
            bits = np.unpackbits(pad[k * 8:h * 8].astype("<u4").view(np.uint8).reshape(-1, 4), axis=1, bitorder="little")
            out += np.packbits(bits[:, :w].reshape(-1), bitorder="little").tobytes()
        k = h
    return bytes(out)


def dictionary(leaf, it0, it1):
    """(entries as PLAIN bytes in first-occurrence order, the entry id of each present item of [it0, it1))"""
    v = leaf.vcol
    ok = np.nonzero(v["valid"][it0:it1])[0] + it0
    if leaf.atype in (UTF8, LARGE_BINARY):
        o, d = v["offsets"], v["data"]
        first = {}
        ids = np.array([first.setdefault(bytes(d[int(o[i]):int(o[i + 1])]), len(first)) for i in ok], dtype=np.uint32)
        return [struct.pack("<I", len(k)) + k for k in first], ids
    if not len(ok):
        return [], np.zeros(0, np.uint32)
    if leaf.atype == UUID:
        rows = np.ascontiguousarray(v["values"][ok]).view("<u8").reshape(-1, 2)
    else:
        rows = np.asarray(v["values"], dtype=NP[leaf.atype])[ok].view("<u4" if WIDTH[leaf.atype] == 4 else "<u8").reshape(-1, 1)
    u, first_at, inv = np.unique(rows, axis=0, return_index=True, return_inverse=True)     # bitwise: ±0, NaN payloads
    order = np.argsort(first_at, kind="stable")
    rank = np.empty(len(order), np.uint32)
    rank[order] = np.arange(len(order), dtype=np.uint32)
    return [u[k].tobytes() for k in order], rank[np.asarray(inv).reshape(-1)]


def chunk_dictionary(leaf, g0, g1):
    """(entries, ids) when the chunk of rows [g0, g1) is dictionary-encoded (a non-Boolean leaf with a present value whose
    entries' PLAIN size is at most DICT_BYTES), else None"""
    if leaf.atype == BOOLEAN:
        return None
    entries, ids = dictionary(leaf, *leaf.items(g0, g1))
    if not len(ids) or sum(len(e) for e in entries) > DICT_BYTES:
        return None
    return entries, ids


def page_payload(leaf, r0, r1, ids=None, width=0):
    """levels + PLAIN values, or with ids (the entry ids of the page's present items) the bit width and the index runs"""
    rep, dfn = leaf.levels(r0, r1)
    out = bytearray()
    if leaf.max_rep:
        b = levels_encode(rep, 1)
        out += struct.pack("<I", len(b)) + b
    if leaf.max_def:
        b = levels_encode(dfn, leaf.w)
        out += struct.pack("<I", len(b)) + b
    if ids is not None:
        out += bytes([width]) + indices_encode(ids, width)
    else:
        out += leaf.plain(*leaf.items(r0, r1))
    return bytes(out), len(dfn)


def footer(leaves, rg_rows, chunks, codec):
    """chunks: row-group major dicts {offset, num_values, usize, csize, null_count, min, max} and, for a dictionary chunk,
    dict=True, data_offset, data_pages; ColumnMetaData.codec is codec & 0xFF"""
    w = TWriter()
    w.i32(1, 1)
    w.list(2, 12, 1 + sum(3 if L.is_list else 1 for L in leaves))
    w.elem(); w.binary(4, b"schema"); w.i32(5, len(leaves)); w.end()
    for L in leaves:
        if not L.is_list:
            _schema_leaf(w, L, False)
            continue
        w.elem(); w.i32(3, 0 if L.required else 1); w.binary(4, L.name.encode()); w.i32(5, 1); w.i32(6, 3); w.i32(9, L.field_id)
        w.begin(10); w.begin(3); w.end(); w.end(); w.end()
        w.elem(); w.i32(3, 2); w.binary(4, b"list"); w.i32(5, 1); w.end()
        _schema_leaf(w, L, True)
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
            w.i32(1, PT[L.atype])
            levels = L.is_list or not L.required
            dic = c.get("dict", False)
            w.list(2, 5, (2 if levels else 1) + dic)
            w.var(0)
            if levels:
                w.var(6)
            if dic:
                w.var(RLE_DICTIONARY << 1)
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
                w.elem(); w.i32(1, 0); w.i32(2, RLE_DICTIONARY); w.i32(3, c["data_pages"]); w.end()
            w.end()
            w.end()
        w.i64(2, sum(c["usize"] for c in cs))
        w.i64(3, rows)
        w.i64(5, cs[0]["offset"])
        w.i64(6, sum(c["csize"] for c in cs))
        w.i16(7, g)
        w.end()
    w.binary(6, CREATED_BY)
    w.list(7, 12, nl)
    for _ in leaves:
        w.elem(); w.begin(1); w.end(); w.end()
    w.end()
    return bytes(w.out)


def write(cols, fields, row_begin, row_end, dictionary=False):
    """(uncompressed file bytes, metrics per leaf, pages [(chunk, header bytes, payload)]); dictionary: ETL_PQ_DICTIONARY"""
    leaves = [Leaf(c, f) for c, f in zip(cols, fields)]
    n = row_end - row_begin
    rg = [(row_begin + g, min(row_end, row_begin + g + ROW_GROUP_ROWS)) for g in range(0, n, ROW_GROUP_ROWS)]
    body = bytearray(b"PAR1")
    chunks, pages = [], []
    metrics = [dict(field_id=L.element_field_id if L.is_list else L.field_id, num_values=0, null_count=0, nan_count=0,
                    compressed_bytes=0, uncompressed_bytes=0, min=None, max=None) for L in leaves]
    for g0, g1 in rg:
        for li, L in enumerate(leaves):
            c = dict(offset=len(body), num_values=0, usize=0, csize=0, null_count=0)
            d = chunk_dictionary(L, g0, g1) if dictionary else None
            if d:
                payload = b"".join(d[0])
                hdr = dict_page_header(len(payload), len(payload), len(d[0]))
                pages.append((len(chunks), hdr, payload))
                body += hdr + payload
                c["usize"] += len(hdr) + len(payload)
                c.update(dict=True, data_offset=len(body), data_pages=0)
                width, seen = dict_width(len(d[0])), 0
            for r0, r1 in pages_of(L, g0, g1):
                it0, it1 = L.items(r0, r1)
                nn = int(np.count_nonzero(L.vcol["valid"][it0:it1]))
                if d:
                    payload, nv = page_payload(L, r0, r1, d[1][seen:seen + nn], width)
                    seen += nn
                    c["data_pages"] += 1
                else:
                    payload, nv = page_payload(L, r0, r1)
                hdr = page_header(len(payload), len(payload), nv, RLE_DICTIONARY if d else 0)
                pages.append((len(chunks), hdr, payload))
                body += hdr + payload
                c["num_values"] += nv
                c["null_count"] += nv - nn
                c["usize"] += len(hdr) + len(payload)
            c["csize"] = c["usize"]
            it0, it1 = L.items(g0, g1)
            c["min"], c["max"], nan = L.stats(it0, it1)
            m = metrics[li]
            for k in ("num_values", "null_count"):
                m[k] += c[k]
            m["nan_count"] += nan
            m["compressed_bytes"] += c["csize"]
            m["uncompressed_bytes"] += c["usize"]
            chunks.append(c)
    for li, L in enumerate(leaves):
        if n:
            metrics[li]["min"], metrics[li]["max"], _ = L.stats(*L.items(row_begin, row_end))
    foot = footer(leaves, [g1 - g0 for g0, g1 in rg], chunks, UNCOMPRESSED)
    body += foot + struct.pack("<I", len(foot)) + b"PAR1"
    return bytes(body), metrics, pages


def walk_pages(data):
    """every page of a file in order: (chunk index, parsed header, header bytes, payload); a dictionary chunk starts at its
    dictionary page"""
    fm, _ = file_footer(data)
    out = []
    ci = 0
    for rg in fm.get(4, []):
        for cc in rg[1]:
            md = cc[3]
            pos = md.get(11, md[9])
            end = pos + md[7]
            while pos < end:
                h, p2 = read_struct(data, pos)
                out.append((ci, h, bytes(data[pos:p2]), bytes(data[p2:p2 + h[3]])))
                pos = p2 + h[3]
            assert pos == end
            ci += 1
    return out
