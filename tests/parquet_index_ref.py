"""Python restatement of the Parquet page index the writer adds with ETL_PQ_PAGE_INDEX (include/etl_decode.h,
etl_dec_parquet_write): each column chunk's ColumnIndex and OffsetIndex, computed from a file's page walk and the emit's
columns, and the file with them (with_index).  The file without the flag comes from tests/parquet_ref.py /
tests/parquet_dict_ref.py (uncompressed) or from the device (any codec); bytes [0, 4 + data end) stay as they are.

It carries its own Thrift compact reader: a list<bool> element is one byte (0x01 true, 0x02 false), which
parquet_ref._read_value does not consume."""
from __future__ import annotations

import struct

import numpy as np

import parquet_ref as PR
from parquet_ref import BOOLEAN, FLOAT32, FLOAT64, LARGE_BINARY, NP, ROW_GROUP_ROWS, UTF8, UUID, Leaf, TWriter

PAGE_INDEX = 0x400                      # codec flag bit (ETL_PQ_PAGE_INDEX)
TRUNCATE = 64                           # arrow-rs's column_index_truncate_length
UNORDERED, ASCENDING, DESCENDING = 0, 1, 2


# ------------------------------------------------------------------------------------------------ Thrift compact reader
def _var(buf, pos):
    v = s = 0
    while True:
        b = buf[pos]
        pos += 1
        v |= (b & 0x7F) << s
        s += 7
        if b < 0x80:
            return v, pos


def _value(buf, pos, t, in_list, ends, path):
    if t in (1, 2):
        if in_list:                                       # a list<bool> element: one byte
            return buf[pos] == 1, pos + 1
        return t == 1, pos
    if t in (3, 4, 5, 6):
        v, pos = _var(buf, pos)
        return (v >> 1) ^ -(v & 1), pos
    if t == 8:
        n, pos = _var(buf, pos)
        return bytes(buf[pos:pos + n]), pos + n
    if t == 9:
        h = buf[pos]
        pos += 1
        n, et = h >> 4, h & 0x0F
        if n == 15:
            n, pos = _var(buf, pos)
        items = []
        for _ in range(n):
            v, pos = _value(buf, pos, et, True, ends, path)
            items.append(v)
        return items, pos
    if t == 12:
        return read_struct(buf, pos, ends, path)
    raise ValueError(f"thrift type {t}")


def read_struct(buf, pos=0, ends=None, path=()):
    """one compact struct: ({field id: value}, next position).  With ends, the position of the stop byte of every
    ColumnChunk of a FileMetaData (path (4, 1)) is appended to it."""
    out, last = {}, 0
    while True:
        b = buf[pos]
        pos += 1
        if b == 0:
            if ends is not None and path == (4, 1):
                ends.append(pos - 1)
            return out, pos
        t, d = b & 0x0F, b >> 4
        if d:
            fid = last + d
        else:
            v, pos = _var(buf, pos)
            fid = (v >> 1) ^ -(v & 1)
        last = fid
        out[fid], pos = _value(buf, pos, t, False, ends, path + (fid,))


def parse(buf, offset, length):
    """the struct at [offset, offset + length), which must end exactly there"""
    s, end = read_struct(buf, offset)
    assert end == offset + length, (offset, length, end)
    return s


def file_footer(data):
    """(parsed FileMetaData, its offset, the stop-byte positions of its ColumnChunks)"""
    assert data[:4] == b"PAR1" and data[-4:] == b"PAR1"
    n = struct.unpack("<I", data[-8:-4])[0]
    at = len(data) - 8 - n
    ends = []
    fm, end = read_struct(data, at, ends)
    assert end == len(data) - 8
    return fm, at, ends


def page_walk(data):
    """per column chunk (row-group major): [(page type, file offset, file bytes)] of its pages"""
    fm, _, _ = file_footer(data)
    out = []
    for rg in fm.get(4, []):
        for cc in rg[1]:
            md = cc[3]
            pos = md.get(11, md[9])
            end = pos + md[7]
            pages = []
            while pos < end:
                h, p2 = read_struct(data, pos)
                pages.append((h[1], pos, p2 + h[3] - pos))
                pos = p2 + h[3]
            assert pos == end
            out.append(pages)
    return out


# ------------------------------------------------------------------------------------------------ bounds
def _boundary(b, i):
    return i >= len(b) or (b[i] & 0xC0) != 0x80


def truncate_min(b, utf8):
    """ColumnIndex minimum of a byte-array bound: itself up to 64 bytes, else its first 64 bytes (Utf8: the longest
    prefix of at most 64 bytes ending on a character boundary)"""
    b = bytes(b)
    if len(b) <= TRUNCATE:
        return b
    if not utf8:
        return b[:TRUNCATE]
    return b[:max(i for i in range(1, TRUNCATE + 1) if _boundary(b, i))]


def truncate_max(b, utf8):
    """ColumnIndex maximum of a byte-array bound: itself up to 64 bytes; else binary: the first 64 bytes with the last
    incremented, 0xFF carrying as 0x00; Utf8: the prefix to the last character boundary <= 64, cut after its last
    character whose code point + 1 is a scalar value of the same UTF-8 length, incremented.  Nothing to increment:
    the value itself."""
    b = bytes(b)
    if len(b) <= TRUNCATE:
        return b
    if not utf8:
        x = bytearray(b[:TRUNCATE])
        for i in range(TRUNCATE - 1, -1, -1):
            if x[i] != 0xFF:
                x[i] += 1
                return bytes(x)
            x[i] = 0
        return b
    prefix = b[:max(i for i in range(TRUNCATE - 3, TRUNCATE + 1) if _boundary(b, i))].decode()
    for k in range(len(prefix) - 1, -1, -1):
        nx = ord(prefix[k]) + 1
        if nx <= 0x10FFFF and not 0xD800 <= nx <= 0xDFFF and len(chr(nx).encode()) == len(prefix[k].encode()):
            return (prefix[:k] + chr(nx)).encode()
    return b


def page_bounds(leaf, it0, it1):
    """(non-null values, bounds) of items [it0, it1): bounds None for a null page, "nan" when every non-null value is
    NaN, else (min key, max key, min bytes, max bytes) with the untruncated PLAIN statistic bytes"""
    v = leaf.vcol
    ok = np.nonzero(v["valid"][it0:it1])[0] + it0
    if not len(ok):
        return 0, None
    t = leaf.atype
    if t in (UTF8, LARGE_BINARY):
        o, d = v["offsets"], v["data"]
        vals = [bytes(d[int(o[i]):int(o[i + 1])]) for i in ok]
        mn, mx = min(vals), max(vals)
        return len(ok), (mn, mx, mn, mx)
    if t == UUID:
        vals = [bytes(v["values"][i]) for i in ok]
        mn, mx = min(vals), max(vals)
        return len(ok), (mn, mx, mn, mx)
    if t == BOOLEAN:
        vals = np.asarray(v["values"])[ok].astype(np.uint8)
        mn, mx = int(vals.min()), int(vals.max())
        return len(ok), (mn, mx, bytes([mn]), bytes([mx]))
    vals = np.asarray(v["values"], dtype=NP[t])[ok]
    if t in (FLOAT32, FLOAT64):
        vals = vals[~np.isnan(vals)]
        if not len(vals):
            return len(ok), "nan"
        mn, mx = vals.min(), vals.max()
        mnb = np.array(-0.0 if mn == 0 else mn, dtype=NP[t]).tobytes()
        mxb = np.array(0.0 if mx == 0 else mx, dtype=NP[t]).tobytes()
        return len(ok), (float(mn), float(mx), mnb, mxb)
    mn, mx = vals.min(), vals.max()
    return len(ok), (int(mn), int(mx), mn.tobytes(), mx.tobytes())


def level_entries(leaf, r0, r1):
    if not leaf.is_list:
        return r1 - r0
    o = np.asarray(leaf.col["offsets"], dtype=np.int64)[r0:r1 + 1]
    n = np.diff(o)
    return int(np.where(np.asarray(leaf.col["valid"][r0:r1]) & (n > 0), n, 1).sum())


def boundary_order(bounds):
    """arrow-rs's two flags over consecutive non-null pages, on the untruncated bounds"""
    asc = desc = True
    prev = None
    for b in bounds:
        if b is None:
            continue
        if prev is not None:
            if b[0] < prev[0] or b[1] < prev[1]:
                asc = False
            if b[0] > prev[0] or b[1] > prev[1]:
                desc = False
        prev = b
    return ASCENDING if asc else DESCENDING if desc else UNORDERED


def column_index_fields(leaf, rows):
    """ColumnIndex fields {1 null_pages, 2 min_values, 3 max_values, 4 boundary_order, 5 null_counts} of the data pages
    with row ranges rows, or None when a page's non-null values are all NaN"""
    utf8 = leaf.atype == UTF8
    byte_array = leaf.atype in (UTF8, LARGE_BINARY)
    nulls, mins, maxs, ncs, bounds = [], [], [], [], []
    for r0, r1 in rows:
        nn, b = page_bounds(leaf, *leaf.items(r0, r1))
        if b == "nan":
            return None
        nulls.append(b is None)
        bounds.append(b)
        mins.append(b"" if b is None else truncate_min(b[2], utf8) if byte_array else b[2])
        maxs.append(b"" if b is None else truncate_max(b[3], utf8) if byte_array else b[3])
        ncs.append(level_entries(leaf, r0, r1) - nn)
    return {1: nulls, 2: mins, 3: maxs, 4: boundary_order(bounds), 5: ncs}


def column_index_bytes(ci):
    w = TWriter()
    k = len(ci[1])
    w.list(1, 1, k)
    w.out += bytes(1 if x else 2 for x in ci[1])
    for fid in (2, 3):
        w.list(fid, 8, k)
        for b in ci[fid]:
            w.var(len(b))
            w.out += b
    w.i32(4, ci[4])
    w.list(5, 6, k)
    for x in ci[5]:
        w.var(TWriter.zz(x))
    w.end()
    return bytes(w.out)


def offset_index_bytes(locs):
    """locs: [(file offset, file bytes, first row in the row group)] of the data pages"""
    w = TWriter()
    w.list(1, 12, len(locs))
    for off, size, first in locs:
        w.elem()
        w.i64(1, off)
        w.i32(2, size)
        w.i64(3, first)
        w.end()
    w.end()
    return bytes(w.out)


def chunk_indexes(data, cols, fields, row_begin, row_end):
    """per column chunk of a file written without the flag: (ColumnIndex fields or None, OffsetIndex locations)"""
    leaves = [Leaf(c, f) for c, f in zip(cols, fields)]
    nl = len(leaves)
    walk = page_walk(data)
    out = []
    for ci, pages in enumerate(walk):
        g, leaf = ci // nl, leaves[ci % nl]
        g0 = row_begin + g * ROW_GROUP_ROWS
        g1 = min(row_end, g0 + ROW_GROUP_ROWS)
        rows = PR.pages_of(leaf, g0, g1)
        data_pages = [(off, size) for typ, off, size in pages if typ == 0]
        assert len(data_pages) == len(rows), (ci, len(data_pages), len(rows))
        locs = [(off, size, r0 - g0) for (off, size), (r0, _) in zip(data_pages, rows)]
        out.append((column_index_fields(leaf, rows), locs))
    return out


def with_index(data, cols, fields, row_begin, row_end):
    """the file with ETL_PQ_PAGE_INDEX, from the same file written without it"""
    fm, foot_at, ends = file_footer(data)
    if not fm.get(4):
        return data
    idx = chunk_indexes(data, cols, fields, row_begin, row_end)
    body = bytearray(data[:foot_at])
    cis, ois = [], []
    for ci, _ in idx:
        b = column_index_bytes(ci) if ci is not None else None
        cis.append((len(body), len(b)) if b is not None else None)
        if b is not None:
            body += b
    for _, locs in idx:
        b = offset_index_bytes(locs)
        ois.append((len(body), len(b)))
        body += b
    foot = bytes(data[foot_at:len(data) - 8])
    out, last = bytearray(), 0
    for end, ci, oi in zip(ends, cis, ois):
        w = TWriter()
        w.last = [3]                                      # after ColumnChunk.meta_data
        w.i64(4, oi[0])
        w.i32(5, oi[1])
        if ci is not None:
            w.i64(6, ci[0])
            w.i32(7, ci[1])
        e = end - foot_at
        out += foot[last:e] + w.out
        last = e
    out += foot[last:]
    return bytes(body + out + struct.pack("<I", len(out)) + b"PAR1")


def read_indexes(data):
    """per column chunk of a file with a page index: (parsed ColumnIndex or None, parsed OffsetIndex or None)"""
    fm, _, _ = file_footer(data)
    out = []
    for rg in fm.get(4, []):
        for cc in rg[1]:
            ci = parse(data, cc[6], cc[7]) if 6 in cc else None
            oi = parse(data, cc[4], cc[5]) if 4 in cc else None
            out.append((ci, oi))
    return out
