"""Python restatement of the split-block bloom filters etl_dec_parquet_write_bloom adds to the Iceberg Parquet file
(include/etl_decode.h): XXH64 of each non-null value's PLAIN bytes, the bitset size from ndv / fpp / max_bytes, the
split-block insert, the BloomFilterHeader, and the file with the filters (with_bloom) from the same file written
without them: the filters go behind the last column chunk, the page index (if any) moves behind them, and the footer
gains ColumnMetaData fields 14 / 15 and the page index's moved offsets.

A bloom entry is (fpp, ndv, max_bytes) per column, as etl_parquet_bloom; fpp 0 is no filter.  Columns and fields are
those of tests/parquet_ref.py.  The Thrift reader is tests/parquet_index_ref.py's."""
from __future__ import annotations

import math
import struct

import numpy as np

import parquet_index_ref as X
from parquet_ref import BOOLEAN, LARGE_BINARY, NP, ROW_GROUP_ROWS, UTF8, UUID, WIDTH, Leaf, TWriter

MIN_BYTES, MAX_BYTES, DEFAULT_MAX_BYTES = 32, 128 << 20, 1 << 20
SALT = np.array([0x47b6137b, 0x44974d91, 0x8824ad5b, 0xa2b7289d, 0x705495c7, 0x2df1424b, 0x9efc4947, 0x5c6bfb31], np.uint64)
_M = (1 << 64) - 1
P1, P2, P3, P4, P5 = 0x9E3779B185EBCA87, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9, 0x85EBCA77C2B2AE63, 0x27D4EB2F165667C5


# ------------------------------------------------------------------------------------------------ XXH64
def _rotl(x, r):
    return ((x << r) | (x >> (64 - r))) & _M


def _round(acc, lane):
    return _rotl((acc + lane * P2) & _M, 31) * P1 & _M


def xxh64(b):
    """XXH64, seed 0, of bytes b (the reference form, one value at a time)"""
    b = bytes(b)
    n, p = len(b), 0
    if n >= 32:
        v = [(P1 + P2) & _M, P2, 0, (-P1) & _M]
        while p + 32 <= n:
            v = [_round(v[i], struct.unpack_from("<Q", b, p + 8 * i)[0]) for i in range(4)]
            p += 32
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & _M
        for x in v:
            h = ((h ^ _round(0, x)) * P1 + P4) & _M
    else:
        h = P5
    h = (h + n) & _M
    while p + 8 <= n:
        h = (_rotl(h ^ _round(0, struct.unpack_from("<Q", b, p)[0]), 27) * P1 + P4) & _M
        p += 8
    if p + 4 <= n:
        h = (_rotl(h ^ (struct.unpack_from("<I", b, p)[0] * P1 & _M), 23) * P2 + P3) & _M
        p += 4
    while p < n:
        h = _rotl(h ^ (b[p] * P5 & _M), 11) * P1 & _M
        p += 1
    h ^= h >> 33
    h = h * P2 & _M
    h ^= h >> 29
    h = h * P3 & _M
    return h ^ (h >> 32)


def _vrotl(x, r):
    return (x << np.uint64(r)) | (x >> np.uint64(64 - r))


def _vround(acc, lane):
    return _vrotl(acc + lane * np.uint64(P2), 31) * np.uint64(P1)


def xxh64_rows(m):
    """XXH64 of every row of a uint8 matrix [k, L] (k values of one length L), vectorised; uint64[k]"""
    m = np.ascontiguousarray(m, dtype=np.uint8)
    k, n = m.shape
    u = lambda x: np.full(k, x, np.uint64)                                # noqa: E731
    q64 = lambda p: m[:, p:p + 8].copy().view("<u8")[:, 0].astype(np.uint64)   # noqa: E731
    with np.errstate(over="ignore"):
        p = 0
        if n >= 32:
            v = [u((P1 + P2) & _M), u(P2), u(0), u((-P1) & _M)]
            while p + 32 <= n:
                v = [_vround(v[i], q64(p + 8 * i)) for i in range(4)]
                p += 32
            h = _vrotl(v[0], 1) + _vrotl(v[1], 7) + _vrotl(v[2], 12) + _vrotl(v[3], 18)
            for x in v:
                h = (h ^ _vround(u(0), x)) * np.uint64(P1) + np.uint64(P4)
        else:
            h = u(P5)
        h = h + np.uint64(n)
        while p + 8 <= n:
            h = _vrotl(h ^ _vround(u(0), q64(p)), 27) * np.uint64(P1) + np.uint64(P4)
            p += 8
        if p + 4 <= n:
            w = m[:, p:p + 4].copy().view("<u4")[:, 0].astype(np.uint64)
            h = _vrotl(h ^ (w * np.uint64(P1)), 23) * np.uint64(P2) + np.uint64(P3)
            p += 4
        while p < n:
            h = _vrotl(h ^ (m[:, p].astype(np.uint64) * np.uint64(P5)), 11) * np.uint64(P1)
            p += 1
        h ^= h >> np.uint64(33)
        h *= np.uint64(P2)
        h ^= h >> np.uint64(29)
        h *= np.uint64(P3)
        h ^= h >> np.uint64(32)
    return h


def hash_values(values):
    """XXH64 of each bytes object of a list, vectorised per length; uint64 array in list order"""
    out = np.zeros(len(values), np.uint64)
    by_len = {}
    for i, v in enumerate(values):
        by_len.setdefault(len(v), []).append(i)
    for n, idx in by_len.items():
        m = np.frombuffer(b"".join(values[i] for i in idx), np.uint8).reshape(len(idx), n) if n else np.zeros((len(idx), 0), np.uint8)
        out[np.array(idx)] = xxh64_rows(m)
    return out


# ------------------------------------------------------------------------------------------------ filter
def bloom_bytes(ndv, fpp, max_bytes=0):
    """bitset bytes: bits = -8 ndv / ln(1 - fpp^(1/8)) truncated, clamped to [256, 2^30], up to a power of two; / 8;
    at most max_bytes (0: 1 MiB)"""
    m = -8.0 * ndv / math.log(1 - math.pow(fpp, 1.0 / 8))
    bits = 8 * MAX_BYTES if not m >= 0 or m > 8 * MAX_BYTES else int(m)
    bits = max(bits, 8 * MIN_BYTES)
    bits = 1 << (bits - 1).bit_length()
    return min(bits // 8, max_bytes or DEFAULT_MAX_BYTES)


def bitset(hashes, nbytes):
    """the split-block bitset (little-endian u32 words) of a uint64 hash array"""
    words = np.zeros(nbytes // 4, np.uint32)
    h = np.asarray(hashes, np.uint64)
    if len(h):
        with np.errstate(over="ignore"):
            blk = ((h >> np.uint64(32)) * np.uint64(nbytes // 32)) >> np.uint64(32)
            key = h & np.uint64(0xFFFFFFFF)
            for i in range(8):
                b = ((key * SALT[i]) & np.uint64(0xFFFFFFFF)) >> np.uint64(27)
                np.bitwise_or.at(words, (blk * np.uint64(8) + np.uint64(i)).astype(np.int64), (np.uint64(1) << b).astype(np.uint32))
    return words.astype("<u4").tobytes()


def contains(bits, h):
    """the filter's probe of one hash"""
    words = np.frombuffer(bits, "<u4")
    blk = ((h >> 32) * (len(bits) // 32)) >> 32
    return all(int(words[8 * blk + i]) >> ((((h & 0xFFFFFFFF) * int(SALT[i])) & 0xFFFFFFFF) >> 27) & 1 for i in range(8))


def header(nbytes):
    """BloomFilterHeader {1 numBytes, 2 algorithm {1 BLOCK}, 3 hash {1 XXHASH}, 4 compression {1 UNCOMPRESSED}}"""
    w = TWriter()
    w.i32(1, nbytes)
    for f in (2, 3, 4):
        w.begin(f)
        w.begin(1)
        w.end()
        w.end()
    w.end()
    return bytes(w.out)


def plain_values(leaf, it0, it1):
    """the PLAIN bytes (no length prefix) of the non-null items of [it0, it1), in item order"""
    v = leaf.vcol
    ok = np.nonzero(np.asarray(v["valid"][it0:it1]))[0] + it0
    t = leaf.atype
    if t in (UTF8, LARGE_BINARY):
        o, d = v["offsets"], v["data"]
        return [bytes(d[int(o[i]):int(o[i + 1])]) for i in ok]
    if t == UUID:
        return [bytes(v["values"][i]) for i in ok]
    raw = np.asarray(v["values"], dtype=NP[t])[ok].tobytes()
    w = WIDTH[t]
    return [raw[k * w:(k + 1) * w] for k in range(len(ok))]


def chunk_hashes(leaf, it0, it1):
    """XXH64 of the non-null items of [it0, it1) (fixed widths vectorised directly)"""
    t = leaf.atype
    v = leaf.vcol
    if t in (UTF8, LARGE_BINARY):
        return hash_values(plain_values(leaf, it0, it1))
    ok = np.nonzero(np.asarray(v["valid"][it0:it1]))[0] + it0
    if t == UUID:
        m = np.asarray(v["values"], np.uint8)[ok]
    else:
        m = np.asarray(v["values"], dtype=NP[t])[ok].view(np.uint8).reshape(len(ok), WIDTH[t])
    return xxh64_rows(m)


def chunk_filter(leaf, g0, g1, b):
    """the filter (header + bitset) of rows [g0, g1) of a leaf under bloom entry b, or None"""
    if b is None or b[0] == 0:
        return None
    assert leaf.atype != BOOLEAN
    h = chunk_hashes(leaf, *leaf.items(g0, g1))
    nb = bloom_bytes(b[1] or max(1, len(h)), b[0], b[2])
    return header(nb) + bitset(h, nb)


def chunk_filters(cols, fields, row_begin, row_end, bloom):
    """per column chunk (row-group major): the filter's bytes (header + bitset), or None"""
    leaves = [Leaf(c, f) for c, f in zip(cols, fields)]
    out = []
    for g0 in range(row_begin, row_end, ROW_GROUP_ROWS):
        g1 = min(row_end, g0 + ROW_GROUP_ROWS)
        for leaf, b in zip(leaves, bloom or [None] * len(leaves)):
            out.append(chunk_filter(leaf, g0, g1, b))
    return out


# ------------------------------------------------------------------------------------------------ file
def _fields(buf, pos):
    """the fields of the compact struct at pos: [(id, type, value start, value end)], and the position after its stop"""
    out, last = [], 0
    while True:
        b = buf[pos]
        pos += 1
        if b == 0:
            return out, pos
        t, d = b & 0x0F, b >> 4
        if d:
            fid = last + d
        else:
            v, pos = X._var(buf, pos)
            fid = (v >> 1) ^ -(v & 1)
        last = fid
        _, end = X._value(buf, pos, t, False, None, ())
        out.append((fid, t, pos, end))
        pos = end


def _list_structs(buf, pos):
    """the element positions of the list<struct> value at pos"""
    h = buf[pos]
    pos += 1
    n = h >> 4
    if n == 15:
        n, pos = X._var(buf, pos)
    out = []
    for _ in range(n):
        _, end = _fields(buf, pos)
        out.append(pos)
        pos = end
    return out


def _field_bytes(fid, last, t, value):
    d = fid - last
    return (bytes([(d << 4) | t]) if 0 < d <= 15 else bytes([t]) + _uv(TWriter.zz(fid))) + value


def _uv(v):
    w = TWriter()
    w.var(v)
    return bytes(w.out)


def data_end(data):
    """the end of the last column chunk (file offset)"""
    fm, _, _ = X.file_footer(data)
    return max((cc[3].get(11, cc[3][9]) + cc[3][7] for rg in fm.get(4, []) for cc in rg[1]), default=4)


def with_bloom(data, cols, fields, row_begin, row_end, bloom, filters=None):
    """the file with the bloom filters, from the same call's file without them (filters: chunk_filters of the same
    arguments, when already computed)"""
    if filters is None:
        filters = chunk_filters(cols, fields, row_begin, row_end, bloom)
    if not any(f is not None for f in filters):
        return data
    fm, foot_at, _ = X.file_footer(data)
    end = data_end(data)
    region, offs = bytearray(), []
    for f in filters:
        offs.append(None if f is None else (end + len(region), len(f)))
        if f is not None:
            region += f
    shift = len(region)
    edits = []                                            # (position in data, bytes removed, bytes inserted)
    top, _ = _fields(data, foot_at)
    rgs = next(f for f in top if f[0] == 4)
    ci = 0
    for rg_at in _list_structs(data, rgs[2]):
        rg_f, _ = _fields(data, rg_at)
        cols_f = next(f for f in rg_f if f[0] == 1)
        for cc_at in _list_structs(data, cols_f[2]):
            cc_f, _ = _fields(data, cc_at)
            for fid, t, a, b in cc_f:
                if fid == 3 and offs[ci] is not None:      # ColumnMetaData: 14 / 15 before its stop byte
                    md_f, _ = _fields(data, a)
                    w = _field_bytes(14, md_f[-1][0], 6, _uv(TWriter.zz(offs[ci][0])))
                    w += _field_bytes(15, 14, 5, _uv(TWriter.zz(offs[ci][1])))
                    edits.append((b - 1, 0, w))
                if fid in (4, 6):                         # the page index's offsets move behind the filters
                    v, _ = X._var(data, a)
                    edits.append((a, b - a, _uv(TWriter.zz(((v >> 1) ^ -(v & 1)) + shift))))
            ci += 1
    foot = bytearray()
    last = foot_at
    for at, rm, ins in sorted(edits, key=lambda e: e[0]):
        foot += data[last:at] + ins
        last = at + rm
    foot += data[last:len(data) - 8]
    return bytes(data[:end]) + bytes(region) + bytes(data[end:foot_at]) + bytes(foot) + struct.pack("<I", len(foot)) + b"PAR1"


def read_filters(data):
    """per column chunk of a file: (offset, stated length, parsed header, header bytes, bitset) or None"""
    fm, _, _ = X.file_footer(data)
    out = []
    for rg in fm.get(4, []):
        for cc in rg[1]:
            md = cc[3]
            if 14 not in md:
                out.append(None)
                continue
            h, p = X.read_struct(data, md[14])
            out.append((md[14], md.get(15), h, bytes(data[md[14]:p]), bytes(data[p:p + h[1]])))
    return out
