"""Python restatement of the Iceberg Parquet data file (include/etl_decode.h, etl_dec_parquet_write): the uncompressed
file and the per-leaf metrics, written from Arrow columns held on the host.

A column is a dict:
  {"type": ETL_ARROW_*, "valid": bool[n], ...}
  fixed width:  "values": numpy array (Boolean: bool, Uuid: uint8[n, 16])
  byte arrays:  "offsets": int64[n + 1], "data": bytes
  List:         "offsets": int64[n + 1], "child": a column of the elements
A field is (name, field_id, element_field_id, required)."""
from __future__ import annotations

import struct

import numpy as np

BOOLEAN, INT32, INT64, FLOAT32, FLOAT64, UTF8, LARGE_BINARY, DATE32, TIME64_US, TIMESTAMP_US, TIMESTAMPTZ_US, UUID, LIST = range(1, 14)
UNCOMPRESSED, SNAPPY = 0, 1
PAGE_ROWS, PAGE_BYTES, ROW_GROUP_ROWS = 20000, 1 << 20, 1 << 20
STAT_MAX = 64
CREATED_BY = b"etl-b200 parquet writer"

# Parquet physical types, converted types
PT = {BOOLEAN: 0, INT32: 1, DATE32: 1, INT64: 2, TIME64_US: 2, TIMESTAMP_US: 2, TIMESTAMPTZ_US: 2, FLOAT32: 4, FLOAT64: 5,
      UTF8: 6, LARGE_BINARY: 6, UUID: 7}
WIDTH = {INT32: 4, DATE32: 4, FLOAT32: 4, INT64: 8, TIME64_US: 8, TIMESTAMP_US: 8, TIMESTAMPTZ_US: 8, FLOAT64: 8, UUID: 16}
NP = {INT32: "<i4", DATE32: "<i4", FLOAT32: "<f4", INT64: "<i8", TIME64_US: "<i8", TIMESTAMP_US: "<i8", TIMESTAMPTZ_US: "<i8",
      FLOAT64: "<f8"}


# ------------------------------------------------------------------------------------------------ Thrift compact
class TWriter:
    def __init__(self):
        self.out = bytearray()
        self.last = [0]

    def var(self, v):
        while v >= 0x80:
            self.out.append((v & 0x7F) | 0x80)
            v >>= 7
        self.out.append(v)

    @staticmethod
    def zz(v):
        return (v << 1) ^ (v >> 63) if v < 0 else v << 1

    def field(self, fid, t):
        d = fid - self.last[-1]
        if 0 < d <= 15:
            self.out.append((d << 4) | t)
        else:
            self.out.append(t)
            self.var(self.zz(fid))
        self.last[-1] = fid

    def i32(self, fid, v):
        self.field(fid, 5)
        self.var(self.zz(v))

    i64 = lambda self, fid, v: (self.field(fid, 6), self.var(self.zz(v)))

    def i16(self, fid, v):
        self.field(fid, 4)
        self.var(self.zz(v))

    def boolean(self, fid, v):
        self.field(fid, 1 if v else 2)

    def binary(self, fid, b):
        self.field(fid, 8)
        self.var(len(b))
        self.out += b

    def begin(self, fid):
        self.field(fid, 12)
        self.last.append(0)

    def end(self):
        self.out.append(0)
        if len(self.last) > 1:
            self.last.pop()

    def list(self, fid, et, n):
        self.field(fid, 9)
        if n < 15:
            self.out.append((n << 4) | et)
        else:
            self.out.append(0xF0 | et)
            self.var(n)

    def elem(self):
        self.last.append(0)


def page_header(usize, csize, num_values):
    w = TWriter()
    w.i32(1, 0)
    w.i32(2, usize)
    w.i32(3, csize)
    w.begin(5)
    w.i32(1, num_values)
    w.i32(2, 0)
    w.i32(3, 3)
    w.i32(4, 3)
    w.end()
    w.end()
    return bytes(w.out)


# ------------------------------------------------------------------------------------------------ levels
def _uvar(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def levels_encode(lv, w):
    """RLE / bit-packed hybrid of the level values lv (no length prefix), with the deterministic run rule"""
    lv = np.asarray(lv, dtype=np.uint8)
    n = len(lv)
    ng = (n + 7) // 8
    if not ng:
        return b""
    pad = np.zeros(ng * 8, dtype=np.uint8)
    pad[:n] = lv
    g = pad.reshape(ng, 8)
    full = (g == g[:, :1]).all(axis=1)
    m = n - (ng - 1) * 8
    cls = np.where(full, g[:, 0].astype(np.int16), -1)
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
            out += _uvar(cnt << 1)
            out.append(c)
        else:
            while h < ng and h - k < 63 and cls[h] < 0:
                h += 1
            out.append(((h - k) << 1) | 1)
            vals = pad[k * 8:h * 8].astype(np.uint32)
            if n < h * 8:
                vals[n - k * 8:] = 0
            bits = np.unpackbits(vals.astype(np.uint8)[:, None], axis=1, bitorder="little")[:, :w].reshape(-1)
            out += np.packbits(bits, bitorder="little").tobytes()
        k = h
    return bytes(out)


# ------------------------------------------------------------------------------------------------ columns → leaves
class Leaf:
    def __init__(self, col, field):
        self.name, self.field_id, self.element_field_id, required = field
        self.required = bool(required)
        self.is_list = col["type"] == LIST
        self.col = col
        self.vcol = col["child"] if self.is_list else col
        self.atype = self.vcol["type"]
        self.max_def = (2 if self.required else 3) if self.is_list else (0 if self.required else 1)
        self.max_rep = 1 if self.is_list else 0
        self.w = int(self.max_def).bit_length()

    def items(self, r0, r1):
        if self.is_list:
            o = self.col["offsets"]
            return int(o[r0]), int(o[r1])
        return r0, r1

    def row_items(self, r):
        return self.items(r, r + 1)

    def levels(self, r0, r1):
        """(rep, def) level arrays of rows [r0, r1)"""
        if not self.is_list:
            return None, self.col["valid"][r0:r1].astype(np.uint8)
        o, lv, cv = self.col["offsets"], self.col["valid"], self.vcol["valid"]
        rep, dfn = [], []
        for r in range(r0, r1):
            a, b = int(o[r]), int(o[r + 1])
            if not lv[r]:
                rep.append(0); dfn.append(0)
            elif a == b:
                rep.append(0); dfn.append(self.max_def - 2)
            else:
                rep += [0] + [1] * (b - a - 1)
                dfn += [self.max_def if cv[k] else self.max_def - 1 for k in range(a, b)]
        return np.array(rep, np.uint8), np.array(dfn, np.uint8)

    def value_bytes(self, i):
        """PLAIN size of item i (bits for Boolean)"""
        v = self.vcol
        if self.atype == BOOLEAN:
            return 1
        if self.atype in (UTF8, LARGE_BINARY):
            return 4 + int(v["offsets"][i + 1] - v["offsets"][i])
        return WIDTH[self.atype]

    def plain(self, it0, it1):
        v = self.vcol
        ok = np.nonzero(v["valid"][it0:it1])[0] + it0
        if self.atype == BOOLEAN:
            return np.packbits(v["values"][ok].astype(np.uint8), bitorder="little").tobytes()
        if self.atype in (UTF8, LARGE_BINARY):
            o, d = v["offsets"], v["data"]
            return b"".join(struct.pack("<I", int(o[i + 1] - o[i])) + d[int(o[i]):int(o[i + 1])] for i in ok)
        if self.atype == UUID:
            return v["values"][ok].tobytes()
        return np.asarray(v["values"], dtype=NP[self.atype])[ok].tobytes()

    def stat_value(self, i):
        """(sort key, PLAIN statistic bytes) of present item i; None for NaN"""
        v = self.vcol
        if self.atype == BOOLEAN:
            b = int(bool(v["values"][i]))
            return b, bytes([b])
        if self.atype in (UTF8, LARGE_BINARY):
            s = v["data"][int(v["offsets"][i]):int(v["offsets"][i + 1])]
            return bytes(s), bytes(s)
        if self.atype == UUID:
            s = bytes(v["values"][i])
            return s, s
        x = np.asarray(v["values"], dtype=NP[self.atype])[i]
        if self.atype in (FLOAT32, FLOAT64) and np.isnan(x):
            return None
        return (float(x) if self.atype in (FLOAT32, FLOAT64) else int(x)), x.tobytes()

    def stats(self, it0, it1):
        """(null-free min bytes, max bytes or None, nan count) over the present items of [it0, it1)"""
        v = self.vcol
        ok = np.nonzero(v["valid"][it0:it1])[0] + it0
        nan = 0
        if self.atype in (FLOAT32, FLOAT64):
            vals = np.asarray(v["values"], dtype=NP[self.atype])[ok]
            isn = np.isnan(vals)
            nan = int(isn.sum())
            vals = vals[~isn]
            if not len(vals):
                return None, None, nan
            mn, mx = vals.min(), vals.max()
            mnb = (np.array(-0.0 if mn == 0 else mn, dtype=NP[self.atype])).tobytes()
            mxb = (np.array(0.0 if mx == 0 else mx, dtype=NP[self.atype])).tobytes()
            return mnb, mxb, nan
        if not len(ok):
            return None, None, 0
        if self.atype in NP:
            vals = np.asarray(v["values"], dtype=NP[self.atype])[ok]
            return vals.min().tobytes(), vals.max().tobytes(), 0
        keys = [self.stat_value(int(i)) for i in ok]
        mn = min(keys, key=lambda k: k[0])[1]
        mx = max(keys, key=lambda k: k[0])[1]
        if self.atype in (UTF8, LARGE_BINARY) and (len(mn) > STAT_MAX or len(mx) > STAT_MAX):
            return None, None, 0
        return mn, mx, 0


def pages_of(leaf, g0, g1):
    """greedy page cuts of rows [g0, g1): list of (r0, r1)"""
    n = g1 - g0
    v = leaf.vcol
    if leaf.atype == BOOLEAN:
        size = v["valid"].astype(np.int64)
    elif leaf.atype in (UTF8, LARGE_BINARY):
        size = np.where(v["valid"], 4 + np.diff(np.asarray(v["offsets"], dtype=np.int64)), 0)
    else:
        size = v["valid"].astype(np.int64) * WIDTH[leaf.atype]
    s_items = np.concatenate([[0], np.cumsum(size)])
    if leaf.is_list:
        o = np.asarray(leaf.col["offsets"], dtype=np.int64)[g0:g1 + 1]
        per_row = np.where(leaf.col["valid"][g0:g1], s_items[o[1:]] - s_items[o[:-1]], 0)
    else:
        per_row = size[g0:g1]
    vb = np.concatenate([[0], np.cumsum(per_row)]).astype(np.int64)
    thresh = 8 * PAGE_BYTES - 7 if leaf.atype == BOOLEAN else PAGE_BYTES
    out, s = [], 0
    while s < n:
        hi = min(n - 1, s + PAGE_ROWS - 1)
        # first e in [s, hi] with vb[e + 1] - vb[s] >= thresh
        e = int(np.searchsorted(vb[s + 1:hi + 2], vb[s] + thresh, side="left")) + s
        end = min(e, hi) + 1
        out.append((g0 + s, g0 + end))
        s = end
    return out


def page_payload(leaf, r0, r1):
    rep, dfn = leaf.levels(r0, r1)
    out = bytearray()
    if leaf.max_rep:
        b = levels_encode(rep, 1)
        out += struct.pack("<I", len(b)) + b
    if leaf.max_def:
        b = levels_encode(dfn, leaf.w)
        out += struct.pack("<I", len(b)) + b
    it0, it1 = leaf.items(r0, r1)
    out += leaf.plain(it0, it1)
    return bytes(out), len(dfn)


LOGICAL = {UTF8: 1, DATE32: 6, TIME64_US: 7, TIMESTAMP_US: 8, TIMESTAMPTZ_US: 8, UUID: 14}
CONVERTED = {UTF8: 0, DATE32: 6, TIMESTAMPTZ_US: 10}


def _schema_leaf(w, leaf, element):
    w.elem()
    w.i32(1, PT[leaf.atype])
    if leaf.atype == UUID:
        w.i32(2, 16)
    w.i32(3, 1 if element or not leaf.required else 0)
    w.binary(4, b"element" if element else leaf.name.encode())
    if leaf.atype in CONVERTED:
        w.i32(6, CONVERTED[leaf.atype])
    w.i32(9, leaf.element_field_id if element else leaf.field_id)
    lg = LOGICAL.get(leaf.atype)
    if lg:
        w.begin(10)
        w.begin(lg)
        if lg in (7, 8):
            w.boolean(1, leaf.atype == TIMESTAMPTZ_US)
            w.begin(2); w.begin(2); w.end(); w.end()
        w.end()
        w.end()
    w.end()


def footer(leaves, rg_rows, chunks, codec):
    """chunks: row-group major dicts {offset, num_values, usize, csize, null_count, min, max}"""
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
            w.list(2, 5, 2 if levels else 1)
            w.var(0)
            if levels:
                w.var(6)
            path = [L.name.encode()] + ([b"list", b"element"] if L.is_list else [])
            w.list(3, 8, len(path))
            for p in path:
                w.var(len(p)); w.out += p
            w.i32(4, codec)
            w.i64(5, c["num_values"])
            w.i64(6, c["usize"])
            w.i64(7, c["csize"])
            w.i64(9, c["offset"])
            w.begin(12)
            w.i64(3, c["null_count"])
            if c["min"] is not None:
                w.binary(5, c["max"])
                w.binary(6, c["min"])
            w.end()
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


def write(cols, fields, row_begin, row_end):
    """(uncompressed file bytes, metrics per leaf, pages [(chunk, header bytes, payload)])"""
    leaves = [Leaf(c, f) for c, f in zip(cols, fields)]
    n = row_end - row_begin
    rg = [(row_begin + g, min(row_end, row_begin + g + ROW_GROUP_ROWS)) for g in range(0, n, ROW_GROUP_ROWS)]
    body = bytearray(b"PAR1")
    chunks, pages = [], []
    metrics = [dict(field_id=L.element_field_id if L.is_list else L.field_id, num_values=0, null_count=0, nan_count=0,
                    compressed_bytes=0, uncompressed_bytes=0, min=None, max=None, _keys=[]) for L in leaves]
    for g0, g1 in rg:
        for li, L in enumerate(leaves):
            c = dict(offset=len(body), num_values=0, usize=0, csize=0, null_count=0)
            for r0, r1 in pages_of(L, g0, g1):
                payload, nv = page_payload(L, r0, r1)
                it0, it1 = L.items(r0, r1)
                nn = int(np.count_nonzero(L.vcol["valid"][it0:it1]))
                hdr = page_header(len(payload), len(payload), nv)
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
        it0, it1 = L.items(row_begin, row_end) if n else (0, 0)
        m = metrics[li]
        m.pop("_keys")
        if n:
            m["min"], m["max"], _ = L.stats(it0, it1)
    foot = footer(leaves, [g1 - g0 for g0, g1 in rg], chunks, UNCOMPRESSED)
    body += foot + struct.pack("<I", len(foot)) + b"PAR1"
    return bytes(body), metrics, pages


# ------------------------------------------------------------------------------------------------ Thrift compact reader
def read_struct(buf, pos=0):
    """parse one compact struct: ({field id: value}, next position); lists become Python lists, binaries bytes"""
    out = {}
    last = 0
    while True:
        b = buf[pos]
        pos += 1
        if b == 0:
            return out, pos
        t, d = b & 0x0F, b >> 4
        if d:
            fid = last + d
        else:
            v, pos = _read_var(buf, pos)
            fid = (v >> 1) ^ -(v & 1)
        last = fid
        out[fid], pos = _read_value(buf, pos, t)


def _read_var(buf, pos):
    v = s = 0
    while True:
        b = buf[pos]
        pos += 1
        v |= (b & 0x7F) << s
        s += 7
        if b < 0x80:
            return v, pos


def _read_value(buf, pos, t):
    if t in (1, 2):
        return t == 1, pos
    if t in (4, 5, 6):
        v, pos = _read_var(buf, pos)
        return (v >> 1) ^ -(v & 1), pos
    if t == 8:
        n, pos = _read_var(buf, pos)
        return bytes(buf[pos:pos + n]), pos + n
    if t == 9:
        h = buf[pos]
        pos += 1
        n, et = h >> 4, h & 0x0F
        if n == 15:
            n, pos = _read_var(buf, pos)
        items = []
        for _ in range(n):
            v, pos = _read_value(buf, pos, et)
            items.append(v)
        return items, pos
    if t == 12:
        return read_struct(buf, pos)
    raise ValueError(f"thrift type {t}")


def file_footer(data):
    """the parsed FileMetaData of a file"""
    assert data[:4] == b"PAR1" and data[-4:] == b"PAR1"
    n = struct.unpack("<I", data[-8:-4])[0]
    fm, end = read_struct(data, len(data) - 8 - n)
    assert end == len(data) - 8
    return fm, len(data) - 8 - n


def walk_pages(data):
    """every page of a file in order: (chunk index, parsed header, header bytes, payload)"""
    fm, foot_at = file_footer(data)
    out = []
    ci = 0
    for rg in fm.get(4, []):
        for cc in rg[1]:
            md = cc[3]
            pos, end = md[9], md[9] + md[7]
            while pos < end:
                h, p2 = read_struct(data, pos)
                out.append((ci, h, bytes(data[pos:p2]), bytes(data[p2:p2 + h[3]])))
                pos = p2 + h[3]
            assert pos == end
            ci += 1
    return out
