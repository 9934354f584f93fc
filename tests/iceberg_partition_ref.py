"""Python restatement of etl_dec_iceberg_partition (include/etl_decode.h, csrc/iceberg_partition.cu): the Iceberg
partition transforms (spec "Partition Transforms", Appendix B's murmur3_x86_32), the grouping of rows by partition
tuple (partitions in first-row order, rows in emit order inside each), the permutation of an emit's columns and the
partition values.  Columns are tests/parquet_ref.py columns, as tests/parquet_io.emit_columns reads them."""
import datetime

import numpy as np

import parquet_ref as R

IDENTITY, BUCKET, TRUNCATE, YEAR, MONTH, DAY, HOUR, VOID = range(8)
MICROS_PER_DAY, MICROS_PER_HOUR = 86400000000, 3600000000
INTEGER = (R.INT32, R.INT64, R.DATE32, R.TIME64_US, R.TIMESTAMP_US, R.TIMESTAMPTZ_US)
BYTES = (R.UTF8, R.LARGE_BINARY, R.UUID)
TIMESTAMPS = (R.TIMESTAMP_US, R.TIMESTAMPTZ_US)


def murmur3_32(data: bytes, seed: int = 0) -> int:
    """MurmurHash3_x86_32 as an unsigned 32-bit value"""
    M = 0xFFFFFFFF
    c1, c2 = 0xCC9E2D51, 0x1B873593

    def rotl(x, r):
        return ((x << r) | (x >> (32 - r))) & M

    def k_of(k):
        return (rotl((k * c1) & M, 15) * c2) & M

    h = seed & M
    nb = len(data) // 4
    for i in range(nb):
        h ^= k_of(int.from_bytes(data[4 * i:4 * i + 4], "little"))
        h = (rotl(h, 13) * 5 + 0xE6546B64) & M
    tail = data[4 * nb:]
    if tail:
        h ^= k_of(int.from_bytes(tail, "little"))
    h ^= len(data)
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & M
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & M
    h ^= h >> 16
    return h


def signed32(h: int) -> int:
    return h - (1 << 32) if h >= 1 << 31 else h


def hash_long(v: int) -> int:
    return murmur3_32((v & 0xFFFFFFFFFFFFFFFF).to_bytes(8, "little"))


def bucket(h: int, n: int) -> int:
    return (h & 0x7FFFFFFF) % n


def _wrap(v: int, bits: int) -> int:
    v &= (1 << bits) - 1
    return v - (1 << bits) if v >> (bits - 1) else v


def truncate_int(v: int, w: int, bits: int) -> int:
    """v - (((v % W) + W) % W) with Java's truncated %, wrapped to the source's width"""
    rem = abs(v) % w * (1 if v >= 0 else -1)
    return _wrap(v - ((rem + w) % w), bits)


def truncate_utf8(b: bytes, w: int) -> bytes:
    """the first w code points of UTF-8 bytes (a code point starts at every non-continuation byte)"""
    starts = 0
    for i, x in enumerate(b):
        if x & 0xC0 != 0x80:
            if starts == w:
                return b[:i]
            starts += 1
    return b


def civil(days: int):
    """(year, month) of a day count since 1970-01-01, proleptic Gregorian, any range (Hinnant's algorithm)"""
    z = days + 719468
    era = z // 146097
    doe = z - era * 146097
    yoe = (doe - doe // 1460 + doe // 36524 - doe // 146096) // 365
    doy = doe - (365 * yoe + yoe // 4 - yoe // 100)
    mp = (5 * doy + 2) // 153
    m = mp + 3 if mp < 10 else mp - 9
    return yoe + era * 400 + (m <= 2), m


def years(days: int) -> int:
    return civil(days)[0] - 1970


def months(days: int) -> int:
    y, m = civil(days)
    return (y - 1970) * 12 + m - 1


def years_dt(d: datetime.date) -> int:
    """the same through Python's datetime (years 1-9999): the cross-check of the integer formulas"""
    return d.year - 1970


def months_dt(d: datetime.date) -> int:
    return (d.year - 1970) * 12 + d.month - 1


def accepts(atype: int, tr: int) -> bool:
    if atype in (R.LIST, 0):
        return False
    flt = atype in (R.FLOAT32, R.FLOAT64)
    return {VOID: True, IDENTITY: not flt, BUCKET: not flt and atype != R.BOOLEAN,
            TRUNCATE: atype in (R.INT32, R.INT64, R.UTF8, R.LARGE_BINARY),
            YEAR: atype in (R.DATE32,) + TIMESTAMPS, MONTH: atype in (R.DATE32,) + TIMESTAMPS,
            DAY: atype in (R.DATE32,) + TIMESTAMPS, HOUR: atype in TIMESTAMPS}.get(tr, False)


def source_value(col, r):
    """row r's value: None, an int (Boolean 0 / 1) or bytes"""
    if not col["valid"][r]:
        return None
    t = col["type"]
    if t == R.BOOLEAN:
        return int(col["values"][r])
    if t in (R.UTF8, R.LARGE_BINARY):
        o = col["offsets"]
        return col["data"][o[r]:o[r + 1]]
    if t == R.UUID:
        return bytes(col["values"][r])
    return int(col["values"][r])


def transform(atype: int, v, tr: int, param: int):
    """a field's result of a source value: None, an int or bytes"""
    if v is None or tr == VOID:
        return None
    if tr == IDENTITY:
        return v
    if tr == BUCKET:
        return bucket(murmur3_32(v) if atype in BYTES else hash_long(v), param)
    if tr == TRUNCATE:
        if atype == R.INT32:
            return truncate_int(v, param, 32)
        if atype == R.INT64:
            return truncate_int(v, param, 64)
        return truncate_utf8(v, param) if atype == R.UTF8 else v[:param]
    days = v if atype == R.DATE32 else v // MICROS_PER_DAY
    if tr == YEAR:
        return years(days)
    if tr == MONTH:
        return months(days)
    if tr == DAY:
        return days
    if tr == HOUR:
        return v // MICROS_PER_HOUR
    raise ValueError(tr)


def partition(cols, spec, rb, re):
    """spec: [(source_column, transform, param)] → (perm: source rows in partitioned order, row offsets (P + 1),
    values: per partition the tuple of field results)"""
    groups = {}
    for r in range(rb, re):
        key = tuple(transform(cols[c]["type"], source_value(cols[c], r), tr, p) for c, tr, p in spec)
        groups.setdefault(key, []).append(r)          # dicts keep insertion order: partitions by first row
    perm, offs, values = [], [0], []
    for key, rows in groups.items():
        perm += rows
        offs.append(len(perm))
        values.append(key)
    return perm, offs, values


def _take_flat(col, idx):
    t = col["type"]
    out = {"type": t, "valid": col["valid"][idx] if len(idx) else np.zeros(0, bool)}
    if t in (R.UTF8, R.LARGE_BINARY):
        o = col["offsets"]
        parts = [col["data"][o[i]:o[i + 1]] for i in idx]
        out["offsets"] = np.concatenate([[0], np.cumsum([len(p) for p in parts], dtype=np.int64)]).astype(np.int64)
        out["data"] = b"".join(parts)
    elif "values" in col:
        out["values"] = col["values"][idx] if len(idx) else col["values"][:0]
    return out


def take(col, idx):
    """the column's rows idx (a list of source rows), in that order"""
    idx = np.asarray(idx, dtype=np.int64)
    if col["type"] != R.LIST:
        return _take_flat(col, idx)
    o = col["offsets"]
    items = [k for i in idx for k in range(o[i], o[i + 1])]
    lens = [o[i + 1] - o[i] for i in idx]
    return {"type": R.LIST, "valid": col["valid"][idx] if len(idx) else np.zeros(0, bool),
            "offsets": np.concatenate([[0], np.cumsum(lens, dtype=np.int64)]).astype(np.int64),
            "child": _take_flat(col["child"], np.asarray(items, dtype=np.int64))}
