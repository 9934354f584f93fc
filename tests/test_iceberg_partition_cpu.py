"""CPU checks of the Iceberg partition transforms of etl_dec_iceberg_partition: the Python restatement
(tests/iceberg_partition_ref.py) against the Iceberg spec's and Austin Appleby's murmur3 known answers and against
Python's datetime; the device's transforms compiled for the host (tests/emul/host_iceberg_partition.cpp) against the
restatement; the grouping order of the restatement; and the layout of the new structs against their ctypes mirror."""
import ctypes as C
import datetime
import os
import subprocess
import tempfile

import numpy as np
import pytest

import iceberg_partition_ref as P
import parquet_ref as R
from etl_b200 import abi

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EPOCH = datetime.date(1970, 1, 1)
I32_MIN, I32_MAX, I64_MIN, I64_MAX = -2**31, 2**31 - 1, -2**63, 2**63 - 1


@pytest.fixture(scope="module")
def host():
    out_dir = tempfile.mkdtemp(prefix="etl_host_iceberg_partition_")
    so = os.path.join(out_dir, "libhost_iceberg_partition.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           "-I", os.path.join(ROOT, "etl_b200", "csrc"), "-o", so, os.path.join(HERE, "emul", "host_iceberg_partition.cpp")])
    lib = C.CDLL(so)
    lib.emu_murmur3.argtypes = [C.c_char_p, C.c_uint64, C.c_uint32]
    lib.emu_murmur3.restype = C.c_uint32
    lib.emu_murmur3_i64.argtypes = [C.c_int64]
    lib.emu_murmur3_i64.restype = C.c_uint32
    lib.emu_bucket.argtypes = [C.c_uint32, C.c_uint32]
    lib.emu_truncate_i32.argtypes = [C.c_int32, C.c_uint32]
    lib.emu_truncate_i64.argtypes = [C.c_int64, C.c_uint32]
    lib.emu_utf8_prefix.argtypes = [C.c_char_p, C.c_uint32, C.c_uint32]
    lib.emu_utf8_prefix.restype = C.c_uint32
    for f in ("emu_bucket", "emu_truncate_i32", "emu_truncate_i64", "emu_years", "emu_months", "emu_days", "emu_hours"):
        getattr(lib, f).restype = C.c_int64
    for f in ("emu_years", "emu_months", "emu_days", "emu_hours"):
        getattr(lib, f).argtypes = [C.c_int64]
    return lib


# ------------------------------------------------------------------------------------------------ known answers
def test_spec_known_answers():
    """Iceberg spec, Appendix B: the hash of each type's bytes"""
    day = (datetime.date(2017, 11, 16) - EPOCH).days
    time_us = (22 * 3600 + 31 * 60 + 8) * 1000000
    ts = day * P.MICROS_PER_DAY + time_us
    cases = [(P.hash_long(34), 2017239379), (P.hash_long(day), -653330422), (P.hash_long(time_us), -662762989),
             (P.hash_long(ts), -2047944441), (P.hash_long(ts + 1), -1207196810),
             (P.murmur3_32(b"iceberg"), 1210000089), (P.murmur3_32(bytes([0, 1, 2, 3])), -188683207),
             (P.murmur3_32(bytes.fromhex("f79c3e09677c4bbda4793f349cb785e7")), 1488055340)]
    for got, want in cases:
        assert P.signed32(got) == want


def test_appleby_known_answers(host):
    fox = b"The quick brown fox jumps over the lazy dog"
    for data, want in ((b"hello", 0x248BFA47), (fox, 0x2E4FF723), (b"", 0)):
        assert P.murmur3_32(data) == want
        assert host.emu_murmur3(data, len(data), 0) == want


# ------------------------------------------------------------------------------------------------ host build vs restatement
def test_murmur3_every_length_and_fuzz(host):
    rng = np.random.default_rng(3)
    base = rng.integers(0, 256, 64, dtype=np.uint8).tobytes()
    for n in range(65):
        for seed in (0, 1, 0xDEADBEEF):
            assert host.emu_murmur3(base[:n], n, seed) == P.murmur3_32(base[:n], seed), (n, seed)
    for _ in range(100000):
        n = int(rng.integers(0, 40))
        data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        assert host.emu_murmur3(data, n, 0) == P.murmur3_32(data)


def test_integer_hash_is_the_long_bytes(host):
    rng = np.random.default_rng(4)
    vals = [0, 1, -1, 34, I32_MIN, I32_MAX, I64_MIN, I64_MAX] + [int(x) for x in rng.integers(I64_MIN, I64_MAX, 20000, dtype=np.int64)]
    for v in vals:
        assert host.emu_murmur3_i64(v) == P.hash_long(v) == P.murmur3_32((v & (2**64 - 1)).to_bytes(8, "little"))


def test_bucket_every_source_type(host):
    """bucket[N] per source type through the restatement's transform, the host build's hash and bucket"""
    rng = np.random.default_rng(5)
    for n in (1, 2, 16, 1000, I32_MAX):
        for atype in P.INTEGER:
            for v in [0, -1, 34, I32_MIN] + [int(x) for x in rng.integers(I32_MIN, I32_MAX, 200)]:
                if atype in (R.INT64, R.TIME64_US) + P.TIMESTAMPS:
                    v *= 1000003
                want = P.transform(atype, v, P.BUCKET, n)
                assert want == host.emu_bucket(host.emu_murmur3_i64(v), n) == (P.hash_long(v) & I32_MAX) % n
        for atype, data in ((R.UTF8, "iceberg ✓ π".encode()), (R.LARGE_BINARY, bytes(range(7))), (R.UUID, bytes(range(16)))):
            want = P.transform(atype, data, P.BUCKET, n)
            assert want == host.emu_bucket(host.emu_murmur3(data, len(data), 0), n)
    assert P.transform(R.UTF8, b"iceberg", P.BUCKET, 16) == 1210000089 % 16


def test_truncate_integers(host):
    rng = np.random.default_rng(6)
    ws = [1, 2, 3, 10, 1000, I32_MAX]
    i32 = [0, 1, -1, 9, -9, 10, -10, 11, -11, I32_MIN, I32_MIN + 1, I32_MAX] + [int(x) for x in rng.integers(I32_MIN, I32_MAX, 3000)]
    i64 = [I64_MIN, I64_MIN + 1, I64_MAX, -1, 0] + [int(x) for x in rng.integers(I64_MIN, I64_MAX, 3000, dtype=np.int64)]
    for w in ws:
        for v in i32:
            want = P.truncate_int(v, w, 32)
            assert host.emu_truncate_i32(v, w) == want == P.transform(R.INT32, v, P.TRUNCATE, w), (v, w)
        for v in i64:
            assert host.emu_truncate_i64(v, w) == P.truncate_int(v, w, 64), (v, w)
    assert P.truncate_int(-1, 10, 32) == -10 and P.truncate_int(5, 10, 32) == 0 and P.truncate_int(-10, 10, 32) == -10
    assert P.truncate_int(I32_MIN, 10, 32) == 2147483646                # -2147483650 wraps
    assert P.truncate_int(I64_MIN, 10, 64) == I64_MAX - 1 and P.truncate_int(I64_MIN, 1, 64) == I64_MIN
    assert P.truncate_int(I32_MIN, I32_MAX, 32) == 2                     # -2^31 - (2^31 - 2) wraps
    assert P.truncate_int(-5, I32_MAX, 32) == -I32_MAX and P.truncate_int(I32_MAX, I32_MAX, 32) == I32_MAX


def test_truncate_utf8_by_code_point(host):
    text = "aé€😀b" * 5                                      # 1-, 2-, 3- and 4-byte code points
    raw = text.encode()
    for w in list(range(0, 30)) + [I32_MAX]:
        want = text[:w].encode()
        if w:
            assert P.truncate_utf8(raw, w) == want
        assert host.emu_utf8_prefix(raw, len(raw), w) == len(want) == len(P.truncate_utf8(raw, w)), w
    assert P.transform(R.UTF8, "iceberg".encode(), P.TRUNCATE, 3) == b"ice"
    assert P.transform(R.LARGE_BINARY, bytes([1, 2, 3]), P.TRUNCATE, 10) == bytes([1, 2, 3])
    assert P.transform(R.LARGE_BINARY, bytes([1, 2, 3]), P.TRUNCATE, 2) == bytes([1, 2])
    assert host.emu_utf8_prefix(b"", 0, 1) == 0


def test_calendar_fields_against_datetime(host):
    """year / month / day / hour for every 7th day of years 1-9999 (pre-1970 included) against datetime, with a
    timestamp per day at a moving time of day"""
    d = datetime.date(1, 1, 1)
    step = datetime.timedelta(days=7)
    k = 0
    while True:
        days = (d - EPOCH).days
        assert host.emu_years(days) == P.years(days) == P.years_dt(d), d
        assert host.emu_months(days) == P.months(days) == P.months_dt(d), d
        us = days * P.MICROS_PER_DAY + (k * 7919 % 86400) * 1000000 + k % 1000000
        dt = datetime.datetime(d.year, d.month, d.day) + datetime.timedelta(microseconds=us - days * P.MICROS_PER_DAY)
        assert host.emu_days(us) == P.transform(R.TIMESTAMP_US, us, P.DAY, 0) == (dt.date() - EPOCH).days
        hours = (dt - datetime.datetime(1970, 1, 1)) // datetime.timedelta(hours=1)
        assert host.emu_hours(us) == P.transform(R.TIMESTAMPTZ_US, us, P.HOUR, 0) == hours
        assert P.transform(R.TIMESTAMP_US, us, P.MONTH, 0) == P.months_dt(dt.date())
        k += 1
        if d > datetime.date(9999, 12, 24):
            break
        d += step
    # 1969-12-31: year -1, month -1, day -1; a microsecond before the epoch is hour -1
    assert P.years(-1) == P.months(-1) == -1 and host.emu_years(-1) == host.emu_months(-1) == -1
    assert host.emu_days(-1) == -1 and host.emu_hours(-1) == -1 and host.emu_hours(0) == 0
    assert P.months(0) == 0 and P.years(365) == 1 and P.months(31) == 1


def test_calendar_fields_beyond_datetime(host):
    """the integer formulas outside years 1-9999: the whole int64 microsecond range and Date32 extremes"""
    rng = np.random.default_rng(8)
    days = [I32_MIN, I32_MAX, -719163, -719162, 2932897] + [int(x) for x in rng.integers(I32_MIN, I32_MAX, 20000)]
    for dd in days:
        assert host.emu_years(dd) == P.years(dd) and host.emu_months(dd) == P.months(dd), dd
        y, m = P.civil(dd)
        assert 1 <= m <= 12
        # the day count of (y, m, 1) is at or before dd and the next month's is after it
        assert P.civil(dd - 31)[0] * 12 + P.civil(dd - 31)[1] < y * 12 + m + 1
    for us in [I64_MIN, I64_MAX, -1, 0, 1] + [int(x) for x in rng.integers(I64_MIN, I64_MAX, 20000, dtype=np.int64)]:
        assert host.emu_days(us) == us // P.MICROS_PER_DAY and host.emu_hours(us) == us // P.MICROS_PER_HOUR, us
        assert host.emu_years(us // P.MICROS_PER_DAY) == P.transform(R.TIMESTAMPTZ_US, us, P.YEAR, 0)


# ------------------------------------------------------------------------------------------------ grouping
def test_grouping_order_of_the_restatement():
    vals = np.array([5, 3, 5, 7, 3, 5, 9], np.int32)
    col = {"type": R.INT32, "valid": np.array([1, 1, 1, 1, 1, 0, 1], bool), "values": vals}
    perm, offs, values = P.partition([col], [(0, P.IDENTITY, 0)], 0, 7)
    assert perm == [0, 2, 1, 4, 3, 5, 6] and offs == [0, 2, 4, 5, 6, 7] and values == [(5,), (3,), (7,), (None,), (9,)]
    perm, offs, values = P.partition([col], [(0, P.IDENTITY, 0)], 2, 5)
    assert perm == [2, 3, 4] and offs == [0, 1, 2, 3]
    assert P.partition([col], [(0, P.VOID, 0)], 0, 7) == (list(range(7)), [0, 7], [(None,)])
    assert P.partition([col], [(0, P.IDENTITY, 0)], 3, 3) == ([], [0], [])
    t = P.take(col, perm)
    assert t["values"].tolist() == [5, 7, 3]


def test_accepted_pairs():
    for at in (R.FLOAT32, R.FLOAT64):
        assert [tr for tr in range(8) if P.accepts(at, tr)] == [P.VOID]
    assert not any(P.accepts(R.LIST, tr) for tr in range(8))
    assert [tr for tr in range(8) if P.accepts(R.BOOLEAN, tr)] == [P.IDENTITY, P.VOID]
    assert [tr for tr in range(8) if P.accepts(R.TIMESTAMPTZ_US, tr)] == [P.IDENTITY, P.BUCKET, P.YEAR, P.MONTH, P.DAY, P.HOUR, P.VOID]
    assert [tr for tr in range(8) if P.accepts(R.UUID, tr)] == [P.IDENTITY, P.BUCKET, P.VOID]
    assert not P.accepts(R.INT32, 8)


# ------------------------------------------------------------------------------------------------ layout
def test_struct_layouts(tmp_path):
    pairs = [("etl_iceberg_partition_field", abi.IcebergPartitionField, 16), ("etl_iceberg_partition_value", abi.IcebergPartitionValue, 24)]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "etl_decode.h"', 'int main(void) {']
    for cname, ct, _ in pairs:
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in ct._fields_:
            lines.append(f'  printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    lines.append('  printf("max %u\\n", ETL_ICE_MAX_FIELDS);')
    lines.append('  printf("void %d hour %d\\n", ETL_ICE_VOID, ETL_ICE_HOUR);')
    lines += ['  return 0;', '}']
    src = tmp_path / "ice_sizes.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "ice_sizes"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    out = subprocess.check_output([str(exe)], text=True).splitlines()
    got = dict(l.split(None, 1) for l in out)
    for cname, ct, size in pairs:
        assert int(got[cname]) == C.sizeof(ct) == size, cname
        for fname, _ in ct._fields_:
            assert int(got[f"{cname}.{fname}"]) == getattr(ct, fname).offset, f"{cname}.{fname}"
    assert int(got["max"]) == abi.ICE_MAX_FIELDS
    assert got["void"] == f"{abi.ICE_VOID} hour {abi.ICE_HOUR}"
    assert (P.IDENTITY, P.BUCKET, P.TRUNCATE, P.YEAR, P.MONTH, P.DAY, P.HOUR, P.VOID) == (
        abi.ICE_IDENTITY, abi.ICE_BUCKET, abi.ICE_TRUNCATE, abi.ICE_YEAR, abi.ICE_MONTH, abi.ICE_DAY, abi.ICE_HOUR, abi.ICE_VOID)
