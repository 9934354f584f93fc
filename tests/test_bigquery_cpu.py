"""BigQuery Storage Write emitter, CPU side:
* the Python restatement (tests/bigquery_ref.py) pinned to the reference's own known answers, transcribed as data from
  crates/etl-destinations/src/bigquery/core.rs:2072-2260, encoding.rs and validation.rs tests;
* the restatement's wire bytes against an independent encoder (google.protobuf, when importable) over a proto2
  descriptor with the same field numbers;
* the device formatters (etl_b200/csrc/bigquery_format.cuh) compiled for the host (tests/emul/host_bigquery.cpp) and
  fuzzed against the restatement: dates over years -262143..262142, timestamps, uuids, signed varints, the scale rule
  and the Json integer rule;
* the ctypes mirrors of the emitter's structs against the C layout of include/etl_decode.h."""
import ctypes as C
import datetime
import os
import random
import struct
import subprocess
import sys
import tempfile

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.normpath(os.path.join(HERE, ".."))
sys.path.insert(0, HERE)
import bigquery_ref as R  # noqa: E402
from arrow_ref import numeric_bytes  # noqa: E402

N_FUZZ = int(os.environ.get("ETL_HOST_FUZZ_N", "100000"))
EPOCH = datetime.date(1970, 1, 1)
DAY_MIN, DAY_MAX = -96465292, 95026236      # -262143-01-01 and +262142-12-31, the years the decoder keeps


def days(y, m, d):
    return (datetime.date(y, m, d) - EPOCH).days


# ------------------------------------------------------------------------------------------------ known answers
def test_sparse_delete_row_known_answer():
    # core.rs:2072-2114: key image I32(42) of a 3-column table, DELETE with sequence "lsn:1": fields 1, 4, 5 only
    row = R.row_bytes([(1, 0, (4, 42)), (4, None, (2, "DELETE")), (5, None, (2, "lsn:1"))], {}, 0)
    assert bytes([0x08, 0x2A]) in row
    assert bytes([0x22, 0x06]) + b"DELETE" in row
    assert bytes([0x2A, 0x05]) + b"lsn:1" in row
    assert 0x12 not in row and 0x18 not in row


def test_update_row_split_known_answers():
    # core.rs:2154-2226: a key change gives DELETE (ordinal 0) then UPSERT (ordinal 1); an unchanged key one UPSERT
    assert R.sequence_key(0x10, 0x2, 0) == b"0000000000000010/0000000000000002/0000000000000000"
    assert len(R.sequence_key(2**64 - 1, 2**64 - 1, 1)) == 50
    assert not R.cells_equal((4, 1), (4, 2)) and R.cells_equal((4, 1), (4, 1))
    assert not R.cells_equal((2, "a"), (0, None))


def test_cell_equality_rules():
    nan = struct.unpack("<Q", struct.pack("<d", float("nan")))[0]
    neg0 = struct.unpack("<Q", struct.pack("<d", -0.0))[0]
    assert not R.cells_equal((8, ("f64", nan)), (8, ("f64", nan)))
    assert R.cells_equal((8, ("f64", neg0)), (8, ("f64", 0)))
    assert not R.cells_equal((9, ("numeric", "+", 0, 1, [1])), (9, ("numeric", "+", 0, 2, [1])))   # 1.0 vs 1.00
    assert R.cells_equal((15, ("json", b'{"a":1, "b":2}')), (15, ("json", b'{"b":2,"a":1}')))
    assert not R.cells_equal((15, ("json", b'{"a":1.0}')), (15, ("json", b'{"a":1}')))
    assert R.cells_equal((17, ("array", 4, [1, None])), (17, ("array", 4, [1, None])))
    assert not R.cells_equal((17, ("array", 4, [1, None])), (17, ("array", 4, [1, 2])))


def test_scalar_encodings_known_answers():
    # encoding.rs: prost int32 of a negative value is 10 bytes, bool / zero / empty string are still written
    assert R.field_bytes(1, 4, -1) == b"\x08" + b"\xff" * 9 + b"\x01"
    assert R.field_bytes(1, 3, -2) == b"\x08" + b"\xfe" + b"\xff" * 8 + b"\x01"
    assert R.field_bytes(2, 1, False) == b"\x10\x00"
    assert R.field_bytes(2, 4, 0) == b"\x10\x00"
    assert R.field_bytes(3, 2, "") == b"\x1a\x00"
    assert R.field_bytes(3, 0, None) == b""
    assert R.field_bytes(1, 5, ("u32", 2**32 - 1)) == b"\x08\xff\xff\xff\xff\x0f"
    assert R.field_bytes(1, 7, ("f32", 0x3FC00000)) == b"\x0d\x00\x00\xc0\x3f"
    assert R.field_bytes(1, 8, ("f64", 0x3FF8000000000000)) == b"\x09" + struct.pack("<d", 1.5)
    assert R.field_bytes(1, 16, ("bytes", b"\x00\xff")) == b"\x0a\x02\x00\xff"
    assert R.field_bytes(1, 17, ("array", 4, [])) == b""
    assert R.field_bytes(1, 17, ("array", 4, [1, -1])) == b"\x0a\x0b\x01" + b"\xff" * 9 + b"\x01"
    assert R.field_bytes(1, 17, ("array", 2, ["a", ""])) == b"\x0a\x01a\x0a\x00"


def test_text_forms_known_answers():
    assert R.date_text(0) == b"1970-01-01"
    assert R.date_text(days(1, 1, 1) - 366) == b"0000-01-01"
    assert R.date_text(days(1, 1, 1) - 366 - 365) == b"-0001-01-01"
    assert R.date_text(days(9999, 12, 31) + 1) == b"+10000-01-01"
    assert R.timestamp_text(-1, 500_000_000, False) == b"1969-12-31 23:59:59.500"
    assert R.timestamp_text(0, 0, True) == b"1970-01-01 00:00:00+00:00"
    assert R.time_text(3723, 123_456_000) == b"01:02:03.123456"
    assert R.uuid_text("550E8400E29B41D4A716446655440000") == b"550e8400-e29b-41d4-a716-446655440000"


def test_validation_known_answers():
    # validation.rs:179-276: scale 38 passes, 39 fails; zero of any scale and the specials pass
    assert not R.numeric_scale_bad(("numeric", "+", -10, 38, [1]))
    assert R.numeric_scale_bad(("numeric", "+", -10, 39, [1]))
    assert not R.numeric_scale_bad(("numeric", "+", 0, 50, []))
    assert not R.numeric_scale_bad(("numeric", "NaN"))
    # i64 / u64 boundary literals; floats and exponents never count
    assert not R.json_int_bad(b"[-9223372036854775808, 18446744073709551615, 1e400, 1.5]")
    assert R.json_int_bad(b"-9223372036854775809")
    assert R.json_int_bad(b'{"a":[18446744073709551616]}')
    assert not R.json_int_bad(b'"18446744073709551616"')
    assert R.cell_issue(17, ("array", 9, [None, ("numeric", "+", -10, 39, [1])])) == (R.ISSUE_ARRAY_NULL, 0)
    assert R.cell_issue(17, ("array", 15, [("json", b"1"), ("json", b"[99999999999999999999]")])) == (R.ISSUE_JSON_INTEGER, 1)


# ------------------------------------------------------------------------------------------------ independent encoder
def test_wire_bytes_against_protobuf():
    pb = pytest.importorskip("google.protobuf")
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    F = descriptor_pb2.FieldDescriptorProto
    fdp = descriptor_pb2.FileDescriptorProto(name="bq_row.proto", package="bq", syntax="proto2")
    m = fdp.message_type.add(name="Row")
    spec = [("b", F.TYPE_BOOL, 0), ("i16", F.TYPE_INT32, 0), ("i32", F.TYPE_INT32, 0), ("i64", F.TYPE_INT64, 0),
            ("u32", F.TYPE_UINT32, 0), ("f32", F.TYPE_FLOAT, 0), ("f64", F.TYPE_DOUBLE, 0), ("s", F.TYPE_STRING, 0),
            ("by", F.TYPE_BYTES, 0), ("ai32", F.TYPE_INT32, 1), ("ai64", F.TYPE_INT64, 1), ("af64", F.TYPE_DOUBLE, 1),
            ("ab", F.TYPE_BOOL, 1), ("as", F.TYPE_STRING, 1), ("aby", F.TYPE_BYTES, 1)]
    for k, (name, t, rep) in enumerate(spec):
        f = m.field.add(name=name, number=k + 1, type=t, label=F.LABEL_REPEATED if rep else F.LABEL_OPTIONAL)
        if rep and t not in (F.TYPE_STRING, F.TYPE_BYTES):
            f.options.packed = True
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fdp)
    Row = message_factory.GetMessageClass(pool.FindMessageTypeByName("bq.Row"))
    rng = random.Random(7)
    for _ in range(2000):
        i16, i32, i64 = rng.randint(-2**15, 2**15 - 1), rng.randint(-2**31, 2**31 - 1), rng.randint(-2**63, 2**63 - 1)
        u32 = rng.randint(0, 2**32 - 1)
        f32 = struct.unpack("<f", struct.pack("<f", rng.uniform(-1e6, 1e6)))[0]
        f64 = rng.uniform(-1e300, 1e300)
        s = "".join(rng.choice("aé✓z") for _ in range(rng.randint(0, 200)))
        by = bytes(rng.randrange(256) for _ in range(rng.randint(0, 140)))
        ai32 = [rng.randint(-2**31, 2**31 - 1) for _ in range(rng.randint(1, 5))]
        ai64 = [rng.randint(-2**63, 2**63 - 1) for _ in range(rng.randint(1, 5))]
        af64 = [rng.uniform(-1, 1) for _ in range(rng.randint(1, 5))]
        ab = [rng.random() < 0.5 for _ in range(rng.randint(1, 5))]
        as_ = ["x" * rng.randint(0, 3) for _ in range(rng.randint(1, 4))]
        aby = [bytes([rng.randrange(256)]) * rng.randint(0, 3) for _ in range(rng.randint(1, 4))]
        msg = Row(b=bool(i16 & 1), i16=i16, i32=i32, i64=i64, u32=u32, f32=f32, f64=f64, s=s, by=by, ai32=ai32, ai64=ai64,
                  af64=af64, ab=ab, **{"as": as_}, aby=aby)
        bits32 = struct.unpack("<I", struct.pack("<f", f32))[0]
        bits64 = lambda x: struct.unpack("<Q", struct.pack("<d", x))[0]  # noqa: E731
        cells = [(1, bool(i16 & 1)), (3, i16), (4, i32), (6, i64), (5, ("u32", u32)), (7, ("f32", bits32)),
                 (8, ("f64", bits64(f64))), (2, s), (16, ("bytes", by)), (17, ("array", 4, ai32)), (17, ("array", 6, ai64)),
                 (17, ("array", 8, [("f64", bits64(x)) for x in af64])), (17, ("array", 1, ab)), (17, ("array", 2, as_)),
                 (17, ("array", 16, [("bytes", x) for x in aby]))]
        ours = R.row_bytes([(k + 1, k, c) for k, c in enumerate(cells)], {}, 0)
        assert ours == msg.SerializeToString(deterministic=True)
    assert pb


# ------------------------------------------------------------------------------------------------ host build of the device formatters
@pytest.fixture(scope="module")
def emu():
    src = os.path.join(HERE, "emul", "host_bigquery.cpp")
    out_dir = tempfile.mkdtemp(prefix="etl_host_bigquery_")
    so = os.path.join(out_dir, "libhost_bigquery.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           "-I", os.path.join(ROOT, "etl_b200", "csrc"), "-o", so, src])
    L = C.CDLL(so)
    L.emu_date.restype = C.c_int64
    L.emu_date.argtypes = [C.c_int64, C.c_char_p]
    L.emu_timestamp.restype = C.c_int64
    L.emu_timestamp.argtypes = [C.c_int64, C.c_uint32, C.c_int, C.c_char_p]
    L.emu_uuid_text.argtypes = [C.c_char_p, C.c_char_p]
    L.emu_int_field.restype = C.c_int64
    L.emu_int_field.argtypes = [C.c_uint32, C.c_uint64, C.c_char_p]
    L.emu_numeric_scale_bad.argtypes = [C.c_char_p, C.c_uint32]
    L.emu_json_int_bad.argtypes = [C.c_char_p, C.c_uint32]
    return L


def test_day_range_ends():
    assert R.date_text(DAY_MIN) == b"-262143-01-01"
    assert R.date_text(DAY_MAX) == b"+262142-12-31"


def test_date_fuzz(emu):
    rng = random.Random(11)
    buf = C.create_string_buffer(32)
    for i in range(N_FUZZ):
        d = rng.randint(DAY_MIN, DAY_MAX) if i % 3 else rng.randint(-800000, 3000000)
        n = emu.emu_date(d, buf)
        assert n >= 0 and buf.raw[:n] == R.date_text(d), d


def test_timestamp_fuzz(emu):
    rng = random.Random(12)
    buf = C.create_string_buffer(64)
    for i in range(N_FUZZ):
        secs = rng.randint(DAY_MIN * 86400, DAY_MAX * 86400 + 86399) if i % 2 else rng.randint(-10**10, 10**10)
        nanos = [0, rng.randrange(1000) * 10**6, rng.randrange(10**6) * 1000, rng.randrange(10**9)][i % 4]
        tz = i % 5 == 0
        n = emu.emu_timestamp(secs, nanos, tz, buf)
        assert n >= 0 and buf.raw[:n] == R.timestamp_text(secs, nanos, tz), (secs, nanos, tz)


def test_uuid_text_fuzz(emu):
    rng = random.Random(13)
    out = C.create_string_buffer(36)
    for _ in range(N_FUZZ):
        be = bytes(rng.randrange(256) for _ in range(16))
        emu.emu_uuid_text(be, out)
        assert out.raw[:36] == R.uuid_text(be.hex())


def test_signed_varint_fuzz(emu):
    rng = random.Random(14)
    buf = C.create_string_buffer(16)
    for i in range(N_FUZZ):
        field = rng.choice([1, 15, 16, 2047, 2048, rng.randint(1, 5000)])
        bits_ = [16, 32, 64][i % 3]
        v = rng.randint(-2**(bits_ - 1), 2**(bits_ - 1) - 1)
        n = emu.emu_int_field(field, v & R.NONE64, buf)
        assert n >= 0 and buf.raw[:n] == R.key(field, R.WT_VARINT) + R.varint(v & R.NONE64), (field, v)


def test_scale_rule_fuzz(emu):
    rng = random.Random(15)
    for i in range(N_FUZZ):
        kind = 0 if i % 7 else rng.randint(1, 3)
        nd = 0 if i % 11 == 0 else rng.randint(1, 4)
        digits = [rng.randint(0, 9999) for _ in range(nd)]
        scale = rng.choice([37, 38, 39, 40, rng.randint(0, 200)])
        weight = rng.randint(-12, 3)
        num = ("numeric", ["NaN", "Infinity", "-Infinity"][kind - 1]) if kind else ("numeric", "+", weight, scale, digits)
        b = numeric_bytes(kind, 0, weight, scale, digits)
        assert bool(emu.emu_numeric_scale_bad(b, nd)) == R.numeric_scale_bad(num), num


def test_json_integer_rule_fuzz(emu):
    rng = random.Random(16)
    edges = [2**63, 2**63 - 1, 2**63 + 1, 2**64 - 1, 2**64, 2**64 + 1, 10**30, 0, 7]

    def num():
        v = rng.choice(edges) if rng.random() < 0.6 else rng.randint(0, 10**25)
        s = ("-" if rng.random() < 0.5 else "") + str(v)
        r = rng.random()
        return s + ".0" if r < 0.1 else (s + "e1" if r < 0.15 else s)

    for _ in range(N_FUZZ):
        doc = "[%s,{\"k\":%s},\"%s\"]" % (num(), num(), rng.choice(edges)) if rng.random() < 0.8 else num()
        b = doc.encode()
        assert bool(emu.emu_json_int_bad(b, len(b))) == R.json_int_bad(b), doc


# ------------------------------------------------------------------------------------------------ ABI
def test_issue_struct_layouts(tmp_path):
    from etl_b200 import abi
    pairs = [("etl_bq_issue", abi.BqIssue), ("etl_bigquery_issues", abi.BigQueryIssues)]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "etl_decode.h"', 'int main(void) {']
    for cname, ct in pairs:
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in ct._fields_:
            lines.append(f'  printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ['  return 0;', '}']
    src = tmp_path / "bq_sizes.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "bq_sizes"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = dict(line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())
    for cname, ct in pairs:
        assert int(got[cname]) == C.sizeof(ct), cname
        for fname, _ in ct._fields_:
            assert int(got[f"{cname}.{fname}"]) == getattr(ct, fname).offset, f"{cname}.{fname}"
