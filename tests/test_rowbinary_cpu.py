"""ClickHouse RowBinary emitter, CPU side:
* the Python restatement (tests/clickhouse_ref.py) pinned to the reference's own known answers, transcribed as data from
  crates/etl-destinations/src/clickhouse/encoding.rs:283-511 and core.rs:1133-1147;
* the device formatters (etl_b200/csrc/rowbinary_format.cuh) compiled for the host (tests/emul/host_rowbinary.cpp) and
  fuzzed against the restatement: varint, NaiveTime's Display, hex, the Date32 range;
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
import clickhouse_ref as R  # noqa: E402

N_FUZZ = int(os.environ.get("ETL_HOST_FUZZ_N", "100000"))
EPOCH = datetime.date(1970, 1, 1)


def days(y, m, d):
    return (datetime.date(y, m, d) - EPOCH).days


# ------------------------------------------------------------------------------------------------ known answers
def test_varint_known_answers():
    # encoding.rs:436-453 varint_encoding
    assert R.varint(0) == bytes([0x00])
    assert R.varint(127) == bytes([0x7F])
    assert R.varint(128) == bytes([0x80, 0x01])
    assert R.varint(300) == bytes([0xAC, 0x02])


def test_hex_known_answers():
    # encoding.rs:455-461 hex_encoding, :367-375 cell_to_clickhouse_value_bytes_hex
    assert R.hex_text(b"") == b""
    assert R.hex_text(b"\x00") == b"00"
    assert R.hex_text(b"\xff") == b"ff"
    assert R.hex_text(bytes([0xDE, 0xAD, 0xBE, 0xEF])) == b"deadbeef"
    assert R.value_bytes(16, ("bytes", bytes([0xDE, 0xAD, 0xBE, 0xEF])), []) == b"\x08deadbeef"


def test_date32_known_answers():
    # encoding.rs:315-345: epoch 0, 1970-01-02 1, 1969-12-31 -1; 1899-12-31 and 2300-01-01 rejected
    for (y, m, d), want in [((1970, 1, 1), 0), ((1970, 1, 2), 1), ((1969, 12, 31), -1)]:
        bad = []
        assert R.value_bytes(10, ("date", days(y, m, d)), bad) == struct.pack("<i", want) and not bad
    for y, m, d in [(1899, 12, 31), (2300, 1, 1)]:
        bad = []
        R.value_bytes(10, ("date", days(y, m, d)), bad)
        assert bad == [None], (y, m, d)
    assert (days(1900, 1, 1), days(2299, 12, 31)) == (R.DATE32_MIN, R.DATE32_MAX)


def test_scalar_known_answers():
    # encoding.rs:377-404 rb_encode_value_scalars, :347-354 timestamp at the epoch
    assert R.value_bytes(1, True, []) == bytes([1])
    assert R.value_bytes(4, -1, []) == (-1).to_bytes(4, "little", signed=True)
    assert R.value_bytes("u64", 2**64 - 1, []) == b"\xff" * 8
    assert R.value_bytes(2, "hi", []) == bytes([2, ord("h"), ord("i")])
    assert R.value_bytes(12, ("timestamp", 0, 0), []) == b"\x00" * 8


def test_uuid_wire_known_answer():
    # encoding.rs:406-420 rb_encode_uuid_wire_format
    be = bytes.fromhex("550e8400e29b41d4a716446655440000")
    want = int.from_bytes(be[:8], "big").to_bytes(8, "little") + int.from_bytes(be[8:], "big").to_bytes(8, "little")
    assert R.value_bytes(14, ("uuid", be.hex()), []) == want
    assert want == bytes.fromhex("d4419be200840e55" "00004455664416a7")


def test_nullable_and_null_known_answers():
    # encoding.rs:422-434 encode_nullable, :471-480 a NULL for a non-nullable column is an error
    issues = {}
    assert R.row_bytes([(0, None)], [True], issues, 0) == b"\x01" and not issues
    assert R.row_bytes([(4, 42)], [True], issues, 0) == b"\x00\x2a\x00\x00\x00" and not issues
    assert R.row_bytes([(0, None)], [False], issues, 7) == b""
    assert issues["null"] == (7, 0, R.NONE32)


def test_cdc_lsn_known_answer():
    # core.rs:1133-1140 cdc_lsn_value_preserves_full_u64_range: UInt64, little-endian on the wire
    row = R.row_bytes([(2, "DELETE"), ("u64", 2**64 - 1)], [False, False], {}, 0)
    assert row == b"\x06DELETE" + b"\xff" * 8


def test_key_row_expansion():
    # core.rs:944-962 / :970-997: pk columns take the key cells, nullable scalars NULL, arrays and NOT NULL columns zero
    kinds = [6, 2, 0x20 | 4, 4, 10, 2]
    col_flags = [2, 1, 1, 0, 0, 3]
    pk = [True, False, False, False, False, True]
    out = R.expand_key_row([(6, 5)], kinds, col_flags, pk)
    assert out == [(6, 5), (0, None), ("default", 0x24), ("default", 4), ("default", 10), (0, None)]
    row = R.row_bytes(out, [False, True, False, False, False, True], {}, 0)
    assert row == struct.pack("<q", 5) + b"\x01" + b"\x00" + b"\x00" * 4 + b"\x00" * 4 + b"\x01"


def test_time_display_known_answers():
    # chrono NaiveTime's Display: fraction by divisibility, leap second as :60
    assert R.time_text(0, 0) == b"00:00:00"
    assert R.time_text(3723, 500_000_000) == b"01:02:03.500"
    assert R.time_text(3723, 123_456_000) == b"01:02:03.123456"
    assert R.time_text(3723, 123_456_789) == b"01:02:03.123456789"
    assert R.time_text(86399, 1_000_000_000) == b"23:59:60"
    assert R.time_text(86399, 1_250_000_000) == b"23:59:60.250"


# ------------------------------------------------------------------------------------------------ host build of the device formatters
@pytest.fixture(scope="module")
def emu():
    src = os.path.join(HERE, "emul", "host_rowbinary.cpp")
    out_dir = tempfile.mkdtemp(prefix="etl_host_rowbinary_")
    so = os.path.join(out_dir, "libhost_rowbinary.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           "-I", os.path.join(ROOT, "etl_b200", "csrc"), "-o", so, src])
    L = C.CDLL(so)
    L.emu_varint.restype = C.c_int64
    L.emu_varint.argtypes = [C.c_uint64, C.c_char_p]
    L.emu_time.restype = C.c_int64
    L.emu_time.argtypes = [C.c_uint64, C.c_uint32, C.c_char_p]
    L.emu_hex.argtypes = [C.c_char_p, C.c_uint32, C.c_char_p]
    L.emu_date32_ok.argtypes = [C.c_int64]
    L.emu_uuid.argtypes = [C.c_char_p, C.c_char_p]
    return L


def test_varint_fuzz(emu):
    rng = random.Random(1)
    buf = C.create_string_buffer(16)
    edges = [1 << 7, 1 << 14, 1 << 21, 1 << 28]
    for i in range(N_FUZZ):
        e = edges[i % 4]
        v = e + rng.randint(-3, 2) if i % 3 else rng.randrange(0, 1 << (7 * (1 + i % 9)))
        n = emu.emu_varint(v, buf)
        assert n >= 0 and buf.raw[:n] == R.varint(v), v


def test_time_fuzz(emu):
    rng = random.Random(2)
    buf = C.create_string_buffer(32)
    for i in range(N_FUZZ):
        secs = rng.randrange(86400) if i % 7 else 86399
        mode = i % 4
        nanos = [0, rng.randrange(1000) * 10**6, rng.randrange(10**6) * 1000, rng.randrange(10**9)][mode]
        if i % 7 == 0:
            nanos += 10**9                              # leap second
        n = emu.emu_time(secs, nanos, buf)
        assert n >= 0 and buf.raw[:n] == R.time_text(secs, nanos), (secs, nanos)


def test_hex_fuzz(emu):
    rng = random.Random(3)
    out = C.create_string_buffer(2 * 64)
    for i in range(N_FUZZ):
        b = bytes(rng.randrange(256) for _ in range(i % 33))
        emu.emu_hex(b, len(b), out)
        assert out.raw[:2 * len(b)] == R.hex_text(b), b


def test_date32_fuzz(emu):
    rng = random.Random(4)
    for i in range(N_FUZZ):
        d = rng.choice([R.DATE32_MIN, R.DATE32_MAX]) + rng.randint(-2, 2) if i % 2 else rng.randint(-(1 << 40), 1 << 40)
        assert bool(emu.emu_date32_ok(d)) == R.date32_ok(d), d


def test_uuid_wire_host(emu):
    rng = random.Random(5)
    out = C.create_string_buffer(16)
    for _ in range(1000):
        be = bytes(rng.randrange(256) for _ in range(16))
        emu.emu_uuid(be, out)
        assert out.raw[:16] == R.uuid_wire(be)


# ------------------------------------------------------------------------------------------------ ABI
def test_issue_struct_layouts(tmp_path):
    from etl_b200 import abi
    pairs = [("etl_rb_issue", abi.RbIssue), ("etl_rowbinary_issues", abi.RowBinaryIssues)]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "etl_decode.h"', 'int main(void) {']
    for cname, ct in pairs:
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in ct._fields_:
            lines.append(f'  printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ['  return 0;', '}']
    src = tmp_path / "rb_sizes.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "rb_sizes"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = dict(line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())
    for cname, ct in pairs:
        assert int(got[cname]) == C.sizeof(ct), cname
        for fname, _ in ct._fields_:
            assert int(got[f"{cname}.{fname}"]) == getattr(ct, fname).offset, f"{cname}.{fname}"
