"""DuckLake emitter, CPU side:
* the Python restatement (tests/ducklake_ref.py) pinned to the reference's own known answers, transcribed as data from
  crates/etl-destinations/src/ducklake/encoding.rs:394-422, batches.rs:2116-2880 and core.rs:1533-1567;
* FNV-1a 64 against its standard vectors;
* the device formatters (etl_b200/csrc/ducklake_format.cuh) compiled for the host (tests/emul/host_ducklake.cpp) and
  fuzzed against the restatement: the shortest digits of doubles and widened floats against Python's repr (Rust's
  Display is assumed to give the same digits; no Rust toolchain checked that), quote_literal, uppercase hex, 6-digit
  times with leap seconds, dates and timestamps with years outside 0..9999, integers, FNV over every alignment;
* the ctypes mirrors of the emitter's structs against the C layout of include/etl_decode.h."""
import ctypes as C
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
import ducklake_ref as R  # noqa: E402

N_FUZZ = int(os.environ.get("ETL_HOST_FUZZ_N", "100000"))
DAY_MIN, DAY_MAX = -96465292, 95026236


def f64(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def f32(x: float) -> int:
    return struct.unpack("<I", struct.pack("<f", x))[0]


# ------------------------------------------------------------------------------------------------ known answers
def test_array_literals_known_answers():
    # encoding.rs:394-422
    assert R.value_literal(17, ("array", 4, [1, None, 3])) == "[1, NULL, 3]"
    assert R.value_literal(17, ("array", 15, [("json", b'{"a": 1}'), None])) == "[CAST('{\"a\":1}' AS JSON), NULL]"
    assert R.row_text([(4, 1), (17, ("array", 4, [1, None, 3]))]) == "(1, [1, NULL, 3])"
    assert R.value_literal(17, ("array", 4, [])) == "[]"


def test_scalar_literals():
    assert R.value_literal(0, None) == "NULL"
    assert R.value_literal(1, True) == "TRUE" and R.value_literal(1, False) == "FALSE"
    assert R.value_literal(5, ("u32", 2**32 - 1)) == "4294967295"
    assert R.value_literal(2, "it's") == "'it''s'"
    assert R.value_literal(2, "a\\b") == "E'a\\\\b'"
    assert R.value_literal(16, ("bytes", b"\x00\xab")) == "from_hex('00AB')"
    assert R.value_literal(14, ("uuid", "550E8400E29B41D4A716446655440000")) == "CAST('550e8400-e29b-41d4-a716-446655440000' AS UUID)"
    assert R.value_literal(11, ("time", 3723, 123_456_789)) == "TIME '01:02:03.123456'"
    assert R.value_literal(11, ("time", 86399, 1_000_000_000)) == "TIME '23:59:60.000000'"
    assert R.value_literal(12, ("timestamp", -1, 500_000_000)) == "TIMESTAMP '1969-12-31 23:59:59.500000'"
    assert R.value_literal(13, ("timestamptz", 0, 0)) == "TIMESTAMPTZ '1970-01-01 00:00:00.000000+00:00'"
    assert R.value_literal(10, ("date", 0)) == "DATE '1970-01-01'"
    assert R.value_literal(9, ("numeric", "+", 0, 1, [1, 5000])) == "'1.5'"


def test_float_literals():
    assert R.value_literal(8, ("f64", f64(1e21))) == "1000000000000000000000"
    assert R.value_literal(8, ("f64", f64(5e-324))) == "0." + "0" * 323 + "5"
    assert R.value_literal(8, ("f64", f64(-0.0))) == "-0"
    assert R.value_literal(8, ("f64", f64(1.0))) == "1"
    assert R.value_literal(8, ("f64", f64(0.1))) == "0.1"
    assert R.value_literal(7, ("f32", f32(0.1))) == "0.10000000149011612"
    assert R.value_literal(8, ("f64", f64(float("nan")))) == "CAST('NaN' AS DOUBLE)"
    assert R.value_literal(7, ("f32", f32(float("-inf")))) == "CAST('-Infinity' AS FLOAT)"
    assert R.value_literal(8, ("f64", f64(float("inf")))) == "CAST('Infinity' AS DOUBLE)"


def test_predicate_known_answers():
    # batches.rs:2116-2205: composite key, a key image, FULL identity (every column, NULL as IS NULL)
    assert R.predicate_text([("tenant_id", (4, 7)), ("id", (6, 42))]) == "tenant_id = 7 AND id = 42"
    assert R.predicate_text([("email", (2, "alice@example.com"))]) == "email = 'alice@example.com'"
    assert R.predicate_text([("id", (4, 1)), ("name", (2, "a")), ("note", (0, None))]) == "id = 1 AND name = 'a' AND note IS NULL"
    # :2208-2380: replace deletes by the new row's identity; assignments of a partial row; an alternative identity
    assert R.predicate_text([("id", (4, 1))]) == "id = 1"
    asg = R.assignments(["id", "name", "note"], [(4, 1), (2, "after"), (254, ("missing",))])
    assert [f"{['id', 'name', 'note'][c]} = {lit}" for c, lit in asg] == ["id = 1", "name = 'after'"]
    assert R.predicate_text([("email", (2, "a@b")), ("region", (2, "eu"))]) == "email = 'a@b' AND region = 'eu'"
    assert R.assignments(["a"], [(0, None)]) == [(0, "NULL")]


def test_key_row_from_partial_row():
    # core.rs:1533-1567: the identity cells of the present columns, in schema order; a missing key column rejects
    cells = [(4, 1), (254, ("missing",)), (2, "k")]
    assert R.key_row_from_partial(cells, [True, False, True]) == [(4, 1), (2, "k")]
    assert R.key_row_from_partial(cells, [True, True, False]) is None


def _want(kinds_texts, commits):
    want = dict(kinds=[], texts=([], [], []), start=[], commit=[], tx=[], seg=[], asg=[], n_cols=2, records=[])
    for m, ((kind, row, pred), (c, t)) in enumerate(zip(kinds_texts, commits)):
        want["kinds"].append(kind)
        want["texts"][0].append(row)
        want["texts"][1].append(pred)
        want["texts"][2].append("")
        want["asg"].append(None)
        want["start"].append(c - 8)
        want["commit"].append(c)
        want["tx"].append(t)
        want["seg"].append(0)
        want["records"].append(m)
    return want


def test_retain_rule_and_identity():
    # batches.rs:2718-2770: only mutations strictly after the persisted key stay
    want = _want([(R.INSERT, "(1, 'a')", "")] * 3, [(10, 0), (10, 1), (20, 0)])
    assert R.retained(want, None) == [0, 1, 2]
    assert R.retained(want, (10, 0)) == [1, 2]
    assert R.retained(want, (10, 1)) == [2]
    assert R.retained(want, (20, 0)) == []
    # :2773-2880: deterministic; changes with the order of the mutations and with an LSN
    a = R.mutation_fingerprint(want, b"public_t", [0, 1, 2])
    assert a == R.mutation_fingerprint(want, b"public_t", [0, 1, 2])
    want2 = _want([(R.INSERT, "(1, 'a')", ""), (R.DELETE, "", "id = 1"), (R.INSERT, "(2, 'b')", "")], [(10, 0), (10, 1), (20, 0)])
    want3 = _want([(R.DELETE, "", "id = 1"), (R.INSERT, "(1, 'a')", ""), (R.INSERT, "(2, 'b')", "")], [(10, 0), (10, 1), (20, 0)])
    assert R.mutation_fingerprint(want2, b"t", [0, 1, 2]) != R.mutation_fingerprint(want3, b"t", [0, 1, 2])
    want4 = _want([(R.INSERT, "(1, 'a')", "")] * 3, [(10, 0), (10, 1), (21, 0)])
    assert R.mutation_fingerprint(want4, b"public_t", [0, 1, 2]) != a
    subs = R.sub_batches(want, b"public_t")
    assert R.batch_id(want, subs[0]) == "mutation:%016x:%016x:%016x" % (2, 20, subs[0][2])


def test_chunks_of_sixteen_within_runs():
    want = _want([(R.INSERT, "(%d)" % i, "") for i in range(40)], [(100 + i, 0) for i in range(40)])
    want["seg"] = [0] * 20 + [1] * 20
    assert [(f, n) for f, n, _ in R.sub_batches(want, b"t")] == [(0, 16), (16, 4), (20, 16), (36, 4)]
    assert [(f, n) for f, n, _ in R.sub_batches(want, b"t", (104, 0))] == [(5, 15), (20, 16), (36, 4)]


def test_fnv_vectors():
    assert R.fnv1a64(b"") == 0xCBF29CE484222325
    assert R.fnv1a64(b"a") == 0xAF63DC4C8601EC8C
    assert R.fnv1a64(b"foobar") == 0x85944171F73967E8


# ------------------------------------------------------------------------------------------------ host build of the device formatters
@pytest.fixture(scope="module")
def emu():
    src = os.path.join(HERE, "emul", "host_ducklake.cpp")
    out_dir = tempfile.mkdtemp(prefix="etl_host_ducklake_")
    so = os.path.join(out_dir, "libhost_ducklake.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           "-I", os.path.join(ROOT, "etl_b200", "csrc"), "-o", so, src])
    L = C.CDLL(so)
    for f, args in (("emu_float_lit", [C.c_uint64, C.c_int, C.c_char_p]), ("emu_quote", [C.c_char_p, C.c_uint32, C.c_char_p]),
                    ("emu_bytes_lit", [C.c_char_p, C.c_uint32, C.c_char_p]), ("emu_time_lit", [C.c_uint64, C.c_uint32, C.c_char_p]),
                    ("emu_date_lit", [C.c_int64, C.c_char_p]), ("emu_ts_lit", [C.c_int64, C.c_uint32, C.c_int, C.c_char_p]),
                    ("emu_int_lit", [C.c_int64, C.c_char_p])):
        getattr(L, f).restype = C.c_int64
        getattr(L, f).argtypes = args
    for f in ("emu_fnv_str", "emu_fnv_bytes"):
        getattr(L, f).restype = C.c_uint64
        getattr(L, f).argtypes = [C.c_char_p, C.c_uint64]
    return L


def _doubles(rng, n):
    fixed = [0.0, -0.0, 5e-324, 1e-323, 2.2250738585072014e-308, 2.225073858507201e-308, 1.7976931348623157e308, 0.1, 1.0,
             float(2**53 - 1), float(2**53), float(2**53 + 2), 9007199254740993.0, 1e15, 1e16, 1e21, 1e22, 1e23, 123.456]
    fixed += [2.0 ** e for e in range(-1074, 1024, 7)] + [10.0 ** e for e in range(-323, 309, 3)]
    fixed += [float(10 ** k) * m for k in range(15, 24) for m in (1, 3, 7, 9.5)]
    for x in fixed:
        yield x
    for i in range(n):
        r = i % 4
        if r == 0:
            yield struct.unpack("<d", struct.pack("<Q", rng.getrandbits(64)))[0]
        elif r == 1:
            yield struct.unpack("<d", struct.pack("<Q", rng.getrandbits(52)))[0]                # subnormals
        elif r == 2:
            yield float(2**53) + rng.randint(-5000, 5000) * rng.choice([1, 2, 4])
        else:
            yield float("%.*g" % (rng.randint(1, 17), rng.uniform(-1e25, 1e25)))


def test_f64_display_fuzz(emu):
    rng = random.Random(21)
    buf = C.create_string_buffer(400)
    for x in _doubles(rng, N_FUZZ):
        b = f64(x)
        n = emu.emu_float_lit(b, 1, buf)
        assert n >= 0 and buf.raw[:n].decode() == R.float_literal(b, True), repr(x)


def test_f32_widened_fuzz(emu):
    rng = random.Random(22)
    buf = C.create_string_buffer(400)
    fixed = [0x7FC00000, 0x7F800000, 0xFF800000, 0x80000000, 0, 1, 0x00800000, 0x7F7FFFFF, f32(0.1), f32(1e10)]
    for i in range(N_FUZZ + len(fixed)):
        b = fixed[i] if i < len(fixed) else rng.getrandbits(32)
        n = emu.emu_float_lit(b, 0, buf)
        assert n >= 0 and buf.raw[:n].decode() == R.float_literal(R.f32_as_f64_bits(b), False), hex(b)


def test_quote_literal_fuzz(emu):
    rng = random.Random(23)
    alphabet = ["a", "'", "\\", "é", "✓", "😀", " ", "''", "\\\\"]
    for _ in range(N_FUZZ):
        s = "".join(rng.choice(alphabet) for _ in range(rng.randint(0, 40)))
        b = s.encode()
        out = C.create_string_buffer(3 * len(b) + 8)
        n = emu.emu_quote(b, len(b), out)
        assert n >= 0 and out.raw[:n].decode() == R.quote_literal(s), s


def test_hex_fuzz(emu):
    rng = random.Random(24)
    for _ in range(N_FUZZ):
        b = bytes(rng.randrange(256) for _ in range(rng.randint(0, 24)))
        out = C.create_string_buffer(2 * len(b) + 16)
        n = emu.emu_bytes_lit(b, len(b), out)
        assert n >= 0 and out.raw[:n].decode() == R.value_literal(16, ("bytes", b))


def test_time_fuzz(emu):
    rng = random.Random(25)
    out = C.create_string_buffer(32)
    for i in range(N_FUZZ):
        secs = rng.randrange(86400)
        nanos = rng.randrange(10**9) if i % 5 else 10**9 + rng.randrange(10**9)       # leap seconds
        if i % 5 == 0:
            secs = secs // 60 * 60 + 59
        n = emu.emu_time_lit(secs, nanos, out)
        assert n >= 0 and out.raw[:n].decode() == R.value_literal(11, ("time", secs, nanos)), (secs, nanos)


def test_date_and_timestamp_fuzz(emu):
    rng = random.Random(26)
    out = C.create_string_buffer(96)
    for i in range(N_FUZZ):
        d = rng.randint(DAY_MIN, DAY_MAX) if i % 3 else rng.randint(-800000, 3000000)
        n = emu.emu_date_lit(d, out)
        assert n >= 0 and out.raw[:n].decode() == R.value_literal(10, ("date", d)), d
        secs = d * 86400 + rng.randrange(86400)
        nanos = [0, rng.randrange(10**9), rng.randrange(1000) * 1000][i % 3]
        tz = i % 2
        n = emu.emu_ts_lit(secs, nanos, tz, out)
        assert n >= 0 and out.raw[:n].decode() == R.value_literal(13 if tz else 12, ("t", secs, nanos)), (secs, nanos, tz)


def test_integer_fuzz(emu):
    rng = random.Random(27)
    out = C.create_string_buffer(32)
    for i in range(N_FUZZ):
        v = rng.choice([-2**63, 2**63 - 1, 0, -1]) if i % 50 == 0 else rng.randint(-2**(i % 64), 2**(i % 64))
        v = max(-2**63, min(2**63 - 1, v))
        n = emu.emu_int_lit(v, out)
        assert n >= 0 and out.raw[:n].decode() == str(v)


def test_fnv_device_code(emu):
    rng = random.Random(28)
    assert emu.emu_fnv_bytes(b"", 0) == 0xCBF29CE484222325
    assert emu.emu_fnv_bytes(b"a", 1) == 0xAF63DC4C8601EC8C
    assert emu.emu_fnv_bytes(b"foobar", 6) == 0x85944171F73967E8
    for _ in range(2000):
        b = bytes(rng.randrange(256) for _ in range(rng.randint(0, 90)))
        off = rng.randrange(8)
        buf = C.create_string_buffer(b"\0" * off + b, off + len(b))     # every alignment of the 8-byte loads
        p = C.cast(C.addressof(buf) + off, C.c_char_p)
        h = R.Hasher()
        h.str(b)
        assert emu.emu_fnv_str(p, len(b)) == h.h


# ------------------------------------------------------------------------------------------------ ABI
def test_struct_layouts(tmp_path):
    from etl_b200 import abi
    pairs = [("etl_ducklake_issues", abi.DuckLakeIssues), ("etl_dl_sub_batch", abi.DlSubBatch)]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "etl_decode.h"', 'int main(void) {']
    for cname, ct in pairs:
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in ct._fields_:
            lines.append(f'  printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ['  printf("kinds %d %d %d %d %d %d\\n", ETL_DL_INSERT, ETL_DL_UPDATE, ETL_DL_UPDATE_PARTIAL, ETL_DL_REPLACE, '
              'ETL_DL_DELETE, ETL_DL_MF_ARRAY);', '  return 0;', '}']
    src = tmp_path / "dl_sizes.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "dl_sizes"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    outp = subprocess.check_output([str(exe)], text=True).splitlines()
    got = dict(line.split(" ", 1) for line in outp)
    for cname, ct in pairs:
        assert int(got[cname]) == C.sizeof(ct), cname
        for fname, _ in ct._fields_:
            assert int(got[f"{cname}.{fname}"]) == getattr(ct, fname).offset, f"{cname}.{fname}"
    assert got["kinds"].split() == [str(x) for x in (R.INSERT, R.UPDATE, R.UPDATE_PARTIAL, R.REPLACE, R.DELETE, R.MF_ARRAY)]
    assert (abi.DL_INSERT, abi.DL_UPDATE, abi.DL_UPDATE_PARTIAL, abi.DL_REPLACE, abi.DL_DELETE, abi.DL_MF_ARRAY) == \
        (R.INSERT, R.UPDATE, R.UPDATE_PARTIAL, R.REPLACE, R.DELETE, R.MF_ARRAY)
