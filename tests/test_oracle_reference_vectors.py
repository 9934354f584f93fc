"""Pins the CPU oracle against every known-answer test the reference holds for the path
(SURVEY.md §8c).  Each block quotes the reference test it restates (file:line under
crates/etl/src/conversions/ of supabase/etl).  Pure CPU; no GPU, no access to the reference checkout.
"""
import datetime as dt
import struct

import pytest

from canon import decode_cell
from oracle import pyoracle as po

BOOL, BYTEA, CHAR, NAME, INT8, INT2, INT4, TEXT, OID, JSON = 16, 17, 18, 19, 20, 21, 23, 25, 26, 114
FLOAT4, FLOAT8, MONEY, BPCHAR, VARCHAR, DATE, TIME, TIMESTAMP, TIMESTAMPTZ = 700, 701, 790, 1042, 1043, 1082, 1083, 1114, 1184
NUMERIC, UUID, JSONB = 1700, 2950, 3802
BOOL_A, INT2_A, INT4_A, INT8_A, TEXT_A, OID_A, FLOAT4_A, FLOAT8_A = 1000, 1005, 1007, 1016, 1009, 1028, 1021, 1022
MONEY_A, NUMERIC_A, TIMESTAMPTZ_A, INTERVAL_A, INET_A = 791, 1231, 1185, 1187, 1041

E_UTF8, E_INT, E_FLOAT, E_DT, E_NUM, E_UUID, E_JSON, E_BOOL, E_BYTEA = 1, 2, 3, 4, 5, 6, 7, 8, 9
E_ARRAY_SHORT, E_ARRAY_BRACES = 20, 21


def parse(oid, text):
    if isinstance(text, str):
        text = text.encode()
    e, tag, val, aux, heap = po.parse_cell(oid, text)
    if e:
        return ("err", e)
    return decode_cell(tag, val, aux, text, heap)


def f32bits(x):
    return struct.unpack("<I", struct.pack("<f", x))[0]


def f64bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def epoch(y, mo, d, h=0, mi=0, s=0):
    return int((dt.datetime(y, mo, d, h, mi, s) - dt.datetime(1970, 1, 1)).total_seconds())


# ---------------------------------------------------------------- text.rs:291-356
def test_bool_text_rs_291():
    assert parse(BOOL, "t") is True
    assert parse(BOOL, "f") is False
    assert parse(BOOL, "invalid") == ("err", E_BOOL)


@pytest.mark.parametrize("s", ["", "true", "false", "0", "1", "T", "F", " t", "t ", " f ", "t\n", "f\t",
                               "t\0", "🤔", "ÿ", "tt", "tf", "ft", "ff"])
def test_bool_rs_26_103_rejects(s):
    assert parse(BOOL, s) == ("err", E_BOOL)


def test_integers_text_rs_302_346():
    assert parse(INT2, "123") == 123
    assert parse(INT4, "-456") == -456
    assert parse(INT8, "9223372036854775807") == 9223372036854775807
    assert parse(OID, "12345") == ("u32", 12345)
    assert parse(INT2, "-32768") == -32768
    assert parse(INT2, "32767") == 32767
    assert parse(INT4, "-2147483648") == -2147483648
    assert parse(INT4, "2147483647") == 2147483647
    assert parse(INT8, "-9223372036854775808") == -9223372036854775808
    assert parse(OID, "4294967295") == ("u32", 4294967295)


def test_integer_overflow_text_rs_349_356():
    for oid, s in [(INT2, "99999"), (INT4, "9999999999"), (INT8, "9223372036854775808"),
                   (INT8, "-9223372036854775809"), (OID, "-1"), (OID, "4294967296")]:
        assert parse(oid, s) == ("err", E_INT), (oid, s)


def test_integer_grammar_rust_core():
    # Rust FromStr for integers: optional single sign, ascii digits only
    assert parse(INT4, "+5") == 5
    assert parse(INT4, "007") == 7
    assert parse(OID, "+7") == ("u32", 7)
    for s in ["", "+", "-", " 1", "1 ", "1_0", "--1", "+-1", "1.0", "0x10", "１"]:
        assert parse(INT4, s) == ("err", E_INT), s
    assert parse(OID, "-0") == ("err", E_INT)


def test_integer_arrays_text_rs_359_381():
    assert parse(INT2_A, "{-32768,32767,NULL}") == ("array", 3, [-32768, 32767, None])
    assert parse(INT4_A, "{-2147483648,2147483647,NULL}") == ("array", 4, [-2147483648, 2147483647, None])
    assert parse(INT8_A, "{-9223372036854775808,9223372036854775807,NULL}") == \
        ("array", 6, [-9223372036854775808, 9223372036854775807, None])
    assert parse(OID_A, "{0,4294967295,NULL}") == ("array", 5, [("u32", 0), ("u32", 4294967295), None])


# ---------------------------------------------------------------- text.rs:383-451 floats
def test_floats_text_rs_383_416():
    assert parse(FLOAT4, "3.15") == ("f32", f32bits(3.15))
    assert parse(FLOAT8, "-2.818") == ("f64", f64bits(-2.818))
    assert parse(FLOAT4, "inf") == ("f32", 0x7F800000)
    assert parse(FLOAT8, "NaN") == ("f64", 0x7FF8000000000000)
    assert parse(FLOAT4, "3.4028235e38") == ("f32", 0x7F7FFFFF)
    assert parse(FLOAT4, "-3.4028235e38") == ("f32", 0xFF7FFFFF)
    assert parse(FLOAT8, "1.7976931348623157e308") == ("f64", 0x7FEFFFFFFFFFFFFF)
    assert parse(FLOAT8, "-1.7976931348623157e308") == ("f64", 0xFFEFFFFFFFFFFFFF)


def test_float_arrays_text_rs_419_451():
    got = parse(FLOAT4_A, "{-3.4028235e38,3.4028235e38,NaN,Infinity,-Infinity,NULL}")
    assert got == ("array", 7, [("f32", 0xFF7FFFFF), ("f32", 0x7F7FFFFF), ("f32", 0x7FC00000),
                               ("f32", 0x7F800000), ("f32", 0xFF800000), None])
    got = parse(FLOAT8_A, "{-1.7976931348623157e308,1.7976931348623157e308,NaN,Infinity,-Infinity,NULL}")
    assert got == ("array", 8, [("f64", 0xFFEFFFFFFFFFFFFF), ("f64", 0x7FEFFFFFFFFFFFFF),
                               ("f64", 0x7FF8000000000000), ("f64", 0x7FF0000000000000),
                               ("f64", 0xFFF0000000000000), None])


def test_float_grammar_rust_dec2flt():
    assert parse(FLOAT8, "1.") == ("f64", f64bits(1.0))
    assert parse(FLOAT8, ".5") == ("f64", f64bits(0.5))
    assert parse(FLOAT8, "+1e3") == ("f64", f64bits(1000.0))
    assert parse(FLOAT8, "1E-2") == ("f64", f64bits(0.01))
    assert parse(FLOAT8, "-nan") == ("f64", 0xFFF8000000000000)
    assert parse(FLOAT8, "+iNfInItY") == ("f64", 0x7FF0000000000000)
    assert parse(FLOAT8, "1e999") == ("f64", 0x7FF0000000000000)      # overflow → inf, not an error
    assert parse(FLOAT8, "1e-999") == ("f64", 0)
    assert parse(FLOAT8, "4.9406564584124654e-324") == ("f64", 1)     # min subnormal
    assert parse(FLOAT8, "2.2250738585072011e-308") == ("f64", 0x000FFFFFFFFFFFFF)  # famous halfway-ish case
    assert parse(FLOAT8, "9007199254740993") == ("f64", f64bits(9007199254740992.0))  # ties-to-even
    assert parse(FLOAT4, "16777217") == ("f32", f32bits(16777216.0))
    assert parse(FLOAT4, "1.00000017881393432617187499") == ("f32", 0x3F800001)  # f32 parsed directly, no double rounding
    for s in ["", ".", "e5", "1e", "1e+", " 1", "1 ", "+", "-", "1_0", "0x1p3", "infinit", "nan(1)", "1.2.3"]:
        assert parse(FLOAT8, s) == ("err", E_FLOAT), s


# ---------------------------------------------------------------- text.rs:454-468 strings
def test_string_types_text_rs_454_468():
    for oid in (TEXT, VARCHAR, CHAR, BPCHAR, NAME):
        assert parse(oid, "Hello, World!") == "Hello, World!"
    assert parse(MONEY, "$1,234.56") == "$1,234.56"
    assert parse(99999, "test") == "test"            # text.rs:798-810 unknown type → string
    assert parse(TEXT, "") == ""
    assert parse(TEXT, "héllo ✓ 🤔") == "héllo ✓ 🤔"


def test_invalid_utf8_event_rs_972():
    for bad in [b"\xff", b"\xc0\x80", b"\xed\xa0\x80", b"\xf4\x90\x80\x80", b"abc\xe2\x82", b"\x80", b"\xf8\x88\x80\x80\x80"]:
        e, *_ = po.parse_cell(TEXT, bad)
        assert e == E_UTF8, bad


# ---------------------------------------------------------------- numeric: text.rs:471-527 + numeric.rs:599-948
def num(s):
    return parse(NUMERIC, s)


def test_numeric_text_rs_471_511():
    assert num("123.45") == ("numeric", "+", 0, 2, [123, 4500])
    assert num("NaN") == ("numeric", "NaN")
    assert num("Infinity") == ("numeric", "Infinity")
    assert num("-Infinity") == ("numeric", "-Infinity")
    assert num("1e131071") == ("numeric", "+", 32767, 0, [1000])
    assert num("1e-16383") == ("numeric", "+", -4096, 16383, [10])
    assert num("1e131072") == ("err", E_NUM)
    assert num("1e-16384") == ("err", E_NUM)


def test_numeric_array_text_rs_514_527():
    assert parse(NUMERIC_A, "{-Infinity,NaN,NULL,123.45}") == \
        ("array", 9, [("numeric", "-Infinity"), ("numeric", "NaN"), None, ("numeric", "+", 0, 2, [123, 4500])])


def test_numeric_rs_599_727():
    assert num("123")[1:] == ("+", 0, 0, [123])
    assert num("-456")[1:] == ("-", 0, 0, [456])
    assert num("NaN   ") == ("numeric", "NaN")
    assert num("+NaN") == ("err", E_NUM)
    assert num("-NaN") == ("err", E_NUM)
    assert num("+Infinity   ") == ("numeric", "Infinity")
    assert num("inf") == ("numeric", "Infinity")
    assert num("-inf") == ("numeric", "-Infinity")
    assert num("1.23e2") == ("numeric", "+", 0, 0, [123])
    for s in ["", "abc", "1.2.3"]:
        assert num(s) == ("err", E_NUM)


def test_numeric_max_shape_numeric_rs_681_705():
    s = "9" * ((32767 + 1) * 4) + "." + "9" * 16383
    got = num(s)
    assert got[1:4] == ("+", 32767, 16383)
    assert len(got[4]) == 36864 and got[4][0] == 9999 and got[4][-1] == 9990


def test_numeric_rs_761_948_canonical_forms():
    for s in ["0", "0.0", "000", "000.000", "-0", "-0.00"]:
        g = num(s)
        assert g[1] == "+" and g[2] == 0 and g[4] == [], s
    assert num("0.000")[3] == 3                                  # zero keeps its scale
    assert num("0.0012000") == ("numeric", "+", -1, 7, [12])
    assert num("9999.9999") == ("numeric", "+", 0, 4, [9999, 9999])
    assert num("10000.0001") == ("numeric", "+", 1, 4, [1, 0, 1])
    assert num("0000120.00") == ("numeric", "+", 0, 2, [120])
    assert num("1200000") == ("numeric", "+", 1, 0, [120])
    assert num("120.00") == ("numeric", "+", 0, 2, [120])
    assert num("1.2000") == ("numeric", "+", 0, 4, [1, 2000])
    assert num("0.0120") == ("numeric", "+", -1, 4, [120])
    assert num("-120.00") == ("numeric", "-", 0, 2, [120])


def test_numeric_grammar_numeric_rs_285_401():
    assert num("  12  ") == ("numeric", "+", 0, 0, [12])            # surrounding whitespace
    assert num("1_000") == ("numeric", "+", 0, 0, [1000])            # digit separators
    assert num("1_0.5") == ("numeric", "+", 0, 1, [10, 5000])
    assert num("1e1_0") == ("numeric", "+", 2, 0, [100])
    assert num(".5") == ("numeric", "+", -1, 1, [5000])
    assert num("5.") == ("numeric", "+", 0, 0, [5])
    assert num("+7") == ("numeric", "+", 0, 0, [7])
    for s in ["1._5", "1_", "_1", "1__0", "1e", "1e+", "1e_1", ".", "-", "+", "1 2", "1e5x", "--1", "0x10"]:
        assert num(s) == ("err", E_NUM), s
    assert num("1e1073741824") == ("err", E_NUM)                     # exponent > i32::MAX/2 → ValueOutOfRange
    assert num("0." + "0" * 16384) == ("err", E_NUM)                 # scale > 16383


# ---------------------------------------------------------------- bytea: text.rs:530-535 + hex.rs:44-190
def test_bytea():
    assert parse(BYTEA, "\\x48656c6c6f") == ("bytes", b"Hello")
    assert parse(BYTEA, "invalid") == ("err", E_BYTEA)
    assert parse(BYTEA, "\\x") == ("bytes", b"")
    assert parse(BYTEA, "\\x41") == ("bytes", b"A")
    assert parse(BYTEA, "\\x0000") == ("bytes", b"\0\0")
    assert parse(BYTEA, "\\xffff") == ("bytes", b"\xff\xff")
    assert parse(BYTEA, "\\xaBcD") == ("bytes", b"\xab\xcd")
    assert parse(BYTEA, "\\x0123456789abcdef") == ("bytes", bytes.fromhex("0123456789abcdef"))
    assert parse(BYTEA, "\\x00010203040506070809") == ("bytes", bytes(range(10)))
    assert parse(BYTEA, "\\x414243444546") == ("bytes", b"ABCDEF")
    for s in ["41", "0x41", "", "\\"]:
        assert parse(BYTEA, s) == ("err", E_BYTEA), s          # Missing '\x' prefix
    for s in ["\\x4", "\\x41424", "\\x4🤔", "\\x4 1", "\\x41-42"]:
        assert parse(BYTEA, s) == ("err", E_BYTEA), s          # Odd number of hexadecimal digits
    for s in ["\\x4g", "\\xgg", "\\x4z", "\\xZZ", "\\x4 12", "\\x41-4"]:
        assert parse(BYTEA, s) == ("err", E_INT), s            # from_str_radix "invalid digit"
    assert parse(BYTEA, "\\x+f") == ("bytes", b"\x0f")          # u8::from_str_radix accepts a leading '+'


# ---------------------------------------------------------------- text.rs:538-592 date/time
def test_date_time_text_rs_538_592():
    assert parse(DATE, "2023-12-25") == ("date", (dt.date(2023, 12, 25) - dt.date(1970, 1, 1)).days)
    assert parse(DATE, "invalid-date") == ("err", E_DT)
    assert parse(TIME, "14:30:45.123") == ("time", 14 * 3600 + 30 * 60 + 45, 123000000)
    assert parse(TIME, "invalid-time") == ("err", E_DT)
    assert parse(TIMESTAMP, "2023-12-25 14:30:45.123") == ("timestamp", epoch(2023, 12, 25, 14, 30, 45), 123000000)
    assert parse(TIMESTAMPTZ, "2023-12-25 14:30:45.123+00:00") == ("timestamptz", epoch(2023, 12, 25, 14, 30, 45), 123000000)
    assert parse(TIMESTAMPTZ, "2023-12-25 14:30:45.123+00") == ("timestamptz", epoch(2023, 12, 25, 14, 30, 45), 123000000)


def test_timestamptz_array_fallback_text_rs_780_795():
    assert parse(TIMESTAMPTZ_A, '{"2023-01-01 12:00:00.000+00"}') == ("array", 13, [("timestamptz", epoch(2023, 1, 1, 12), 0)])


def test_chrono_semantics_unpinned():
    """chrono 0.4 leniency restated from the crate's parser (parity unpinned in-tree)."""
    assert parse(TIMESTAMPTZ, "2024-02-29 23:59:59.999999+05:30") == ("timestamptz", epoch(2024, 2, 29, 18, 29, 59), 999999000)
    assert parse(TIMESTAMPTZ, "2024-02-29 23:59:59-0800") == ("timestamptz", epoch(2024, 3, 1, 7, 59, 59), 0)
    assert parse(TIMESTAMPTZ, "2024-02-29 23:59:59Z") == ("timestamptz", epoch(2024, 2, 29, 23, 59, 59), 0)
    assert parse(TIMESTAMP, "2024-1-5 3:4:5") == ("timestamp", epoch(2024, 1, 5, 3, 4, 5), 0)       # 1..=width digits
    assert parse(TIMESTAMP, "2024-01-05    03:04:05") == ("timestamp", epoch(2024, 1, 5, 3, 4, 5), 0)  # space = \s*
    assert parse(TIMESTAMP, "2024-01-0503:04:05") == ("timestamp", epoch(2024, 1, 5, 3, 4, 5), 0)
    assert parse(TIME, "23:59:59.1234567891234") == ("time", 86399, 123456789)                       # >9 digits dropped
    assert parse(TIME, "23:59:60") == ("time", 86399, 1000000000)                                     # leap second
    assert parse(DATE, "0001-01-01") == ("date", -719162)
    assert parse(DATE, "+12345-01-01") == ("date", (12345 - 1970) * 365 + sum(1 for y in range(1970, 12345) if (y % 4 == 0 and y % 100 != 0) or y % 400 == 0))
    for s in ["2023-02-29", "2023-13-01", "2023-00-10", "2023-01-32", "12345-01-01", "2023-12-25 BC", "infinity",
              "2023-12-25x", "", "2023-12"]:
        assert parse(DATE, s) == ("err", E_DT), s
    for s in ["24:00:00", "12:60:00", "12:00:61", "12:00", "12:00:00.", "12:00:00 ", "1:2:3x"]:
        assert parse(TIME, s) == ("err", E_DT), s
    for s in ["2024-01-01 00:00:00", "2024-01-01 00:00:00+", "2024-01-01 00:00:00+1", "2024-01-01 00:00:00+01:6",
              "2024-01-01 00:00:00+01:60", "2024-01-01 00:00:00+24", "2024-01-01 00:00:00+05:30:15"]:
        assert parse(TIMESTAMPTZ, s) == ("err", E_DT), s


# ---------------------------------------------------------------- text.rs:595-636 uuid / json
def test_uuid_text_rs_595_605():
    assert parse(UUID, "550e8400-e29b-41d4-a716-446655440000") == ("uuid", "550e8400e29b41d4a716446655440000")
    assert parse(UUID, "invalid-uuid") == ("err", E_UUID)
    # uuid 1.x alternate spellings (parity unpinned)
    assert parse(UUID, "550E8400-E29B-41D4-A716-446655440000") == ("uuid", "550e8400e29b41d4a716446655440000")
    assert parse(UUID, "550e8400e29b41d4a716446655440000") == ("uuid", "550e8400e29b41d4a716446655440000")
    assert parse(UUID, "{550e8400-e29b-41d4-a716-446655440000}") == ("uuid", "550e8400e29b41d4a716446655440000")
    assert parse(UUID, "urn:uuid:550e8400-e29b-41d4-a716-446655440000") == ("uuid", "550e8400e29b41d4a716446655440000")
    for s in ["", "550e8400-e29b-41d4-a716-44665544000", "550e8400-e29b-41d4-a716-4466554400000",
              "550e8400-e29b-41d4-a716_446655440000", "g50e8400-e29b-41d4-a716-446655440000"]:
        assert parse(UUID, s) == ("err", E_UUID), s


def test_json_text_rs_607_636():
    js = '{"key": "value", "number": 42}'
    assert parse(JSON, js) == ("json", js.encode())
    assert parse(JSONB, js) == ("json", js.encode())
    assert parse(JSON, "invalid json") == ("err", E_JSON)
    assert parse(JSON, '{"value":1e309}') == ("json", b'{"value":1e309}')   # arbitrary_precision
    assert parse(JSONB, '{"value":1e309}') == ("json", b'{"value":1e309}')


def test_json_grammar_serde_json():
    ok = ['null', ' true ', '[]', '{}', '[1,2.5e-3,-0,"a\\u00e9\\n",{"k":[null]}]', '"\\ud83d\\ude00"', '0', '-0.0e+5',
          '\t\n\r [ ] ', '"é"', '1E5', '123456789012345678901234567890', "[" * 127 + "]" * 127]
    for s in ok:
        assert parse(JSON, s) == ("json", s.encode()), s
    bad = ['', ' ', '{', '[1,]', '{"a":1,}', "{'a':1}", '01', '1.', '.5', '+1', '1e', 'tru', 'nul', 'True', '"\\x"',
           '"\\ud800"', '"\\udc00"', '"\\ud800\\u0041"', '"a\nb"', '"unterminated', '[1 2]', '{"a" 1}', '{1:2}',
           '1 2', 'NaN', '-', '--1', '"\\u12g4"', "[" * 128 + "]" * 128]
    for s in bad:
        assert parse(JSON, s) == ("err", E_JSON), s


# ---------------------------------------------------------------- arrays text.rs:259-288, 639-795
def test_arrays_text_rs():
    assert parse(TEXT_A, '{"a","null"}') == ("array", 2, ["a", "null"])                   # :259-267
    assert parse(TEXT_A, "{a,NULL}") == ("array", 2, ["a", None])                          # :270-278
    assert parse(INT4_A, "{1,invalid,3}") == ("err", E_INT)                                 # :281-288
    assert parse(INT4_A, "{1,2,3}") == ("array", 4, [1, 2, 3])                              # :639-647
    assert parse(INT4_A, "{1,NULL,3}") == ("array", 4, [1, None, 3])                        # :650-658
    assert parse(TEXT_A, r'{"hello","world with spaces","with\"quotes"}') == \
        ("array", 2, ["hello", "world with spaces", 'with"quotes'])                         # :661-680
    assert parse(MONEY_A, r'{"$1,234.56",NULL,"-$0.01"}') == ("array", 2, ["$1,234.56", None, "-$0.01"])  # :683-695
    assert parse(INTERVAL_A, r'{"1 day",NULL,"2 hours"}') == ("array", 2, ["1 day", None, "2 hours"])     # :698-709
    assert parse(INET_A, "{127.0.0.1,NULL,192.168.0.1}") == ("array", 2, ["127.0.0.1", None, "192.168.0.1"])
    assert parse(INT4_A, "{}") == ("array", 4, [])                                          # :725-733
    assert parse(BOOL_A, "{t}") == ("array", 1, [True])                                     # :736-744
    assert parse(INT4_A, "1,2,3}") == ("err", E_ARRAY_BRACES)                               # :747-758
    assert parse(INT4_A, "{1,2,3") == ("err", E_ARRAY_BRACES)
    assert parse(INT4_A, "{") == ("err", E_ARRAY_SHORT)
    assert parse(INT4_A, "}") == ("err", E_ARRAY_SHORT)
    assert parse(INT4_A, "") == ("err", E_ARRAY_SHORT)
    assert parse(TEXT_A, r'{"line1\\nline2","tab\\there"}') == ("array", 2, ["line1\\nline2", "tab\\there"])  # :761-778
    assert parse(TEXT_A, "{nUlL,\"\",x}") == ("array", 2, [None, "", "x"])
    assert parse(TEXT_A, "{a,}") == ("array", 2, ["a", ""])       # trailing comma → one more (empty) element


# ---------------------------------------------------------------- frames: replication_trace.txt:481-485
def test_keepalive_golden_frame_replication_trace_481():
    from etl_b200 import pgoutput as pg
    golden = bytes([107, 0, 0, 0, 0, 1, 155, 217, 232, 0, 2, 179, 42, 70, 55, 56, 220, 0])
    wal_end = int.from_bytes(golden[1:9], "big")
    ts = int.from_bytes(golden[9:17], "big", signed=True)
    assert pg.keepalive(wal_end, ts, 0) == golden
    o = po.Oracle()
    p = o.decode(pg.frame(golden))
    assert p.first_error[0] is None and p.n_records == 1
    assert chr(p.rec_kind[0]) == "k" and int(p.rec_start_lsn[0]) == wal_end and int(p.rec_rel[0]) == 0
    assert p.n_events == 0
