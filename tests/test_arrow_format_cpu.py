"""The device formatters of the columnar emitter (etl_b200/csrc/arrow_format.cuh), compiled for the host
(tests/emul/host_format.cpp — test infrastructure, not a product path), against the Python restatements of PgNumeric's
and serde_json's Display (tests/arrow_ref.py), which are first pinned to the reference's own known answers
(crates/etl/src/conversions/numeric.rs tests, crates/etl-destinations/src/iceberg/encoding.rs cell_to_string test)."""
import ctypes as C
import json
import os
import random
import subprocess
import sys
import tempfile

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.normpath(os.path.join(HERE, ".."))
sys.path.insert(0, HERE)
from arrow_ref import json_display, numeric_bytes, numeric_display  # noqa: E402
from canon import numeric_from_heap  # noqa: E402

N_FUZZ = int(os.environ.get("ETL_HOST_FUZZ_N", "100000"))


@pytest.fixture(scope="module")
def fmt():
    src = os.path.join(HERE, "emul", "host_format.cpp")
    out_dir = tempfile.mkdtemp(prefix="etl_host_format_")
    so = os.path.join(out_dir, "libhost_format.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           "-I", os.path.join(ROOT, "etl_b200", "csrc"), "-o", so, src])
    L = C.CDLL(so)
    L.emu_numeric_text.restype = C.c_int64
    L.emu_numeric_text.argtypes = [C.c_char_p, C.c_uint32, C.c_char_p, C.c_uint32]
    L.emu_json_canon.restype = C.c_int64
    L.emu_json_canon.argtypes = [C.c_char_p, C.c_uint32, C.c_char_p]
    out = C.create_string_buffer(1 << 20)

    def numeric(entry: bytes, nd: int):
        n = L.emu_numeric_text(entry, nd, out, len(out))
        assert n >= 0, ("numeric_write and numeric_len disagree" if n == -1 else "too long", entry)
        return out.raw[:n].decode()

    def canon(doc: bytes):
        buf = C.create_string_buffer(len(doc) + 1) if len(doc) >= len(out) else out
        n = L.emu_json_canon(doc, len(doc), buf)
        return None if n < 0 else buf.raw[:n]
    return numeric, canon


def num(sign, weight, scale, digits):
    return ("numeric", "-" if sign else "+", weight, scale, list(digits))


# ------------------------------------------------------------------------------------------------ restatements pinned
def test_numeric_restatement_known_answers(oracle_mod):
    assert numeric_display(("numeric", "NaN")) == "NaN"
    assert numeric_display(("numeric", "Infinity")) == "Infinity"
    assert numeric_display(("numeric", "-Infinity")) == "-Infinity"
    assert numeric_display(num(0, 0, 0, [123])) == "123"                    # display_simple_integers
    assert numeric_display(num(1, 0, 0, [456])) == "-456"
    assert numeric_display(num(0, 0, 2, [1234, 5000])) == "1234.50"         # display_decimals
    assert numeric_display(num(0, 0, 0, [])) == "0"                         # display_zero
    assert numeric_display(num(0, 1, 0, [1234, 5678])) == "12345678"
    assert numeric_display(num(0, -1, 4, [1234])) == "0.1234"
    assert numeric_display(num(0, 1, 4, [1200, 0])).endswith("0000")
    # parsed by the oracle (parse_cell(1700, ...)), printed back: numeric.rs's string cases and round trips
    cases = {"0.0012000": "0.0012000", "9999.9999": "9999.9999", "10000.0001": "10000.0001", "0000120.00": "120.00",
             "-0": "0", "-0.00": "0", "0": "0", "0.000": "0", "000.000": "0", "1200000": "1200000", "NaN": "NaN"}
    for text, want in cases.items():
        e, tag, val, aux, heap = oracle_mod.parse_cell(1700, text.encode())
        assert e == 0 and tag == 9, text
        assert numeric_display(numeric_from_heap(heap, val, aux)) == want, text
    for case in ["120.00", "1.2000", "0.0120", "9999.9999", "10000.0001", "-120.00", "1200000"]:
        e, tag, val, aux, heap = oracle_mod.parse_cell(1700, case.encode())
        printed = numeric_display(numeric_from_heap(heap, val, aux))
        e2, _, val2, aux2, heap2 = oracle_mod.parse_cell(1700, printed.encode())
        assert printed == numeric_display(numeric_from_heap(heap2, val2, aux2)), case
        assert numeric_from_heap(heap, val, aux) == numeric_from_heap(heap2, val2, aux2), case


def test_json_restatement_known_answers():
    assert json_display(b'{"key": "value"}') == b'{"key":"value"}'                       # encoding.rs cell_to_string
    assert json_display(b' {"b":1, "a":[1 ,2,{"z":null}],"b":2} ') == b'{"a":[1,2,{"z":null}],"b":2}'
    assert json_display(b'[1.50, -0, 1E+5, 12345678901234567890123]') == b'[1.50,-0,1E+5,12345678901234567890123]'
    assert json_display(b'"\\u00e9\\ud83d\\ude00\\/\\u0000\\u001f\\b\\u007f"') == '"é😀/\\u0000\\u001f\\b\x7f"'.encode()
    assert json_display(b'{"k10":1,"k2":2,"\\u00e9":3,"z":4,"":5}') == '{"":5,"k10":1,"k2":2,"z":4,"é":3}'.encode()
    assert json_display(b'{"a":1,"a":{"x":1,"x":[]}}') == b'{"a":{"x":[]}}'


# ------------------------------------------------------------------------------------------------ device formatters
def test_numeric_formatter_edges(fmt):
    numeric, _ = fmt
    for kind, want in ((1, "NaN"), (2, "Infinity"), (3, "-Infinity")):
        assert numeric(numeric_bytes(kind, 0, 0, 0, []), 0) == want
    edges = [(0, 0, 0, [123]), (1, 0, 0, [456]), (0, 0, 2, [1234, 5000]), (0, 0, 0, []), (1, 5, 9, []), (0, 1, 0, [1234, 5678]),
             (0, -1, 4, [1234]), (0, 1, 4, [1200, 0]), (0, -1, 7, [12]), (0, 0, 4, [9999, 9999]), (0, 1, 4, [1, 0, 1]), (0, 0, 2, [120]),
             (1, -1, 0, [5]), (0, 24, 0, [1]), (0, -25, 100, [1]), (0, -3, 6, [7]), (0, 2, 1, [9]), (1, 0, 16383, [1, 2, 3])]
    for sign, weight, scale, digits in edges:
        got = numeric(numeric_bytes(0, sign, weight, scale, digits), len(digits))
        assert got == numeric_display(num(sign, weight, scale, digits)), (sign, weight, scale, digits)


def test_numeric_formatter_fuzz_against_oracle_parses(fmt, oracle_mod):
    """numerics parsed by the oracle (parse_cell(1700, ...)): the heap entry the decode writes, printed by the device
    formatter and by the restatement"""
    numeric, _ = fmt
    rng = random.Random(1700)

    def digits(n):
        return "".join(rng.choice("0123456789") for _ in range(n))
    n_ok = 0
    for it in range(N_FUZZ):
        k = it % 5
        if k == 0:
            text = rng.choice(["", "-", "+"]) + digits(rng.randint(1, 40)) + rng.choice(["", ".", "." + digits(rng.randint(1, 30))])
        elif k == 1:
            text = rng.choice(["", "-"]) + "0." + "0" * rng.randint(0, 12) + digits(rng.randint(1, 12)) + "0" * rng.randint(0, 8)
        elif k == 2:
            text = rng.choice(["", "-"]) + digits(rng.randint(1, 6)) + "e" + str(rng.randint(-120, 120))
        elif k == 3:
            text = rng.choice(["NaN", "Infinity", "-Infinity", "inf", "-inf", "0", "-0.00", "1e100", "1e-100"])
        else:
            text = rng.choice(["", "-"]) + "0" * rng.randint(0, 6) + digits(rng.randint(0, 9)) + "." + digits(rng.randint(0, 9)) + "0" * rng.randint(0, 9)
        e, tag, val, aux, heap = oracle_mod.parse_cell(1700, text.encode())
        if e:
            continue
        n_ok += 1
        entry = bytes(heap[val:val + 8 + 2 * aux])
        assert numeric(entry, aux) == numeric_display(numeric_from_heap(heap, val, aux)), text
    assert n_ok > N_FUZZ // 2


def _gen_json(rng, max_depth):
    """a random JSON document with its whitespace, escapes, duplicate keys and number spellings"""
    ws = lambda: rng.choice(["", "", "", " ", "\n", "\t", " \r\n "])  # noqa: E731
    strings = ["", "abc", "\\/", "é", "\\u00e9", "😀", "\\ud83d\\ude00", "\\u0000", "\\u001f", "\\b\\f\\n\\r\\t", '\\"', "\\\\",
               "a\\u0041b", "\\u007f", "✓✓", "\\u2028", "sp ace"]
    keys = ["k2", "k10", "k1", "k", "", "a", "b", "é", "\\u00e9", "z\\u0000", "😀", "\\ud83d\\ude00", "K", "kk", "k\\/", "ab", "a\\u0062"]
    numbers = ["0", "-0", "1", "-1", "1.50", "1E+5", "1e-7", "-0.0", "12345678901234567890123", "3.25e10", "2E3", "10"]

    def value(d):
        k = rng.randint(0, 9 if d < max_depth else 4)
        if k == 0:
            return rng.choice(numbers)
        if k == 1:
            return rng.choice(["true", "false", "null"])
        if k in (2, 3, 4):
            return '"' + "".join(rng.choice(strings) for _ in range(rng.randint(0, 3))) + '"'
        if k in (5, 6):
            return "[" + ws() + ("," + ws()).join(value(d + 1) + ws() for _ in range(rng.randint(0, 4))) + "]"
        members = []
        for _ in range(rng.randint(0, 6)):
            key = rng.choice(keys) if rng.random() < 0.8 else "k%d" % rng.randint(0, 30)
            members.append(ws() + '"' + key + '"' + ws() + ":" + ws() + value(d + 1) + ws())
        return "{" + ",".join(members) + ws() + "}"
    return ws() + value(0) + ws()


def _deep(rng, depth):
    """one chain of `depth` nested containers with duplicates and siblings along it"""
    s = '"leaf"'
    for d in range(depth - 1):
        if rng.random() < 0.5:
            s = "[" + rng.choice(["", "1,", '"x",']) + s + "]"
        else:
            s = '{"k%d":%s,"a":%d,"k%d":%s}' % (d % 3, rng.choice(["1", "[]", "{}"]), d, d % 3, s)
    return s


def test_json_canon_known_answers(fmt):
    _, canon = fmt
    cases = [b'{"key": "value"}', b'  [1e309, -0.0, 12345678901234567890123, "\\u00e9\\ud83e\\udd14\\n"] ', b'"x"', b"true",
             b'{"k":{"k":{"k":[[],{}]}},"":""}', b'{"esc":"a\\\\b\\"c\\/d"}', b'{"b":1,"a":[1,2,{"z":null}],"b":2}', b"{}", b"[]",
             b'{"\\u0061":1,"a":2}', b'{"a":2,"\\u0061":1}', b'"\\u0000\\u001F\\u0008\\u000a"', b"-0", b"1E+5", b"[ ]", b"{ }"]
    for d in cases:
        assert canon(d) == json_display(d), d
    assert canon(_deep(random.Random(1), 127).encode()) == json_display(_deep(random.Random(1), 127).encode())
    assert canon(b"[" * 128 + b"]" * 128) is None                  # beyond json_valid's depth
    for bad in [b"", b"{", b'{"a"}', b"[1,]", b'"\\x"', b'"\\ud800"', b'"a\x01"', b"tru", b"[1 2]", b"{} {}", b'"\\udc00"']:
        assert canon(bad) is None, bad


def test_json_canon_fuzz(fmt):
    _, canon = fmt
    rng = random.Random(3802)
    n_long = 0
    for it in range(N_FUZZ):
        if it % 1000 == 0:
            doc = _deep(rng, rng.randint(100, 127))
        else:
            doc = _gen_json(rng, rng.choice([2, 3, 4, 6]))
        raw = doc.encode()
        json.loads(doc)                                      # the generator makes valid documents only
        got = canon(raw)
        assert got == json_display(raw), doc
        assert len(got) <= len(raw)
        n_long += len(raw) > 200
    assert n_long > N_FUZZ // 50


def test_json_canon_large_document(fmt):
    """a TOAST-sized document (>= 256 KiB) with one wide object and long strings"""
    _, canon = fmt
    rng = random.Random(7)
    members = ['"k%d":%s' % (rng.randint(0, 30000), _gen_json(rng, 3)) for _ in range(12000)]
    doc = ("{" + ", ".join(members) + ', "long":"' + "x\\n" * 20000 + '"}').encode()
    assert len(doc) >= 256 * 1024
    assert canon(doc) == json_display(doc)
