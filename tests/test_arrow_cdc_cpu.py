"""The CDC columns of the columnar emitter (ETL_ARROW_CDC_COLUMNS): the device formatters of sequence_number and
cdc_operation (etl_b200/csrc/arrow_format.cuh), compiled for the host (tests/emul/host_cdc.cpp — test
infrastructure, not a product path), against Python restatements of the reference's formatting, which are first pinned
to the reference's own known answers."""
import ctypes as C
import os
import random
import subprocess
import sys
import tempfile

import pytest

from etl_b200 import abi

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.normpath(os.path.join(HERE, ".."))
sys.path.insert(0, HERE)
from arrow_copy_ref import CDC_COLUMNS, CDC_OP, sequence_key  # noqa: E402

N_FUZZ = int(os.environ.get("ETL_HOST_FUZZ_N", "100000"))
U64 = (1 << 64) - 1


# ------------------------------------------------------------------------------------------------ restatements
def generate_sequence_number(start_lsn: int, commit_lsn: int) -> bytes:
    """etl-postgres/src/types/utils.rs:35-40: the commit LSN first"""
    return ("%016x/%016x" % (commit_lsn, start_lsn)).encode()


COPY_ROW_KEY = generate_sequence_number(0, 0)       # write_table_rows, iceberg/core.rs:252


def test_restatement_known_answers():
    # generate_sequence_number_fn, etl-postgres/src/types/utils.rs:119-139
    assert generate_sequence_number(0, 0) == b"0000000000000000/0000000000000000"
    assert generate_sequence_number(1, 0) == b"0000000000000000/0000000000000001"
    assert generate_sequence_number(255, 0) == b"0000000000000000/00000000000000ff"
    assert generate_sequence_number(65535, 0) == b"0000000000000000/000000000000ffff"
    assert generate_sequence_number(U64, 0) == b"0000000000000000/ffffffffffffffff"
    # the COPY rows of etl-destinations/tests/iceberg/destination.rs:134-171: INSERT and the (0, 0) key
    assert COPY_ROW_KEY == b"0000000000000000/0000000000000000"
    assert CDC_OP[ord("I")] == b"INSERT"
    # the operation values of destination.rs:369-404
    assert (CDC_OP[ord("U")], CDC_OP[ord("D")]) == (b"UPDATE", b"DELETE")
    # EventSequenceKey puts the commit LSN first, like generate_sequence_number
    assert sequence_key(0x16B3748, 3) == generate_sequence_number(3, 0x16B3748) == b"00000000016b3748/0000000000000003"
    assert all(len(sequence_key(a, b)) == 33 for a, b in ((0, 0), (U64, U64), (1 << 63, 1)))
    assert {len(v) for v in CDC_OP.values()} == {6}


def test_abi_mirror():
    assert abi.ARROW_CDC_COLUMNS == CDC_COLUMNS == 0x200
    assert abi.ARROW_CDC_COLUMNS & abi.ARROW_ALL_COLUMNS == 0
    header = open(os.path.join(ROOT, "include", "etl_decode.h")).read()
    assert "#define ETL_ARROW_CDC_COLUMNS 0x200u" in header


# ------------------------------------------------------------------------------------------------ device formatters
@pytest.fixture(scope="module")
def fmt():
    src = os.path.join(HERE, "emul", "host_cdc.cpp")
    out_dir = tempfile.mkdtemp(prefix="etl_host_cdc_")
    so = os.path.join(out_dir, "libhost_cdc.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                           "-I", os.path.join(ROOT, "etl_b200", "csrc"), "-o", so, src])
    L = C.CDLL(so)
    L.emu_seq_key.restype = None
    L.emu_seq_key.argtypes = [C.c_uint64, C.c_uint64, C.c_char_p]
    L.emu_cdc_op.restype = None
    L.emu_cdc_op.argtypes = [C.c_uint32, C.c_char_p]
    out = C.create_string_buffer(64)

    def key(lsn, ord_):
        C.memset(out, 0x55, 64)
        L.emu_seq_key(lsn, ord_, out)
        assert out.raw[33:64] == b"\x55" * 31, "wrote past 33 bytes"
        return out.raw[:33]

    def op(kind):
        C.memset(out, 0x55, 64)
        L.emu_cdc_op(kind, out)
        assert out.raw[6:64] == b"\x55" * 58, "wrote past 6 bytes"
        return out.raw[:6]
    return key, op


def test_operation_names(fmt):
    _, op = fmt
    for kind, want in CDC_OP.items():
        assert op(kind) == want
    assert op(0) == b"INSERT"          # rec_kind NULL (COPY rows) reaches the formatter as an insert


def test_sequence_key_edges(fmt):
    key, _ = fmt
    edges = [0, 1, 9, 10, 15, 16, 255, 256, 0xA, 0xF0, U64, U64 - 1, 1 << 63, (1 << 63) - 1, 0x0123456789ABCDEF, 0xFEDCBA9876543210]
    edges += [d << (4 * k) for k in range(16) for d in (1, 9, 0xA, 0xF)]          # one nibble set, at every position
    edges += [U64 ^ (0xF << (4 * k)) for k in range(16)]                          # one nibble cleared
    for a in edges:
        for b in (0, a, U64, 1):
            assert key(a, b) == sequence_key(a, b), (hex(a), hex(b))
            assert key(b, a) == sequence_key(b, a), (hex(b), hex(a))
    assert key(0, 0) == COPY_ROW_KEY


def test_sequence_key_fuzz(fmt):
    key, _ = fmt
    rng = random.Random(0x5E0)
    for it in range(N_FUZZ):
        k = it % 4
        if k == 0:
            a, b = rng.getrandbits(64), rng.getrandbits(64)
        elif k == 1:                                   # LSN-like: a few GiB of WAL, small ordinals
            a, b = rng.getrandbits(rng.randint(1, 40)), rng.getrandbits(rng.randint(0, 20))
        elif k == 2:                                   # single-nibble values
            a, b = rng.randint(0, 15) << (4 * rng.randint(0, 15)), rng.randint(0, 15) << (4 * rng.randint(0, 15))
        else:
            a, b = rng.choice([0, U64, 1 << 63]), rng.getrandbits(64)
        assert key(a, b) == sequence_key(a, b), (hex(a), hex(b))
