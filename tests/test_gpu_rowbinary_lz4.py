"""ClickHouse INSERT bodies (csrc/clickhouse_lz4.cu, etl_dec_rowbinary_lz4) on RowBinary emits (test_gpu_rowbinary.py's
harness) against the restatement (tests/clickhouse_lz4_ref.py): for every INSERT the rows of the greedy split; every
block's method, sizes and checksum; blocks of at most KBLOCK bytes; each payload decoded by pyarrow's lz4_raw (liblz4) and
by the restatement's strict decoder to the emit's bytes of those rows; to_host 0 and 1 and a repeated call giving the
same bytes; and the argument checks.  Inputs: c1-c5 (every schema version), the COPY reference vectors and 200 000
COPY rows, the every-type stream, a random-bytea table and a constant-text table of long runs; max_bytes_per_insert 1,
about one row, 1 MiB, 64 MiB and more than the emit; the whole emit, a range that starts and ends mid-emit, an empty
range and a 1-row range.
The checksum of every block is computed by the device helpers compiled for the host (tests/emul/host_ch_lz4.cpp, which
the CPU suite pins to the restatement); the restatement's own CityHash128 and strict decoder run on every block of an
emit up to 2000 blocks and on every 16th block (and each INSERT's first and last) beyond, to bound the Python time."""
import ctypes as C
import os
import random
import struct
import subprocess
import tempfile

import numpy as np
import pytest

import clickhouse_lz4_ref as Z
import scenarios as sc
from etl_b200 import abi, pgoutput as pg, workloads as wl
from test_gpu_arrow_copy import copy_batch
from test_gpu_arrow_formatted import arr, decode
from test_gpu_copy import BYTEA, INT4, REF_ROWS, TEXT, cols_of, synth_rows
from test_gpu_rowbinary import flag_sets, hand_built, rb_emit

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.normpath(os.path.join(HERE, ".."))
ERR_INVALID_ARG = 1
MIB = 1 << 20


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from etl_b200 import decoder
    return decoder


@pytest.fixture(scope="module")
def tools():
    import pyarrow as pa
    codec = pa.Codec("lz4_raw")
    src = os.path.join(HERE, "emul", "host_ch_lz4.cpp")
    so = os.path.join(tempfile.mkdtemp(prefix="etl_host_ch_lz4_"), "libhost_ch_lz4.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I", os.path.join(ROOT, "include"),
                           "-I", os.path.join(ROOT, "etl_b200", "csrc"), "-o", so, src])
    emu = C.CDLL(so)
    emu.emu_city128.argtypes = [C.c_char_p, C.c_uint64, C.POINTER(C.c_uint64)]
    emu.emu_block_size.restype = C.c_uint32
    assert emu.emu_block_size() == Z.KBLOCK
    abi.load()
    rt = C.CDLL("libcudart.so.12")
    rt.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
    return codec, emu, rt


def emit_view(lib, h):
    n = lib.etl_dec_rowbinary_rows(h)
    nbytes = lib.etl_dec_rowbinary_bytes(h)
    offs = [int(x) for x in arr(lib.etl_dec_rowbinary_row_offsets(h, 1), C.c_uint64, np.uint64, n + 1)]
    data = bytes((C.c_uint8 * nbytes).from_address(lib.etl_dec_rowbinary_data(h, 1))) if nbytes else b""
    return n, offs, data


def lz4_call(lib, h, b, e, mx, to_host=1):
    z = C.c_void_p()
    rc = lib.etl_dec_rowbinary_lz4(h, b, e, mx, to_host, C.byref(z))
    return rc, z


def fetch_host(lib, z):
    n = lib.etl_dec_rowbinary_lz4_inserts(z)
    rows = [int(x) for x in arr(lib.etl_dec_rowbinary_lz4_insert_rows(z, 1), C.c_uint64, np.uint64, n + 1)]
    offs = [int(x) for x in arr(lib.etl_dec_rowbinary_lz4_insert_offsets(z, 1), C.c_uint64, np.uint64, n + 1)]
    nbytes = lib.etl_dec_rowbinary_lz4_bytes(z)
    data = bytes((C.c_uint8 * nbytes).from_address(lib.etl_dec_rowbinary_lz4_data(z, 1))) if nbytes else b""
    return rows, offs, data


def fetch_device(lib, rt, z):
    n = lib.etl_dec_rowbinary_lz4_inserts(z)
    out = []
    for ptr, nb in ((lib.etl_dec_rowbinary_lz4_insert_rows(z, 0), 8 * (n + 1)), (lib.etl_dec_rowbinary_lz4_insert_offsets(z, 0), 8 * (n + 1)),
                    (lib.etl_dec_rowbinary_lz4_data(z, 0), lib.etl_dec_rowbinary_lz4_bytes(z))):
        buf = C.create_string_buffer(max(1, nb))
        if nb:
            assert rt.cudaMemcpy(buf, ptr, nb, 2) == 0            # cudaMemcpyDeviceToHost
        out.append(buf.raw[:nb])
    rows = [int(x) for x in np.frombuffer(out[0], dtype=np.uint64)]
    offs = [int(x) for x in np.frombuffer(out[1], dtype=np.uint64)]
    return rows, offs, out[2]


def check_bodies(tools, rows, offs, body, e_offs, e_data, want_rows, what):
    codec, emu, _ = tools
    assert rows == want_rows, (what, rows[:8], want_rows[:8])
    assert offs[0] == 0 and offs[-1] == len(body) and all(a <= b for a, b in zip(offs, offs[1:])), what
    blocks = []
    for k in range(len(rows) - 1):
        parsed = Z.parse_blocks(body[offs[k]:offs[k + 1]])
        assert parsed, (what, k)
        blocks.append(parsed)
    n_blocks = sum(len(p) for p in blocks)
    full = n_blocks <= 2000
    h = (C.c_uint64 * 2)()
    i = 0
    for k, parsed in enumerate(blocks):
        got = []
        for j, (csum, method, csize, raw, payload, hp) in enumerate(parsed):
            assert method == Z.METHOD_LZ4 and csize == 9 + len(payload), (what, k, j)
            assert 0 < raw <= Z.KBLOCK and (raw == Z.KBLOCK or j == len(parsed) - 1), (what, k, j, raw)
            emu.emu_city128(hp, len(hp), h)
            assert csum == struct.pack("<QQ", h[0], h[1]), (what, k, j, "checksum")
            dec = codec.decompress(payload, decompressed_size=raw, asbytes=True)
            if full or i % 16 == 0 or j in (0, len(parsed) - 1):
                assert csum == Z.checksum(hp), (what, k, j, "restated checksum")
                assert Z.lz4_decode(payload, raw) == dec, (what, k, j)
            got.append(dec)
            i += 1
        want = e_data[e_offs[rows[k]]:e_offs[rows[k + 1]]]
        assert b"".join(got) == want, (what, k)
    return n_blocks


def sweep(lib, tools, h, what, ranges=True):
    """every max_bytes_per_insert over the whole emit, then the row ranges at about one row and 1 MiB"""
    n, e_offs, e_data = emit_view(lib, h)
    row = max(1, len(e_data) // max(1, n))
    maxes = [1, row, MIB, 64 * MIB, len(e_data) + 1]
    cases = [(0, n, mx) for mx in maxes]
    if ranges and n:
        for mx in (row, MIB):
            cases += [(n // 3, max(n // 3, 2 * n // 3), mx), (n // 2, n // 2, mx), (n // 2, n // 2 + 1, mx)]
    stats = dict(rows=n, bytes=len(e_data), blocks=0, z=0)
    for b, e, mx in cases:
        rc, z = lz4_call(lib, h, b, e, mx)
        assert rc == 0, (what, b, e, mx, rc)
        try:
            rows, offs, body = fetch_host(lib, z)
            stats["blocks"] += check_bodies(tools, rows, offs, body, e_offs, e_data, Z.split(e_offs, b, e, mx), f"{what} [{b},{e}) max {mx}")
            if mx == 64 * MIB and (b, e) == (0, n):
                stats["z"] = len(body)
        finally:
            lib.etl_dec_rowbinary_lz4_free(z)
    return stats


def repeat_and_device(lib, tools, h, mx):
    """a second call gives the same bytes; to_host 0 gives them in device memory, which outlive the emit"""
    n = lib.etl_dec_rowbinary_rows(h)
    rc, z1 = lz4_call(lib, h, 0, n, mx)
    rc2, z2 = lz4_call(lib, h, 0, n, mx)
    rc3, z3 = lz4_call(lib, h, 0, n, mx, to_host=0)
    assert rc == rc2 == rc3 == 0
    try:
        first = fetch_host(lib, z1)
        assert fetch_host(lib, z2) == first
        assert lib.etl_dec_rowbinary_lz4_data(z3, 1) is None and lib.etl_dec_rowbinary_lz4_insert_rows(z3, 1) is None
        return first, z3
    finally:
        lib.etl_dec_rowbinary_lz4_free(z1)
        lib.etl_dec_rowbinary_lz4_free(z2)


# ------------------------------------------------------------------------------------------------ workloads
@pytest.mark.parametrize("name,scale", [("c1", 0.01), ("c2", 0.0005), ("c3", 0.001), ("c4", 0.002), ("c5", 0.0005)])
def test_workloads(gpu, oracle_mod, tools, name, scale):
    w = wl.make(name, scale, n_segments=1)
    stream, _ = w.generate()
    raw = stream.tobytes()
    tables = w.table_schemas()
    planes, dec, st = decode(gpu, oracle_mod, tables, raw)
    lib = abi.load()
    total = 0
    with dec.decode_input(st.view(), to_host=True) as bh:
        for si in range(len(planes.schemas)):                     # c4: every schema version
            rc, h = rb_emit(lib, bh, si, flag_sets(planes, si)["create_table"])
            assert rc == 0
            try:
                total += sweep(lib, tools, h, f"{name} schema {si}", ranges=si < 3)["rows"]
            finally:
                lib.etl_dec_rowbinary_free(h)
    assert total > 0
    st.close()
    dec.close()


def test_hand_built_every_type(gpu, oracle_mod, tools):
    cols, row, n_rows = hand_built(oracle_mod)
    rel = pg.relation(95, "public", "rb", "f", sc.rel_cols(cols, set()))
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(rel)
    for r in range(n_rows):
        w.emit(pg.insert(95, row(r)))
        if r % 3 == 1:
            w.emit(pg.update(95, row(r + 1), old=row(r)))
        if r % 5 == 2:
            w.emit(pg.delete(95, old=row(r)))
    tx.commit()
    raw = w.bytes()
    planes, dec, st = decode(gpu, oracle_mod, {95: cols}, raw)
    lib = abi.load()
    with dec.decode_input(st.view(), to_host=True) as bh:
        rc, h = rb_emit(lib, bh, 0, [True] * (len(cols) + 2))
        assert rc == 0
        try:
            assert sweep(lib, tools, h, "every type")["rows"] > 0
        finally:
            lib.etl_dec_rowbinary_free(h)
    st.close()
    dec.close()


# ------------------------------------------------------------------------------------------------ COPY batches
@pytest.mark.parametrize("idx", range(len(REF_ROWS)))
def test_copy_reference_vectors(gpu, tools, idx):
    oids, row = REF_ROWS[idx]
    lib = abi.load()
    dec = gpu.Decoder(0)
    dec.put_table_schema(7, cols_of(oids))
    with copy_batch(gpu, dec, 7, [row]) as bh:
        rc, h = rb_emit(lib, bh, 0, [True] * (len(oids) + 2))
        assert rc == 0
        try:
            sweep(lib, tools, h, f"vector {idx}")
        finally:
            lib.etl_dec_rowbinary_free(h)
    dec.close()


def copy_table(gpu, tools, oids, rows, what, flags=None):
    lib = abi.load()
    dec = gpu.Decoder(0)
    dec.put_table_schema(7, cols_of(oids))
    with copy_batch(gpu, dec, 7, rows) as bh:
        rc, h = rb_emit(lib, bh, 0, flags or [True] * len(oids) + [False, False])
        assert rc == 0
        try:
            stats = sweep(lib, tools, h, what)
            (rows_, offs, body), z3 = repeat_and_device(lib, tools, h, MIB)
        finally:
            lib.etl_dec_rowbinary_free(h)
        try:                                                       # the emit is gone: the output is the call's own
            assert fetch_device(lib, tools[2], z3) == (rows_, offs, body)
        finally:
            lib.etl_dec_rowbinary_lz4_free(z3)
    dec.close()
    return stats


def test_copy_200k_rows(gpu, tools):
    oids, rows = synth_rows(200000, 4321)
    s = copy_table(gpu, tools, oids, rows, "copy 200k")
    assert s["rows"] == 200000 and s["z"] < s["bytes"]


def test_random_bytea_does_not_compress(gpu, tools):
    rng = random.Random(7)
    rows = [b"%d\t\\\\x%s\n" % (i, bytes(rng.randrange(256) for _ in range(rng.randrange(50, 400))).hex().encode()) for i in range(3000)]
    s = copy_table(gpu, tools, [INT4, BYTEA], rows, "random bytea")
    assert s["z"] > 0.5 * s["bytes"]                     # hex text of random bytes: little for LZ4 to find


def test_constant_text_long_runs(gpu, tools):
    rows = [b"%d\t%s\n" % (i, b"a" * (1000 + 37 * (i % 300))) for i in range(3000)]
    s = copy_table(gpu, tools, [INT4, TEXT], rows, "constant text")
    assert s["z"] * 50 < s["bytes"], s


# ------------------------------------------------------------------------------------------------ arguments
def test_argument_checks(gpu, tools):
    oids, rows = synth_rows(100, 99)
    lib = abi.load()
    dec = gpu.Decoder(0)
    dec.put_table_schema(7, cols_of(oids))
    with copy_batch(gpu, dec, 7, rows) as bh:
        rc, h = rb_emit(lib, bh, 0, [True] * (len(oids) + 2))
        assert rc == 0
        z = C.c_void_p()
        for b, e, mx in ((0, 100, 0), (5, 4, MIB), (0, 101, MIB), (101, 101, MIB)):
            assert lib.etl_dec_rowbinary_lz4(h, b, e, mx, 1, C.byref(z)) == ERR_INVALID_ARG, (b, e, mx)
        assert lib.etl_dec_rowbinary_lz4(None, 0, 0, MIB, 1, C.byref(z)) == ERR_INVALID_ARG
        assert lib.etl_dec_rowbinary_lz4(h, 0, 100, MIB, 1, None) == ERR_INVALID_ARG
        rc, z = lz4_call(lib, h, 100, 100, 1)                  # an empty range at the end: zero INSERTs
        assert rc == 0 and lib.etl_dec_rowbinary_lz4_inserts(z) == 0 and fetch_host(lib, z) == ([100], [0], b"")
        lib.etl_dec_rowbinary_lz4_free(z)
        lib.etl_dec_rowbinary_free(h)
    dec.close()
