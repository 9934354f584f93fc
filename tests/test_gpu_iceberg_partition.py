"""etl_dec_iceberg_partition (csrc/iceberg_partition.cu) against the Python restatement (tests/iceberg_partition_ref.py)
fed the same Arrow emit's columns: the partition row offsets and values, every column of the partitioned emit (List
children included) and its row records against the source rows in the restatement's permutation, and the data files of
the partitions: the uncompressed file byte for byte and the Snappy file page by page against parquet_ref.write of the
permuted columns (test_gpu_parquet.check_write), a Snappy + dictionary + page-index file read back by pyarrow with
sequence_number's ColumnIndex ASCENDING, and one file with bloom filters.  The source emit is freed before the
partitioned one is written.  Inputs: c1, c2, c3, c5, a 200 000-row COPY batch, the every-type hand-built table, an edge
table (pre-1970 dates and timestamps, INT32_MIN, multi-byte text, nulls in every source, all-null and void fields, a
multi-field spec), single-partition and all-distinct specs, row slices and zero rows; then the argument checks and
partition/free cycles."""
import ctypes as C

import numpy as np
import pytest

import iceberg_partition_ref as P
import parquet_index_ref as X
import parquet_ref as R
import scenarios as sc
from parquet_io import emit_columns, fields_for, file_bytes, pq_write, pq_write_bloom
from etl_b200 import abi, pgoutput as pg, workloads as wl
from test_gpu_arrow_copy import copy_batch
from test_gpu_copy import synth_rows
from test_gpu_parquet import ERR_INVALID_ARG, INT4, TEXT, _decode_stream, _emit, _norm_ref, check_pyarrow, check_write
from test_gpu_rowbinary import hand_built

pytestmark = pytest.mark.gpu

BOOL, BYTEA, DATE, TS, TSTZ, FLOAT8, INT4_ARR, TEXT_ARR = 16, 17, 1082, 1114, 1184, 701, 1007, 1009


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from etl_b200 import decoder
    return decoder


def partition(lib, a, spec, rb, re, to_host=1):
    """etl_dec_iceberg_partition; spec: [(source_column, transform, param)]"""
    arr = (abi.IcebergPartitionField * max(1, len(spec)))()
    for i, (c, tr, p) in enumerate(spec):
        arr[i].source_column, arr[i].transform, arr[i].param = c, tr, p
    h = C.c_void_p()
    rc = lib.etl_dec_iceberg_partition(a, arr, len(spec), rb, re, to_host, C.byref(h))
    return rc, h


def _u64(ptr, n):
    return np.frombuffer((C.c_uint64 * n).from_address(ptr), dtype=np.uint64).copy() if n else np.zeros(0, np.uint64)


def read_values(lib, h, n_parts, n_fields):
    out = []
    v = abi.IcebergPartitionValue()
    for k in range(n_parts):
        row = []
        for f in range(n_fields):
            assert lib.etl_dec_iceberg_partition_value(h, k, f, C.byref(v)) == 0
            if v.is_null:
                row.append(None)
            elif v.data:
                row.append(bytes((C.c_uint8 * v.len).from_address(v.data)) if v.len else b"")
            else:
                row.append(v.value)
        out.append(tuple(row))
    return out


def check_partition(lib, a, cols, spec, rb, re, what, fields=None, writes=3, free_source=None):
    """partition a's rows [rb, re) by spec and check everything against the restatement; with fields, write the first
    `writes` partitions and the last (every partition when writes is None).  free_source(): called after the call and
    before any read of the result (the source emit must not be needed any more)."""
    perm, offs, values = P.partition(cols, spec, rb, re)
    src_recs = _u64(lib.etl_dec_arrow_row_records(a, 1), lib.etl_dec_arrow_rows(a))
    first_skipped = lib.etl_dec_arrow_first_skipped(a)
    rc, h = partition(lib, a, spec, rb, re)
    assert rc == 0, what
    if free_source:
        free_source()
    n_parts = lib.etl_dec_iceberg_partitions(h)
    assert n_parts == len(values), (what, n_parts, len(values))
    rows = _u64(lib.etl_dec_iceberg_partition_rows(h, 1), n_parts + 1)
    assert rows.tolist() == offs, what
    assert lib.etl_dec_iceberg_partition_rows(h, 0)
    assert read_values(lib, h, n_parts, len(spec)) == values, what
    pa = lib.etl_dec_iceberg_partitioned_arrow(h)
    n = re - rb
    assert lib.etl_dec_arrow_rows(pa) == n and lib.etl_dec_arrow_cols(pa) == len(cols), what
    assert lib.etl_dec_arrow_first_skipped(pa) == first_skipped, what
    got = emit_columns(lib, pa)
    want = [P.take(c, perm) for c in cols]
    for c, (g, w) in enumerate(zip(got, want)):
        assert g["type"] == w["type"], (what, c)
        assert _norm_ref(g) == _norm_ref(w), f"{what}: column {c}"
    assert _u64(lib.etl_dec_arrow_row_records(pa, 1), n).tolist() == src_recs[perm].tolist(), what
    if fields is not None and n:
        ks = range(n_parts) if writes is None else sorted(set(list(range(min(writes, n_parts))) + [n_parts - 1]))
        for k in ks:
            check_write(lib, pa, want, fields, offs[k], offs[k + 1], f"{what} partition {k}")
            codec = abi.PQ_SNAPPY | abi.PQ_DICTIONARY | abi.PQ_PAGE_INDEX
            rc, fh = pq_write(lib, pa, fields, offs[k], offs[k + 1], codec)
            assert rc == 0, what
            data = file_bytes(lib, fh)
            lib.etl_dec_parquet_free(fh)
            check_pyarrow(data, want, fields, offs[k], offs[k + 1])
            seq = X.read_indexes(data)[len(fields) - 1][0]                  # sequence_number, first row group
            assert seq is not None and seq[4] == X.ASCENDING, (what, k)
    lib.etl_dec_iceberg_partition_free(h)
    return n_parts


def run_stream(gpu, tables, raw, what, specs, write=True):
    """specs(schema_index, cols) → [spec]: each checked over the whole emit, and the first over a slice and zero rows"""
    lib = abi.load()
    dec, st = _decode_stream(gpu, tables, raw)
    n_total = 0
    with dec.decode_input(st.view(), to_host=True) as bh:
        for si in range(len(bh.schemas())):
            a = _emit(lib, bh, si)
            cols = emit_columns(lib, a)
            n = lib.etl_dec_arrow_rows(a)
            fields = fields_for(cols) if write else None
            for j, spec in enumerate(specs(si, cols)):
                check_partition(lib, a, cols, spec, 0, n, f"{what} v{si} spec {j}", fields if j < 3 else None)
                if j == 0 and n > 2:
                    check_partition(lib, a, cols, spec, n // 3, n - n // 4, f"{what} v{si} slice", fields, writes=1)
                    check_partition(lib, a, cols, spec, n // 2, n // 2, f"{what} v{si} empty", fields)
            n_total += n
            lib.etl_dec_arrow_free(a)
    st.close()
    dec.close()
    return n_total


def test_c1(gpu):
    w = wl.make("c1", 0.01, n_segments=1)
    stream, _ = w.generate()
    specs = lambda si, cols: [[(4, P.DAY, 0), (0, P.BUCKET, 16)], [(4, P.DAY, 0)], [(0, P.BUCKET, 16)]]
    assert run_stream(gpu, w.table_schemas(), stream.tobytes(), "c1", specs) > 0


def test_c2(gpu):
    """bucket[16](id); truncate on text and on int4 columns holding negatives"""
    w = wl.make("c2", 0.0005, n_segments=1)
    stream, _ = w.generate()
    specs = lambda si, cols: [[(0, P.BUCKET, 16)], [(5, P.TRUNCATE, 1), (1, P.TRUNCATE, 1 << 30)], [(6, P.TRUNCATE, 2)]]
    assert run_stream(gpu, w.table_schemas(), stream.tobytes(), "c2", specs) > 0


def test_c3_timestamptz(gpu):
    w = wl.make("c3", 0.001, n_segments=1)
    stream, _ = w.generate()
    specs = lambda si, cols: [[(4, P.HOUR, 0)], [(10, P.MONTH, 0), (16, P.YEAR, 0)]]
    assert run_stream(gpu, w.table_schemas(), stream.tobytes(), "c3", specs) > 0


def test_c5_toast(gpu):
    w = wl.make("c5", 0.0005, n_segments=1)
    stream, _ = w.generate()
    assert run_stream(gpu, w.table_schemas(), stream.tobytes(), "c5", lambda si, cols: [[(0, P.BUCKET, 16)]]) > 0


def test_hand_built_every_type(gpu, oracle_mod):
    """identity and bucket on every column whose type accepts them, one field at a time and all at once"""
    cols_s, row, n_rows = hand_built(oracle_mod)
    rel = pg.relation(95, "public", "ice", "f", sc.rel_cols(cols_s, set()))
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
    seen = set()

    def specs(si, cols):
        out, every = [], []
        for c, col in enumerate(cols):
            for tr, p in ((P.IDENTITY, 0), (P.BUCKET, 7)):
                if P.accepts(col["type"], tr):
                    out.append([(c, tr, p)])
                    seen.add((col["type"], tr))
                    if len(every) < 16:
                        every.append((c, tr, p))
        return [every] + out
    assert run_stream(gpu, {95: cols_s}, w.bytes(), "hand-built", specs) > 0
    for at in (R.INT32, R.INT64, R.DATE32, R.TIME64_US, R.TIMESTAMP_US, R.TIMESTAMPTZ_US, R.UTF8, R.LARGE_BINARY, R.UUID):
        assert (at, P.IDENTITY) in seen and (at, P.BUCKET) in seen, at
    assert (R.BOOLEAN, P.IDENTITY) in seen


def _copy_emit(gpu, dec, oids, rows):
    dec.put_table_schema(7, [dict(name=f"c{i}", type_oid=o, pk=1 if i == 0 else None, nullable=True) for i, o in enumerate(oids)])
    return copy_batch(gpu, dec, 7, rows)


def test_copy_batch_200k(gpu):
    lib = abi.load()
    dec = gpu.Decoder(0)
    oids, rows = synth_rows(200000, 41)
    with _copy_emit(gpu, dec, oids, rows) as bh:
        a = _emit(lib, bh, 0)
        cols = emit_columns(lib, a)
        n = lib.etl_dec_arrow_rows(a)
        fields = fields_for(cols, required=(0,))
        check_partition(lib, a, cols, [(6, P.BUCKET, 4), (2, P.IDENTITY, 0)], 0, n, "copy 200k", fields, writes=2)
        check_partition(lib, a, cols, [(5, P.DAY, 0), (0, P.BUCKET, 3)], 0, n, "copy 200k day", None)
        check_partition(lib, a, cols, [(9, P.TRUNCATE, 1 << 20)], 5, 150000, "copy 200k slice", fields, writes=1)
        lib.etl_dec_arrow_free(a)
    dec.close()


def _edge_rows(n):
    rows = []
    for r in range(n):
        k = r % 9
        i4 = "\\N" if r % 13 == 0 else str((-2**31, 2**31 - 1, -1, 0, -10, -11, 7, 9, 123456)[k] if r % 2 else (r % 40) - 20)
        text = "\\N" if r % 11 == 0 else ("", "a", "é", "€uro", "😀😀x", "naïve%d" % (r % 3), "x" * 70, "ab", "abc")[k]
        date = "\\N" if r % 7 == 0 else ("0001-01-01", "1969-12-31", "1970-01-01", "1900-02-28", "2000-02-29", "1969-01-01",
                                         "9999-12-31", "1582-10-15", "2024-%02d-01" % (1 + r % 12))[k]
        ts = "\\N" if r % 17 == 0 else ("1969-12-31 23:59:59.999999", "1970-01-01 00:00:00", "1960-06-15 12:30:00",
                                        "2024-03-10 0%d:00:00" % (r % 10), "0100-01-01 00:00:00")[r % 5]
        tstz = "\\N" if r % 19 == 0 else ts + "+00" if ts != "\\N" else "\\N"
        byt = "\\N" if r % 23 == 0 else "\\\\x" + "%02x" % (r % 5) * (r % 4)
        ints = "\\N" if r % 29 == 0 else "{%s}" % ",".join(str(r - j) for j in range(r % 4))
        texts = "{%s}" % ",".join('"s%d"' % (r + j) if (r + j) % 3 else "NULL" for j in range(r % 3))
        rows.append(("%d\t%s\t%s\t%s\t%s\t%s\t%s\t\\N\t%s\t%s\t%s\t%s\n" % (
            r, i4, text, date, ts, tstz, byt, "1.5" if r % 2 else "-0", "t" if r % 3 else "f", ints, texts)).encode())
    return rows


EDGE_OIDS = [INT4, INT4, TEXT, DATE, TS, TSTZ, BYTEA, INT4, FLOAT8, BOOL, INT4_ARR, TEXT_ARR]


def test_edges(gpu):
    """pre-1970 dates and timestamps, INT32_MIN / INT32_MAX, multi-byte text, nulls in every source, an all-null column,
    void fields, multi-field specs, one partition, every row its own partition, slices and zero rows"""
    lib = abi.load()
    dec = gpu.Decoder(0)
    n = 20000
    with _copy_emit(gpu, dec, EDGE_OIDS, _edge_rows(n)) as bh:
        a = _emit(lib, bh, 0)
        cols = emit_columns(lib, a)
        fields = fields_for(cols, required=(0,))
        specs = [
            [(3, P.YEAR, 0), (3, P.MONTH, 0), (3, P.DAY, 0)],
            [(4, P.YEAR, 0), (4, P.MONTH, 0), (4, P.DAY, 0), (4, P.HOUR, 0)],
            [(5, P.HOUR, 0), (5, P.DAY, 0), (1, P.TRUNCATE, 10)],
            [(1, P.TRUNCATE, 10), (1, P.IDENTITY, 0), (1, P.BUCKET, 5)],
            [(2, P.TRUNCATE, 1), (2, P.TRUNCATE, 3), (2, P.BUCKET, 4), (6, P.TRUNCATE, 2), (6, P.IDENTITY, 0)],
            [(7, P.IDENTITY, 0), (7, P.BUCKET, 2), (8, P.VOID, 0), (0, P.VOID, 0)],   # all-null column and void fields
            [(9, P.IDENTITY, 0), (len(cols) - 2, P.IDENTITY, 0)],                        # Boolean and cdc_operation
            [(1, P.TRUNCATE, 2**31 - 1), (3, P.BUCKET, 2**31 - 1), (4, P.BUCKET, 1)],
            [(len(cols) - 1, P.VOID, 0)] * 16,                                           # one partition
        ]
        for j, spec in enumerate(specs):
            check_partition(lib, a, cols, spec, 0, n, f"edges spec {j}", fields if j in (0, 5, 8) else None)
        for rb, re in ((19990, 20000), (1, 2), (7, 7), (0, 0)):
            check_partition(lib, a, cols, specs[4], rb, re, f"edges [{rb}, {re})", fields)
        # every row its own partition: identity on the key
        check_partition(lib, a, cols, [(0, P.IDENTITY, 0)], 0, n, "edges all distinct", fields, writes=2)
        check_partition(lib, a, cols, [(len(cols) - 1, P.IDENTITY, 0)], 100, 5000, "edges sequence_number", None)
        # bloom filters on one partition's file
        rc, h = partition(lib, a, specs[3], 0, n)
        assert rc == 0
        pa = lib.etl_dec_iceberg_partitioned_arrow(h)
        rows = _u64(lib.etl_dec_iceberg_partition_rows(h, 1), lib.etl_dec_iceberg_partitions(h) + 1)
        bloom = [(0.0, 0, 0) if c["type"] in (R.BOOLEAN,) else (0.01, 0, 0) for c in cols]
        for codec in (abi.PQ_SNAPPY, abi.PQ_SNAPPY | abi.PQ_DICTIONARY | abi.PQ_PAGE_INDEX):
            rc, fh = pq_write_bloom(lib, pa, fields, bloom, int(rows[1]), int(rows[2]), codec)
            assert rc == 0
            data = file_bytes(lib, fh)
            lib.etl_dec_parquet_free(fh)
            check_pyarrow(data, [P.take(c, P.partition(cols, specs[3], 0, n)[0]) for c in cols], fields, int(rows[1]), int(rows[2]))
        lib.etl_dec_iceberg_partition_free(h)
        lib.etl_dec_arrow_free(a)
    dec.close()


def test_source_freed_before_write(gpu):
    lib = abi.load()
    dec = gpu.Decoder(0)
    with _copy_emit(gpu, dec, EDGE_OIDS, _edge_rows(5000)) as bh:
        a = _emit(lib, bh, 0)
        cols = emit_columns(lib, a)
        fields = fields_for(cols, required=(0,))
        check_partition(lib, a, cols, [(3, P.MONTH, 0), (2, P.TRUNCATE, 1)], 0, 5000, "freed source", fields, writes=None,
                        free_source=lambda: lib.etl_dec_arrow_free(a))
    dec.close()


def test_arguments(gpu):
    lib = abi.load()
    dec = gpu.Decoder(0)
    with _copy_emit(gpu, dec, EDGE_OIDS, _edge_rows(1000)) as bh:
        a = _emit(lib, bh, 0)
        nc = lib.etl_dec_arrow_cols(a)
        ok = [(0, P.BUCKET, 16)]
        bad_specs = [[], [(0, P.BUCKET, 16)] * 17, [(nc, P.IDENTITY, 0)], [(10, P.IDENTITY, 0)], [(11, P.VOID, 0)],
                     [(8, P.IDENTITY, 0)], [(8, P.BUCKET, 4)], [(8, P.TRUNCATE, 4)], [(9, P.BUCKET, 2)], [(2, P.YEAR, 0)],
                     [(0, P.HOUR, 0)], [(3, P.HOUR, 0)], [(6, P.DAY, 0)], [(0, 8, 0)], [(0, P.BUCKET, 0)],
                     [(0, P.BUCKET, 2**31)], [(0, P.TRUNCATE, 0)], [(0, P.TRUNCATE, 2**32 - 1)], [(0, P.IDENTITY, 1)],
                     [(0, P.VOID, 3)], [(3, P.DAY, 1)], ok + [(2, P.TRUNCATE, 0)]]
        for spec in bad_specs:
            assert partition(lib, a, spec, 0, 1000)[0] == ERR_INVALID_ARG, spec
        for rb, re in ((5, 4), (0, 1001), (1001, 1001)):
            assert partition(lib, a, ok, rb, re)[0] == ERR_INVALID_ARG, (rb, re)
        h = C.c_void_p()
        arr = (abi.IcebergPartitionField * 1)()
        assert lib.etl_dec_iceberg_partition(None, arr, 1, 0, 10, 1, C.byref(h)) == ERR_INVALID_ARG
        assert lib.etl_dec_iceberg_partition(a, None, 1, 0, 10, 1, C.byref(h)) == ERR_INVALID_ARG
        assert lib.etl_dec_iceberg_partition(a, arr, 1, 0, 10, 1, None) == ERR_INVALID_ARG
        rc, h = partition(lib, a, [(1, P.IDENTITY, 0)] * 16, 0, 1000, to_host=0)       # 16 fields, no host image
        assert rc == 0
        pa = lib.etl_dec_iceberg_partitioned_arrow(h)
        assert not lib.etl_dec_arrow_row_records(pa, 1) and lib.etl_dec_arrow_row_records(pa, 0)
        v = abi.IcebergPartitionValue()
        n_parts = lib.etl_dec_iceberg_partitions(h)
        assert lib.etl_dec_iceberg_partition_value(h, n_parts, 0, C.byref(v)) == ERR_INVALID_ARG
        assert lib.etl_dec_iceberg_partition_value(h, 0, 16, C.byref(v)) == ERR_INVALID_ARG
        lib.etl_dec_iceberg_partition_free(h)
        lib.etl_dec_iceberg_partition_free(None)
        lib.etl_dec_arrow_free(a)
        # an emit without ETL_ARROW_ALL_COLUMNS: its List columns are unsupported and rejected
        plain = C.c_void_p()
        assert lib.etl_dec_arrow_emit(bh._h, 0, 1, 1, C.byref(plain)) == 0
        assert partition(lib, plain, [(10, P.VOID, 0)], 0, 1000)[0] == ERR_INVALID_ARG
        lib.etl_dec_arrow_free(plain)
    dec.close()


def test_partition_free_cycles_keep_memory_stable(gpu):
    lib = abi.load()
    dec = gpu.Decoder(0)
    free, total = C.c_uint64(), C.c_uint64()
    with _copy_emit(gpu, dec, EDGE_OIDS, _edge_rows(3000)) as bh:
        a = _emit(lib, bh, 0)
        for i in range(100):
            rc, h = partition(lib, a, [(2, P.TRUNCATE, 1), (3, P.YEAR, 0)], 0, 3000, to_host=i % 3 == 0)
            assert rc == 0 and lib.etl_dec_iceberg_partitions(h) > 1
            lib.etl_dec_iceberg_partition_free(h)
            assert lib.etl_dec_mem_info(dec._ctx, C.byref(free), C.byref(total)) == 0
            if i == 1:
                base = free.value
        assert abs(free.value - base) <= 4 << 20, (free.value, base)
        lib.etl_dec_arrow_free(a)
    dec.close()
