"""etl_dec_parquet_write_files (csrc/parquet_write.cu): every file of one call is byte for byte the file
etl_dec_parquet_write_bloom writes for its row range, with the same metrics per leaf; the byte offsets are packed and the
host image equals the device bytes.  Inputs: partitioned emits of c1 (day, and day + bucket[16]), c2, c3, c5 (two
schema versions), the 200 000-row COPY batch, the every-type hand-built table and the edge table; the codec matrix
(uncompressed, Snappy, ZSTD, each with and without dictionary and page index) and bloom filters on some columns;
arbitrary offsets over an unpartitioned emit (one file, empty files among others, a two-row-group file between small
ones, no file); every row its own file (the edge table's key: 20 000 files, a sample checked against single calls,
every file read by pyarrow); the required-null rule; the partition result's emit written after its source is freed;
the argument checks and write/free cycles."""
import ctypes as C

import numpy as np
import pytest

import iceberg_partition_ref as P
from parquet_io import device_bytes, emit_columns, fields_for, file_bytes, metrics, pq_write_bloom, write_files
from etl_b200 import abi, pgoutput as pg, workloads as wl
from test_gpu_copy import synth_rows
from test_gpu_iceberg_partition import EDGE_OIDS, _copy_emit, _edge_rows, _u64, partition
from test_gpu_parquet import ERR_INVALID_ARG, _decode_stream, _emit
from test_gpu_rowbinary import hand_built
import scenarios as sc

pytestmark = pytest.mark.gpu

SNAPPY_ALL = abi.PQ_SNAPPY | abi.PQ_DICTIONARY | abi.PQ_PAGE_INDEX
CODECS = [cc | d | i for cc in (abi.PQ_UNCOMPRESSED, abi.PQ_SNAPPY, abi.PQ_ZSTD) for d in (0, abi.PQ_DICTIONARY)
          for i in (0, abi.PQ_PAGE_INDEX)]


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from etl_b200 import decoder
    return decoder


def files_offsets(lib, h):
    k = lib.etl_dec_parquet_files_count(h)
    return _u64(lib.etl_dec_parquet_files_offsets(h), k + 1).tolist()


def files_image(lib, h, host=1):
    offs = files_offsets(lib, h)
    n = offs[-1]
    if not n:
        return b""
    if host:
        return bytes((C.c_uint8 * n).from_address(lib.etl_dec_parquet_files_bytes(h, 1)))
    return device_bytes(lib.etl_dec_parquet_files_bytes(h, 0), n)


def files_metrics(lib, h, k, n_leaves):
    out = []
    for l in range(n_leaves):
        m = abi.ParquetMetrics()
        assert lib.etl_dec_parquet_files_metrics(h, k, l, C.byref(m)) == 0
        has = bool(m.flags & abi.PQ_HAS_MIN_MAX)
        out.append(dict(field_id=m.field_id, num_values=m.num_values, null_count=m.null_count, nan_count=m.nan_count,
                        compressed_bytes=m.compressed_bytes, uncompressed_bytes=m.uncompressed_bytes,
                        min=bytes((C.c_uint8 * m.min_len).from_address(m.min)) if has else None,
                        max=bytes((C.c_uint8 * m.max_len).from_address(m.max)) if has else None))
    return out


def check_files(lib, a, fields, ro, codec, what, bloom=None, sample=None, device=False):
    """one call over ro against single calls over each range (every file, or `sample` of them); returns the files"""
    rc, h = write_files(lib, a, fields, bloom, ro, codec)
    assert rc == 0, what
    K = len(ro) - 1
    assert lib.etl_dec_parquet_files_count(h) == K, what
    offs = files_offsets(lib, h)
    assert offs[0] == 0 and all(offs[k] < offs[k + 1] for k in range(K)), what     # packed, every file non-empty
    img = files_image(lib, h)
    if device:
        assert files_image(lib, h, 0) == img, what
    files = [img[offs[k]:offs[k + 1]] for k in range(K)]
    ks = range(K) if sample is None else sorted(set(k for k in sample if 0 <= k < K))
    for k in ks:
        rc, fh = pq_write_bloom(lib, a, fields, bloom, int(ro[k]), int(ro[k + 1]), codec)
        assert rc == 0, what
        assert files[k] == file_bytes(lib, fh), f"{what}: file {k} of {K}, rows [{ro[k]}, {ro[k + 1]}), codec {codec:#x}"
        assert files_metrics(lib, h, k, len(fields)) == metrics(lib, fh, len(fields)), f"{what}: metrics of file {k}"
        lib.etl_dec_parquet_free(fh)
    m = abi.ParquetMetrics()
    assert lib.etl_dec_parquet_files_metrics(h, K, 0, C.byref(m)) == ERR_INVALID_ARG
    assert lib.etl_dec_parquet_files_metrics(h, 0, len(fields), C.byref(m)) == ERR_INVALID_ARG
    lib.etl_dec_parquet_files_free(h)
    return files


def partitioned(lib, a, spec, rb, re):
    """the partition result of a's rows [rb, re) by spec: (handle, its emit, its row offsets)"""
    rc, h = partition(lib, a, spec, rb, re)
    assert rc == 0
    return h, lib.etl_dec_iceberg_partitioned_arrow(h), _u64(lib.etl_dec_iceberg_partition_rows(h, 1),
                                                             lib.etl_dec_iceberg_partitions(h) + 1).tolist()


def check_partitioned(lib, a, fields, spec, what, codecs=(abi.PQ_SNAPPY, SNAPPY_ALL), bloom=None, sample=None):
    n = lib.etl_dec_arrow_rows(a)
    h, pa, ro = partitioned(lib, a, spec, 0, n)
    for codec in codecs:
        check_files(lib, pa, fields, ro, codec, f"{what} codec {codec:#x}", bloom=bloom, sample=sample)
    lib.etl_dec_iceberg_partition_free(h)
    return len(ro) - 1


def run_stream(gpu, tables, raw, what, specs):
    lib = abi.load()
    dec, st = _decode_stream(gpu, tables, raw)
    n_total = 0
    with dec.decode_input(st.view(), to_host=True) as bh:
        for si in range(len(bh.schemas())):
            a = _emit(lib, bh, si)
            cols = emit_columns(lib, a)
            fields = fields_for(cols)
            for j, spec in enumerate(specs(si, cols)):
                n_total += check_partitioned(lib, a, fields, spec, f"{what} v{si} spec {j}")
            lib.etl_dec_arrow_free(a)
    st.close()
    dec.close()
    return n_total


def test_c1(gpu):
    w = wl.make("c1", 0.01, n_segments=1)
    stream, _ = w.generate()
    assert run_stream(gpu, w.table_schemas(), stream.tobytes(), "c1",
                      lambda si, cols: [[(4, P.DAY, 0)], [(4, P.DAY, 0), (0, P.BUCKET, 16)]]) > 1


@pytest.mark.parametrize("name,scale,spec", [("c2", 0.0005, [(0, P.BUCKET, 16)]), ("c3", 0.001, [(4, P.HOUR, 0)])])
def test_workloads(gpu, name, scale, spec):
    w = wl.make(name, scale, n_segments=1)
    stream, _ = w.generate()
    assert run_stream(gpu, w.table_schemas(), stream.tobytes(), name, lambda si, cols: [spec]) > 1


def test_c5_versions(gpu):
    """every schema version of the c5 stream, each version's emit partitioned and written on its own"""
    w = wl.make("c5", 0.02, n_segments=1)
    stream, _ = w.generate()
    assert run_stream(gpu, w.table_schemas(), stream.tobytes(), "c5", lambda si, cols: [[(0, P.BUCKET, 16)]]) > 1


def test_hand_built_every_type(gpu, oracle_mod):
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
    tx.commit()

    def specs(si, cols):
        return [[(c, P.BUCKET, 7)] for c, col in enumerate(cols) if P.accepts(col["type"], P.BUCKET)][:1] + \
               [[(len(cols) - 2, P.IDENTITY, 0)]]
    assert run_stream(gpu, {95: cols_s}, w.bytes(), "hand-built", specs) > 1


def _copy200k(gpu, dec):
    oids, rows = synth_rows(200000, 41)
    return _copy_emit(gpu, dec, oids, rows)


def test_copy_batch_200k_codec_matrix_and_bloom(gpu):
    lib = abi.load()
    dec = gpu.Decoder(0)
    with _copy200k(gpu, dec) as bh:
        a = _emit(lib, bh, 0)
        cols = emit_columns(lib, a)
        fields = fields_for(cols, required=(0,))
        n = check_partitioned(lib, a, fields, [(6, P.BUCKET, 4), (2, P.IDENTITY, 0)], "copy 200k", codecs=CODECS)
        assert n > 1
        bloom = [(0.0, 0, 0) if c["type"] == P.R.BOOLEAN or i % 2 else (0.01, 0, 0) for i, c in enumerate(cols)]
        check_partitioned(lib, a, fields, [(0, P.BUCKET, 16)], "copy 200k bloom", codecs=(abi.PQ_SNAPPY, SNAPPY_ALL, abi.PQ_ZSTD),
                          bloom=bloom)
        bloom_ndv = [(0.05, 100, 4096) if c["type"] != P.R.BOOLEAN else (0.0, 0, 0) for c in cols]
        check_partitioned(lib, a, fields, [(0, P.BUCKET, 16)], "copy 200k bloom ndv", codecs=(SNAPPY_ALL,), bloom=bloom_ndv)
        lib.etl_dec_arrow_free(a)
    dec.close()


def test_edges_partitioned(gpu):
    lib = abi.load()
    dec = gpu.Decoder(0)
    with _copy_emit(gpu, dec, EDGE_OIDS, _edge_rows(20000)) as bh:
        a = _emit(lib, bh, 0)
        cols = emit_columns(lib, a)
        fields = fields_for(cols, required=(0,))
        check_partitioned(lib, a, fields, [(3, P.YEAR, 0), (3, P.MONTH, 0)], "edges month", codecs=(abi.PQ_SNAPPY, SNAPPY_ALL, abi.PQ_ZSTD))
        check_partitioned(lib, a, fields, [(2, P.TRUNCATE, 1), (6, P.TRUNCATE, 2)], "edges text", codecs=(SNAPPY_ALL,),
                          bloom=[(0.01, 0, 0) if c["type"] != P.R.BOOLEAN else (0.0, 0, 0) for c in cols])
        lib.etl_dec_arrow_free(a)
    dec.close()


def test_every_row_its_own_file(gpu):
    """the edge table's all-distinct key: 20 000 one-row files in one call"""
    import pyarrow as pa
    import pyarrow.parquet as pq
    lib = abi.load()
    dec = gpu.Decoder(0)
    n = 20000
    with _copy_emit(gpu, dec, EDGE_OIDS, _edge_rows(n)) as bh:
        a = _emit(lib, bh, 0)
        cols = emit_columns(lib, a)
        fields = fields_for(cols, required=(0,))
        h, pa_emit, ro = partitioned(lib, a, [(0, P.IDENTITY, 0)], 0, n)
        assert len(ro) == n + 1
        rng = np.random.default_rng(5)
        sample = [0, 1, n - 1] + rng.integers(0, n, 40).tolist()
        # the device memory the result keeps: its output buffer is sized by bounds that grow with the pages' bytes (a
        # compressed slot per page is the bound of its own fragments), not by a 64 KiB fragment per page
        free0, free1, total = C.c_uint64(), C.c_uint64(), C.c_uint64()
        assert lib.etl_dec_mem_info(dec._ctx, C.byref(free0), C.byref(total)) == 0
        rc, fh = write_files(lib, pa_emit, fields, None, ro, SNAPPY_ALL, to_host=0)
        assert rc == 0
        assert lib.etl_dec_mem_info(dec._ctx, C.byref(free1), C.byref(total)) == 0
        kept, image = free0.value - free1.value, files_offsets(lib, fh)[-1]
        lib.etl_dec_parquet_files_free(fh)
        print(f"every row its own file: {n} files, {image} B of files, {kept} B of device memory kept by the result")
        assert kept <= 8 * image + (64 << 20), (kept, image)
        for codec in (abi.PQ_SNAPPY, SNAPPY_ALL):
            files = check_files(lib, pa_emit, fields, ro, codec, f"every row codec {codec:#x}", sample=sample, device=True)
            total = 0
            for f in files:
                t = pq.read_table(pa.BufferReader(f))
                assert t.num_rows == 1
                total += t.num_rows
            assert total == n
        lib.etl_dec_iceberg_partition_free(h)
        lib.etl_dec_arrow_free(a)
    dec.close()


def test_arbitrary_offsets(gpu):
    """an unpartitioned emit cut into files: one file, empty files among others, a file of two row groups between small
    files, a slice starting above 0, and no file at all"""
    lib = abi.load()
    dec = gpu.Decoder(0)
    n_big = (1 << 20) + 1000
    with _copy_emit(gpu, dec, [23, 25, 20], [b"%d\t%s\t%d\n" % (r, b"t%d" % (r % 97) if r % 5 else b"\\N", r * 7)
                                                for r in range(n_big + 2000)]) as bh:
        a = _emit(lib, bh, 0)
        cols = emit_columns(lib, a)
        fields = fields_for(cols, required=(0,))
        n = lib.etl_dec_arrow_rows(a)
        assert n == n_big + 2000
        for codec in (abi.PQ_SNAPPY, SNAPPY_ALL, abi.PQ_ZSTD | abi.PQ_DICTIONARY):
            check_files(lib, a, fields, [0, n], codec, "one file", device=True)
            check_files(lib, a, fields, [10, 10, 500, 500, 500, 501, 4000, 4000], codec, "empty files among others")
            check_files(lib, a, fields, [3, 700, 700 + n_big, n - 5, n - 5], codec, "two row groups between small files")
        check_files(lib, a, fields, [1 << 20, (1 << 20) + 1, n], abi.PQ_SNAPPY, "a slice above 0", bloom=[(0.01, 0, 0)] * len(fields))
        rc, h = write_files(lib, a, fields, None, [17], abi.PQ_SNAPPY)
        assert rc == 0 and lib.etl_dec_parquet_files_count(h) == 0 and files_offsets(lib, h) == [0]
        m = abi.ParquetMetrics()
        assert lib.etl_dec_parquet_files_metrics(h, 0, 0, C.byref(m)) == ERR_INVALID_ARG
        lib.etl_dec_parquet_files_free(h)
        lib.etl_dec_arrow_free(a)
    dec.close()


def test_zero_row_partition_result(gpu):
    lib = abi.load()
    dec = gpu.Decoder(0)
    with _copy_emit(gpu, dec, EDGE_OIDS, _edge_rows(100)) as bh:
        a = _emit(lib, bh, 0)
        fields = fields_for(emit_columns(lib, a), required=(0,))
        h, pa_emit, ro = partitioned(lib, a, [(0, P.BUCKET, 4)], 7, 7)
        assert ro == [0]
        rc, fh = write_files(lib, pa_emit, fields, None, ro, SNAPPY_ALL)
        assert rc == 0 and lib.etl_dec_parquet_files_count(fh) == 0
        lib.etl_dec_parquet_files_free(fh)
        lib.etl_dec_iceberg_partition_free(h)
        lib.etl_dec_arrow_free(a)
    dec.close()


def test_required_null(gpu):
    """a null inside some file's range writes nothing and reports the whole-range call's column and row; one before
    row_offsets[0] does not count"""
    lib = abi.load()
    dec = gpu.Decoder(0)
    rows = [b"%d\t%s\n" % (r, b"\\N" if r in (50, 3000) else b"x%d" % r) for r in range(4000)]
    with _copy_emit(gpu, dec, [23, 25], rows) as bh:
        a = _emit(lib, bh, 0)
        fields = fields_for(emit_columns(lib, a), required=(0, 1))
        col, row = C.c_uint32(), C.c_uint64()
        for ro in ([0, 10, 2000, 3500], [100, 2999, 3001, 4000], [60, 60, 3000, 3001]):
            rc, h = write_files(lib, a, fields, None, ro, abi.PQ_SNAPPY)
            assert rc == 0
            assert files_offsets(lib, h) == [0] * len(ro) and not lib.etl_dec_parquet_files_bytes(h, 0)
            assert lib.etl_dec_parquet_files_required_null(h, C.byref(col), C.byref(row)) == 0
            rc, fh = pq_write_bloom(lib, a, fields, None, ro[0], ro[-1], abi.PQ_SNAPPY)
            wc, wr = C.c_uint32(), C.c_uint64()
            assert rc == 0 and lib.etl_dec_parquet_required_null(fh, C.byref(wc), C.byref(wr)) == 0
            assert (col.value, row.value) == (wc.value, wr.value) == (1, 50 if ro[0] <= 50 else 3000), ro
            lib.etl_dec_parquet_free(fh)
            lib.etl_dec_parquet_files_free(h)
        files = check_files(lib, a, fields, [51, 1000, 2999], abi.PQ_SNAPPY, "null before the range")
        assert len(files) == 2
        rc, h = write_files(lib, a, fields, None, [51, 1000, 2999], abi.PQ_SNAPPY)
        assert lib.etl_dec_parquet_files_required_null(h, C.byref(col), C.byref(row)) == 0
        assert (col.value, row.value) == (2**32 - 1, 2**64 - 1)
        lib.etl_dec_parquet_files_free(h)
        lib.etl_dec_arrow_free(a)
    dec.close()


def test_source_freed_before_write(gpu):
    lib = abi.load()
    dec = gpu.Decoder(0)
    with _copy_emit(gpu, dec, EDGE_OIDS, _edge_rows(5000)) as bh:
        a = _emit(lib, bh, 0)
        cols = emit_columns(lib, a)
        fields = fields_for(cols, required=(0,))
        h, pa_emit, ro = partitioned(lib, a, [(3, P.MONTH, 0), (2, P.TRUNCATE, 1)], 0, 5000)
        lib.etl_dec_arrow_free(a)
        check_files(lib, pa_emit, fields, ro, SNAPPY_ALL, "freed source", device=True)
        lib.etl_dec_iceberg_partition_free(h)
    dec.close()


def test_arguments_and_cycles(gpu):
    lib = abi.load()
    dec = gpu.Decoder(0)
    free, total = C.c_uint64(), C.c_uint64()
    with _copy_emit(gpu, dec, EDGE_OIDS, _edge_rows(3000)) as bh:
        a = _emit(lib, bh, 0)
        cols = emit_columns(lib, a)
        fields = fields_for(cols, required=(0,))
        ok = [0, 1000, 3000]
        for ro in ([0, 2000, 1000], [0, 3001], [3001, 3001], [5, 4]):
            assert write_files(lib, a, fields, None, ro, abi.PQ_SNAPPY)[0] == ERR_INVALID_ARG, ro
        for codec in (2, abi.PQ_SNAPPY | 0x200, 0xFF):
            assert write_files(lib, a, fields, None, ok, codec)[0] == ERR_INVALID_ARG, codec
        assert write_files(lib, a, fields[:-1], None, ok, abi.PQ_SNAPPY)[0] == ERR_INVALID_ARG
        assert write_files(lib, a, [("", 1, 2, 0)] + fields[1:], None, ok, abi.PQ_SNAPPY)[0] == ERR_INVALID_ARG
        bad_bloom = [(1.0, 0, 0)] + [(0.0, 0, 0)] * (len(fields) - 1)
        assert write_files(lib, a, fields, bad_bloom, ok, abi.PQ_SNAPPY)[0] == ERR_INVALID_ARG
        arr = (abi.ParquetField * len(fields))()
        for i, f in enumerate(fields):
            arr[i].name, arr[i].field_id, arr[i].element_field_id, arr[i].required = f[0].encode(), f[1], f[2], f[3]
        offs = (C.c_uint64 * 3)(*ok)
        h = C.c_void_p()
        assert lib.etl_dec_parquet_write_files(None, arr, None, len(fields), offs, 2, 1, 1, C.byref(h)) == ERR_INVALID_ARG
        assert lib.etl_dec_parquet_write_files(a, arr, None, len(fields), None, 2, 1, 1, C.byref(h)) == ERR_INVALID_ARG
        assert lib.etl_dec_parquet_write_files(a, arr, None, len(fields), offs, 2, 1, 1, None) == ERR_INVALID_ARG
        m = abi.ParquetMetrics()
        assert lib.etl_dec_parquet_files_metrics(None, 0, 0, C.byref(m)) == ERR_INVALID_ARG
        assert lib.etl_dec_parquet_files_count(None) == 0 and not lib.etl_dec_parquet_files_offsets(None)
        lib.etl_dec_parquet_files_free(None)
        # write/free cycles keep device memory stable
        for i in range(100):
            rc, h = write_files(lib, a, fields, None, ok, SNAPPY_ALL if i % 2 else abi.PQ_ZSTD, to_host=i % 3 == 0)
            assert rc == 0 and lib.etl_dec_parquet_files_count(h) == 2
            lib.etl_dec_parquet_files_free(h)
            assert lib.etl_dec_mem_info(dec._ctx, C.byref(free), C.byref(total)) == 0
            if i == 1:
                base = free.value
        assert abs(free.value - base) <= 4 << 20, (free.value, base)
        lib.etl_dec_arrow_free(a)
    dec.close()
