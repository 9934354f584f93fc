#!/usr/bin/env python
"""Time the Iceberg Parquet writer (etl_dec_parquet_write) on resident Arrow emits, against pyarrow's CPU writer.

  python tools/parquet_measure.py [--copy-rows 1000000] [--c3-scale 1] [--c4-scale 0.1] [--reps 7] [--warmup 2]
                                  [--plain-only] [--no-pyarrow] [--tag NAME]
  python tools/parquet_measure.py --page-index [--copy-rows 1000000] [--c5-scale 0.02] [--c4-scale 0.1] [--reps 7]
  python tools/parquet_measure.py --bloom [--copy-rows 1000000] [--c5-scale 0.02] [--c4-scale 0.1] [--reps 7]
  python tools/parquet_measure.py --zstd [--copy-rows 1000000] [--c2-scale 0.05] [--c3-scale 1] [--c5-scale 0.02] [--reps 7]
  python tools/parquet_measure.py --partition [--copy-rows 1000000] [--c1-scale 10] [--c2-scale 0.05] [--c5-scale 0.02]

Workloads: bench.py's 10-column COPY table, C3 (one schema version) and C4 (every schema version: times and sizes are
sums over the versions), each emitted once with 7 | ETL_ARROW_ALL_COLUMNS | ETL_ARROW_CDC_COLUMNS and kept in HBM.
Every time is median / min / max over the repetitions of wall time around the call (the call syncs before it returns),
to_host 0:
  * write_ms_uncompressed / write_ms_snappy: the whole call, file in HBM;
  * snappy_GBps: page payload bytes before compression / the median Snappy call;
  * file_bytes_* and the pyarrow baseline: pyarrow.parquet.write_table(compression="snappy") with its defaults
    (dictionary encoding on) over the same columns on the host, into memory;
  * the dictionary leg (codec | ETL_PQ_DICTIONARY): write_ms_dict_* and file_bytes_dict_*, uncompressed and Snappy.
A low-cardinality COPY table (status text of a dozen values, small int codes, dates, uuids from a pool of nine and a
text[] of three tags) runs beside the COPY table.  --plain-only skips the dictionary leg, so that a library without
ETL_PQ_DICTIONARY can be timed by the same script (ETL_LIB_SUFFIX selects it); --tag labels the lines.
--page-index instead writes each emit of the COPY table, C5 and C4 with and without ETL_PQ_PAGE_INDEX, alternating the
two in every repetition, with Snappy and with Snappy | ETL_PQ_DICTIONARY: the CUDA-event time of the call (median over
the repetitions, summed over the emits) and the index bytes as a share of the file.
--bloom does the same with and without bloom filters (etl_dec_parquet_write_bloom) on every eligible column (fpp 0.01,
ndv 0: the chunk's non-null count, max_bytes 0: 1 MiB): the call's CUDA-event time and the filter bytes' share.
--zstd writes each emit of the COPY table, C2, C3 and C5 uncompressed, with Snappy and with ETL_PQ_ZSTD, each with and
without ETL_PQ_DICTIONARY, the six calls alternated in every repetition: the call's CUDA-event time (median, summed over
the emits), the file bytes, and from one torch.profiler pass per codec the device time of the compression kernel
(k_snappy / k_zstd) against the call's other kernels.
--partition partitions each emit with etl_dec_iceberg_partition (C1 day(created), C2 bucket[16](id), the COPY table
bucket[16](c0) + truncate[1](c5), C5 bucket[16](id)) and writes every partition's Snappy file from the partitioned emit;
the unpartitioned Snappy write of the same rows is alternated with it in every repetition.  Reported: the partition
call's CUDA-event time, its device time from one torch.profiler pass split into transform + group (k_ice_transform …
k_ice_reps and the radix sort), the length scans and the gather (k_ice_gather_*), the gather's bytes moved (the
partitioned emit read from the source and written once: 2 × its column bytes) per second as a kernel share of the
3.35 TB/s data sheet figure, P, and the whole partitioned write (partition + P file writes) against the unpartitioned
write.  Before timing, the partition offsets, values and every column of the partitioned emit are compared with
tests/iceberg_partition_ref.py; every timed file must have the bytes of the first repetition's.  The one-call leg writes
the same files with one etl_dec_parquet_write_files call over the partition offsets, alternated with the per-partition
loop and the unpartitioned write in every repetition (its file sizes must be the loop's); one torch.profiler pass
splits it into kernel time, copies, launches and the call's wall time. A --c1-scale, --c2-scale or --c5-scale of 0 leaves that
workload out of the --partition run.
Prints the card name and power limit in the same run.
"""
import argparse
import ctypes as C
import io
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import pyarrow as pa  # noqa: E402
import pyarrow.parquet as pq  # noqa: E402
import torch  # noqa: E402

import parquet_ref as R  # noqa: E402
from arrow_emit_measure import bench_copy_table, card, timed  # noqa: E402
from etl_b200 import abi, decoder, workloads as wl  # noqa: E402
from rowbinary_measure import sum_stats  # noqa: E402
from parquet_io import emit_columns, fields_for, pq_write  # noqa: E402

KINDS = 7 | abi.ARROW_ALL_COLUMNS | abi.ARROW_CDC_COLUMNS
PA_TYPE = {R.BOOLEAN: pa.bool_(), R.INT32: pa.int32(), R.INT64: pa.int64(), R.FLOAT32: pa.float32(), R.FLOAT64: pa.float64(),
           R.DATE32: pa.date32(), R.TIME64_US: pa.time64("us"), R.TIMESTAMP_US: pa.timestamp("us"),
           R.TIMESTAMPTZ_US: pa.timestamp("us", tz="UTC")}


def to_arrow(col):
    """a parquet_ref column as a pyarrow array (host copy of the emit)"""
    t, valid = col["type"], col["valid"]
    mask = pa.py_buffer(np.packbits(valid, bitorder="little").tobytes())
    n = len(valid)
    if t == R.LIST:
        kid = to_arrow(col["child"])
        return pa.Array.from_buffers(pa.list_(kid.type), n, [mask, pa.py_buffer(col["offsets"].astype(np.int32).tobytes())],
                                     children=[kid])
    if t in (R.UTF8, R.LARGE_BINARY):
        ty, ow = (pa.string(), np.int32) if t == R.UTF8 else (pa.large_binary(), np.int64)
        return pa.Array.from_buffers(ty, n, [mask, pa.py_buffer(col["offsets"].astype(ow).tobytes()), pa.py_buffer(col["data"])])
    if t == R.UUID:
        return pa.Array.from_buffers(pa.binary(16), n, [mask, pa.py_buffer(col["values"].tobytes())])
    if t == R.BOOLEAN:
        return pa.Array.from_buffers(pa.bool_(), n, [mask, pa.py_buffer(np.packbits(col["values"], bitorder="little").tobytes())])
    return pa.Array.from_buffers(PA_TYPE[t], n, [mask, pa.py_buffer(np.ascontiguousarray(col["values"]).tobytes())])


OPTS = dict(plain_only=False, pyarrow=True, page_index=False, bloom=False, zstd=False, partition=False, spec=None)


def write_bloom(lib, a, fields, bloom, n, codec):
    """etl_dec_parquet_write_bloom of rows [0, n), file in HBM; bloom None: a NULL array"""
    arr = (abi.ParquetField * len(fields))()
    names = [f[0].encode() for f in fields]
    for i, (f, nm) in enumerate(zip(fields, names)):
        arr[i].name, arr[i].field_id, arr[i].element_field_id, arr[i].required = nm, f[1], f[2], f[3]
    barr = None
    if bloom is not None:
        barr = (abi.ParquetBloom * len(bloom))()
        for i, (fpp, ndv, mb) in enumerate(bloom):
            barr[i].fpp, barr[i].ndv, barr[i].max_bytes = fpp, ndv, mb
    h = C.c_void_p()
    rc = lib.etl_dec_parquet_write_bloom(a, arr, barr, len(fields), 0, n, codec, 0, C.byref(h))
    return rc, h


def bloom_emits(lib, emits, reps, warmup):
    """bloom filters: per codec, the call's CUDA-event time without / with them, alternated, and their bytes"""
    out = {}
    for codec, name in ((abi.PQ_SNAPPY, "snappy"), (abi.PQ_SNAPPY | abi.PQ_DICTIONARY, "snappy_dict")):
        ms, size = {0: [], 1: []}, {0: 0, 1: 0}
        for a in emits:
            cols = emit_columns(lib, a)
            fields = fields_for(cols)
            leaf_type = [c["child"]["type"] if c["type"] == R.LIST else c["type"] for c in cols]
            bloom = [(0.0 if t == R.BOOLEAN else 0.01, 0, 0) for t in leaf_type]
            n = lib.etl_dec_arrow_rows(a)
            t = {0: [], 1: []}
            for r in range(warmup + reps):
                for on in (0, 1):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    rc, h = write_bloom(lib, a, fields, bloom if on else None, n, codec)
                    e1.record()
                    e1.synchronize()
                    assert rc == 0
                    if r == 0:
                        size[on] += lib.etl_dec_parquet_size(h)
                    lib.etl_dec_parquet_free(h)
                    if r >= warmup:
                        t[on].append(e0.elapsed_time(e1))
            for on in t:
                ms[on].append(float(np.median(t[on])))
        base, with_b = sum(ms[0]), sum(ms[1])
        out[name] = dict(write_ms=round(base, 3), write_ms_bloom=round(with_b, 3),
                         cost_pct=round(100 * (with_b - base) / base, 1) if base else None,
                         file_bytes=int(size[0]), file_bytes_bloom=int(size[1]),
                         bloom_share_pct=round(100 * (size[1] - size[0]) / size[1], 3) if size[1] else None)
    return out


ZSTD_LEGS = [(c | d, n + ("_dict" if d else "")) for d in (0, abi.PQ_DICTIONARY)
             for c, n in ((abi.PQ_UNCOMPRESSED, "uncompressed"), (abi.PQ_SNAPPY, "snappy"), (abi.PQ_ZSTD, "zstd"))]


def _kernel_ms(lib, emits, codec):
    """device time of one call per emit under torch.profiler: (compression kernel, every other kernel), ms"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for a in emits:
            cols = emit_columns(lib, a)
            rc, h = write_bloom(lib, a, fields_for(cols), None, lib.etl_dec_arrow_rows(a), codec)
            assert rc == 0
            lib.etl_dec_parquet_free(h)
        torch.cuda.synchronize()
    comp = other = 0.0
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if e.device_type is not None and str(e.device_type).endswith("CUDA") and us:
            if "k_zstd" in e.key or "k_snappy" in e.key:
                comp += us
            elif "k_" in e.key:
                other += us
    return round(comp / 1e3, 3), round(other / 1e3, 3)


def zstd_emits(lib, emits, reps, warmup):
    """ETL_PQ_ZSTD: per codec and dictionary flag, the call's CUDA-event time (six calls alternated) and file bytes"""
    ms = {n: [] for _, n in ZSTD_LEGS}
    size = {n: 0 for _, n in ZSTD_LEGS}
    for a in emits:
        fields = fields_for(emit_columns(lib, a))
        n = lib.etl_dec_arrow_rows(a)
        t = {name: [] for _, name in ZSTD_LEGS}
        for r in range(warmup + reps):
            for codec, name in ZSTD_LEGS:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                rc, h = write_bloom(lib, a, fields, None, n, codec)
                e1.record()
                e1.synchronize()
                assert rc == 0
                if r == 0:
                    size[name] += lib.etl_dec_parquet_size(h)
                lib.etl_dec_parquet_free(h)
                if r >= warmup:
                    t[name].append(e0.elapsed_time(e1))
        for name in t:
            ms[name].append(float(np.median(t[name])))
    out = {name: dict(write_ms=round(sum(ms[name]), 3), file_bytes=int(size[name])) for _, name in ZSTD_LEGS}
    for codec, name in ((abi.PQ_SNAPPY, "snappy"), (abi.PQ_ZSTD, "zstd")):
        out[name]["compress_kernel_ms"], out[name]["other_kernels_ms"] = _kernel_ms(lib, emits, codec)
    return out


def _emit_bytes(lib, a):
    """bytes of an emit's column buffers: validity, values, offsets and data, List children included"""
    n = lib.etl_dec_arrow_rows(a)

    def flat(col, items):
        b = (items + 7) // 8
        t = col.arrow_type
        if t == R.BOOLEAN:
            return 2 * b
        if t in R.WIDTH:
            return b + items * R.WIDTH[t]
        return b + (items + 1) * (8 if t == R.LARGE_BINARY else 4) + col.data_bytes
    total = 8 * n                                          # row records
    for c in range(lib.etl_dec_arrow_cols(a)):
        col = abi.ArrowColumn()
        lib.etl_dec_arrow_column(a, c, 0, C.byref(col))
        total += flat(col, n)
        if col.arrow_type == R.LIST:
            kid, ne = abi.ArrowColumn(), C.c_uint64()
            lib.etl_dec_arrow_list_child(a, c, 0, C.byref(kid), C.byref(ne))
            total += flat(kid, ne.value)
    return total


def _partition(lib, a, spec, n, to_host=0):
    arr = (abi.IcebergPartitionField * len(spec))()
    for i, (c, tr, p) in enumerate(spec):
        arr[i].source_column, arr[i].transform, arr[i].param = c, tr, p
    h = C.c_void_p()
    assert lib.etl_dec_iceberg_partition(a, arr, len(spec), 0, n, to_host, C.byref(h)) == 0
    return h


def _check_partition(lib, a, spec):
    """the partition of the whole emit against tests/iceberg_partition_ref.py; returns the partition count"""
    import iceberg_partition_ref as IP
    from test_gpu_parquet import _norm_ref
    cols = emit_columns(lib, a)
    n = lib.etl_dec_arrow_rows(a)
    perm, offs, values = IP.partition(cols, spec, 0, n)
    h = _partition(lib, a, spec, n, 1)
    P = lib.etl_dec_iceberg_partitions(h)
    rows = np.frombuffer((C.c_uint64 * (P + 1)).from_address(lib.etl_dec_iceberg_partition_rows(h, 1)), dtype=np.uint64)
    assert rows.tolist() == offs
    v = abi.IcebergPartitionValue()
    for k in range(P):
        for f in range(len(spec)):
            assert lib.etl_dec_iceberg_partition_value(h, k, f, C.byref(v)) == 0
            got = None if v.is_null else bytes((C.c_uint8 * v.len).from_address(v.data)) if v.data else v.value
            assert got == values[k][f], (k, f)
    got = emit_columns(lib, lib.etl_dec_iceberg_partitioned_arrow(h))
    for g, c in zip(got, cols):
        assert _norm_ref(g) == _norm_ref(IP.take(c, perm))
    lib.etl_dec_iceberg_partition_free(h)
    return P


def _partition_kernel_ms(lib, a, spec, n):
    """device time of one partition call under torch.profiler: (transform + group, scans, gather), ms"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        lib.etl_dec_iceberg_partition_free(_partition(lib, a, spec, n))
        torch.cuda.synchronize()
    group = scan = gather = 0.0
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if e.device_type is None or not str(e.device_type).endswith("CUDA") or not us:
            continue
        if "k_ice_gather" in e.key:
            gather += us
        elif "k_ice_" in e.key or "RadixSort" in e.key:
            group += us
        elif "k_len_blocks" in e.key or "k_blk_scan" in e.key or "k_offsets" in e.key:
            scan += us
    return group / 1e3, scan / 1e3, gather / 1e3


def partition_emits(lib, emits, reps, warmup):
    """--partition: see the module docstring; sums over the emits"""
    spec = OPTS["spec"]
    codec = abi.PQ_SNAPPY
    call, whole, plain, files, parts, moved, group, scan, gather = [], [], [], 0, 0, 0, 0.0, 0.0, 0.0
    one, one_spread, prof = [], [], dict(kernel_ms=0.0, memcpy_ms=0.0, launches=0, wall_ms=0.0)
    for a in emits:
        fields = fields_for(emit_columns(lib, a))
        n = lib.etl_dec_arrow_rows(a)
        parts += _check_partition(lib, a, spec)
        g, s, k = _partition_kernel_ms(lib, a, spec, n)
        group, scan, gather = group + g, scan + s, gather + k
        moved += 2 * _emit_bytes(lib, a)
        first, t_call, t_whole, t_plain, t_one = None, [], [], [], []
        for r in range(warmup + reps):
            e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            e[0].record()
            h = _partition(lib, a, spec, n)
            e[1].record()
            pa_ = lib.etl_dec_iceberg_partitioned_arrow(h)
            P = lib.etl_dec_iceberg_partitions(h)
            rows = np.frombuffer((C.c_uint64 * (P + 1)).from_address(lib.etl_dec_iceberg_partition_rows(h, 1)), dtype=np.uint64).copy()
            sizes = []
            for k in range(P):
                rc, fh = pq_write(lib, pa_, fields, int(rows[k]), int(rows[k + 1]), codec, 0)
                assert rc == 0
                sizes.append(lib.etl_dec_parquet_size(fh))
                lib.etl_dec_parquet_free(fh)
            e[2].record()
            e[2].synchronize()
            lib.etl_dec_iceberg_partition_free(h)
            if first is None:
                first = sizes
                files += P
            assert sizes == first
            # the one-call leg: every partition's file in one etl_dec_parquet_write_files over the same offsets
            h = _partition(lib, a, spec, n)
            pa_ = lib.etl_dec_iceberg_partitioned_arrow(h)
            rows = np.frombuffer((C.c_uint64 * (P + 1)).from_address(lib.etl_dec_iceberg_partition_rows(h, 1)), dtype=np.uint64).copy()
            o0, o1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            o0.record()
            rc, fs = write_files(lib, pa_, fields, None, rows, codec, 0)
            o1.record()
            o1.synchronize()
            assert rc == 0
            offs = np.frombuffer((C.c_uint64 * (P + 1)).from_address(lib.etl_dec_parquet_files_offsets(fs)), dtype=np.uint64)
            assert np.diff(offs).tolist() == first
            lib.etl_dec_parquet_files_free(fs)
            if r == warmup:                                  # one torch.profiler pass (not timed)
                prof_one(lib, pa_, fields, rows, codec, prof)
            lib.etl_dec_iceberg_partition_free(h)
            p0, p1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            p0.record()
            rc, fh = pq_write(lib, a, fields, 0, n, codec, 0)
            p1.record()
            p1.synchronize()
            assert rc == 0
            lib.etl_dec_parquet_free(fh)
            if r >= warmup:
                t_call.append(e[0].elapsed_time(e[1]))
                t_whole.append(e[0].elapsed_time(e[2]))
                t_plain.append(p0.elapsed_time(p1))
                t_one.append(o0.elapsed_time(o1))
        call.append(float(np.median(t_call)))
        one.append(float(np.median(t_one)))
        one_spread.append([round(min(t_one), 3), round(max(t_one), 3)])
        whole.append(float(np.median(t_whole)))
        plain.append(float(np.median(t_plain)))
    c, w, p = sum(call), sum(whole), sum(plain)
    gbps = moved / (gather * 1e-3) / 1e9 if gather else None
    return dict(spec=spec, partitions=int(parts), files=int(files), partition_call_ms=round(c, 3),
                device_ms=dict(transform_group=round(group, 3), scans=round(scan, 3), gather=round(gather, 3)),
                gather_bytes_moved=int(moved), gather_GBps=round(gbps, 1) if gbps else None,
                gather_kernel_share_of_3_35TBps_pct=round(100 * gbps / 3350, 1) if gbps else None,
                partitioned_write_ms=round(w, 3), unpartitioned_snappy_write_ms=round(p, 3),
                ratio=round(w / p, 2) if p else None, ms_per_file=round((w - c) / files, 3) if files else None,
                one_call_write_ms=round(sum(one), 3), one_call_min_max_per_emit=one_spread,
                loop_over_one_call=round((w - c) / sum(one), 1) if sum(one) else None,
                one_call_over_unpartitioned=round(sum(one) / p, 2) if p else None,
                one_call_profile={k: round(v, 3) if isinstance(v, float) else v for k, v in prof.items()})


def write_files(lib, a, fields, bloom, ro, codec, to_host):
    arr = (abi.ParquetField * max(1, len(fields)))()
    for i, f in enumerate(fields):
        arr[i].name, arr[i].field_id, arr[i].element_field_id, arr[i].required = f[0].encode(), f[1], f[2], f[3]
    offs = np.ascontiguousarray(ro, dtype=np.uint64)
    h = C.c_void_p()
    rc = lib.etl_dec_parquet_write_files(a, arr, None, len(fields), offs.ctypes.data_as(C.POINTER(C.c_uint64)), len(offs) - 1,
                                         codec, to_host, C.byref(h))
    return rc, h


def prof_one(lib, a, fields, ro, codec, acc):
    """one torch.profiler pass over one etl_dec_parquet_write_files call: the kernels' device time, the copies', the
    launches and the call's wall time (the rest is host work and the syncs' waits)"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as p:
        t0 = time.perf_counter()
        rc, fs = write_files(lib, a, fields, None, ro, codec, 0)
        acc["wall_ms"] += (time.perf_counter() - t0) * 1e3
    assert rc == 0
    lib.etl_dec_parquet_files_free(fs)
    for e in p.key_averages():
        us = getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0)
        if "Memcpy" in e.key or "Memset" in e.key:
            acc["memcpy_ms"] += us / 1e3
        elif e.key.startswith(("void", "k_")) or "k_" in e.key:
            acc["kernel_ms"] += us / 1e3
            acc["launches"] += e.count


def leg(lib, emits, reps, warmup):
    if OPTS["partition"]:
        return partition_emits(lib, emits, reps, warmup)
    if OPTS["zstd"]:
        return zstd_emits(lib, emits, reps, warmup)
    if OPTS["bloom"]:
        return bloom_emits(lib, emits, reps, warmup)
    if OPTS["page_index"]:
        return page_index_emits(lib, emits, reps, warmup)
    return measure_emits(lib, emits, reps, warmup)


def measure_emits(lib, emits, reps, warmup):
    """emits: Arrow batch handles of one workload; sums over them"""
    t0, t1, tp, sizes, payload, rows = [], [], [], [0, 0, 0], 0, 0
    td, dsizes = {abi.PQ_UNCOMPRESSED: [], abi.PQ_SNAPPY: []}, [0, 0]
    for a in emits:
        cols = emit_columns(lib, a)
        fields = fields_for(cols)
        n = lib.etl_dec_arrow_rows(a)
        rows += n
        for codec, acc in ((abi.PQ_UNCOMPRESSED, t0), (abi.PQ_SNAPPY, t1)):
            acc.append(timed(lambda: lib.etl_dec_parquet_free(pq_write(lib, a, fields, 0, n, codec, 0)[1]), reps, warmup))
            rc, h = pq_write(lib, a, fields, 0, n, codec, 0)
            assert rc == 0
            sizes[codec] += lib.etl_dec_parquet_size(h)
            if codec == abi.PQ_UNCOMPRESSED:
                for l in range(len(fields)):
                    m = abi.ParquetMetrics()
                    lib.etl_dec_parquet_metrics(h, l, C.byref(m))
                    payload += m.uncompressed_bytes
            lib.etl_dec_parquet_free(h)
            if OPTS["plain_only"]:
                continue
            dc = codec | abi.PQ_DICTIONARY
            td[codec].append(timed(lambda: lib.etl_dec_parquet_free(pq_write(lib, a, fields, 0, n, dc, 0)[1]), reps, warmup))
            rc, h = pq_write(lib, a, fields, 0, n, dc, 0)
            assert rc == 0
            dsizes[codec] += lib.etl_dec_parquet_size(h)
            lib.etl_dec_parquet_free(h)
        if not OPTS["pyarrow"]:
            continue
        table = pa.table({f[0]: to_arrow(c) for c, f in zip(cols, fields)})
        sink = io.BytesIO()
        pq.write_table(table, sink, compression="snappy")
        sizes[2] += len(sink.getvalue())

        def cpu():
            pq.write_table(table, io.BytesIO(), compression="snappy")
        tp.append(timed(cpu, max(3, reps // 2), 1))
    s1 = sum_stats(t1)
    out = dict(rows=int(rows), write_ms_uncompressed=sum_stats(t0), write_ms_snappy=s1,
               snappy_GBps=round(payload / (s1["median"] * 1e-3) / 1e9, 2) if s1["median"] else None,
               file_bytes_uncompressed=int(sizes[0]), file_bytes_snappy=int(sizes[1]))
    if OPTS["pyarrow"]:
        out.update(pyarrow_snappy_ms=sum_stats(tp), pyarrow_file_bytes=int(sizes[2]))
    if not OPTS["plain_only"]:
        out.update(write_ms_dict_uncompressed=sum_stats(td[abi.PQ_UNCOMPRESSED]), write_ms_dict_snappy=sum_stats(td[abi.PQ_SNAPPY]),
                   file_bytes_dict_uncompressed=int(dsizes[0]), file_bytes_dict_snappy=int(dsizes[1]))
    return out


def page_index_emits(lib, emits, reps, warmup):
    """ETL_PQ_PAGE_INDEX: per codec, the call's CUDA-event time without / with the flag, alternated, and the index's bytes"""
    out = {}
    for codec, name in ((abi.PQ_SNAPPY, "snappy"), (abi.PQ_SNAPPY | abi.PQ_DICTIONARY, "snappy_dict")):
        ms, size = {0: [], abi.PQ_PAGE_INDEX: []}, {0: 0, abi.PQ_PAGE_INDEX: 0}
        for a in emits:
            fields = fields_for(emit_columns(lib, a))
            n = lib.etl_dec_arrow_rows(a)
            t = {0: [], abi.PQ_PAGE_INDEX: []}
            for r in range(warmup + reps):
                for flag in (0, abi.PQ_PAGE_INDEX):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    rc, h = pq_write(lib, a, fields, 0, n, codec | flag, 0)
                    e1.record()
                    e1.synchronize()
                    assert rc == 0
                    if r == 0:
                        size[flag] += lib.etl_dec_parquet_size(h)
                    lib.etl_dec_parquet_free(h)
                    if r >= warmup:
                        t[flag].append(e0.elapsed_time(e1))
            for flag in t:
                ms[flag].append(float(np.median(t[flag])))
        base, with_idx = sum(ms[0]), sum(ms[abi.PQ_PAGE_INDEX])
        out[name] = dict(write_ms=round(base, 3), write_ms_page_index=round(with_idx, 3),
                         cost_pct=round(100 * (with_idx - base) / base, 1) if base else None,
                         file_bytes=int(size[0]), file_bytes_page_index=int(size[abi.PQ_PAGE_INDEX]),
                         index_share_pct=round(100 * (size[abi.PQ_PAGE_INDEX] - size[0]) / size[abi.PQ_PAGE_INDEX], 3)
                         if size[abi.PQ_PAGE_INDEX] else None)
    return out


def low_cardinality_rows(n_rows):
    """(oids, COPY rows) of the low-cardinality table, seeded"""
    rng = np.random.default_rng(29)
    words = ["active", "pending", "shipped", "cancelled", "returned", "on hold", "lost", "refunded", "draft", "open",
             "closed", "archived"]
    uuids = ["%08x-0000-4000-8000-%012x" % (k * 7919, k) for k in range(9)]
    w, code, day, u, nt = (rng.integers(0, 12, n_rows), rng.integers(0, 7, n_rows), rng.integers(1, 29, n_rows),
                           rng.integers(0, 9, n_rows), rng.integers(0, 4, n_rows))
    tags = ["{}", "{red}", "{red,green}", "{blue,green,red}"]
    rows = [("%d\t%s\t%d\t2024-03-%02d\t%s\t%s\n" % (r, words[w[r]], code[r], day[r], uuids[u[r]], tags[nt[r]])).encode()
            for r in range(n_rows)]
    return [23, 25, 23, 1082, 2950, 1009], rows


def copy_table(n_rows, reps, warmup, tag, low_card=False):
    oids, rows = low_cardinality_rows(n_rows) if low_card else bench_copy_table(n_rows)
    lib = abi.load()
    blob = b"".join(rows)
    offs = np.zeros(len(rows) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(r) for r in rows])
    d_buf = torch.zeros(len(blob) + 64, dtype=torch.uint8, device="cuda")
    d_buf[:len(blob)].copy_(torch.from_numpy(np.frombuffer(blob, dtype=np.uint8).copy()))
    d_off = torch.from_numpy(offs.view(np.int64).copy()).cuda()
    torch.cuda.synchronize()
    dec = decoder.Decoder(0)
    dec.put_table_schema(9, [dict(name=f"c{i}", type_oid=o, pk=1 if i == 0 else None, nullable=i != 0) for i, o in enumerate(oids)])
    inp = abi.CopyInput()
    inp.dev_buf, inp.dev_row_offsets, inp.len, inp.n_rows, inp.row_offsets = d_buf.data_ptr(), d_off.data_ptr(), len(blob), len(rows), offs.ctypes.data
    h = C.c_void_p()
    assert lib.etl_dec_copy_decode(dec._ctx, 9, C.byref(inp), 0, C.byref(h)) == 0, lib.etl_dec_last_error(dec._ctx)
    with decoder.BatchHandle(dec, h) as bh:
        a = C.c_void_p()
        assert lib.etl_dec_arrow_emit(bh._h, 0, KINDS, 1, C.byref(a)) == 0
        res = dict(tag=tag, workload="low-cardinality COPY table (int4, text, int4, date, uuid, text[])" if low_card
                   else "bench.py COPY table (5 x int4, 5 x text)", input_bytes=len(blob))
        res.update(leg(lib, [a], reps, warmup))
        lib.etl_dec_arrow_free(a)
        print(json.dumps(res), flush=True)
    dec.close()


def streaming(name, scale, reps, warmup, tag):
    w = wl.make(name, scale, n_segments=1)
    stream, stats = w.generate()
    st = decoder.Stager(stream.nbytes, 2048)
    st.append_framed(stream)
    dec = decoder.Decoder(0)
    for tid, cols in w.table_schemas().items():
        dec.put_table_schema(tid, cols)
    lib = abi.load()
    res = dict(tag=tag, workload=name, scale=scale, stream_bytes=int(stream.nbytes))
    with dec.decode_input(st.view(), to_host=False) as bh:
        emits = []
        for si in range(bh.summary().n_schemas):
            a = C.c_void_p()
            assert lib.etl_dec_arrow_emit(bh._h, si, KINDS, 1, C.byref(a)) == 0
            emits.append(a)
        res.update(leg(lib, emits, reps, warmup), versions=len(emits))
        for a in emits:
            lib.etl_dec_arrow_free(a)
    st.close()
    dec.close()
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--copy-rows", type=int, default=1_000_000)
    ap.add_argument("--c3-scale", type=float, default=1.0)
    ap.add_argument("--c4-scale", type=float, default=0.1)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--plain-only", action="store_true")
    ap.add_argument("--no-pyarrow", action="store_true")
    ap.add_argument("--tag", default="")
    ap.add_argument("--page-index", action="store_true")
    ap.add_argument("--bloom", action="store_true")
    ap.add_argument("--c5-scale", type=float, default=0.02)
    ap.add_argument("--zstd", action="store_true")
    ap.add_argument("--c2-scale", type=float, default=0.05)
    ap.add_argument("--partition", action="store_true")
    ap.add_argument("--c1-scale", type=float, default=10.0)
    a = ap.parse_args()
    OPTS.update(plain_only=a.plain_only, pyarrow=not a.no_pyarrow, page_index=a.page_index, bloom=a.bloom, zstd=a.zstd,
                partition=a.partition)
    if not torch.cuda.is_available():
        raise SystemExit("parquet_measure needs a CUDA device")
    t = time.time()
    print(json.dumps(dict(card=card(), torch_device=torch.cuda.get_device_name(0))), flush=True)
    if a.partition:
        for name, scale, spec in (("c1", a.c1_scale, [(4, abi.ICE_DAY, 0)]), ("c2", a.c2_scale, [(0, abi.ICE_BUCKET, 16)]),
                                  ("copy", 0, [(0, abi.ICE_BUCKET, 16), (5, abi.ICE_TRUNCATE, 1)]),
                                  ("c5", a.c5_scale, [(0, abi.ICE_BUCKET, 16)])):
            OPTS["spec"] = spec
            if name != "copy" and not scale:                 # a scale of 0 skips the workload
                continue
            if name == "copy":
                copy_table(a.copy_rows, a.reps, a.warmup, a.tag)
            else:
                streaming(name, scale, a.reps, a.warmup, a.tag)
        print(json.dumps(dict(wall_s=round(time.time() - t, 1))), flush=True)
        return
    copy_table(a.copy_rows, a.reps, a.warmup, a.tag)
    if a.zstd:
        for name, scale in (("c2", a.c2_scale), ("c3", a.c3_scale), ("c5", a.c5_scale)):
            streaming(name, scale, a.reps, a.warmup, a.tag)
        print(json.dumps(dict(wall_s=round(time.time() - t, 1))), flush=True)
        return
    if a.page_index or a.bloom:
        for name, scale in (("c5", a.c5_scale), ("c4", a.c4_scale)):
            streaming(name, scale, a.reps, a.warmup, a.tag)
        print(json.dumps(dict(wall_s=round(time.time() - t, 1))), flush=True)
        return
    if not a.plain_only:
        copy_table(a.copy_rows, a.reps, a.warmup, a.tag, low_card=True)
    for name, scale in (("c3", a.c3_scale), ("c4", a.c4_scale)):
        streaming(name, scale, a.reps, a.warmup, a.tag)
    print(json.dumps(dict(wall_s=round(time.time() - t, 1))), flush=True)


if __name__ == "__main__":
    main()
