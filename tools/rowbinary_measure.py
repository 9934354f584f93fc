#!/usr/bin/env python
"""Time the ClickHouse RowBinary emitter (etl_dec_rowbinary_emit) on resident decoded batches, beside the Arrow emit
(row_kinds 3|ALL|CDC, COPY: 1|ALL|CDC) and etl_shim_materialise of the same batch.

  python tools/rowbinary_measure.py [--c2-scale 1] [--c3-scale 1] [--c4-scale 0.1] [--c5-scale 0.1] [--copy-rows 1000000]
                                    [--reps 7] [--warmup 2] [--profile OUT_DIR] [--lz4]

Workloads: C2, C3 (one batch, one schema version), C4 (one batch, every schema version: times are sums over the
versions), C5 at 0.1, about 1 GiB (both tables: TOAST, key-only deletes, partial updates), and bench.py's 10-column COPY table.  The stream
(or the COPY rows) is resident in HBM; every emit gets the Nullable flags build_create_table_sql would give the table
(source-nullable non-array columns; the CDC columns not nullable).  Every time is median / min / max over the repetitions
of wall time around the call (each emit syncs before it returns), with to_host 0 and 1; GB/s = RowBinary bytes / median
time with to_host 0.  Prints the card name and power limit in the same run.
--profile: one emit per workload under torch.profiler instead (separate run), written to OUT_DIR as a table of CUDA
kernel time and CUDA runtime API time (cudaMallocAsync / cudaFreeAsync / cudaMalloc / cudaFree / syncs) per workload.
--lz4: instead, the compressed INSERT bodies (etl_dec_rowbinary_lz4) of each emit at the 64 MiB default
max_bytes_per_insert: the call's time with to_host 0 and 1, uncompressed GB/s (RowBinary bytes / median to_host 0 time),
the compression ratio (RowBinary bytes / body bytes), and the same INSERTs cut at the same block size compressed on one
host thread by pyarrow's lz4_raw (liblz4, standing in for the clickhouse crate's lz4_flex): its time and ratio.  With
--profile, the LZ4 call's kernels under torch.profiler.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import torch  # noqa: E402

from arrow_emit_measure import bench_copy_table, card, timed  # noqa: E402
from etl_b200 import abi, decoder, workloads as wl  # noqa: E402

ALL, CDC = abi.ARROW_ALL_COLUMNS, abi.ARROW_CDC_COLUMNS


def create_table_flags(lib, bh, si, copy_kinds=None):
    """build_create_table_sql's Nullable wrappers: source-nullable, non-array columns; CDC columns not nullable"""
    if copy_kinds is not None:
        return [0] + [1] * (len(copy_kinds) - 1) + [0, 0]        # measure_copy's table: column 0 NOT NULL
    info = abi.SchemaInfo()
    lib.etl_dec_batch_schema(bh._h, si, C.byref(info))
    kinds = np.ctypeslib.as_array(info.col_kind, shape=(info.n_cols,))
    fl = np.ctypeslib.as_array(info.col_flags, shape=(info.n_cols,))
    return [int(bool(f & 1) and not k & 0x20) for k, f in zip(kinds, fl)] + [0, 0]


def rb_once(lib, bh, si, flags, to_host):
    fl = (C.c_uint8 * len(flags))(*flags)
    h = C.c_void_p()
    assert lib.etl_dec_rowbinary_emit(bh._h, si, fl, len(flags), to_host, C.byref(h)) == 0
    return h


def sum_stats(parts):
    return {k: round(sum(p[k] for p in parts), 3) for k in ("median", "min", "max")}


LZ4_MAX = 64 << 20        # the destination's default max_bytes_per_insert


def lz4_once(lib, h, to_host):
    z = C.c_void_p()
    assert lib.etl_dec_rowbinary_lz4(h, 0, lib.etl_dec_rowbinary_rows(h), LZ4_MAX, to_host, C.byref(z)) == 0
    return z


def measure_lz4(lib, bh, versions, flags_of, reps, warmup):
    """per version: etl_dec_rowbinary_lz4 over the whole emit (to_host 0 / 1) and liblz4 on one host thread over the
    same INSERTs and block cuts; summed over the versions"""
    import pyarrow as pa
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))
    import clickhouse_lz4_ref as Z
    codec = pa.Codec("lz4_raw")
    t0s, t1s, host_ms, raw, dev_z, host_z = [], [], 0.0, 0, 0, 0
    for si in versions:
        h = rb_once(lib, bh, si, flags_of(si), 1)
        t0s.append(timed(lambda: lib.etl_dec_rowbinary_lz4_free(lz4_once(lib, h, 0)), reps, warmup))
        t1s.append(timed(lambda: lib.etl_dec_rowbinary_lz4_free(lz4_once(lib, h, 1)), reps, warmup))
        z = lz4_once(lib, h, 1)
        n_ins = lib.etl_dec_rowbinary_lz4_inserts(z)
        cuts = np.ctypeslib.as_array(C.cast(lib.etl_dec_rowbinary_lz4_insert_rows(z, 1), C.POINTER(C.c_uint64)), shape=(n_ins + 1,)).copy()
        dev_z += lib.etl_dec_rowbinary_lz4_bytes(z)
        lib.etl_dec_rowbinary_lz4_free(z)
        n = lib.etl_dec_rowbinary_rows(h)
        nbytes = lib.etl_dec_rowbinary_bytes(h)
        raw += nbytes
        if nbytes:
            offs = np.ctypeslib.as_array(C.cast(lib.etl_dec_rowbinary_row_offsets(h, 1), C.POINTER(C.c_uint64)), shape=(n + 1,))
            data = bytes((C.c_uint8 * nbytes).from_address(lib.etl_dec_rowbinary_data(h, 1)))
            blocks = [data[a:min(a + Z.KBLOCK, int(offs[cuts[k + 1]]))]
                      for k in range(n_ins) for a in range(int(offs[cuts[k]]), int(offs[cuts[k + 1]]), Z.KBLOCK)]
            t = time.perf_counter()
            host_z += sum(Z.HEADER + len(codec.compress(b, asbytes=True)) for b in blocks)
            host_ms += (time.perf_counter() - t) * 1e3
        lib.etl_dec_rowbinary_free(h)
    t0 = sum_stats(t0s)
    return dict(rowbinary_bytes=int(raw), lz4_bytes=int(dev_z), lz4_block=Z.KBLOCK, lz4_ms_to_host0=t0, lz4_ms_to_host1=sum_stats(t1s),
                lz4_GBps_uncompressed=round(raw / (t0["median"] * 1e-3) / 1e9, 2) if t0["median"] else None,
                lz4_ratio=round(raw / dev_z, 3) if dev_z else None, liblz4_1thread_ms=round(host_ms, 1),
                liblz4_ratio=round(raw / host_z, 3) if host_z else None, versions=len(versions))


def profile_lz4(lib, bh, versions, flags_of, label, out_dir):
    """one warm etl_dec_rowbinary_lz4 call per version under torch.profiler: kernel time by name"""
    from torch.profiler import ProfilerActivity, profile
    hs = [rb_once(lib, bh, si, flags_of(si), 0) for si in versions]
    for h in hs:
        lib.etl_dec_rowbinary_lz4_free(lz4_once(lib, h, 0))
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for h in hs:
            lib.etl_dec_rowbinary_lz4_free(lz4_once(lib, h, 0))
        torch.cuda.synchronize()
    for h in hs:
        lib.etl_dec_rowbinary_free(h)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, f"lz4_profile_{label}.txt"), "w") as f:
        f.write(prof.key_averages().table(sort_by="self_cuda_time_total", row_limit=30) + "\n")
    kern = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0)
        if t and not e.key.startswith("cu"):
            kern[e.key[:60]] = round(t / 1e3, 3)
    res = dict(profile=label, lz4_kernel_ms=kern)
    print(json.dumps(res), flush=True)
    return res


def measure_batch(lib, bh, versions, flags_of, arrow_kinds, reps, warmup):
    """per version: RowBinary emit (to_host 0 / 1) and the Arrow emit; summed over the versions"""
    rb0, rb1, ar, rows, nbytes = [], [], [], 0, 0
    for si in versions:
        flags = flags_of(si)
        rb0.append(timed(lambda: lib.etl_dec_rowbinary_free(rb_once(lib, bh, si, flags, 0)), reps, warmup))
        rb1.append(timed(lambda: lib.etl_dec_rowbinary_free(rb_once(lib, bh, si, flags, 1)), reps, warmup))

        def arrow():
            a = C.c_void_p()
            assert lib.etl_dec_arrow_emit(bh._h, si, arrow_kinds, 0, C.byref(a)) == 0
            lib.etl_dec_arrow_free(a)
        ar.append(timed(arrow, reps, warmup))
        h = rb_once(lib, bh, si, flags, 0)
        rows += lib.etl_dec_rowbinary_rows(h)
        nbytes += lib.etl_dec_rowbinary_bytes(h)
        lib.etl_dec_rowbinary_free(h)
    t0 = sum_stats(rb0)
    return dict(rows=int(rows), rowbinary_bytes=int(nbytes), rowbinary_ms_to_host0=t0, rowbinary_ms_to_host1=sum_stats(rb1),
                rowbinary_GBps=round(nbytes / (t0["median"] * 1e-3) / 1e9, 2) if t0["median"] else None,
                arrow_all_cdc_ms=sum_stats(ar), versions=len(versions))


def streaming(name, scale, reps, warmup, profile=None, lz4=False):
    w = wl.make(name, scale, n_segments=1)
    stream, stats = w.generate()
    st = decoder.Stager(stream.nbytes, 2048)
    st.append_framed(stream)
    dec = decoder.Decoder(0)
    for tid, cols in w.table_schemas().items():
        dec.put_table_schema(tid, cols)
    d_stream = torch.empty(stream.nbytes + 64, dtype=torch.uint8, device="cuda")
    d_stream[:stream.nbytes].copy_(torch.from_numpy(st.host_array()))
    torch.cuda.synchronize()
    lib = abi.load()
    inp = st.view()
    inp.dev_buf = d_stream.data_ptr()
    res = dict(workload=name, scale=scale, stream_bytes=int(stream.nbytes), frames=int(stats["frames"]))
    with dec.decode_input(inp, to_host=profile is None) as bh:
        s = bh.summary()
        versions = list(range(s.n_schemas))
        if lz4:
            flags_of = lambda si: create_table_flags(lib, bh, si)  # noqa: E731
            res.update(profile_lz4(lib, bh, versions, flags_of, name, profile) if profile else measure_lz4(lib, bh, versions, flags_of, reps, warmup))
            print(json.dumps(res), flush=True)
            return res
        if profile is not None:
            return profile_emits(lib, bh, versions, lambda si: create_table_flags(lib, bh, si), name, profile)
        res["decode_kernel_ms"] = round(s.kernel_ms, 3)
        res.update(measure_batch(lib, bh, versions, lambda si: create_table_flags(lib, bh, si), 3 | ALL | CDC, reps, warmup))
        lst = C.c_void_p()
        t0 = time.perf_counter()
        assert lib.etl_shim_materialise(bh._h, st.view().host_buf, None, C.byref(lst)) == 0
        res["shim_materialise_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
        lib.etl_shim_event_list_free(lst)
    st.close()
    dec.close()
    print(json.dumps(res), flush=True)
    return res


def copy_table(n_rows, reps, warmup, profile=None, lz4=False):
    oids, rows = bench_copy_table(n_rows)
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
    flags = create_table_flags(lib, None, 0, oids)
    with decoder.BatchHandle(dec, h) as bh:
        if lz4:
            res = dict(workload="bench.py COPY table (5 x int4, 5 x text)", input_bytes=len(blob))
            res.update(profile_lz4(lib, bh, [0], lambda si: flags, "copy", profile) if profile else measure_lz4(lib, bh, [0], lambda si: flags, reps, warmup))
            dec.close()
            print(json.dumps(res), flush=True)
            return res
        if profile is not None:
            return profile_emits(lib, bh, [0], lambda si: flags, "copy", profile)
        res = dict(workload="bench.py COPY table (5 x int4, 5 x text)", input_bytes=len(blob))
        res.update(measure_batch(lib, bh, [0], lambda si: flags, 1 | ALL | CDC, reps, warmup))
    dec.close()
    print(json.dumps(res), flush=True)
    return res


def profile_emits(lib, bh, versions, flags_of, label, out_dir):
    """one warm RowBinary emit per version under torch.profiler: kernel time by name, CUDA API time by name"""
    from torch.profiler import ProfilerActivity, profile
    for si in versions:
        lib.etl_dec_rowbinary_free(rb_once(lib, bh, si, flags_of(si), 0))
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for si in versions:
            lib.etl_dec_rowbinary_free(rb_once(lib, bh, si, flags_of(si), 0))
        torch.cuda.synchronize()
    os.makedirs(out_dir, exist_ok=True)
    table = prof.key_averages().table(sort_by="self_cuda_time_total", row_limit=40)
    with open(os.path.join(out_dir, f"rowbinary_profile_{label}.txt"), "w") as f:
        f.write(table + "\n")
    kern, api = {}, {}
    for e in prof.key_averages():
        name = e.key
        if name.startswith("cuda") or name.startswith("cu"):
            api[name] = round(e.cpu_time_total / 1e3, 3)
        elif getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0):
            kern[name[:60]] = round((getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0)) / 1e3, 3)
    res = dict(profile=label, kernel_ms=kern, api_ms=api)
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--c2-scale", type=float, default=1.0)
    ap.add_argument("--c3-scale", type=float, default=1.0)
    ap.add_argument("--c4-scale", type=float, default=0.1)
    ap.add_argument("--c5-scale", type=float, default=0.1)
    ap.add_argument("--copy-rows", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", default=None)
    ap.add_argument("--lz4", action="store_true")
    a = ap.parse_args()
    print(json.dumps(dict(card=card(), torch_device=torch.cuda.get_device_name(0))), flush=True)
    copy_table(a.copy_rows, a.reps, a.warmup, a.profile, a.lz4)
    for name, scale in (("c2", a.c2_scale), ("c3", a.c3_scale), ("c4", a.c4_scale), ("c5", a.c5_scale)):
        streaming(name, scale, a.reps, a.warmup, a.profile, a.lz4)


if __name__ == "__main__":
    main()
