#!/usr/bin/env python
"""Time the BigQuery Storage Write emitter (etl_dec_bigquery_emit) on resident decoded batches, beside the ClickHouse
RowBinary emit of the same schema versions.

  python tools/bigquery_measure.py [--c2-scale 1] [--c3-scale 1] [--c4-scale 0.1] [--c5-scale 0.1] [--copy-rows 1000000]
                                   [--reps 7] [--warmup 2] [--profile OUT_DIR]

Workloads: those of tools/rowbinary_measure.py — C2, C3 (one batch, one schema version), C4 (one batch, every schema
version: times are sums over the versions), C5 at 0.1 and bench.py's 10-column COPY table, resident in HBM.  Every time
is median / min / max over the repetitions of wall time around the call (each emit syncs before it returns), with
to_host 0 and 1; GB/s = proto bytes / median time with to_host 0.  Prints the card name and power limit in the same run.
--profile: one emit per workload under torch.profiler instead (separate run), written to OUT_DIR as a table of CUDA
kernel time and CUDA runtime API time per workload.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import torch  # noqa: E402

from arrow_emit_measure import bench_copy_table, card, timed  # noqa: E402
from etl_b200 import abi, decoder, workloads as wl  # noqa: E402
from rowbinary_measure import create_table_flags, rb_once, sum_stats  # noqa: E402


def bq_once(lib, bh, si, to_host):
    h = C.c_void_p()
    assert lib.etl_dec_bigquery_emit(bh._h, si, to_host, C.byref(h)) == 0
    return h


def measure_batch(lib, bh, versions, flags_of, reps, warmup):
    """per version: BigQuery emit (to_host 0 / 1) and the RowBinary emit (to_host 0); summed over the versions"""
    bq0, bq1, rb, rows, nbytes = [], [], [], 0, 0
    for si in versions:
        flags = flags_of(si)
        bq0.append(timed(lambda: lib.etl_dec_bigquery_free(bq_once(lib, bh, si, 0)), reps, warmup))
        bq1.append(timed(lambda: lib.etl_dec_bigquery_free(bq_once(lib, bh, si, 1)), reps, warmup))
        rb.append(timed(lambda: lib.etl_dec_rowbinary_free(rb_once(lib, bh, si, flags, 0)), reps, warmup))
        h = bq_once(lib, bh, si, 0)
        rows += lib.etl_dec_bigquery_rows(h)
        nbytes += lib.etl_dec_bigquery_bytes(h)
        lib.etl_dec_bigquery_free(h)
    t0 = sum_stats(bq0)
    return dict(rows=int(rows), proto_bytes=int(nbytes), bigquery_ms_to_host0=t0, bigquery_ms_to_host1=sum_stats(bq1),
                bigquery_GBps=round(nbytes / (t0["median"] * 1e-3) / 1e9, 2) if t0["median"] else None,
                rowbinary_ms=sum_stats(rb), versions=len(versions))


def streaming(name, scale, reps, warmup, profile=None):
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
    with dec.decode_input(inp, to_host=False) as bh:
        versions = list(range(bh.summary().n_schemas))
        if profile is not None:
            res = profile_emits(lib, bh, versions, name, profile)
        else:
            res.update(measure_batch(lib, bh, versions, lambda si: create_table_flags(lib, bh, si), reps, warmup))
    st.close()
    dec.close()
    if profile is None:
        print(json.dumps(res), flush=True)
    return res


def copy_table(n_rows, reps, warmup, profile=None):
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
        if profile is not None:
            res = profile_emits(lib, bh, [0], "copy", profile)
        else:
            res = dict(workload="bench.py COPY table (5 x int4, 5 x text)", input_bytes=len(blob))
            res.update(measure_batch(lib, bh, [0], lambda si: flags, reps, warmup))
            print(json.dumps(res), flush=True)
    dec.close()
    return res


def profile_emits(lib, bh, versions, label, out_dir):
    """one warm BigQuery emit per version under torch.profiler: kernel time by name, CUDA API time by name"""
    from torch.profiler import ProfilerActivity, profile
    for si in versions:
        lib.etl_dec_bigquery_free(bq_once(lib, bh, si, 0))
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for si in versions:
            lib.etl_dec_bigquery_free(bq_once(lib, bh, si, 0))
        torch.cuda.synchronize()
    os.makedirs(out_dir, exist_ok=True)
    table = prof.key_averages().table(sort_by="self_cuda_time_total", row_limit=40)
    with open(os.path.join(out_dir, f"bigquery_profile_{label}.txt"), "w") as f:
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
    a = ap.parse_args()
    print(json.dumps(dict(card=card(), torch_device=torch.cuda.get_device_name(0))), flush=True)
    copy_table(a.copy_rows, a.reps, a.warmup, a.profile)
    for name, scale in (("c2", a.c2_scale), ("c3", a.c3_scale), ("c4", a.c4_scale), ("c5", a.c5_scale)):
        streaming(name, scale, a.reps, a.warmup, a.profile)


if __name__ == "__main__":
    main()
