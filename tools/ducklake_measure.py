#!/usr/bin/env python
"""Time the DuckLake emitter (etl_dec_ducklake_emit), its sub-batch fingerprints (etl_dec_ducklake_sub_batches) and
the host COPY fingerprint (etl_dec_ducklake_copy_fingerprint) on resident decoded batches.

  python tools/ducklake_measure.py [--c2-scale 1] [--c3-scale 1] [--c4-scale 0.1] [--c5-scale 0.1] [--copy-rows 1000000]
                                   [--reps 7] [--warmup 2]

Workloads: those of tools/bigquery_measure.py — C2, C3 (one batch, one schema version), C4 (one batch, every schema
version: times are sums over the versions), C5 at 0.1 and bench.py's 10-column COPY table, resident in HBM.  Every time
is median / min / max over the repetitions of wall time around the call (each call syncs before it returns): the emit
with to_host 0 and 1, the sub-batch call (no last_key, results on the host) and, for COPY, the host fingerprint over the
pinned texts.  GB/s = text bytes (row + predicate + assignments) / median time.  Prints the card name and power limit in
the same run.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from arrow_emit_measure import bench_copy_table, card, timed  # noqa: E402
from etl_b200 import abi, decoder, workloads as wl  # noqa: E402
from rowbinary_measure import sum_stats  # noqa: E402


def names_of(bh, si, tables):
    lib = abi.load()
    info = abi.SchemaInfo()
    assert lib.etl_dec_batch_schema(bh._h, si, C.byref(info)) == 0
    cols = tables[info.table_id]
    names = [f'"{cols[info.col_index[c]]["name"]}"' for c in range(info.n_cols)]
    return (C.c_char_p * max(1, len(names)))(*[n.encode() for n in names]), len(names)


def dl_once(lib, bh, si, names, to_host):
    h = C.c_void_p()
    assert lib.etl_dec_ducklake_emit(bh._h, si, names[0], names[1], to_host, C.byref(h)) == 0
    return h


def text_bytes(lib, h, host):
    total = 0
    for which in range(3):
        d, o, nb = C.c_void_p(), C.c_void_p(), C.c_uint64()
        assert lib.etl_dec_ducklake_text(h, which, host, C.byref(d), C.byref(o), C.byref(nb)) == 0
        total += nb.value
    return total


def sub_once(lib, h):
    out, n = C.c_void_p(), C.c_uint64()
    assert lib.etl_dec_ducklake_sub_batches(h, b"public_t", 8, None, 1, C.byref(out), C.byref(n)) == 0
    return n.value


def measure_batch(lib, bh, versions, names_for, reps, warmup, copy=False):
    e0, e1, sb, fp, muts, nbytes, chunks = [], [], [], [], 0, 0, 0
    for si in versions:
        names = names_for(si)
        e0.append(timed(lambda: lib.etl_dec_ducklake_free(dl_once(lib, bh, si, names, 0)), reps, warmup))
        e1.append(timed(lambda: lib.etl_dec_ducklake_free(dl_once(lib, bh, si, names, 1)), reps, warmup))
        h = dl_once(lib, bh, si, names, 1)
        muts += lib.etl_dec_ducklake_mutations(h)
        nbytes += text_bytes(lib, h, 1)
        if copy:
            out = C.c_uint64()
            fp.append(timed(lambda: lib.etl_dec_ducklake_copy_fingerprint(h, b"public_t", 8, C.byref(out)), reps, warmup))
        else:
            sb.append(timed(lambda: sub_once(lib, h), reps, warmup))
            chunks += sub_once(lib, h)
        lib.etl_dec_ducklake_free(h)
    t0 = sum_stats(e0)
    res = dict(mutations=int(muts), text_bytes=int(nbytes), emit_ms_to_host0=t0, emit_ms_to_host1=sum_stats(e1),
               emit_GBps=round(nbytes / (t0["median"] * 1e-3) / 1e9, 2) if t0["median"] else None, versions=len(versions))
    if copy:
        f = sum_stats(fp)
        res.update(copy_fingerprint_ms=f, copy_fingerprint_GBps=round(nbytes / (f["median"] * 1e-3) / 1e9, 2) if f["median"] else None)
    else:
        s = sum_stats(sb)
        res.update(sub_batches=int(chunks), sub_batches_ms=s,
                   sub_batches_GBps=round(nbytes / (s["median"] * 1e-3) / 1e9, 2) if s["median"] else None)
    return res


def streaming(name, scale, reps, warmup):
    w = wl.make(name, scale, n_segments=1)
    stream, stats = w.generate()
    st = decoder.Stager(stream.nbytes, 2048)
    st.append_framed(stream)
    dec = decoder.Decoder(0)
    tables = w.table_schemas()
    for tid, cols in tables.items():
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
        res.update(measure_batch(lib, bh, versions, lambda si: names_of(bh, si, tables), reps, warmup))
    st.close()
    dec.close()
    print(json.dumps(res), flush=True)
    return res


def copy_table(n_rows, reps, warmup):
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
    cols = [dict(name=f"c{i}", type_oid=o, pk=1 if i == 0 else None, nullable=i != 0) for i, o in enumerate(oids)]
    dec.put_table_schema(9, cols)
    inp = abi.CopyInput()
    inp.dev_buf, inp.dev_row_offsets, inp.len, inp.n_rows, inp.row_offsets = d_buf.data_ptr(), d_off.data_ptr(), len(blob), len(rows), offs.ctypes.data
    h = C.c_void_p()
    assert lib.etl_dec_copy_decode(dec._ctx, 9, C.byref(inp), 0, C.byref(h)) == 0, lib.etl_dec_last_error(dec._ctx)
    names = (C.c_char_p * len(cols))(*[c["name"].encode() for c in cols]), len(cols)
    with decoder.BatchHandle(dec, h) as bh:
        res = dict(workload="bench.py COPY table (5 x int4, 5 x text)", input_bytes=len(blob))
        res.update(measure_batch(lib, bh, [0], lambda si: names, reps, warmup, copy=True))
        print(json.dumps(res), flush=True)
    dec.close()
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
    a = ap.parse_args()
    t = time.time()
    print(json.dumps(dict(card=card(), torch_device=torch.cuda.get_device_name(0))), flush=True)
    copy_table(a.copy_rows, a.reps, a.warmup)
    for name, scale in (("c2", a.c2_scale), ("c3", a.c3_scale), ("c4", a.c4_scale), ("c5", a.c5_scale)):
        streaming(name, scale, a.reps, a.warmup)
    print(json.dumps(dict(wall_s=round(time.time() - t, 1))), flush=True)


if __name__ == "__main__":
    main()
