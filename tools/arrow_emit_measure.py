#!/usr/bin/env python
"""Time the columnar emitter (etl_dec_arrow_emit) with and without ETL_ARROW_ALL_COLUMNS / ETL_ARROW_CDC_COLUMNS on a
resident decoded batch.

  python tools/arrow_emit_measure.py [--c3-scale 1.0] [--c4-scale 0.1] [--copy-rows 1000000] [--reps 7] [--warmup 2]

COPY rows: bench.py's COPY table and a synth_rows-shaped table, both resident in HBM; times etl_dec_copy_decode and the
emit of its batch with row_kinds 1, 1|ALL and 1|ALL|CDC.
For C3 (one batch, its one schema version) and C4 (one batch, every schema version): decode the workload with the stream
resident in HBM, then per schema version time the emit (rows 3 = inserts + updates, to_host = 0) with and without each
bit.  Every time is median / min / max over the repetitions of wall time around the call (the decode and the emit sync
before they return).  Reports rows, output bytes per column class and the decode time of the same batch; times
etl_shim_materialise of the C3 batch once for comparison.  Prints the card name and power limit (read-only nvidia-smi
query) in the same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from etl_b200 import abi, decoder, workloads as wl  # noqa: E402

ALL = abi.ARROW_ALL_COLUMNS
CDC = abi.ARROW_CDC_COLUMNS
CLASS = {1: "fixed", 2: "fixed", 3: "fixed", 4: "fixed", 5: "fixed", 8: "fixed", 9: "fixed", 10: "fixed", 11: "fixed", 12: "fixed",
         6: "utf8", 7: "binary", 13: "list"}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def out_bytes(lib, a, kinds_all, schema_kinds):
    """output bytes per column class: fixed-width values + validity, Utf8 / LargeBinary data + offsets, Numeric and Json
    text, List offsets + children"""
    n = lib.etl_dec_arrow_rows(a)
    acc = {}
    for c in range(lib.etl_dec_arrow_cols(a)):
        col = abi.ArrowColumn()
        lib.etl_dec_arrow_column(a, c, 0, C.byref(col))
        if not col.arrow_type:
            acc["unsupported"] = acc.get("unsupported", 0)
            continue
        k = int(schema_kinds[c]) if c < len(schema_kinds) else -1
        cls = "cdc" if k < 0 else "numeric" if k == 9 else "json" if k == 15 else CLASS[col.arrow_type]
        b = (n + 7) // 8
        if col.arrow_type in (6, 7):
            b += col.data_bytes + (n + 1) * (4 if col.arrow_type == 6 else 8)
        elif col.arrow_type == 13:
            kid, ne = abi.ArrowColumn(), C.c_uint64()
            lib.etl_dec_arrow_list_child(a, c, 0, C.byref(kid), C.byref(ne))
            b += (n + 1) * 4 + (ne.value + 7) // 8 + kid.data_bytes
        elif col.arrow_type == 1:
            b += (n + 7) // 8
        else:
            b += n * {2: 4, 3: 8, 4: 4, 5: 8, 8: 4, 9: 8, 10: 8, 11: 8, 12: 16}[col.arrow_type]
        acc[cls] = acc.get(cls, 0) + b
    return n, acc


def measure(name, scale, reps, warmup, materialise):
    w = wl.make(name, scale, n_segments=1)
    stream, stats = w.generate()
    st = decoder.Stager(stream.nbytes, 2048)
    st.append_framed(stream)
    dec = decoder.Decoder(0)
    for tid, cols in w.table_schemas().items():
        dec.put_table_schema(tid, cols)
    v = st.view()
    d_stream = torch.empty(stream.nbytes + 64, dtype=torch.uint8, device="cuda")
    d_stream[:stream.nbytes].copy_(torch.from_numpy(st.host_array()))
    torch.cuda.synchronize()
    lib = abi.load()
    res = dict(workload=name, scale=scale, stream_bytes=int(stream.nbytes), frames=int(stats["frames"]), versions=[])
    inp = st.view()
    inp.dev_buf = d_stream.data_ptr()
    with dec.decode_input(inp, to_host=materialise) as bh:
        s = bh.summary()
        res["decode_kernel_ms"] = round(s.kernel_ms, 3)
        for si in range(s.n_schemas):
            info = abi.SchemaInfo()
            lib.etl_dec_batch_schema(bh._h, si, C.byref(info))
            kinds = np.ctypeslib.as_array(info.col_kind, shape=(info.n_cols,)).copy()
            row = dict(schema=si, n_cols=int(info.n_cols))
            for label, rk in (("plain", 3), ("plain_cdc", 3 | CDC), ("all_columns", 3 | ALL), ("all_columns_cdc", 3 | ALL | CDC)):
                ts = []
                for it in range(warmup + reps):
                    a = C.c_void_p()
                    t0 = time.perf_counter()
                    rc = lib.etl_dec_arrow_emit(bh._h, si, rk, 0, C.byref(a))
                    t1 = time.perf_counter()
                    assert rc == 0, rc
                    if it >= warmup:
                        ts.append((t1 - t0) * 1e3)
                    if it == warmup + reps - 1:
                        row["rows"], row[label + "_bytes"] = out_bytes(lib, a, rk, kinds)
                    lib.etl_dec_arrow_free(a)
                row[label + "_ms"] = dict(median=round(float(np.median(ts)), 3), min=round(min(ts), 3), max=round(max(ts), 3))
            res["versions"].append(row)
            print(json.dumps(dict(workload=name, **row)), flush=True)
        if materialise:
            lst = C.c_void_p()
            t0 = time.perf_counter()
            assert lib.etl_shim_materialise(bh._h, st.view().host_buf, None, C.byref(lst)) == 0
            res["shim_materialise_s"] = round(time.perf_counter() - t0, 2)
            lib.etl_shim_event_list_free(lst)
    st.close()
    dec.close()
    return res


def bench_copy_table(n_rows):
    """bench.py's COPY table: 5 x int4 + 5 x text, 5 % NULL (same generator, same seed)"""
    rng = np.random.default_rng(0xC0B7)
    ints = rng.integers(-2**31, 2**31, size=(n_rows, 5))
    lens = np.minimum(256, np.maximum(1, np.exp(np.log(16) + 0.8 * rng.standard_normal((n_rows, 5))).astype(np.int64)))
    alnum = np.frombuffer(b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789      ", dtype=np.uint8)
    pool = alnum[rng.integers(0, len(alnum), size=1 << 20)].tobytes()
    starts = rng.integers(0, (1 << 20) - 256, size=(n_rows, 5))
    nulls = rng.integers(0, 20, size=(n_rows, 9)) == 0
    rows = []
    for r in range(n_rows):
        f = [str(ints[r, 0])] + ["\\N" if nulls[r, c - 1] else str(ints[r, c]) for c in range(1, 5)]
        f += ["\\N" if nulls[r, 4 + c] else pool[starts[r, c]:starts[r, c] + lens[r, c]].decode() for c in range(5)]
        rows.append(("\t".join(f) + "\n").encode())
    return [23] * 5 + [25] * 5, rows


def synth_table(n_rows, distinct=100_000):
    """tests/test_gpu_copy.py's synth_rows shape (int4, text with escapes, bool, numeric, jsonb, timestamptz, uuid, bytea,
    float8, int8; NULLs): `distinct` generated rows repeated to n_rows (the generator is slow in Python)"""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    from test_gpu_copy import synth_rows
    oids, rows = synth_rows(min(n_rows, distinct), 0x5E7)
    return oids, (rows * (-(-n_rows // len(rows))))[:n_rows]


def timed(fn, reps, warmup):
    ts = []
    for it in range(warmup + reps):
        t0 = time.perf_counter()
        fn()
        if it >= warmup:
            ts.append((time.perf_counter() - t0) * 1e3)
    return dict(median=round(float(np.median(ts)), 3), min=round(min(ts), 3), max=round(max(ts), 3))


def measure_copy(label, oids, rows, reps, warmup):
    """COPY rows resident in HBM: etl_dec_copy_decode (planes stay on the device), then the emit of the batch with
    row_kinds 1, 1|ALL and 1|ALL|CDC (to_host = 0); wall time around each call (both sync before they return)"""
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

    def decode():
        h = C.c_void_p()
        assert lib.etl_dec_copy_decode(dec._ctx, 9, C.byref(inp), 0, C.byref(h)) == 0, lib.etl_dec_last_error(dec._ctx)
        return decoder.BatchHandle(dec, h)
    res = dict(table=label, rows=len(rows), bytes=len(blob), copy_decode_ms=timed(lambda: decode().free(), reps, warmup))
    kinds = [dec._l.etl_dec_kind_for_type_oid(o) for o in oids]
    with decode() as bh:
        assert bh.summary().first_error.record_index == 2**64 - 1
        for name, rk in (("emit", 1), ("emit_all", 1 | ALL), ("emit_all_cdc", 1 | ALL | CDC)):
            def once():
                a = C.c_void_p()
                assert lib.etl_dec_arrow_emit(bh._h, 0, rk, 0, C.byref(a)) == 0
                lib.etl_dec_arrow_free(a)
            res[name + "_ms"] = timed(once, reps, warmup)
            a = C.c_void_p()
            assert lib.etl_dec_arrow_emit(bh._h, 0, rk, 0, C.byref(a)) == 0
            res[name + "_bytes"] = out_bytes(lib, a, rk, kinds)[1]
            lib.etl_dec_arrow_free(a)
    dec.close()
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--c3-scale", type=float, default=1.0)
    ap.add_argument("--c4-scale", type=float, default=0.1)
    ap.add_argument("--copy-rows", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-materialise", action="store_true")
    a = ap.parse_args()
    print(json.dumps(dict(card=card(), torch_device=torch.cuda.get_device_name(0))), flush=True)
    measure_copy("bench.py COPY table (5 x int4, 5 x text)", *bench_copy_table(a.copy_rows), a.reps, a.warmup)
    measure_copy("synth_rows shape (numeric, jsonb, uuid, bytea, floats, ...)", *synth_table(a.copy_rows), a.reps, a.warmup)
    for name, scale, mat in (("c3", a.c3_scale, not a.no_materialise), ("c4", a.c4_scale, False)):
        r = measure(name, scale, a.reps, a.warmup, mat)
        r.pop("versions")
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
