#!/usr/bin/env python
"""Time the columnar emitter (etl_dec_arrow_emit) with and without ETL_ARROW_ALL_COLUMNS on a resident decoded batch.

  python tools/arrow_emit_measure.py [--c3-scale 1.0] [--c4-scale 0.1] [--reps 7] [--warmup 2]

For C3 (one batch, its one schema version) and C4 (one batch, every schema version): decode the workload with the stream
resident in HBM, then per schema version time the emit (rows 3 = inserts + updates, to_host = 0) with and without the
bit: median / min / max over the repetitions of wall time around the call (the emit syncs before it returns).  Reports
rows, output bytes per column class and the decode time of the same batch; times etl_shim_materialise of the C3 batch
once for comparison.  Prints the card name and power limit (read-only nvidia-smi query) in the same run.
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
        k = int(schema_kinds[c])
        cls = "numeric" if k == 9 else "json" if k == 15 else CLASS[col.arrow_type]
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
            for label, rk in (("plain", 3), ("all_columns", 3 | ALL)):
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--c3-scale", type=float, default=1.0)
    ap.add_argument("--c4-scale", type=float, default=0.1)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-materialise", action="store_true")
    a = ap.parse_args()
    print(json.dumps(dict(card=card(), torch_device=torch.cuda.get_device_name(0))), flush=True)
    for name, scale, mat in (("c3", a.c3_scale, not a.no_materialise), ("c4", a.c4_scale, False)):
        r = measure(name, scale, a.reps, a.warmup, mat)
        r.pop("versions")
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
