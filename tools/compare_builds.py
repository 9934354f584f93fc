"""Run the same seeded decodes through two builds of the decode library and compare what they return.

    python tools/compare_builds.py --a _parent --b ""

Each build is selected by its ETL_LIB_SUFFIX (etl_b200/build.py): etl_b200/libetl_decode<suffix>.so must exist, and is
loaded as it is.  Every build runs in a process of its own through the sequences of tests/test_gpu_batch_sequence.py
(every sizing branch: optimistic, exact, record and cell re-runs, scratch restart, array-heap retry, late long-value
passes, decode_begin / decode_finish, COPY rows between replication batches), COPY batches over the heap corpora of
tests/test_gpu_copy_edges.py, and one context per workload (C2 to C5 at small scale) decoding two batches with and
without the host copy and the timings.  Every batch freed is recorded: each etl_dec_summary field except the *_ms
timings, which planes are null, a digest of each host plane, and the oracle's canonical digest of the cells (cell_val
and the heap are compared through it alone: the kernels bump-allocate heap slots in no fixed order).  Exit status 0 when
the two records are equal.  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (plane, bytes per entry); rec_cell_base, with its n_records + 1 entries, is listed on its own
REC_PLANES = [("rec_off", 8), ("rec_kind", 1), ("rec_flags", 1), ("rec_rel", 4), ("rec_schema", 4), ("rec_start_lsn", 8),
              ("rec_commit_lsn", 8), ("rec_tx_ordinal", 8), ("rec_tuple_bytes", 4), ("rec_heap_hint", 4)]
CELL_PLANES = [("cell_tag", 1), ("cell_val", 8), ("cell_aux", 4)]


def record_of(bh, abi, C, pyoracle, copy_stream):
    s = bh.summary()
    out = {}
    for name, _ in abi.Summary._fields_:
        if name.endswith("_ms"):
            continue
        v = getattr(s, name)
        out[name] = [getattr(v, f) for f, _ in v._fields_ if f != "_pad"] if isinstance(v, C.Structure) else int(v)
    dev = bh.planes(False)
    out["null_planes"] = [n for n, _ in abi.Planes._fields_ if n.startswith(("rec_", "cell_", "heap")) and n != "heap_bytes"
                          and not getattr(dev, n)]
    out["counts"] = [int(dev.n_records), int(dev.n_cells), int(dev.heap_bytes)]
    try:
        p = bh.planes(True)
    except Exception:  # noqa: BLE001 — decoded without ETL_DECODE_RESULTS_TO_HOST
        return out
    import numpy as np
    from etl_b200.decoder import _np_from
    n, m = int(p.n_records), int(p.n_cells)
    sizes = [(k, w * n) for k, w in REC_PLANES] + [("rec_cell_base", 8 * (n + 1))] + [(k, w * m) for k, w in CELL_PLANES
                                                                                      if k != "cell_val"]
    fe = s.first_error.record_index
    n_valid = n if fe == 2**64 - 1 else int(fe - s.record_index_base)
    if p.rec_kind:
        out["canonical"] = pyoracle.planes_digest(p, n_valid)
    else:
        out["canonical"] = pyoracle.copy_planes_digest(
            _np_from(p.cell_tag, m, np.uint8), _np_from(p.cell_val, m, np.uint64), _np_from(p.cell_aux, m, np.uint32),
            n_valid, m // n if n else 0, copy_stream, _np_from(p.heap, p.heap_bytes, np.uint8))
    digests = {}
    for k, nbytes in sizes:
        ptr = getattr(p, k)
        digests[k] = None if not ptr else hashlib.sha256(C.string_at(ptr, nbytes) if nbytes else b"").hexdigest()[:16]
    out["host_null_planes"] = sorted(k for k, v in digests.items() if v is None)
    out["host"] = digests
    return out


def child(out_path: str) -> None:
    import ctypes as C
    import types

    import numpy as np
    for p in (ROOT, os.path.join(ROOT, "tests")):
        sys.path.insert(0, p)
    from etl_b200 import abi, decoder, workloads
    from oracle import pyoracle
    import test_gpu_batch_sequence as T
    import test_gpu_copy_edges as E
    from test_gpu_copy import cols_of

    pyoracle.build()
    records = []
    label = ["?"]
    copy_stream = [np.zeros(0, np.uint8)]         # the rows of the last COPY decode
    free = decoder.BatchHandle.free
    copy_decode = decoder.Decoder.copy_decode

    def recording_free(self):
        if self._h:
            r = record_of(self, abi, C, pyoracle, copy_stream[0])
            r["label"] = label[0]
            records.append(r)
        free(self)
    decoder.BatchHandle.free = recording_free

    def stashing_copy_decode(self, table_id, rows, row_offsets=None):
        copy_stream[0] = np.frombuffer(b"".join(bytes(r) for r in rows) if isinstance(rows, (list, tuple)) else bytes(rows),
                                       dtype=np.uint8)
        return copy_decode(self, table_id, rows, row_offsets)
    decoder.Decoder.copy_decode = stashing_copy_decode
    gpu = types.SimpleNamespace(Decoder=decoder.Decoder, Stager=decoder.Stager)

    def run(name, fn, *args):
        label[0] = name
        fn(*args)
        print(f"{name}: {sum(r['label'] == name for r in records)} batches", flush=True)

    run("steady c2", T.test_steady_state_sequence, gpu, pyoracle, "c2", 0.06, 11)
    run("steady c4", T.test_steady_state_sequence, gpu, pyoracle, "c4", 0.004, 12)
    run("rerun records", T.test_rerun_records_after_sparse_history, gpu, pyoracle)
    run("rerun cells", T.test_rerun_cells_only_after_sparse_history, gpu, pyoracle)
    run("scratch restart", T.test_scratch_restart_then_normal_batch, gpu, pyoracle)
    run("array heap", T.test_array_heap_retry_with_history, gpu, pyoracle)
    run("wrong hint", T.test_wrong_frame_hint_with_history, gpu, pyoracle, False)
    run("wrong hint poisoned", T.test_wrong_frame_hint_with_history, gpu, pyoracle, True)
    run("interleaved + COPY", T.test_interleaved_entry_points, gpu, pyoracle)
    run("size swings", T.test_size_swings, gpu, pyoracle)
    run("empty batch", T.test_empty_batch_on_a_used_context, gpu, pyoracle)
    for corpus in sorted(E.HEAP_CORPORA):
        for n in (13, 100000):
            run(f"COPY {corpus} {n}", E.test_heap_corpora, gpu, pyoracle, corpus, n)

    def workload(name, scale):
        w = workloads.make(name, scale, n_segments=2)
        dec = decoder.Decoder(0)
        try:
            for tid, cols in w.table_schemas().items():
                dec.put_table_schema(tid, cols)
            for seg, (to_host, timing) in enumerate([(True, True), (False, False)]):
                stream, _ = w.generate(range(seg, seg + 1))
                st = decoder.Stager(max(stream.nbytes, 1), 2048)
                try:
                    st.append_framed(stream.tobytes())
                    dec.decode_input(st.view(), to_host=to_host, timing=timing).free()
                finally:
                    st.close()
        finally:
            dec.close()
    for name, scale in (("c2", 0.02), ("c3", 0.002), ("c4", 0.004), ("c5", 0.0004)):
        run(f"workload {name}", workload, name, scale)

    def copy_flags():
        # etl_dec_copy_decode with and without the host copy and the timings, on one context
        oids, rows = E.heap_corpus("heavy", 1000)
        dec = decoder.Decoder(0)
        try:
            dec.put_table_schema(7, cols_of(oids))
            offs = np.zeros(len(rows) + 1, dtype=np.uint64)
            offs[1:] = np.cumsum([len(r) for r in rows])
            buf = np.frombuffer(b"".join(bytes(r) for r in rows) + bytes(64), dtype=np.uint8)
            copy_stream[0] = buf[:int(offs[-1])]
            for flags in (abi.RESULTS_TO_HOST, 0, abi.NO_TIMING, abi.RESULTS_TO_HOST | abi.NO_TIMING):
                inp = abi.CopyInput()
                inp.host_buf = buf.ctypes.data
                inp.len = int(offs[-1])
                inp.row_offsets = offs.ctypes.data
                inp.n_rows = len(rows)
                h = C.c_void_p()
                dec._check(dec._l.etl_dec_copy_decode(dec._ctx, 7, C.byref(inp), flags, C.byref(h)))
                decoder.BatchHandle(dec, h).free()
        finally:
            dec.close()
    run("COPY flags", copy_flags)

    with open(out_path, "w") as f:
        json.dump(records, f)


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--a", required=True, help="ETL_LIB_SUFFIX of the first build (e.g. _parent)")
    ap.add_argument("--b", default="", help="ETL_LIB_SUFFIX of the second build (default: the in-tree library)")
    ap.add_argument("--child", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        child(args.child)
        return 0
    runs = []
    with tempfile.TemporaryDirectory() as tmp:
        for suffix in (args.a, args.b):
            lib = os.path.join(ROOT, "etl_b200", f"libetl_decode{suffix}.so")
            if not os.path.exists(lib):
                sys.exit(f"{lib} does not exist")
            out = os.path.join(tmp, f"run{len(runs)}.json")
            print(f"== build '{suffix}'", flush=True)
            subprocess.run([sys.executable, __file__, "--a", args.a, "--child", out], check=True,
                           env={**os.environ, "ETL_LIB_SUFFIX": suffix})
            with open(out) as f:
                runs.append(json.load(f))
    a, b = runs
    bad = 0
    if len(a) != len(b):
        print(f"batch counts differ: {len(a)} against {len(b)}")
        bad += 1
    for i, (x, y) in enumerate(zip(a, b)):
        if x != y:
            bad += 1
            keys = sorted(k for k in set(x) | set(y) if x.get(k) != y.get(k))
            print(f"batch {i} ({x['label']}): " + "; ".join(f"{k}: {x.get(k)} | {y.get(k)}" for k in keys))
    sizing = sorted({r["sizing"] for r in a})
    print(f"{len(a)} batches, sizing values {sizing}: " + ("equal" if not bad else f"{bad} differ"))
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
