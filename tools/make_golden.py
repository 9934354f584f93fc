#!/usr/bin/env python
"""Writes tests/golden/workload_digests.json: SHA-256 of the canonical event list the oracle produces for
small instances of the five BASELINE workloads.  The digest is over `repr(planes_to_events(...))` (typed
values dereferenced from the stream / heap, so heap placement does not matter).

The reference is a Rust workspace that the build does not compile (no Rust toolchain needed), so these fixtures pin the
ORACLE (which is itself pinned to the reference's known-answer tests, see tests/test_oracle_*.py) and
let the GPU path be checked against committed bytes instead of against a freshly built checker.
Usage: python tools/make_golden.py"""
import hashlib
import json
import os
import sys

ROOT = os.path.normpath(os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

CASES = [("c1", 1.0, None), ("c2", 0.004, 1), ("c3", 0.0005, 1), ("c4", 0.0004, 2), ("c5", 0.0004, 2)]


def digest_events(planes, stream: bytes) -> str:
    from canon import planes_to_events
    return hashlib.sha256(repr(planes_to_events(planes, stream)).encode()).hexdigest()


def main():
    from etl_b200 import workloads as wl
    from oracle import pyoracle
    out = {}
    for name, scale, segs in CASES:
        w = wl.make(name, scale, n_segments=segs)
        stream, stats = w.generate()
        o = pyoracle.Oracle()
        for tid, cols in w.table_schemas().items():
            o.put_table_schema(tid, cols)
        planes = o.decode(stream.tobytes())
        assert planes.first_error[0] is None
        out[name] = {"scale": scale, "n_segments": segs, "stream_sha256": hashlib.sha256(stream.tobytes()).hexdigest(),
                     "stream_bytes": int(stream.nbytes), "n_records": int(planes.n_records), "n_cells": int(planes.rec_cell_base[planes.n_records]),
                     "events_sha256": digest_events(planes, stream.tobytes())}
    path = os.path.join(ROOT, "tests", "golden", "workload_digests.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print("wrote", path)


if __name__ == "__main__":
    main()
