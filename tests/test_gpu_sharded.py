"""Sharded decode on several GPUs of one box (etl_dec_decode_sharded: NCCL seam all-gather + device-side fold +
relation-update exchange, all inside the library), checked against the oracle's decode of the whole stream.
The NCCL cases need one GPU per rank and skip on a smaller machine.  Also: context leak check and parity at BASELINE sizes."""
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest

from canon import assert_planes_equal
from etl_b200 import workloads as wl
from shard_util import mid_tx_cuts, schema_maps, stitch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gpus():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


def _load_rank(path):
    z = np.load(path)
    m = z["meta"]
    fe = (None if m[2] < 0 else int(m[2]), int(m[3]), int(m[4]), int(m[5]))
    schemas = [SimpleNamespace(table_id=int(t), effective_off=int(o), n_identity=int(i)) for t, o, i in zip(z["schema_tables"], z["schema_offs"], z["schema_ident"])]
    return SimpleNamespace(n_records=int(m[0]), n_cells=int(m[1]), first_error=fe, carry_out=(int(m[6]), int(m[7]), int(m[8])),
                           insert_bytes=int(m[9]), update_bytes=int(m[10]), delete_bytes=int(m[11]), n_events=int(m[12]),
                           record_index_base=int(m[13]), schemas=schemas, **{k: z[k] for k in z.files if k not in ("meta", "schema_tables", "schema_offs", "schema_ident")})


@pytest.mark.parametrize("name,scale,world,exchange", [("c2", 0.02, 2, "host"), ("c4", 0.002, 3, "host"), ("c5", 0.004, 4, "host"),
                                                      ("c2", 0.02, 2, "nccl"), ("c4", 0.002, 2, "nccl"), ("c4", 0.004, 4, "nccl"), ("c5", 0.004, 8, "nccl")])
def test_sharded_decode_matches_oracle(oracle_mod, tmp_path, name, scale, world, exchange):
    """ONE stream cut into `world` byte ranges inside transactions.  c4: 64 tables whose Relation messages all sit in
    the first range, plus mid-stream schema bumps (replica identity flips) that later ranges must honour.
    exchange = "nccl": one process per GPU, the library's own communicator (needs `world` GPUs); "host": every rank
    on GPU 0 with the two exchanges carried by gloo (etl_dec_comm_init_host) — the whole protocol on a one-GPU box."""
    if _gpus() < (world if exchange == "nccl" else 1):
        pytest.skip(f"needs {world} GPUs")
    w = wl.make(name, scale, n_segments=1)
    if name == "c4":
        w.schema_bump_ppm = 3000
    stream, _ = w.generate()
    raw = stream.tobytes()
    orc = oracle_mod.Oracle()
    for tid, cols in w.table_schemas().items():
        orc.put_table_schema(tid, cols)
    full = orc.decode(raw)
    assert full.first_error[0] is None
    cuts = mid_tx_cuts(full, world) + [len(raw)]
    np.save(tmp_path / "cuts.npy", np.array(cuts, dtype=np.int64))
    env = dict(os.environ, ETL_TEST_BUMP="3000" if name == "c4" else "0", ETL_TEST_HOST_EXCHANGE="1" if exchange == "host" else "0")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", "29611", os.path.join(ROOT, "tests", "sharded_worker.py"), str(tmp_path), name, str(scale)]
    r = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=240)
    assert r.returncode == 0, r.stdout[-4000:]
    print(r.stdout[-3000:])
    parts = [_load_rank(tmp_path / f"rank{k}.npz") for k in range(world)]
    base = 0
    for k, p in enumerate(parts):
        assert p.first_error[0] is None, (k, p.first_error)
        assert p.record_index_base == base
        base += p.n_records
    assert base == full.n_records
    # schema numbering is per range (carried-in versions first): map every range's indices to the whole-stream numbering
    got = stitch(parts, cuts, schema_maps(full, parts, cuts))
    got.schemas = full.schemas                          # compared through the mapping above
    got.carry_out = parts[-1].carry_out
    assert_planes_equal(got, full, raw)
    assert all(p.carry_out == full.carry_out for p in parts)   # every rank reports the state after the LAST range


def test_context_create_decode_destroy_does_not_leak():
    """etl_dec_destroy releases every device buffer of the context (ADVICE r1: half of them used to stay)."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from etl_b200 import decoder
    w = wl.make("c3", 0.002, n_segments=1)
    stream, _ = w.generate()

    def once():
        dec = decoder.Decoder(0)
        for tid, cols in w.table_schemas().items():
            dec.put_table_schema(tid, cols)
        p = dec.decode(stream)
        assert p.first_error[0] is None
        free, _ = dec.mem_info()
        dec.close()
        return free

    for _ in range(3):
        once()
    torch.cuda.synchronize()
    first = once()
    for _ in range(100):
        last = once()
    assert first - last < (8 << 20), f"free device memory shrank by {first - last} bytes over 100 create/decode/destroy cycles"


@pytest.mark.parametrize("name,scale", [("c2", 1.0), ("c4", 0.1)])
def test_workload_parity_at_size(oracle_mod, name, scale):
    """BASELINE sizes (c2: 1M msgs; c4: 1M msgs over 64 tables with Relation re-sends and schema bumps) decoded as ONE
    batch, every plane compared with the oracle by canonical digest (oracle/oracle_digest.c)."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from etl_b200 import decoder
    w = wl.make(name, scale)
    stream, stats = w.generate()
    orc = oracle_mod.Oracle()
    dec = decoder.Decoder(0)
    for tid, cols in w.table_schemas().items():
        orc.put_table_schema(tid, cols)
        dec.put_table_schema(tid, cols)
    want, n_want, fe = orc.digest(stream)
    assert fe is None and n_want == stats["frames"]
    st = decoder.Stager(stream.nbytes, 2048)
    st.append_framed(stream)
    for _ in range(2):                                  # second pass takes the optimistic single-sync path
        dec.reset_relations()
        with dec.decode_input(st.view(), to_host=True) as bh:
            assert bh.summary().first_error.record_index == 2**64 - 1
            p = bh.planes(True)
            assert int(p.n_records) == n_want
            assert oracle_mod.planes_digest(p, int(p.n_records)) == want
    st.close()
    dec.close()
