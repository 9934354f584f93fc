"""Shape bins per tile of consecutive records (k_records counts per (tile, bin), k_bin_scan lays the bins out tile after
tile, k_perm fills them and writes the warp padding, k_rows walks the order): batches whose record counts straddle tile
edges, shapes that occur in one tile only, clamped bins across several tiles, the sizing reruns (which recompute the
tiles) and two-phase shards, each checked against the oracle.

A tile holds max(16 Ki, 1024 · n_bins) records and n_bins = min(4096, 16 · column layouts): a one-table stream has 16 Ki
records per tile.  Records are frames, Begin and Commit included, so the batches below are cut by frame count.
"""
import numpy as np
import pytest

import scenarios as sc
from canon import assert_planes_equal
from etl_b200 import pgoutput as pg
from etl_b200 import workloads as wl
from seq_util import SIZING, Decode, run_sequence, sizing_names
from shard_util import mid_tx_cuts, stitch
from test_gpu_batch_sequence import HIST_COLS, HIST_TABLE, history_batch, oracle_of, reservations
from test_gpu_parity import _two_phase

pytestmark = pytest.mark.gpu

TILE = 16384                                      # records per tile of a batch with one column layout


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from etl_b200 import decoder
    return decoder


@pytest.fixture(scope="module")
def c2_stream(oracle_mod):
    w = wl.make("c2", 0.07, n_segments=1)
    raw = w.generate()[0].tobytes()
    full = oracle_of(oracle_mod, w.table_schemas(), raw)
    assert full.n_records > 65537
    return w.table_schemas(), raw, full


def decode_both(gpu, oracle_mod, tables, stream):
    dec = gpu.Decoder(0)
    for tid, cols in tables.items():
        dec.put_table_schema(tid, cols)
    got = dec.decode(stream)
    dec.close()
    return got, oracle_of(oracle_mod, tables, stream)


@pytest.mark.parametrize("n_records", [16383, 16384, 16385, 32767, 32769, 65537])
def test_record_counts_around_tile_edges(gpu, oracle_mod, c2_stream, n_records):
    """c2 cut after exactly n_records frames (mid-transaction): the last tile is one record short of full, full, or
    holds a single record."""
    tables, raw, full = c2_stream
    stream = raw[:int(full.rec_off[n_records])]
    got, want = decode_both(gpu, oracle_mod, tables, stream)
    assert want.n_records == n_records and want.first_error[0] is None
    assert_planes_equal(got, want, stream)


def test_shape_once_per_tile_and_only_in_last_tile(gpu, oracle_mod):
    """Inserts fill the tiles; an update with a key image (a shape bin of its own) is the only one of its shape in every
    tile, deletes with a full old image occur only in the last tile: one-record bins, each padded by 31 lanes."""
    cols = [sc.col("id", sc.INT8, 1), sc.col("n", sc.INT4, None, True), sc.col("t", sc.TEXT, None, True)]
    tables = {70: cols}
    rng = np.random.default_rng(70)
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(pg.relation(70, "public", "d", "d", sc.rel_cols(cols, {"id"})))
    tx.commit()
    keyed = []
    i = 0
    while len(w.chunks) < 3 * TILE + 5000:
        tx.begin()
        for _ in range(int(rng.integers(1, 60))):
            t = rng.integers(97, 123, size=int(rng.integers(0, 40)), dtype=np.uint8).tobytes()
            if len(w.chunks) // TILE == len(keyed):
                keyed.append(len(w.chunks))
                w.emit(pg.update(70, [str(i), str(i % 1000), t], key=[str(i - 1), None, None]))
            else:
                w.emit(pg.insert(70, [str(i), None if i % 7 == 0 else str(i % 1000), t]))
            i += 1
        tx.commit()
    tx.begin()
    last = [w.emit(pg.delete(70, old=[str(j), str(j), b"gone"])) for j in range(3)]
    tx.commit()
    stream = w.bytes()
    got, want = decode_both(gpu, oracle_mod, tables, stream)
    assert want.first_error[0] is None
    assert [r // TILE for r in keyed] == list(range(4))
    first_delete = int(np.searchsorted(np.asarray(want.rec_off[:want.n_records]), last[0]))
    assert first_delete // TILE == (want.n_records - 1) // TILE == 3
    assert_planes_equal(got, want, stream)


def test_clamped_bins_across_tiles(gpu, oracle_mod):
    """300 tables with 300 column layouts: more layouts than the 256 the bins can tell apart, so n_bins = 4096, the
    last 16 bins hold warps of mixed shapes, and a tile holds 4 Mi records.  4.5 M messages span two tiles; every
    plane is compared by canonical digest."""
    tables = []
    for k in range(300):
        cols = [wl.ColSpec("id", "int8", wl.SEQ_INT8, False, 1)]
        cols += [wl.ColSpec(f"c{j}", "int2", wl.INT2G, True) if (k >> j) & 1 else wl.ColSpec(f"c{j}", "bool", wl.BOOLG, True)
                 for j in range(9)]
        tables.append(wl.TableSpec(20000 + k, f"t{k}", "f" if k % 3 == 0 else "d", cols))
    w = wl.Workload("clamp", tables, 0xB1A5, msgs_per_segment=4_500_000 // 8, n_segments=8, mix=(5000, 3500, 1500),
                    pct_key_change=1000, tx_mean=20, null_pct=500)
    stream, stats = w.generate()
    assert stats["frames"] > 1024 * 4096
    orc = oracle_mod.Oracle()
    dec = gpu.Decoder(0)
    for tid, cols in w.table_schemas().items():
        orc.put_table_schema(tid, cols)
        dec.put_table_schema(tid, cols)
    want, n_want, fe = orc.digest(stream)
    orc.close()
    assert fe is None and n_want == stats["frames"]
    st = gpu.Stager(stream.nbytes, 2048)
    st.append_framed(stream)
    try:
        with dec.decode_input(st.view(), to_host=True) as bh:
            assert bh.summary().first_error.record_index == 2**64 - 1
            p = bh.planes(True)
            assert int(p.n_records) == n_want
            assert oracle_mod.planes_digest(p, n_want) == want
    finally:
        st.close()
        dec.close()


def test_rerun_records_multi_tile(gpu, oracle_mod):
    """After the sparse history batch, 8 MiB of c2 (several tiles) overflows the record reservation: pass C runs again
    with exact sizes, and with tiles recomputed for the larger record plane."""
    hist = history_batch()
    hp = oracle_of(oracle_mod, {HIST_TABLE: HIST_COLS}, hist)
    w = wl.make("c2", 0.08, n_segments=1)
    raw = w.generate()[0].tobytes()
    tables = {HIST_TABLE: HIST_COLS, **w.table_schemas()}
    full = oracle_of(oracle_mod, tables, raw)
    end = int(full.rec_off[np.searchsorted(full.rec_off[:full.n_records], 8 << 20)])
    n_rec = int(np.searchsorted(full.rec_off[:full.n_records], end))
    cap_r, _, cap_scratch = reservations(hp.n_records, hp.n_cells, len(hist), end)
    assert cap_r < TILE < 2 * TILE < n_rec < cap_scratch, (cap_r, n_rec, cap_scratch)
    res = run_sequence(gpu, oracle_mod, [Decode(hist, label="hist"), Decode(raw[:end], label="c2 8 MiB"),
                                         Decode(raw[end:], label="c2 rest")], tables)
    assert res.sizing[1] & SIZING["RERUN_RECORDS"] and res.sizing[1] & SIZING["OPTIMISTIC"], sizing_names(res.sizing[1])
    assert not res.sizing[1] & SIZING["SCRATCH_RESTART"]


def test_rerun_cells_multi_tile(gpu, oracle_mod):
    """A history of keepalives (many records, almost no cells per byte), then 8 MiB of c2: its records fit the record
    reservation and span several tiles, its cells do not fit, so only the cell plane is resized and pass C runs
    again."""
    hist = history_batch() + pg.frame(pg.keepalive(0, 0, 0)) * 100_000
    hp = oracle_of(oracle_mod, {HIST_TABLE: HIST_COLS}, hist)
    w = wl.make("c2", 0.08, n_segments=1)
    raw = w.generate()[0].tobytes()
    tables = {HIST_TABLE: HIST_COLS, **w.table_schemas()}
    full = oracle_of(oracle_mod, tables, raw)
    end = int(full.rec_off[np.searchsorted(full.rec_off[:full.n_records], 8 << 20)])
    n_rec = int(np.searchsorted(full.rec_off[:full.n_records], end))
    cap_r, cap_c, _ = reservations(hp.n_records, hp.n_cells, len(hist), end)
    assert 2 * TILE < n_rec < cap_r and int(full.rec_cell_base[n_rec]) > cap_c, (n_rec, cap_r, cap_c)
    res = run_sequence(gpu, oracle_mod, [Decode(hist, label="keepalives"), Decode(raw[:end], label="c2 8 MiB"),
                                         Decode(raw[end:], label="c2 rest")], tables)
    s = res.sizing[1]
    assert s & SIZING["RERUN_CELLS"] and not s & SIZING["RERUN_RECORDS"], sizing_names(s)


def test_two_phase_shards_multi_tile(gpu, oracle_mod):
    """decode_begin / decode_finish over three mid-transaction ranges of ~80 k records each (five tiles per range):
    stitched, every plane equals the oracle's decode of the whole stream."""
    w = wl.make("c2", 0.22, n_segments=1)
    raw = w.generate()[0].tobytes()
    full = oracle_of(oracle_mod, w.table_schemas(), raw)
    cuts = mid_tx_cuts(full, 3) + [len(raw)]
    parts, base = _two_phase(gpu, w.table_schemas(), raw, cuts)
    assert base == full.n_records
    assert all(p.first_error[0] is None and p.n_records > 4 * TILE for p in parts)
    assert_planes_equal(stitch(parts, cuts), full, raw)
