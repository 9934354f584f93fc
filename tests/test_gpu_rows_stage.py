"""k_rows writes each lane's output cells into a per-warp stage in shared memory and flushes them to the cell planes as
runs of consecutive cells (a run holds 4 cells; a flush also happens at the end of an old image and of the walk).
These streams put the run edges where they matter, each checked plane for plane against the oracle:

  - tables wider than two runs (inserts, full old images, deletes);
  - a data error in the middle of a run (the failing record's cells past the error stay unwritten);
  - unchanged-TOAST cells whose source in the old image was flushed a run or more earlier, light and pending ones;
  - key-only old images, dense and full width, with more identity columns than one run holds;
  - shape bins whose last warp has padding lanes next to live ones.
"""
import pytest

import scenarios as sc
from canon import assert_planes_equal
from etl_b200 import pgoutput as pg
from etl_b200.pgoutput import UNCHANGED

pytestmark = pytest.mark.gpu

STAGE = 4                                         # cells per lane in one run of the stage (rows_kernel.cuh)
KINDS = [sc.INT8, sc.TEXT, sc.INT4, sc.BOOL, sc.DATE, sc.TEXT, sc.NUMERIC, sc.TIMESTAMPTZ, sc.FLOAT8, sc.TEXT, sc.JSONB, sc.UUID]


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from etl_b200 import decoder
    return decoder


def wide_cols(n, identity=()):
    """n columns cycling through light and pending kinds; the identity columns are NOT NULL, the others nullable."""
    return [sc.col(f"c{i}", KINDS[i % len(KINDS)], pk=(identity.index(i) + 1) if i in identity else None,
                   nullable=i not in identity) for i in range(n)]


def value(oid, rec, i):
    if oid == sc.INT8:
        return str(rec * 1000003 + i)
    if oid == sc.INT4:
        return str((rec * 31 + i) % 100000 - 5000)
    if oid == sc.BOOL:
        return "t" if (rec + i) & 1 else "f"
    if oid == sc.DATE:
        return f"20{10 + rec % 20}-0{1 + i % 9}-1{rec % 10}"
    if oid == sc.NUMERIC:
        return f"{rec}.{i:02d}"
    if oid == sc.TIMESTAMPTZ:
        return f"2024-03-1{rec % 10} 12:{i % 60:02d}:0{rec % 10}.25+00"
    if oid == sc.FLOAT8:
        return f"{rec}.5e{i % 7}"
    if oid == sc.JSONB:
        return '{"r": %d, "c": [%d, "x"]}' % (rec, i)
    if oid == sc.UUID:
        return "%08x-0000-4000-8000-%012x" % (rec, i)
    return "v%d_%d_" % (rec, i) + "x" * ((rec * 7 + i * 3) % 40)


def row(cols, rec, nulls=()):
    return [None if i in nulls else value(c["type_oid"], rec, i) for i, c in enumerate(cols)]


def decode_both(gpu, oracle_mod, tables, stream):
    dec = gpu.Decoder(0)
    orc = oracle_mod.Oracle()
    for tid, cols in tables.items():
        dec.put_table_schema(tid, cols)
        orc.put_table_schema(tid, cols)
    got = dec.decode(stream)
    want = orc.decode(stream)
    dec.close()
    orc.close()
    return got, want


@pytest.mark.parametrize("n_cols", [2 * STAGE + 1, 3 * STAGE, 41])
@pytest.mark.parametrize("n_rec", [33, 70])
def test_wide_full_old_image(gpu, oracle_mod, n_cols, n_rec):
    """Inserts, updates with a full old image and unchanged-TOAST cells at and around the run edges, deletes with a full
    old image; the record counts leave padding lanes in each bin's last warp."""
    cols = wide_cols(n_cols)
    rel = pg.relation(70, "public", "wide", "f", sc.rel_cols(cols, set()))
    toast = {STAGE - 1, STAGE, 2 * STAGE - 1, 2 * STAGE, n_cols - 1, 6, 10}   # 6 / 10: numeric / jsonb (pending sources)
    msgs = []
    for r in range(n_rec):
        msgs.append(pg.insert(70, row(cols, r, nulls={(r + 3) % n_cols} - {0})))
    for r in range(n_rec):
        new = row(cols, r + 5000)
        for i in toast:
            if (r + i) % 3 and i < n_cols:
                new[i] = UNCHANGED
        msgs.append(pg.update(70, new, old=row(cols, r, nulls={(r + 5) % n_cols} - {0})))
    for r in range(n_rec):
        msgs.append(pg.delete(70, old=row(cols, r + 9000)))
    stream = sc.stream_with(None, [rel], msgs).bytes()
    got, want = decode_both(gpu, oracle_mod, {70: cols}, stream)
    assert want.first_error[0] is None
    assert_planes_equal(got, want, stream)


@pytest.mark.parametrize("bad_col", [2, STAGE + 3, 2 * STAGE + 2])
def test_data_error_inside_a_run(gpu, oracle_mod, bad_col):
    """One record of a full warp fails at a cell in the middle of a run (a NOT NULL violation, or an integer that does
    not parse); the records before it, in the same warps, keep their cells."""
    cols = wide_cols(3 * STAGE)
    cols[bad_col] = dict(cols[bad_col], nullable=False)
    rel = pg.relation(71, "public", "wide", "f", sc.rel_cols(cols, set()))
    msgs = [pg.insert(71, row(cols, r)) for r in range(45)]
    bad = row(cols, 45)
    bad[bad_col] = None if cols[bad_col]["type_oid"] not in (sc.INT8, sc.INT4) else "12x"
    msgs.append(pg.insert(71, bad))
    msgs += [pg.insert(71, row(cols, r)) for r in range(46, 80)]
    msgs += [pg.update(71, row(cols, r + 100), old=row(cols, r)) for r in range(40)]
    stream = sc.stream_with(None, [rel], msgs).bytes()
    got, want = decode_both(gpu, oracle_mod, {71: cols}, stream)
    assert want.first_error[0] == 2 + 45
    assert_planes_equal(got, want, stream)


@pytest.mark.parametrize("dense", [True, False], ids=["dense_key", "full_width_key"])
def test_key_only_old_image(gpu, oracle_mod, dense):
    """Updates and deletes with a key-only old image: 11 identity columns (more than one run) spread over 30 columns;
    the new tuples leave identity columns unchanged, so their values come from the key image flushed before."""
    ident = (0, 1, 3, 7, 8, 9, 14, 15, 16, 22, 29)
    cols = wide_cols(30, ident)
    rel = pg.relation(72, "public", "keyed", "d", sc.rel_cols(cols, {cols[i]["name"] for i in ident}))

    def key(rec):
        full = row(cols, rec)
        return [full[i] for i in ident] if dense else [full[i] if i in ident else None for i in range(len(cols))]

    msgs = []
    for r in range(50):
        new = row(cols, r + 700)
        for i in ident:
            if (r + i) % 2:
                new[i] = UNCHANGED
        msgs.append(pg.update(72, new, key=key(r)))
    msgs += [pg.delete(72, key=key(r + 50)) for r in range(37)]
    msgs += [pg.insert(72, row(cols, r + 2000)) for r in range(20)]
    stream = sc.stream_with(None, [rel], msgs).bytes()
    got, want = decode_both(gpu, oracle_mod, {72: cols}, stream)
    assert want.first_error[0] is None
    assert_planes_equal(got, want, stream)


def test_padding_lanes_in_mixed_bins(gpu, oracle_mod):
    """Several tables and shapes with a few records each, interleaved: every bin's only warp is mostly padding lanes."""
    tables, rels, msgs = {}, [], []
    for t in range(6):
        cols = wide_cols(STAGE * (t % 3) + 5 + t)
        tables[80 + t] = cols
        rels.append(pg.relation(80 + t, "public", f"t{t}", "f", sc.rel_cols(cols, set())))
    for r in range(40):
        tid = 80 + r % 6
        cols = tables[tid]
        if r % 3 == 0:
            msgs.append(pg.insert(tid, row(cols, r)))
        elif r % 3 == 1:
            new = row(cols, r + 1)
            new[-1] = UNCHANGED
            msgs.append(pg.update(tid, new, old=row(cols, r)))
        else:
            msgs.append(pg.delete(tid, old=row(cols, r)))
    stream = sc.stream_with(None, rels, msgs).bytes()
    got, want = decode_both(gpu, oracle_mod, tables, stream)
    assert want.first_error[0] is None
    assert_planes_equal(got, want, stream)
