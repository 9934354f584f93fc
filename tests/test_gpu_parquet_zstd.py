"""Zstandard pages of etl_dec_parquet_write / _bloom (ETL_PQ_ZSTD, csrc/parquet_write.cu, k_zstd) against the file
written UNCOMPRESSED with the same flags and against the host build of the same block compressor
(tests/emul/host_parquet_zstd.cpp).  Every input is written in ZSTD × {with, without ETL_PQ_DICTIONARY} × {with, without
ETL_PQ_PAGE_INDEX}, and with bloom filters on the key column, and checked: the pages line up 1:1 with the uncompressed
file's, every header field but compressed_page_size is equal, every payload decodes with pyarrow's zstd to the
uncompressed payload and equals the host encoder's frame byte for byte (so the structural and re-framing checks of
tests/test_parquet_zstd_cpu.py hold for it, and are repeated here); the footer equals the uncompressed file's but for
the sizes and offsets, with codec 6 and consistent offsets; the metrics equal the uncompressed file's but
the byte totals, which count this file's page headers (compressed_bytes: the chunk's page bytes); the ColumnIndex equals the Snappy file's, the OffsetIndex gives the
pages' positions and the bytes before the index are the file without the flag; the bloom filters equal the Snappy
file's; pyarrow reads the columns; repeated writes and to_host 0 / 1 give the same bytes; and ZSTD's page bytes are
below Snappy's.  Inputs: c1–c5 (every schema version), a 200 000-row COPY batch, a hand-built table of every leaf type,
an edge table, two row groups, row slices and zero rows; then the argument checks."""
import ctypes as C

import pytest

import parquet_bloom_ref as B
import parquet_index_ref as X
import scenarios as sc
from parquet_io import device_bytes, emit_columns, fields_for, file_bytes, metrics, pq_write, pq_write_bloom
from etl_b200 import abi, pgoutput as pg, workloads as wl
from test_gpu_arrow_copy import copy_batch
from test_gpu_copy import synth_rows
from test_gpu_parquet import ERR_INVALID_ARG, INT4, TEXT, _decode_stream, _emit, check_pyarrow
from test_gpu_rowbinary import hand_built
from test_parquet_zstd_cpu import CODEC, FRAG, _build, walk, zstd

pytestmark = pytest.mark.gpu

PIDX, DICT, ZSTD, SNAPPY = abi.PQ_PAGE_INDEX, abi.PQ_DICTIONARY, abi.PQ_ZSTD, abi.PQ_SNAPPY
FLOAT8, BYTEA, BOOL, INT4_ARR, TEXT_ARR = 701, 17, 16, 1007, 1009
FLAGS = [d | p for d in (0, DICT) for p in (0, PIDX)]
TOTALS = {"zstd": 0, "snappy": 0}


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from etl_b200 import decoder
    return decoder


@pytest.fixture(scope="module")
def host():
    lib = _build("libhost_parquet_zstd.so", "host_parquet_zstd.cpp")
    lib.emu_zstd.argtypes = [C.c_char_p, C.c_uint64, C.c_void_p]
    lib.emu_zstd.restype = C.c_uint64
    lib.emu_zstd_bound.argtypes = [C.c_uint64]
    lib.emu_zstd_bound.restype = C.c_uint64
    return lib


def _write(lib, a, fields, rb, re, codec, bloom=None, to_host=1):
    rc, h = pq_write_bloom(lib, a, fields, bloom, rb, re, codec, to_host)
    assert rc == 0, hex(codec)
    if to_host:
        data = file_bytes(lib, h)
    else:                                                # the device copy
        data = device_bytes(lib.etl_dec_parquet_bytes(h, 0), lib.etl_dec_parquet_size(h))
    m = metrics(lib, h, len(fields))
    lib.etl_dec_parquet_free(h)
    return data, m


def pages(data):
    """every page in file order: (chunk, parsed header, header bytes, payload), dictionary pages included"""
    fm, _, _ = X.file_footer(data)
    out, ci = [], 0
    for rg in fm.get(4, []):
        for cc in rg[1]:
            md = cc[3]
            pos = md.get(11, md[9])
            end = pos + md[7]
            while pos < end:
                h, p2 = X.read_struct(data, pos)
                out.append((ci, h, bytes(data[pos:p2]), bytes(data[p2:p2 + h[3]]), pos))
                pos = p2 + h[3]
            assert pos == end
            ci += 1
    return out


def _masked(fm):
    fm = dict(fm)
    rgs = []
    for rg in fm.get(4, []):
        rg = {k: v for k, v in rg.items() if k not in (2, 5, 6)}   # byte totals count the page headers, whose
        rg[1] = [{k: ({f: x for f, x in v.items() if f not in (4, 6, 7, 9, 11, 14)} if k == 3 else v)   # varints vary
                  for k, v in cc.items() if k not in (2, 4, 5, 6)} for cc in rg[1]]
        rgs.append(rg)
    fm[4] = rgs
    return fm


def check_frame(host, payload, frame):
    assert CODEC.decompress(frame, decompressed_size=len(payload)).to_pybytes() == payload
    assert frame == zstd(host, payload)
    blocks = walk(frame, len(payload))
    if len(blocks) > 1:
        for k, (_, blk, _, _) in enumerate(blocks):
            frag = payload[k * FRAG:(k + 1) * FRAG]
            h = int.from_bytes(blk[:3], "little") | 1
            alone = b"\x28\xb5\x2f\xfd\xa0" + len(frag).to_bytes(4, "little") + h.to_bytes(3, "little") + blk[3:]
            assert CODEC.decompress(alone, decompressed_size=len(frag)).to_pybytes() == frag


def check_zstd(lib, host, a, cols, fields, rb, re, what, flags=FLAGS, pyarrow=True, key=0):
    for fl in flags:
        w = f"{what} flags {fl:#x}"
        got, got_m = _write(lib, a, fields, rb, re, ZSTD | fl)
        base, base_m = _write(lib, a, fields, rb, re, abi.PQ_UNCOMPRESSED | fl)
        snap, _ = _write(lib, a, fields, rb, re, SNAPPY | fl)
        gp, bp = pages(got), pages(base)
        assert len(gp) == len(bp), w
        for (gc, gh, _, gpl, _), (bc, bh, _, bpl, _) in zip(gp, bp):
            assert gc == bc and {k: v for k, v in gh.items() if k != 3} == {k: v for k, v in bh.items() if k != 3}, w
            assert gh[3] == len(gpl)
            check_frame(host, bpl, gpl)
        gfm, bfm = X.file_footer(got)[0], X.file_footer(base)[0]
        assert _masked(gfm) == _masked(bfm), w
        csize, usize = {}, {}
        ci = 0
        for rg in gfm.get(4, []):
            for li, cc in enumerate(rg[1]):
                md = cc[3]
                assert md[4] == 6 and cc[2] == md.get(11, md[9]), w
                chunk_pages = [p for p in gp if p[0] == ci]
                assert md[7] == sum(len(p[2]) + len(p[3]) for p in chunk_pages) and chunk_pages[0][4] == md.get(11, md[9]), w
                assert md[6] == sum(len(p[2]) + p[1][2] for p in chunk_pages), w   # headers + uncompressed payloads
                csize[li] = csize.get(li, 0) + md[7]
                usize[li] = usize.get(li, 0) + md[6]
                ci += 1
            assert rg[2] == sum(cc[3][6] for cc in rg[1]) and rg[6] == sum(cc[3][7] for cc in rg[1]), w
        sizes = ("compressed_bytes", "uncompressed_bytes")
        for li, (gm, bm) in enumerate(zip(got_m, base_m)):
            assert {k: v for k, v in gm.items() if k not in sizes} == {k: v for k, v in bm.items() if k not in sizes}, w
            assert gm["compressed_bytes"] == csize.get(li, 0) and gm["uncompressed_bytes"] == usize.get(li, 0), w
        if fl & PIDX and rb != re:
            plain, _ = _write(lib, a, fields, rb, re, ZSTD | (fl & ~PIDX))
            end = B.data_end(got)
            assert got[:end] == plain[:end], w
            gi, si = X.read_indexes(got), X.read_indexes(snap)
            assert [c for c, _ in gi] == [c for c, _ in si], w
            for ci, (_, oi) in enumerate(gi):
                locs = [p for p in gp if p[0] == ci and p[1][1] == 0]
                assert [(e[1], e[2]) for e in oi[1]] == [(p[4], len(p[2]) + len(p[3])) for p in locs], w
        if rb != re:
            bloom = [(0.01, 0, 0) if i == key else (0.0, 0, 0) for i in range(len(fields))]
            gb, _ = _write(lib, a, fields, rb, re, ZSTD | fl, bloom)
            sb, _ = _write(lib, a, fields, rb, re, SNAPPY | fl, bloom)
            assert [f and (f[2], f[4]) for f in B.read_filters(gb)] == [f and (f[2], f[4]) for f in B.read_filters(sb)], w
            assert gb[:B.data_end(gb)] == got[:B.data_end(got)], w
        if fl == flags[0]:
            assert _write(lib, a, fields, rb, re, ZSTD | fl)[0] == got, f"{w}: a second write differs"
            assert _write(lib, a, fields, rb, re, ZSTD | fl, to_host=0)[0] == got, f"{w}: to_host 0 differs"
            TOTALS["zstd"] += sum(len(p[3]) for p in gp)
            TOTALS["snappy"] += sum(len(p[3]) for p in pages(snap))
            if pyarrow and rb != re:
                check_pyarrow(got, cols, fields, rb, re)


def run_stream(gpu, host, tables, raw, what, required=()):
    lib = abi.load()
    dec, st = _decode_stream(gpu, tables, raw)
    n_total = 0
    with dec.decode_input(st.view(), to_host=True) as bh:
        for si in range(len(bh.schemas())):
            a = _emit(lib, bh, si)
            cols = emit_columns(lib, a)
            n = lib.etl_dec_arrow_rows(a)
            fields = fields_for(cols, required)
            check_zstd(lib, host, a, cols, fields, 0, n, f"{what} v{si}")
            if n > 2:
                check_zstd(lib, host, a, cols, fields, n // 3, n - n // 4, f"{what} v{si} slice", flags=FLAGS[::3])
                check_zstd(lib, host, a, cols, fields, n // 2, n // 2, f"{what} v{si} empty", flags=FLAGS[:1])
            n_total += n
            lib.etl_dec_arrow_free(a)
    st.close()
    dec.close()
    return n_total


@pytest.mark.parametrize("name,scale", [("c1", 0.01), ("c2", 0.0005), ("c3", 0.001), ("c4", 0.002), ("c5", 0.0005)])
def test_workloads(gpu, host, name, scale):
    w = wl.make(name, scale, n_segments=1)
    stream, _ = w.generate()
    TOTALS["zstd"] = TOTALS["snappy"] = 0
    assert run_stream(gpu, host, w.table_schemas(), stream.tobytes(), name) > 0
    print(f"{name}: page bytes Snappy {TOTALS['snappy']}, ZSTD {TOTALS['zstd']}")
    assert TOTALS["zstd"] < TOTALS["snappy"]


def test_hand_built_every_type(gpu, host, oracle_mod):
    cols, row, n_rows = hand_built(oracle_mod)
    rel = pg.relation(95, "public", "pq", "f", sc.rel_cols(cols, set()))
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(rel)
    for r in range(n_rows):
        w.emit(pg.insert(95, row(r)))
        if r % 3 == 1:
            w.emit(pg.update(95, row(r + 1), old=row(r)))
    tx.commit()
    assert run_stream(gpu, host, {95: cols}, w.bytes(), "hand-built", required=(0,)) > 0


def _copy_check(gpu, host, oids, rows, what, required=(), slices=(), flags=FLAGS, pyarrow=True):
    lib = abi.load()
    dec = gpu.Decoder(0)
    dec.put_table_schema(7, [dict(name=f"c{i}", type_oid=o, pk=1 if i == 0 else None, nullable=True) for i, o in enumerate(oids)])
    with copy_batch(gpu, dec, 7, rows) as bh:
        a = _emit(lib, bh, 0)
        cols = emit_columns(lib, a)
        n = lib.etl_dec_arrow_rows(a)
        fields = fields_for(cols, required)
        check_zstd(lib, host, a, cols, fields, 0, n, what, flags, pyarrow)
        for rb, re in slices:
            check_zstd(lib, host, a, cols, fields, rb, re, f"{what} [{rb}, {re})", flags[::3], pyarrow)
        lib.etl_dec_arrow_free(a)
    dec.close()


def test_copy_batch_200k(gpu, host):
    oids, rows = synth_rows(200000, 41)
    TOTALS["zstd"] = TOTALS["snappy"] = 0
    _copy_check(gpu, host, oids, rows, "copy 200k", required=(0,), slices=[(19999, 20001), (5, 150000), (7, 7)])
    print(f"copy 200k: page bytes Snappy {TOTALS['snappy']}, ZSTD {TOTALS['zstd']}")
    assert TOTALS["zstd"] < TOTALS["snappy"]


def test_edges(gpu, host):
    """−0.0 / NaN, empty, short and long text and bytea, null and empty lists, an all-null column, a Boolean column"""
    n = 30000
    rows = []
    for r in range(n):
        k = r % 7
        text = "\\N" if r % 13 == 0 else "" if k == 0 else "t" if k == 1 else ("é%d" % r) * (300 if k == 2 else 3)
        byt = "\\\\x" + ("" if k == 0 else "%02x" % (r % 256) * (1100 if k == 1 else 5))
        fl = ("NaN", "0", "-0", "-%d.5" % r, "%d.25" % (r % 500))[r % 5]
        ints = "\\N" if r % 17 == 0 else "{}" if r % 19 == 0 else "{%s}" % ",".join("NULL" if (r + j) % 11 == 0 else str(r - j) for j in range(r % 5))
        texts = "{%s}" % ",".join('"%s"' % ("w" * (j * 40) + str(r)) if (r + j) % 3 else "NULL" for j in range(r % 3))
        rows.append(("%d\t%s\t%s\t%s\t\\N\t%s\t%s\t%s\n" % (r, text, byt, fl, "t" if r % 2 else "f", ints, texts)).encode())
    _copy_check(gpu, host, [INT4, TEXT, BYTEA, FLOAT8, INT4, BOOL, INT4_ARR, TEXT_ARR], rows, "edges", required=(0,),
                slices=[(19990, 20010), (1, 2)])


def test_two_row_groups(gpu, host):
    n = (1 << 20) + 4321
    rows = [b"%d\tv%d\n" % (i * 7 - 5, i % 1000) if i % 17 else b"\\N\t\\N\n" for i in range(n)]
    _copy_check(gpu, host, [INT4, TEXT], rows, "two row groups", slices=[((1 << 20) - 3, (1 << 20) + 3)],
                flags=[0, DICT | PIDX], pyarrow=False)


def test_arguments(gpu):
    lib = abi.load()
    dec = gpu.Decoder(0)
    dec.put_table_schema(7, [dict(name="c0", type_oid=INT4, pk=None, nullable=True), dict(name="c1", type_oid=TEXT, pk=None, nullable=True)])
    rows = [b"%d\tt%d\n" % (i % 4, i % 3) for i in range(1000)]
    with copy_batch(gpu, dec, 7, rows) as bh:
        a = _emit(lib, bh, 0)
        fields = fields_for(emit_columns(lib, a))
        for fl in FLAGS:
            rc, h = pq_write(lib, a, fields, 0, 1000, ZSTD | fl)
            assert rc == 0 and lib.etl_dec_parquet_size(h) > 0
            lib.etl_dec_parquet_free(h)
        for bad in (2, 3, 4, 5, 7, 8, 0xFF, ZSTD | 0x200):
            assert pq_write(lib, a, fields, 0, 1000, bad)[0] == ERR_INVALID_ARG, bad
        lib.etl_dec_arrow_free(a)
    dec.close()
