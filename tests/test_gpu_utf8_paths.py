"""Every path that answers "is this cell valid UTF-8" (core::str::from_utf8, event.rs:972) on the device, against Python's
strict decoder and the oracle:

* long text at anchor strides 256 to 32768: the cell starts 0-5 bytes before a segment boundary, ends on one or 1-3 bytes
  after one, covers 0, 1 or 2 whole segments (one segment of several 2 KiB dead-pass items above 2048); invalid and
  near-miss sequences at the cell ends, around S0 and S1 (the first and last byte k_long_cells takes from the line
  bitmap), at the 64-byte lane and 128-byte line edges of the first dead item and at every 2 KiB item edge;
* long Json, text[], bytea and int4 cells, whose interior is judged by the bitmap alone: the verdict is UTF-8 (code 1) at
  that (record, seq), never the kind's own parse error;
* text and Json cells at the lengths where k_rows changes strategy (the window, kWideLen, kCoopLen);
* COPY rows of 1 to 5000 bytes;
* which error wins: a long cell's UTF-8 error against a short cell's parse error, the old and the new image of one update,
  two long cells megabytes apart; a wrong max_frame_len hint (the long passes run late); one decoder across batches.

A poisoned case must report (that record, that cell's seq, 1) exactly when Python rejects the cell's bytes; a clean case
must report nothing.  The valid near-miss cases of one stride share one stream."""
import os
import re

import numpy as np
import pytest

import scenarios as sc
from canon import assert_planes_equal
from etl_b200 import abi
from etl_b200 import pgoutput as pg
from test_gpu_copy import INT4, TEXT
from test_gpu_copy_edges import check_rows

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "etl_b200", "csrc")


def _const(fname, pattern):
    with open(os.path.join(CSRC, fname)) as f:
        return int(re.search(pattern, f.read()).group(1))


K_COOP = _const("wal_kernels.cuh", r"constexpr int kCoopLen = (\d+);")
K_WIDE = _const("wal_kernels.cuh", r"constexpr int kWideLen = (\d+);")
K_MAX_IN_WIN = _const("rows_kernel.cuh", r"#define ETL_TUPLE_WIN (\d+)") - _const("rows_kernel.cuh", r"kRowsMaxInWin = kRowsWin - (\d+);")
DEAD_ITEM = 2048                               # bytes of one dead-segment pass item (k_utf8_dead)
E_UTF8 = 1


def new_seq(col):
    """first_error.seq of column `col` of the new image (old-image cells come first: 0x10001 + col)"""
    return 0x20001 + col


def old_seq(col):
    return 0x10001 + col

REDUCED = [b"\xff", b"\x80", b"\xf0\x9f\x98", b"\xed\xa0\x80", b"\xf4\x90\x80\x80"]
FULL = [b"\x80", b"\xbf", b"\xc0\x80", b"\xc1\xbf", b"\xe0\x80\x80", b"\xe0\x9f\xbf", b"\xed\xa0\x80", b"\xed\xbf\xbf",
        b"\xf0\x80\x80\x80", b"\xf0\x8f\xbf\xbf", b"\xf4\x90\x80\x80", b"\xf5\x80\x80\x80", b"\xf8", b"\xfe", b"\xff",
        b"\xc2", b"\xe2\x82", b"\xf0\x9f\x98", b"\xc2\x80\x80"]
NEAR_OK = [b"\xc2\x80", b"\xdf\xbf", b"\xe0\xa0\x80", b"\xed\x9f\xbf", b"\xee\x80\x80", b"\xf0\x90\x80\x80", b"\xf4\x8f\xbf\xbf",
           b"\xef\xbf\xbf"]

REL_TEXT = 97
TEXT_COLS = [sc.col("id", sc.INT8, 1), sc.col("doc", sc.TEXT, None, True), sc.col("n", sc.INT4, None, True)]
REL_KINDS = 98
KIND_COLS = [sc.col("id", sc.INT8, 1), sc.col("js", sc.JSONB, None, True), sc.col("arr", 1009, None, True),
             sc.col("by", sc.BYTEA, None, True), sc.col("n", sc.INT4, None, True), sc.col("doc", sc.TEXT, None, True)]
TABLES = {REL_TEXT: TEXT_COLS, REL_KINDS: KIND_COLS}


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from etl_b200 import decoder
    return decoder


def strict_ok(b: bytes) -> bool:
    try:
        b.decode("utf-8")
        return True
    except UnicodeDecodeError:
        return False


def ascii_fill(n, seed):
    rng = np.random.default_rng(seed)
    return bytearray(rng.integers(97, 123, size=n, dtype=np.uint8).tobytes())


def _value_offset(cells, col):
    """offset of cells[col]'s value inside an insert message body"""
    o = 1 + 4 + 1 + 2
    for c in cells[:col]:
        o += 1 if c is None else 5 + len(c)
    return o + 5


class Layout:
    """One transaction of inserts; put() can first emit a filler insert so that a chosen cell starts at a chosen offset
    modulo the anchor stride."""

    def __init__(self):
        self.w = pg.StreamWriter()
        self.tx = sc.Tx(self.w)
        self.tx.begin()
        self.w.emit(pg.relation(REL_TEXT, "public", "u8text", "d", sc.rel_cols(TEXT_COLS, {"id"})))
        self.w.emit(pg.relation(REL_KINDS, "public", "u8kinds", "d", sc.rel_cols(KIND_COLS, {"id"})))
        self.n = 3

    def _filler(self, rel, n):
        return pg.insert(rel, ["0", b"f" * n, None] if rel == REL_TEXT else ["0", None, None, None, None, b"f" * n])

    def put(self, rel, cells, col, stride=None, start=None, update_old=None):
        """insert `cells` (or an update with old image `update_old`); returns (record, stream offset of cells[col])"""
        body = pg.insert(rel, cells) if update_old is None else pg.update(rel, cells, old=update_old)
        voff = _value_offset(cells, col) if update_old is None else None
        if stride is not None:
            base = self.w.size + 30 + len(self._filler(rel, 0)) + 30 + voff
            self.w.emit(self._filler(rel, (start - base) % stride))
            self.n += 1
        off = self.w.emit(body)
        self.n += 1
        return self.n - 1, (off + 30 + voff if voff is not None else None)

    def bytes(self):
        self.tx.commit()
        return self.w.bytes()


def text_cells(payload):
    return ["1", payload, "7"]


class Runner:
    """one Decoder per stride, paired with one Oracle that sees the same batches (the Relation messages of every batch
    move both to a new schema version); every decode compared with the oracle's"""

    def __init__(self, gpu, oracle_mod):
        self.gpu, self.orc_mod, self.ctx, self.n = gpu, oracle_mod, {}, 0

    def pair(self, stride):
        if stride not in self.ctx:
            d, o = self.gpu.Decoder(0), self.orc_mod.Oracle()
            for tid, cols in TABLES.items():
                d.put_table_schema(tid, cols)
                o.put_table_schema(tid, cols)
            self.ctx[stride] = (d, o)
        return self.ctx[stride]

    def run(self, stream, stride, hint=None, what=None, planes=False, ctx=None):
        self.n += 1
        dec, orc = self.pair(stride if ctx is None else ctx)
        got = dec.decode(stream, anchor_stride=stride, max_frame_len=hint)
        want = orc.decode(stream)
        assert got.first_error == want.first_error, (what, got.first_error, want.first_error)
        if planes:
            assert_planes_equal(got, want, stream)
        return got, want

    def poisoned(self, stream, stride, rec, seq, cell, what, hint=None):
        got, want = self.run(stream, stride, hint, what)
        if strict_ok(cell):
            assert want.first_error[0] is None, (what, want.first_error)
        else:
            assert want.first_error[:3] == (rec, seq, E_UTF8), (what, want.first_error)
        return got

    def close(self):
        for d, _ in self.ctx.values():
            d.close()


@pytest.fixture(scope="module")
def runner(gpu, oracle_mod):
    r = Runner(gpu, oracle_mod)
    yield r
    r.close()


# ------------------------------------------------------------------------------------------------ long text matrix
STRIDES = [256, 512, 2048, 4096, 16384, 32768]


def placements(S):
    """(name, d, m, e): the cell starts d bytes before boundary B, ends e bytes after boundary B + m*S (e < 0: before it).
    The start placements end 0xF5 - d bytes into a segment: the length's low byte is then 0xF5, and the byte before the
    cell (the low byte of its length field) is a lead byte, which a stream-wide verdict at the cell's first bytes would
    (wrongly) see — S0 must skip at least three bytes of the cell."""
    out = [(f"start-{d}", d, 2, 0xF5 - d) for d in range(6)]
    out += [(f"end+{e}/m{m}", 3, m, e) for m in (1, 2) for e in range(4)]
    out.append(("short-cover", 1, 1, 0xF5 - 1))                # S0 == S1 when S >= 512: no whole segment inside the cell
    return out


def geometry(S, d, m, e):
    B = 8 * S                                                      # the first boundary the cell crosses
    soff = B - d
    n = m * S + e + d
    S0 = (soff + 3 + S - 1) // S * S
    S1 = (soff + n) // S * S
    return soff, n, S0 - soff, S1 - soff


def spots(S, d, m, e, name):
    """(cell-relative position, catalog): where the poison goes for one placement.  Around an edge every reduced entry
    goes at the edge and one byte before it, one entry (in turn) at the other offsets up to 3 bytes away."""
    soff, n, s0, s1 = geometry(S, d, m, e)
    out = []

    def around(x, ks=range(-3, 4)):
        for i, k in enumerate(ks):
            out.append((x + k, REDUCED if k in (-1, 0) else [REDUCED[(i + x) % len(REDUCED)]]))

    if name.startswith("start") or name == "short-cover":
        around(s0)
    if name.startswith("end") and s1 > s0:
        around(s1)
    if name in ("start-0", "end+0/m1", "short-cover"):             # the first and last bytes of the cell
        for p in (0, 1, 2, 3, n - 4, n - 3, n - 2, n - 1):
            out.append((p, [REDUCED[p % len(REDUCED)], b"\xc2"]))
    if name == "start-3":                                          # the full catalog at S0 and at the cell ends
        out += [(s0 - 1, FULL), (s0, FULL), (0, FULL), (-1, FULL)]
    if name == "end+2/m1" and s1 > s0:                             # ... and at S1
        out += [(s1 - 1, FULL), (s1, FULL)]
    if name == "start-4" and s1 > s0:                              # lane and line edges of the first dead item
        for edge in sorted({64, 128, 192, min(1024, S - 64)}):
            around(s0 + edge, (-3, -1, 0, 1))
    if name == "end+1/m1" and S > DEAD_ITEM:                       # every 2 KiB item edge of one segment
        for i in range(1, S // DEAD_ITEM):
            around(s0 + i * DEAD_ITEM, (-3, -1, 0, 1, 3) if i in (1, S // DEAD_ITEM - 1) else (-1, 1))
        out.append((s0 + DEAD_ITEM - 1, FULL))
    return n, out


def real_edges(S, d, m, e):
    """(label, cell-relative position) of every seam of one placement: S0, S1 and the segment boundaries between them,
    the 64-byte lane and 128-byte line edges of the first dead item, every 2 KiB item edge of every dead segment, and the
    cell's two ends"""
    soff, n, s0, s1 = geometry(S, d, m, e)
    out = [("start", 0), ("end", n)]
    if s1 > s0:
        out += [("S0", s0), ("S1", s1)] + [(f"segment {k}", s0 + k * S) for k in range(1, (s1 - s0) // S)]
        out += [(f"line {x}", s0 + x) for x in (64, 128, 192, 1024) if x < min(S, DEAD_ITEM)]
        if S > DEAD_ITEM:
            out += [(f"item {k}.{i}", s0 + k * S + i * DEAD_ITEM) for k in range((s1 - s0) // S) for i in range(1, S // DEAD_ITEM)]
    else:
        out.append(("S0 (no whole segment)", s0))
    return out


def straddle_cells(base, edges):
    """valid 2-4 byte sequences across every edge at every split point j (the sequence starts j bytes before the edge, j
    from 0 to its length).  One (entry, j) goes to every edge it fits at in one cell; an edge whose bytes are taken moves
    on to the next cell.  Returns the cells and the set of (edge label, entry, j) placed."""
    n = len(base)
    cells, placed = [], set()
    for entry in NEAR_OK:
        L = len(entry)
        for j in range(L + 1):
            pending = [(lab, x - j) for lab, x in edges if (lab != "start" or j == 0) and (lab != "end" or j == L)
                       and 0 <= x - j and x - j + L <= n]
            while pending:
                b, taken, later = bytearray(base), [], []
                for lab, q in pending:
                    if any(q < t1 + 1 and t0 < q + L + 1 for t0, t1 in taken):
                        later.append((lab, q))
                        continue
                    b[q:q + L] = entry
                    taken.append((q, q + L))
                    placed.add((lab, entry, j))
                cells.append(bytes(b))
                pending = later
    return cells, placed


def place(buf, p, entry):
    """entry at position p (p = -1: ending at the last byte); None when it does not fit"""
    if p == -1:
        p = len(buf) - len(entry)
    if p < 0 or p + len(entry) > len(buf):
        return None
    b = bytearray(buf)
    b[p:p + len(entry)] = entry
    return bytes(b)


@pytest.mark.parametrize("stride", STRIDES)
def test_long_text_stride_matrix(runner, stride):
    S = stride
    n_poison, clean = 0, []
    for name, d, m, e in placements(S):
        soff, n, s0, s1 = geometry(S, d, m, e)
        base = bytes(ascii_fill(n, S + d * 7 + m * 3 + e))
        n_cell, todo = spots(S, d, m, e, name)
        seen = set()
        for p, cat in todo:
            for entry in cat:
                cell = place(base, p, entry)
                if cell is None or cell in seen:
                    continue
                seen.add(cell)
                L = Layout()
                rec, at = L.put(REL_TEXT, text_cells(cell), 1, S, soff)
                stream = L.bytes()
                assert stream[at:at + n] == cell and at % S == soff % S
                runner.poisoned(stream, S, rec, new_seq(1), cell, (S, name, p, entry.hex()))
                n_poison += 1
        # the valid near misses straddling every real edge at every split point: one stream for the whole stride
        edges = real_edges(S, d, m, e)
        cells, placed = straddle_cells(base, edges)
        for lab, x in edges:
            for entry in NEAR_OK:
                for j in range(len(entry) + 1):
                    fits = 0 <= x - j and x - j + len(entry) <= n and (lab != "start" or j == 0) and (lab != "end" or j == len(entry))
                    assert not fits or (lab, entry, j) in placed, (S, name, lab, entry.hex(), j)
        assert any(lab == "S0" for lab, _, _ in placed) or s1 <= s0
        clean += [(name, soff, c) for c in cells]
    L = Layout()
    for name, soff, cell in clean:
        assert strict_ok(cell)
        L.put(REL_TEXT, text_cells(cell), 1, S, soff)
    stream = L.bytes()
    got, want = runner.run(stream, S, what=(S, "near misses"), planes=True)
    assert want.first_error[0] is None
    assert n_poison > 150


# ------------------------------------------------------------------------------------------------ long non-text cells
def kind_values(S):
    """(column index, name, clean value, (lo, hi) of the bytes that may be poisoned): about three segments each"""
    n = max(3 * S + 100, 700)
    body = bytes(ascii_fill(n, 5))
    return [(1, "json", b'"' + body + b'"', (1, n + 1)),
            (2, "text[]", b'{"' + body + b'"}', (2, n + 2)),
            (3, "bytea", b"\\x" + bytes(ascii_fill(n, 6).hex()[:n].encode()), (2, n + 2))]


@pytest.mark.parametrize("stride", [256, 2048, 16384])
def test_long_non_text_cells(runner, stride):
    S = stride
    for col, kname, clean, (lo, hi) in kind_values(S):
        cells = ["1", None, None, None, None, None]
        cells[col] = clean
        L = Layout()
        L.put(REL_KINDS, cells, col, S, 5)
        s = L.bytes()
        runner.run(s, S, what=(S, kname, "clean"), planes=True)
        n = len(clean)
        for where, p in (("head", lo + 1), ("interior", n // 2), ("segment end", (n // 2 + 5) // S * S - 5 - 2), ("tail", hi - 2)):
            for entry in (b"\xff", b"\xed\xa0\x80"):
                v = place(clean, min(p, hi - len(entry)), entry)
                cells[col] = v
                L = Layout()
                rec, at = L.put(REL_KINDS, cells, col, S, 5)
                s = L.bytes()
                assert s[at:at + n] == v
                got = runner.poisoned(s, S, rec, new_seq(col), v, (S, kname, where, entry.hex()))
                assert got.first_error[2] == E_UTF8
        cells[col] = None
    # a light kind: an int4 of about 600 digits with a poisoned interior — UTF-8 wins over the integer parse error
    digits = b"0" * 599 + b"7"
    for p in (1, 300, 598):
        cells = ["1", None, None, None, place(digits, p, b"\xff"), None]
        L = Layout()
        rec, _ = L.put(REL_KINDS, cells, 4, S, S - 2)
        s = L.bytes()
        runner.poisoned(s, S, rec, new_seq(4), cells[4], (S, "int4", p))


@pytest.mark.parametrize("stride", [256, 2048, 16384])
def test_long_non_text_cell_ending_on_a_boundary(runner, stride):
    """A long Json, text[], bytea or int4 cell that ends exactly on a segment boundary, with a sequence left open in its
    last bytes: everything before the boundary is judged by the line bitmap, and the open sequence is a violation only
    past the cell's end, so k_rows must still check the cell's last bytes — the verdict is UTF-8, not the kind's own
    parse error.  The same cells closed with a valid sequence decode cleanly."""
    S = stride
    n = 2 * S + 40
    body = bytes(ascii_fill(n, 8))
    for col, kname, make in ((1, "json", lambda t: b'"' + body[:n - 2 - len(t)] + t + b'"'),
                             (2, "text[]", lambda t: b'{"' + body[:n - 4 - len(t)] + t + b'"}'),
                             (3, "bytea", lambda t: b"\\x" + body[:n - 2].hex().encode()[:n - 2]),
                             (4, "int4", lambda t: b"0" * (n - 1) + b"7"),
                             (5, "text", lambda t: body[:n - len(t)] + t)):
        clean = make(b"\xc3\xa9")
        assert len(clean) == n
        cells = ["1", None, None, None, None, None]
        cells[col] = clean
        L = Layout()
        L.put(REL_KINDS, cells, col, S, -n % S)
        s = L.bytes()
        runner.run(s, S, what=(S, kname, "clean, ends on a boundary"), planes=True)
        for tail in (b"\xc2", b"\xe2\x82", b"\xf0\x9f\x98"):
            v = clean[:n - len(tail)] + tail
            cells[col] = v
            L = Layout()
            rec, at = L.put(REL_KINDS, cells, col, S, -n % S)
            s = L.bytes()
            assert s[at:at + n] == v and (at + n) % S == 0
            got = runner.poisoned(s, S, rec, new_seq(col), v, (S, kname, "open at a boundary", tail.hex()))
            assert got.first_error[2] == E_UTF8


# ------------------------------------------------------------------------------------------------ length classes
LENGTHS = list(range(1, 9)) + [K_WIDE - 1, K_WIDE, K_WIDE + 1, K_MAX_IN_WIN - 1, K_MAX_IN_WIN, K_MAX_IN_WIN + 1,
                               239, 240, 241, 255, 256, 257, K_COOP - 1, K_COOP, K_COOP + 1]


@pytest.mark.parametrize("kind", ["text", "json"])
def test_length_classes(runner, kind):
    S = 2048
    for n in LENGTHS:
        inner = n - 2 if kind == "json" else n
        if inner < 1:
            continue
        base = ascii_fill(inner, n)
        wrap = (lambda b: b'"' + b + b'"') if kind == "json" else (lambda b: b)
        if n <= K_WIDE + 1:
            pos = range(inner)
        else:
            pos = sorted({0, 1, 14, 15, 16, 17, 31, 32, inner // 2, inner - 17, inner - 16, inner - 1} & set(range(inner)))
        for i, p in enumerate(pos):
            for entry in ([(REDUCED + [b"\xe2\x82"])[(i + n) % 6]] if n > 8 else REDUCED):
                v = place(bytes(base), p, entry) if p + len(entry) <= inner else place(bytes(base), -1, entry)
                if v is None:
                    continue
                v = wrap(v)
                L = Layout()
                if kind == "json":
                    rec, _ = L.put(REL_KINDS, ["1", v, None, None, None, None], 1, S, 100 + n)
                else:
                    rec, _ = L.put(REL_TEXT, text_cells(v), 1, S, 100 + n)
                runner.poisoned(L.bytes(), S, rec, new_seq(1), v, (kind, n, p, entry.hex()))
    # the valid near misses at every length: one stream
    L = Layout()
    for n in LENGTHS:
        for j, entry in enumerate(NEAR_OK):
            inner = n - 2 if kind == "json" else n
            v = place(bytes(ascii_fill(max(inner, 0), j)), (j * 7) % max(inner - len(entry) + 1, 1), entry)
            if v is None:
                continue
            if kind == "json":
                L.put(REL_KINDS, ["1", b'"' + v + b'"', None, None, None, None], 1)
            else:
                L.put(REL_TEXT, text_cells(v), 1)
    s = L.bytes()
    _, want = runner.run(s, S, what=(kind, "near misses"), planes=True)
    assert want.first_error[0] is None


# ------------------------------------------------------------------------------------------------ COPY rows
def test_copy_rows(gpu, oracle_mod):
    dec = gpu.Decoder(0)
    try:
        lengths = list(range(1, 41)) + [100, 511, 512, 513, 5000]
        for n in lengths:
            base = bytes(ascii_fill(n, n))
            pos = sorted({0, n - 1} | ({15, 16, 31, 32, n // 2} if n > 32 else set()))
            for i, p in enumerate(pos):
                for entry in (REDUCED[(i + n) % len(REDUCED)], b"\xc2"):
                    v = place(base, p, entry) if p + len(entry) <= n else place(base, -1, entry)
                    if v is None:
                        continue
                    rows = [b"ok\t1\n", v + b"\t2\n"]
                    err = check_rows(gpu, oracle_mod, [TEXT, INT4], rows, ("copy", n, p, entry.hex()), dec=dec,
                                     expect_error=not strict_ok(v))
                    if err is not None:
                        assert err == (1, 0, E_UTF8), (n, p, err)
            rows = [place(base, (j * 5) % max(n - len(e) + 1, 1), e) for j, e in enumerate(NEAR_OK)]
            rows = [r + b"\t3\n" for r in rows if r is not None]
            if rows:
                check_rows(gpu, oracle_mod, [TEXT, INT4], rows, ("copy near misses", n), dec=dec, expect_error=False)
    finally:
        dec.close()


# ------------------------------------------------------------------------------------------------ error order
def test_error_order(runner):
    S = 2048
    long_bad = place(bytes(ascii_fill(5000, 1)), 2500, b"\xed\xa0\x80")

    for i_long, i_short in ((3, 5), (5, 3)):             # record order among the six inserts
        L = Layout()
        recs = {}
        for r in range(6):
            if r == i_long:
                recs[r], _ = L.put(REL_TEXT, text_cells(long_bad), 1, S, 3)
            elif r == i_short:
                recs[r], _ = L.put(REL_TEXT, ["1", "short", "x1"], 2)    # int4 parse error in a short cell
            else:
                recs[r], _ = L.put(REL_TEXT, text_cells(b"fine"), 1)
        _, want = runner.run(L.bytes(), S, what=("long vs short", i_long, i_short))
        if i_long < i_short:
            assert want.first_error[:3] == (recs[i_long], new_seq(1), E_UTF8)
        else:
            assert want.first_error[:2] == (recs[i_short], new_seq(2)) and want.first_error[2] != E_UTF8

    # an update whose old and new image both carry a poisoned long cell: the lower seq (the old image) wins
    L = Layout()
    old = place(bytes(ascii_fill(6000, 2)), 4000, b"\xff")
    new = place(bytes(ascii_fill(7000, 3)), 3000, b"\xf4\x90\x80\x80")
    rec, _ = L.put(REL_TEXT, ["1", new, "2"], 1, update_old=["1", old, "2"])
    _, want = runner.run(L.bytes(), S, what="update old/new")
    assert want.first_error[:3] == (rec, old_seq(1), E_UTF8)

    # two poisoned long cells megabytes apart (their dead segments on different warps): the earlier one wins
    L = Layout()
    first = None
    for r in range(40):
        cell = bytes(ascii_fill(100_000, 10 + r))
        if r in (5, 35):
            cell = place(cell, 50_000 + r, b"\xe0\x80\x80")
        rec, _ = L.put(REL_TEXT, text_cells(cell), 1)
        if r == 5:
            first = rec
    _, want = runner.run(L.bytes(), S, what="two far apart")
    assert want.first_error[:3] == (first, new_seq(1), E_UTF8)

    # a poisoned long cell after a valid prefix of about 10 k records: the prefix's planes equal the oracle's
    L = Layout()
    for r in range(10_000):
        L.put(REL_TEXT, ["%d" % r, "v%d é" % r, str(r)], 1)
    rec, _ = L.put(REL_TEXT, text_cells(place(bytes(ascii_fill(9000, 4)), 6000, b"\x80")), 1)
    s = L.bytes()
    _, want = runner.run(s, S, what="prefix", planes=True)
    assert want.first_error[:3] == (rec, new_seq(1), E_UTF8)


# ------------------------------------------------------------------------------------------------ late passes, history
@pytest.mark.parametrize("stride", [256, 2048, 16384])
def test_wrong_hint_runs_the_long_passes_late(runner, stride):
    S = stride
    n = 3 * S + 700
    base = bytes(ascii_fill(n, 9))
    for entry in REDUCED:
        v = place(base, n // 2, entry)
        L = Layout()
        rec, _ = L.put(REL_TEXT, text_cells(v), 1, S, 1)
        got = runner.poisoned(L.bytes(), S, rec, new_seq(1), v, (S, "hint 64", entry.hex()), hint=64)
        assert got.sizing & abi.SIZING_LONG_PASSES_LATE


def test_one_decoder_across_batches(gpu, oracle_mod):
    """poisoned → clean shorter → clean longer → poisoned at another stride, on one context: bitmap bits of an earlier
    batch never become a false positive, and the long passes run in time (no late rerun) with the stager's own hint"""
    r = Runner(gpu, oracle_mod)
    try:
        def batch(n_cells, size, poison_at=None, stride=2048):
            L = Layout()
            recs = []
            for i in range(n_cells):
                cell = bytes(ascii_fill(size, 20 + i))
                if poison_at is not None and i == poison_at[0]:
                    cell = place(cell, poison_at[1], b"\xff")
                recs.append(L.put(REL_TEXT, text_cells(cell), 1, stride, 7)[0])
            return L.bytes(), recs

        seq = [(batch(8, 40_000, (5, 30_000)), 2048, True), (batch(4, 9_000), 2048, False), (batch(12, 60_000), 2048, False),
               (batch(6, 50_000, (2, 20_000), 16384), 16384, True)]
        for (s, recs), stride, bad in seq:
            got, want = r.run(s, stride, what=(stride, bad), planes=not bad, ctx="one")
            assert (want.first_error[0] is not None) == bad
            assert not got.sizing & abi.SIZING_LONG_PASSES_LATE, abi.SIZING_NAMES
    finally:
        r.close()
