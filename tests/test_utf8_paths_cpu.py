"""The DEVICE UTF-8 validators — utf8_valid, utf8_chunk_valid, utf8_chunk_valid_at (cell_parsers.cuh), has_high_bits and
utf8_range_bad (utf8.cuh) — compiled for the host (tests/emul/host_utf8.cpp, test infrastructure) and checked against
Python's strict decoder, which accepts exactly what core::str::from_utf8 accepts: no overlongs, no surrogates, nothing
above U+10FFFF, noncharacters allowed.

* every 1- and 2-byte string, every 3-byte string with a lead byte >= 0xC0, every string of up to 4 bytes over a boundary
  alphabet — alone, after an ASCII prefix and before an ASCII suffix;
* chunking invariance: a cell cut into random ranges, each range checked by utf8_range_bad with 1, 16 or 32 threads at
  every alignment mod 16 (the device ORs over threads and ranges), by utf8_chunk_valid, and by utf8_chunk_valid_at with
  the cell inside a longer stream — the OR must be Python's verdict, negated;
* every error and near-miss sequence of a catalog at every position of cells of 1-100, 127-129 and 511-513 bytes, at
  every alignment, as one range and split in two at every point near the sequence;
* the work split of utf8_range_bad: the head goes to thread 0 and the tail to the last thread, so that no thread carries
  both byte-serial edges of a range."""
import ctypes as C
import itertools
import os
import random
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.normpath(os.path.join(HERE, ".."))

# sequences Python rejects, each followed by ASCII (or by the end of the cell) where it is placed
CATALOG_BAD = [b"\x80", b"\xbf", b"\xc0\x80", b"\xc1\xbf", b"\xe0\x80\x80", b"\xe0\x9f\xbf", b"\xed\xa0\x80", b"\xed\xbf\xbf",
               b"\xf0\x80\x80\x80", b"\xf0\x8f\xbf\xbf", b"\xf4\x90\x80\x80", b"\xf5\x80\x80\x80", b"\xf8", b"\xfe", b"\xff",
               b"\xc2", b"\xe2\x82", b"\xf0\x9f\x98", b"\xc2\x80\x80"]
# the valid sequences right next to them
CATALOG_OK = [b"\xc2\x80", b"\xdf\xbf", b"\xe0\xa0\x80", b"\xed\x9f\xbf", b"\xee\x80\x80", b"\xf0\x90\x80\x80", b"\xf4\x8f\xbf\xbf",
              b"\xef\xbf\xbf"]
CATALOG = CATALOG_BAD + CATALOG_OK
VALID_MULTI = [b"\xc3\xa9", b"\xdf\xbf", b"\xe2\x9c\x93", b"\xef\xbf\xbd", b"\xf0\x9f\xa4\x94", b"\xf4\x8f\xbf\xbf", b"\xe0\xa0\x80"]
ALPHABET = bytes([0x00, 0x41, 0x7F, 0x80, 0x8F, 0x90, 0x9F, 0xA0, 0xBF, 0xC0, 0xC1, 0xC2, 0xDF, 0xE0, 0xE1, 0xEC, 0xED, 0xEE, 0xEF,
                  0xF0, 0xF1, 0xF3, 0xF4, 0xF5, 0xF8, 0xFF])
NTHREADS = (1, 16, 32)


@pytest.fixture(scope="module")
def emu():
    src = os.path.join(HERE, "emul", "host_utf8.cpp")
    so = os.path.join(HERE, "emul", "libhost_utf8.so")
    deps = [src] + [os.path.join(ROOT, "etl_b200", "csrc", f) for f in ("cell_parsers.cuh", "utf8.cuh", "json_tables.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "include"),
                               "-I", os.path.join(ROOT, "etl_b200", "csrc"), "-o", so, src])
    L = C.CDLL(so)
    vp = C.c_void_p
    L.emu_utf8_valid_batch.argtypes = [vp, vp, C.c_uint64, vp]
    L.emu_utf8_ranges.argtypes = [C.c_int, vp, vp, vp, vp, vp, C.c_uint64, C.c_uint32, C.c_uint32, vp, vp, vp]
    L.emu_has_high_bits.argtypes = [vp, vp, vp, vp, vp, C.c_uint64, C.c_uint32, vp]
    return L


def _ptr(a):
    return a.ctypes.data


class Arena:
    """cells back to back (offsets into one buffer) with 64 readable bytes on each side, as on the device"""

    def __init__(self, cells):
        lens = np.fromiter((len(c) for c in cells), dtype=np.uint64, count=len(cells))
        self.off = np.zeros(len(cells) + 1, dtype=np.uint64)
        np.cumsum(lens, out=self.off[1:])
        self.off += 64
        self.buf = np.frombuffer(b"\xff" * 64 + b"".join(cells) + b"\xff" * 64, dtype=np.uint8)
        self.n = len(cells)


def python_valid(cells):
    """Python's strict UTF-8 verdict per cell, vectorised: the cells are decoded as one buffer with a NUL between them
    (no sequence spans an ASCII byte, so every cell is judged alone); surrogateescape maps each byte the strict decoder
    rejects to one code point U+DC80..U+DCFF — a cell is valid when none of its bytes was escaped."""
    lens = np.fromiter((len(c) for c in cells), dtype=np.int64, count=len(cells))
    starts = np.zeros(len(cells), dtype=np.int64)
    np.cumsum(lens[:-1] + 1, out=starts[1:])
    text = b"\x00".join(cells).decode("utf-8", "surrogateescape")
    cps = np.frombuffer(text.encode("utf-32-le", "surrogatepass"), dtype=np.uint32)
    esc = (cps >= 0xDC80) & (cps <= 0xDCFF)
    nbytes = np.where(esc | (cps < 0x80), 1, np.where(cps < 0x800, 2, np.where(cps < 0x10000, 3, 4)))
    at = np.concatenate(([0], np.cumsum(nbytes)[:-1]))
    bad_cells = np.searchsorted(starts, at[esc], side="right") - 1
    ok = np.ones(len(cells), dtype=bool)
    ok[bad_cells] = False
    return ok


def strict(b):
    try:
        b.decode("utf-8")
        return True
    except UnicodeDecodeError:
        return False


def test_python_reference_is_the_strict_decoder():
    """the vectorised verdict above is bytes.decode('utf-8') cell by cell"""
    rng = random.Random(3)
    cells = [bytes(rng.choice(ALPHABET + b"ab") for _ in range(rng.randint(0, 9))) for _ in range(20000)]
    cells += CATALOG + [b"x" + e + b"y" for e in CATALOG] + [b"", b"\xed\xa0\x80", b"\xef\xbf\xbe", b"\xf4\x90"]
    assert python_valid(cells).tolist() == [strict(c) for c in cells]
    assert not any(strict(e + b"a") for e in CATALOG_BAD) and all(strict(e + b"a") for e in CATALOG_OK)


def valid_batch(emu, cells):
    a = Arena(cells)
    out = np.zeros(a.n, dtype=np.uint8)
    emu.emu_utf8_valid_batch(_ptr(a.buf), _ptr(a.off), a.n, _ptr(out))
    return out.astype(bool)


def fixed_cells(arr):
    """rows of a 2-D uint8 array as byte strings"""
    raw = arr.tobytes()
    w = arr.shape[1]
    return [raw[i:i + w] for i in range(0, len(raw), w)]


@pytest.mark.parametrize("space", ["len1", "len2", "len3_lead_c0", "alphabet_le4"])
def test_utf8_valid_exhaustive_short(emu, space):
    if space == "len1":
        cells = fixed_cells(np.arange(256, dtype=np.uint8).reshape(-1, 1))
    elif space == "len2":
        g = np.indices((256, 256)).reshape(2, -1).T.astype(np.uint8)
        cells = fixed_cells(g)
    elif space == "len3_lead_c0":
        g = np.indices((64, 256, 256)).reshape(3, -1).T
        g[:, 0] += 0xC0
        cells = fixed_cells(g.astype(np.uint8))
    else:
        cells = [bytes(t) for k in range(1, 5) for t in itertools.product(ALPHABET, repeat=k)]
    want = python_valid(cells)
    assert 0 < want.sum() < len(cells)
    for ctx, wrap in (("alone", lambda c: c), ("after ASCII", lambda c: b"ab" + c), ("before ASCII", lambda c: c + b"yz")):
        got = valid_batch(emu, [wrap(c) for c in cells])
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (space, ctx, [cells[i].hex() for i in bad[:8]])


# ---------------------------------------------------------------------------------------------- ranges
def run_ranges(emu, arena, cell_of, lo, hi, mode, align, nthreads=1, lead=None, tail=None):
    cell_of = np.ascontiguousarray(cell_of, dtype=np.uint32)
    lo = np.ascontiguousarray(lo, dtype=np.uint32)
    hi = np.ascontiguousarray(hi, dtype=np.uint32)
    n = len(cell_of)
    lead = np.zeros(n, dtype=np.uint8) if lead is None else np.ascontiguousarray(lead, dtype=np.uint8)
    tail = np.zeros(n, dtype=np.uint8) if tail is None else np.ascontiguousarray(tail, dtype=np.uint8)
    out = np.zeros(n, dtype=np.uint32)
    emu.emu_utf8_ranges(mode, _ptr(arena.buf), _ptr(arena.off), _ptr(cell_of), _ptr(lo), _ptr(hi), n, align, nthreads,
                        _ptr(lead), _ptr(tail), _ptr(out))
    assert not (out == 0xFFFFFFFF).any()
    return out


def cell_verdicts(n_cells, cell_of, bad_per_range):
    """OR of the range verdicts per cell"""
    v = np.zeros(n_cells, dtype=bool)
    np.logical_or.at(v, cell_of, bad_per_range != 0)
    return v


def catalog_heavy(rng, n):
    out = bytearray()
    while len(out) < n:
        k = rng.random()
        if k < 0.35:
            out += rng.choice(CATALOG)
        elif k < 0.6:
            out += rng.choice(VALID_MULTI)
        else:
            out += bytes(rng.randint(0x20, 0x7E) for _ in range(rng.randint(1, 24)))
    return bytes(out[:n])


def random_cuts(rng, n):
    if n == 0:
        return [(0, 0)]
    k = rng.choice([0, 0, 1, 2, 3, 6, 12])
    pts = sorted(set(rng.randint(1, n - 1) for _ in range(k))) if n > 1 else []
    b = [0] + pts + [n]
    return list(zip(b[:-1], b[1:]))


def test_chunking_invariance(emu):
    rng = random.Random(1009)
    cells = []
    for i in range(3000):
        n = rng.choice([rng.randint(0, 40), rng.randint(0, 700), rng.randint(0, 700)])
        c = catalog_heavy(rng, n)
        if i % 3 == 0:                                    # a third of the cells clean: the verdict must not fire on them
            c = c.decode("utf-8", "ignore").encode()
        cells.append(c)
    want_bad = ~python_valid(cells)
    assert 0.2 < want_bad.mean() < 0.9
    a = Arena(cells)
    cell_of, lo, hi = [], [], []
    for i, c in enumerate(cells):
        for r0, r1 in random_cuts(rng, len(c)):
            cell_of.append(i); lo.append(r0); hi.append(r1)
    cell_of = np.array(cell_of)
    for align in range(16):
        for nt in NTHREADS:
            got = cell_verdicts(a.n, cell_of, run_ranges(emu, a, cell_of, lo, hi, 0, align, nt))
            bad = np.flatnonzero(got != want_bad)
            assert bad.size == 0, ("utf8_range_bad", align, nt, [cells[i].hex() for i in bad[:4]])
    got = cell_verdicts(a.n, cell_of, run_ranges(emu, a, cell_of, lo, hi, 1, 0))
    assert (got == want_bad).all(), "utf8_chunk_valid"
    for lead in range(20):
        tails = np.array([(i + lead) % 4 for i in cell_of], dtype=np.uint8)      # the stream runs on 0-3 ASCII bytes
        got = cell_verdicts(a.n, cell_of, run_ranges(emu, a, cell_of, lo, hi, 2, lead % 16, 1, np.full(len(cell_of), lead), tails))
        assert (got == want_bad).all(), ("utf8_chunk_valid_at", lead)


def test_has_high_bits_every_window(emu):
    """has_high_bits reads whole aligned words: every window of a 40-byte cell with one high byte, at every alignment"""
    cells = [b"a" * p + b"\x80" + b"a" * (39 - p) for p in range(40)]
    a = Arena(cells)
    cell_of, lo, hi, want = [], [], [], []
    for i in range(len(cells)):
        for x in range(41):
            for y in range(x, 41):
                cell_of.append(i); lo.append(x); hi.append(y); want.append(x <= i < y)
    cell_of, lo, hi = (np.array(v, dtype=np.uint32) for v in (cell_of, lo, hi))
    for align in range(16):
        out = np.zeros(len(cell_of), dtype=np.uint8)
        emu.emu_has_high_bits(_ptr(a.buf), _ptr(a.off), _ptr(cell_of), _ptr(lo), _ptr(hi), len(cell_of), align, _ptr(out))
        assert (out.astype(bool) == np.array(want)).all(), align


CATALOG_LENGTHS = list(range(1, 101)) + [127, 128, 129, 511, 512, 513]


def catalog_cells():
    """(cell, entry index, position): the entry at every position of ASCII cells of every catalog length"""
    out = []
    for ei, e in enumerate(CATALOG):
        for n in CATALOG_LENGTHS:
            for p in range(0, n - len(e) + 1):
                out.append((b"q" * p + e + b"r" * (n - p - len(e)), ei, p))
    return out


def test_catalog_at_every_position(emu):
    cases = catalog_cells()
    cells = [c for c, _, _ in cases]
    want_bad = ~python_valid(cells)
    assert want_bad.sum() == sum(1 for _, ei, _ in cases if ei < len(CATALOG_BAD))
    a = Arena(cells)
    whole_of = np.arange(len(cells), dtype=np.uint32)
    whole_lo = np.zeros(len(cells), dtype=np.uint32)
    whole_hi = (a.off[1:] - a.off[:-1]).astype(np.uint32)
    split_of, split_lo, split_hi, split_id = [], [], [], []       # [0, k) and [k, n) for every k near the entry
    sid = 0
    for i, (c, ei, p) in enumerate(cases):
        n = len(c)
        for k in range(max(1, p - 3), min(n - 1, p + len(CATALOG[ei]) + 3) + 1):
            split_of += [i, i]; split_lo += [0, k]; split_hi += [k, n]; split_id += [sid, sid]
            sid += 1
    split_of, split_id = np.array(split_of, dtype=np.uint32), np.array(split_id)
    split_cell = split_of[::2]
    for align in range(16):
        nt = NTHREADS[align % 3]
        for mode in (0, 1):
            if mode == 1 and align:
                continue
            got = run_ranges(emu, a, whole_of, whole_lo, whole_hi, mode, align, nt) != 0
            bad = np.flatnonzero(got != want_bad)
            assert bad.size == 0, ("whole", mode, align, nt, [(cases[i][0][:40].hex(), cases[i][2]) for i in bad[:4]])
            r = run_ranges(emu, a, split_of, split_lo, split_hi, mode, align, nt) != 0
            got = np.zeros(sid, dtype=bool)
            np.logical_or.at(got, split_id, r)
            bad = np.flatnonzero(got != want_bad[split_cell])
            assert bad.size == 0, ("split", mode, align, nt, [(cases[split_cell[i]][2], len(cases[split_cell[i]][0]),
                                                               CATALOG[cases[split_cell[i]][1]].hex()) for i in bad[:4]])


def test_range_work_split(emu):
    """utf8_range_bad with several threads: a violation in the range's head (before its first 16-byte boundary) is
    reported by thread 0, one in its tail (after its last whole chunk) by the last thread, and one inside a chunk by the
    thread that owns the chunk — so the two byte-serial edges of a range never fall on one thread.  Positions within
    reach of the head's 19-byte look-ahead or of a neighbour's 3-byte look-back are left out: two threads may see them."""
    cells = []
    for n in (40, 100, 129, 300, 513):
        for p in range(n):
            c = bytearray(b"s" * n)
            c[p] = 0xFF
            cells.append(bytes(c))
    a = Arena(cells)
    n_tail = 0
    for align in range(16):
        for nt in (2, 16, 32):
            cell_of, lo, hi, want = [], [], [], []
            for i, c in enumerate(cells):
                n, p = len(c), c.index(0xFF)
                for r0 in (0, 1, 5):
                    if p < r0:
                        continue
                    body0 = r0 + min(n - r0, (16 - (align + r0) % 16) % 16)
                    tail0 = body0 + (n - body0) // 16 * 16
                    if p < body0:
                        owner = 0
                    elif body0 + 18 <= p < tail0 - 3:
                        owner = ((p - body0) // 16) % nt
                    elif p >= max(tail0, body0 + 18):
                        owner = nt - 1
                        n_tail += 1
                    else:
                        continue
                    cell_of.append(i); lo.append(r0); hi.append(n); want.append(1 << owner)
            got = run_ranges(emu, a, cell_of, lo, hi, 0, align, nt)
            bad = np.flatnonzero(got != np.array(want, dtype=np.uint32))
            assert bad.size == 0, (align, nt, [(len(cells[cell_of[i]]), cells[cell_of[i]].index(0xFF), lo[i], bin(got[i]), bin(want[i]))
                                               for i in bad[:4]])
    assert n_tail > 1000
