"""Restatement of the ClickHouse INSERT bodies (etl_dec_rowbinary_lz4, csrc/clickhouse_lz4.cu):
* insert_rows's greedy split over an emit's row offsets (INTEGRATION.md §8);
* the framing of one ClickHouse compressed block: 16 bytes of checksum (low64 then high64, each little-endian), method
  0x82, u32 LE compressed size (9 + payload), u32 LE decompressed size, the LZ4 payload;
* CityHash128 v1.0.2, the version ClickHouse checks its blocks with (not 1.1: the seed CityHash128 derives from the first
  16 bytes, HashLen0to16 / HashLen17to32, and the long-input loop and tail differ), in 64-bit-masked Python, written
  from the published v1.0.2 algorithm;
* a strict LZ4 block decoder: besides decoding, it rejects an offset of 0 or one reaching before the output, a block whose
  last sequence carries a match, a match that starts fewer than 12 bytes before the end of the block or ends within its
  last 5 bytes, and any trailing or truncated input."""
import struct

M64 = (1 << 64) - 1
K0, K1, K2, K3 = 0xc3a5c85c97cb3127, 0xb492b66fbe98f273, 0x9ae16a3b2f90404f, 0xc949d7c7509e6557
KBLOCK = 16384                 # uncompressed bytes per block (clickhouse_lz4.cuh kBlock)
HEADER = 25
METHOD_LZ4 = 0x82
MFLIMIT, LAST_LITERALS, MIN_MATCH = 12, 5, 4


# ------------------------------------------------------------------------------------------------ split
def split(off, row_begin, row_end, max_bytes):
    """insert_rows's loop from row_begin: n_inserts + 1 row boundaries"""
    assert max_bytes > 0
    cuts, i = [row_begin], row_begin
    while i < row_end:
        start = i
        while i < row_end and off[i] - off[start] < max_bytes:
            i += 1
        cuts.append(i)
    return cuts


# ------------------------------------------------------------------------------------------------ CityHash128 v1.0.2
def _f64(s, i):
    return int.from_bytes(s[i:i + 8], "little")


def _f32(s, i):
    return int.from_bytes(s[i:i + 4], "little")


def _rot(v, s):
    return v if s == 0 else ((v >> s) | (v << (64 - s))) & M64


def _smix(v):
    return v ^ (v >> 47)


def _h16(u, v):
    kmul = 0x9ddfea08eb382d69
    a = ((u ^ v) * kmul) & M64
    a ^= a >> 47
    b = ((v ^ a) * kmul) & M64
    b ^= b >> 47
    return (b * kmul) & M64


def _len0to16(s, i, n):
    if n > 8:
        a, b = _f64(s, i), _f64(s, i + n - 8)
        return _h16(a, _rot((b + n) & M64, n)) ^ b
    if n >= 4:
        a = _f32(s, i)
        return _h16((n + (a << 3)) & M64, _f32(s, i + n - 4))
    if n > 0:
        y = s[i] + (s[i + (n >> 1)] << 8)
        z = n + (s[i + n - 1] << 2)
        return (_smix(((y * K2) ^ (z * K3)) & M64) * K2) & M64
    return K2


def _weak32(s, i, a, b):
    w, x, y, z = _f64(s, i), _f64(s, i + 8), _f64(s, i + 16), _f64(s, i + 24)
    a = (a + w) & M64
    b = _rot((b + a + z) & M64, 21)
    c = a
    a = (a + x + y) & M64
    b = (b + _rot(a, 44)) & M64
    return (a + z) & M64, (b + c) & M64


def _murmur(s, i, n, seed):
    a, b = seed
    if n <= 16:
        a = (_smix((a * K1) & M64) * K1) & M64
        c = (b * K1 + _len0to16(s, i, n)) & M64
        d = _smix((a + (_f64(s, i) if n >= 8 else c)) & M64)
    else:
        c = _h16((_f64(s, i + n - 8) + K1) & M64, a)
        d = _h16((b + n) & M64, (c + _f64(s, i + n - 16)) & M64)
        a = (a + d) & M64
        l = n - 16
        while True:
            a ^= (_smix((_f64(s, i) * K1) & M64) * K1) & M64
            a = (a * K1) & M64
            b ^= a
            c ^= (_smix((_f64(s, i + 8) * K1) & M64) * K1) & M64
            c = (c * K1) & M64
            d ^= c
            i += 16
            l -= 16
            if l <= 0:
                break
    a = _h16(a, c)
    b = _h16(d, b)
    return a ^ b, _h16(b, a)


def _city128_seed(s, i, n, seed):
    if n < 128:
        return _murmur(s, i, n, seed)
    x, y = seed
    z = (n * K1) & M64
    v1 = (_rot(y ^ K1, 49) * K1 + _f64(s, i)) & M64
    v2 = (_rot(v1, 42) * K1 + _f64(s, i + 8)) & M64
    w1 = (_rot((y + z) & M64, 35) * K1 + x) & M64
    w2 = (_rot((x + _f64(s, i + 88)) & M64, 53) * K1) & M64
    while True:
        for _ in range(2):
            x = (_rot((x + y + v1 + _f64(s, i + 16)) & M64, 37) * K1) & M64
            y = (_rot((y + v2 + _f64(s, i + 48)) & M64, 42) * K1) & M64
            x ^= w2
            y ^= v1
            z = _rot(z ^ w1, 33)
            v1, v2 = _weak32(s, i, (v2 * K1) & M64, (x + w1) & M64)
            w1, w2 = _weak32(s, i + 32, (z + w2) & M64, y)
            z, x = x, z
            i += 64
        n -= 128
        if n < 128:
            break
    y = (y + _rot(w1, 37) * K0 + z) & M64
    x = (x + _rot((v1 + z) & M64, 49) * K0) & M64
    done = 0
    while done < n:
        done += 32
        y = (_rot((y - x) & M64, 42) * K0 + v2) & M64
        w1 = (w1 + _f64(s, i + n - done + 16)) & M64
        x = (_rot(x, 49) * K0 + w1) & M64
        w1 = (w1 + v1) & M64
        v1, v2 = _weak32(s, i + n - done, v1, v2)
    x = _h16(x, v1)
    y = _h16(y, w1)
    return (_h16((x + v2) & M64, w2) + y) & M64, _h16((x + w2) & M64, (y + v2) & M64)


def city128(s):
    """CityHash128 v1.0.2 of bytes s: (low64, high64)"""
    s = bytes(s)
    n = len(s)
    if n >= 16:
        return _city128_seed(s, 16, n - 16, (_f64(s, 0) ^ K3, _f64(s, 8)))
    if n >= 8:
        return _city128_seed(b"", 0, 0, (_f64(s, 0) ^ ((n * K0) & M64), _f64(s, n - 8) ^ K1))
    return _city128_seed(s, 0, n, (K0, K1))


def checksum(header_and_payload):
    lo, hi = city128(header_and_payload)
    return struct.pack("<QQ", lo, hi)


# ------------------------------------------------------------------------------------------------ framing
def frame(payload, raw_len):
    """one ClickHouse compressed block around an LZ4 payload"""
    hdr = bytes([METHOD_LZ4]) + struct.pack("<II", 9 + len(payload), raw_len)
    return checksum(hdr + payload) + hdr + payload


def parse_blocks(body):
    """a body → [(checksum, method, compressed size, decompressed size, payload, header and payload)]"""
    out, pos = [], 0
    while pos < len(body):
        assert len(body) - pos >= HEADER, ("truncated block header", pos)
        csum = body[pos:pos + 16]
        method = body[pos + 16]
        csize, raw = struct.unpack_from("<II", body, pos + 17)
        assert csize >= 9 and pos + 16 + csize <= len(body), ("bad compressed size", pos, csize)
        out.append((csum, method, csize, raw, body[pos + HEADER:pos + 16 + csize], body[pos + 16:pos + 16 + csize]))
        pos += 16 + csize
    return out


# ------------------------------------------------------------------------------------------------ LZ4 sequences
def _ext(v):
    out = bytearray()
    while v >= 255:
        out.append(255)
        v -= 255
    out.append(v)
    return bytes(out)


def sequence(lit, offset=0, match_len=0):
    """one LZ4 sequence: token, literal-length extension, literals, and (match_len > 0) offset and match-length
    extension; match_len 0 is the last sequence of a block"""
    ml = match_len - MIN_MATCH if match_len else 0
    out = bytes([min(len(lit), 15) << 4 | min(ml, 15)])
    if len(lit) >= 15:
        out += _ext(len(lit) - 15)
    out += bytes(lit)
    if match_len:
        assert match_len >= MIN_MATCH and 0 < offset < 65536
        out += struct.pack("<H", offset)
        if ml >= 15:
            out += _ext(ml - 15)
    return out


# ------------------------------------------------------------------------------------------------ strict LZ4 decoder
class Lz4Error(ValueError):
    pass


def lz4_decode(src, raw_len=None):
    """one LZ4 block → its bytes; raises Lz4Error on a malformed block or one that breaks the end-of-block rules
    (raw_len, when given, must equal the decoded length)"""
    src = bytes(src)
    out, matches = bytearray(), []
    i, n = 0, len(src)
    if n == 0:
        raise Lz4Error("empty block")
    while True:
        if i >= n:
            raise Lz4Error("truncated: missing token")
        tok = src[i]
        i += 1
        lit = tok >> 4
        if lit == 15:
            while True:
                if i >= n:
                    raise Lz4Error("truncated literal length")
                b = src[i]
                i += 1
                lit += b
                if b != 255:
                    break
        if i + lit > n:
            raise Lz4Error("literals past the end of the input")
        out += src[i:i + lit]
        i += lit
        if i == n:                                   # the last sequence: literals only
            break
        if i + 2 > n:
            raise Lz4Error("truncated offset")
        off = src[i] | (src[i + 1] << 8)
        i += 2
        if off == 0:
            raise Lz4Error("offset 0")
        if off > len(out):
            raise Lz4Error("offset reaches before the output")
        ml = tok & 15
        if ml == 15:
            while True:
                if i >= n:
                    raise Lz4Error("truncated match length")
                b = src[i]
                i += 1
                ml += b
                if b != 255:
                    break
        ml += MIN_MATCH
        start = len(out) - off
        if off >= ml:
            out += out[start:start + ml]
        else:                                        # overlapping: the pattern of `off` bytes repeats
            pat = bytes(out[start:])
            out += (pat * (ml // off + 1))[:ml]
        if i == n:
            raise Lz4Error("the last sequence carries a match")
        matches.append((len(out) - ml, len(out)))   # checked once the total is known
    total = len(out)
    for s, e in matches:
        if total - s < MFLIMIT:
            raise Lz4Error(f"a match starts {total - s} bytes before the end")
        if total - e < LAST_LITERALS:
            raise Lz4Error(f"a match ends {total - e} bytes before the end")
    if raw_len is not None and total != raw_len:
        raise Lz4Error(f"decoded {total} bytes, the header says {raw_len}")
    return bytes(out)


def body_bytes(body, kblock=KBLOCK):
    """check every block of a body (method, sizes, checksum, strict decode) and return the decompressed bytes"""
    out = []
    for csum, method, csize, raw, payload, hp in parse_blocks(body):
        assert method == METHOD_LZ4, method
        assert 0 < raw <= kblock, raw
        assert csum == checksum(hp), "checksum"
        out.append(lz4_decode(payload, raw))
    return b"".join(out)
