"""Value streams for checking the GPU decoders byte for byte, and relation images that carry them.

  image_with_streams   a relation (rowid int8, x) whose x value streams are exactly the given (codec, stream, raw
                       length) chunks, one chunk per stripe: arbitrary and hand-assembled streams, and several codecs in
                       one relation
  recompress           an uncompressed relation image with every value stream recompressed by the codec its stripe
                       names, like ALTER TABLE ... SET (compression ...) between inserts
  HAND_LZ4 / HAND_PGLZ / HAND_ZSTD / MALFORMED
                       streams assembled from the published formats, with the bytes they decode to (computed while
                       assembling, not by a decoder)
  readback_desc        the query that returns every row's decoded values: GROUP BY rowid, bit_or(x1) ... bit_or(x7)

The page arithmetic is the reference's (columnar_storage.c): logical offset L lives in block L / 8168 at byte
24 + L % 8168.
"""
import ctypes as C
import struct

import numpy as np

BLCKSZ, PAGE_HEADER = 8192, 24
BYTES_PER_PAGE = BLCKSZ - PAGE_HEADER
COMP_NONE, COMP_PGLZ, COMP_LZ4, COMP_ZSTD = 0, 1, 2, 3


# --------------------------------------------------------------------------- page images
def storage_write(pages, logical, data):
    done = 0
    while done < len(data):
        blk, off = divmod(logical + done, BYTES_PER_PAGE)
        off += PAGE_HEADER
        n = min(len(data) - done, BLCKSZ - off)
        at = blk * BLCKSZ + off
        pages[at:at + n] = np.frombuffer(bytes(data[done:done + n]), np.uint8)
        done += n


def storage_read(pages, logical, amount):
    out = bytearray()
    while len(out) < amount:
        blk, off = divmod(logical + len(out), BYTES_PER_PAGE)
        off += PAGE_HEADER
        n = min(amount - len(out), BLCKSZ - off)
        out += pages[blk * BLCKSZ + off: blk * BLCKSZ + off + n].tobytes()
    return bytes(out)


def _node_view(oracle, nodes):
    return (oracle.SkipNode * (len(nodes) // C.sizeof(oracle.SkipNode))).from_buffer(nodes)


def image_with_streams(oracle, chunks, attlen=1):
    """chunks: [(kind, stream, raw_len)] -> (pages, stripes, nodes, chunk_row_limit, rows per chunk).

    The oracle writes (rowid int8, room int8) uncompressed, one insert -- so one stripe of one chunk -- per stream, with
    raw_len / attlen rows (at least one): 8 bytes of room per row.  The stream is written over the start of the room
    column's value stream, its skip node gets the codec, value_length = len(stream), decompressed_size = raw_len and no
    min / max, and the column is read as attlen bytes wide.  A chunk with raw_len 0 keeps one row and marks it NULL in
    the exists bitmap.  The page framing does not change, so the result is a valid image."""
    rows = [max(raw // attlen, 1) for _, _, raw in chunks]
    for (kind, stream, raw), r in zip(chunks, rows):
        assert raw % attlen == 0 and len(stream) <= 8 * r, (kind, len(stream), raw)
    limit = max(rows)
    t = oracle.Table([8, 8], stripe_row_limit=limit, chunk_row_limit=limit)
    first = 0
    for r in rows:
        t.insert([np.arange(first, first + r), np.zeros(r, np.int64)])
        first += r
    pages = t.pages()
    nodes = t.nodes_array()
    nv = _node_view(oracle, nodes)
    stripes = t.stripes()
    assert len(stripes) == len(chunks)
    for st, (kind, stream, raw) in zip(stripes, chunks):
        assert st.chunk_count == 1
        n = nv[st.skipnode_base + 1]
        storage_write(pages, st.file_offset + n.value_offset, stream)
        present = raw // attlen
        bits = np.packbits(np.arange(n.exists_length * 8) < present, bitorder="little")
        storage_write(pages, st.file_offset + n.exists_offset, bits.tobytes())
        n.compression_type = kind
        n.value_length = len(stream)
        n.decompressed_size = raw
        n.has_minmax, n.min_value, n.max_value = 0, 0, 0
    return pages, t.stripes_array(), nodes, limit, rows


def expected_values(raw_bytes, attlen, rows):
    """the column a decoded stream holds: its values (sign-extended) in the first rows, NULL in the others"""
    vals = np.zeros(rows, np.int64)
    nulls = np.ones(rows, np.uint8)
    v = np.frombuffer(raw_bytes, {1: np.int8, 2: np.int16, 4: np.int32, 8: np.int64}[attlen]).astype(np.int64)
    vals[:len(v)] = v
    nulls[:len(v)] = 0
    return vals, nulls


def recompress(oracle, t, kinds, level=3):
    """the image of oracle Table t (written uncompressed) with the value streams of stripe s compressed by kinds[s]
    (a codec that does not shrink a stream leaves it stored raw, as CompressBuffer does)"""
    pages = t.pages()
    nodes = t.nodes_array()
    nv = _node_view(oracle, nodes)
    for st, kind in zip(t.stripes(), kinds):
        for i in range(st.skipnode_base, st.skipnode_base + st.column_count * st.chunk_count):
            n = nv[i]
            assert n.compression_type == COMP_NONE
            if kind == COMP_NONE or n.value_length == 0:
                continue
            raw = storage_read(pages, st.file_offset + n.value_offset, n.value_length)
            comp = oracle.codec_compress(kind, raw, level)
            if comp is None or len(comp) >= len(raw):
                continue
            storage_write(pages, st.file_offset + n.value_offset, comp)
            n.compression_type = kind
            n.compression_level = level
            n.value_length = len(comp)
    return pages, t.stripes_array(), nodes


# --------------------------------------------------------------------------- codec-written relations
ATTLENS = [8, 8, 8, 8, 4, 2, 1, 1]        # rowid + 7 payload columns: one readback query reads them all
# row counts of the inserts of a "small chunks" relation (one stripe each; chunk_row_limit 2064): raw stream lengths on
# and around 16, 128, 256, 2048 and 2064 bytes for the 1-, 2-, 4- and 8-byte columns, single-row chunks, ragged last chunks
SMALL_INSERTS = [1, 2, 15, 16, 17, 32, 33, 127, 128, 129, 255, 256, 257, 258, 1024, 2047, 2048, 2049, 2063, 2064, 2065, 5000]


def codec_columns(n, seed, all_null_rows=()):
    """(values, nulls) of the 8 columns for n rows: long overlapping matches, short matches, a period of 65528 bytes
    (LZ4 offsets up to 65535), incompressible int8 (pglz stores it raw), int4 with 10 % NULLs, int2 with 50 % NULLs,
    an int1 period of 2049 bytes (beyond the 2 KB windows), int1 runs; the last column is NULL on all_null_rows"""
    rng = np.random.default_rng(seed)
    base = rng.integers(-2**40, 2**40, 8191)
    period = rng.integers(-128, 128, 2049)
    vals = [
        np.zeros(n, np.int64),
        np.arange(n) % 7,
        base[np.arange(n) % 8191],
        rng.integers(-2**63, 2**63 - 1, n, endpoint=True),
        rng.integers(-2**31, 2**31, n),
        rng.integers(-2**15, 2**15, n) // 7,
        period[np.arange(n) % 2049],
        np.repeat(rng.integers(-128, 128, n // 300 + 1), 300)[:n],
    ]
    nulls = [np.zeros(n, np.uint8) for _ in vals]
    nulls[4] = (rng.random(n) < 0.1).astype(np.uint8)
    nulls[5] = (rng.random(n) < 0.5).astype(np.uint8)
    nulls[7][list(all_null_rows)] = 1
    return vals, nulls


def codec_table(oracle, kind, level, inserts, chunk_row_limit, seed, first_rowid=0):
    """an oracle-written relation of ATTLENS columns, one insert -- one stripe -- per entry of `inserts` (the second
    insert's last column all NULL); returns (table, values, nulls) with rowid = first_rowid, first_rowid + 1, ..."""
    total = sum(inserts)
    stripe_row_limit = max(inserts)
    second = range(inserts[0], inserts[0] + inserts[1]) if len(inserts) > 1 else ()
    vals, nulls = codec_columns(total, seed, second)
    vals[0] = np.arange(first_rowid, first_rowid + total)
    t = oracle.Table(ATTLENS, stripe_row_limit=stripe_row_limit, chunk_row_limit=chunk_row_limit, compression=kind,
                     compression_level=level)
    at = 0
    for n in inserts:
        t.insert([v[at:at + n] for v in vals], [m[at:at + n] for m in nulls])
        at += n
    return t, vals, nulls


# --------------------------------------------------------------------------- LZ4 blocks by hand
def _lz4_ext(n):
    out = bytearray()
    while n >= 255:
        out.append(255)
        n -= 255
    out.append(n)
    return bytes(out)


class Lz4Block:
    """an LZ4 block assembled sequence by sequence (token = literal length << 4 | match length - 4, 255-continued
    lengths, literals, 16-bit little-endian offset); `out` is what it decodes to, copied byte by byte"""

    def __init__(self):
        self.s, self.out = bytearray(), bytearray()

    def seq(self, lits, off, ml):
        lits = bytes(lits)
        L, m = len(lits), ml - 4
        self.s.append((min(L, 15) << 4) | min(m, 15))
        if L >= 15:
            self.s += _lz4_ext(L - 15)
        self.s += lits + struct.pack("<H", off)
        if m >= 15:
            self.s += _lz4_ext(m - 15)
        self.out += lits
        for _ in range(ml):
            self.out.append(self.out[-off])
        return self

    def end(self, lits):
        lits = bytes(lits)
        L = len(lits)
        self.s.append(min(L, 15) << 4)
        if L >= 15:
            self.s += _lz4_ext(L - 15)
        self.s += lits
        self.out += lits
        return bytes(self.s), bytes(self.out)


def _noise(seed, n):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()


def _hand_lz4():
    cases = {}
    cases["16 x a"] = (bytes([0x16, ord("a"), 1, 0, 0x50]) + b"aaaaa", b"a" * 16)
    lits = bytes((i * 7) & 0xff for i in range(273))
    cases["273 literals, 536-byte match at offset 273"] = (
        bytes([0xFF, 255, 3]) + lits + bytes([273 & 0xff, 273 >> 8, 255, 255, 7]) + bytes([0x50]) + b"vwxyz",
        lits + (lits * 2)[:536] + b"vwxyz")
    tail = _noise(1, 12)
    # 255-continued literal and match lengths whose last length byte sits at stream position 128k + d, d = -2 .. 1:
    # just before, on and just after a refill of the decoders' 256-byte input ring (128 bytes per refill)
    for k in (1, 2, 3):
        for d in (-2, -1, 0, 1):
            q = 128 * k + d - 2                     # the second token; its two literal-length bytes end at 128k + d
            L = q - 3 - len(_lz4_ext(q - 4 - 15))                        # token, literal length bytes, L literals, offset
            b = Lz4Block().seq(_noise(k * 10 + d, L), 1, 4)
            assert len(b.s) == q
            b.seq(_noise(k * 100 + d, 379), 3, 4 + 15 + 255 + 255 + 9)  # its three match-length bytes end at 128(k + 3) + d
            assert len(b.s) == 128 * (k + 3) + d + 1
            cases[f"continued lengths at ring refill k={k} d={d}"] = b.end(tail)
    for L in (1, 4, 15, 16, 300):
        cases[f"offset == position {L}"] = Lz4Block().seq(_noise(L, L), L, 40).end(tail)
    for off in range(1, 9):
        for ml in (4, 19, 270, 5000):
            cases[f"offset {off} match {ml}"] = Lz4Block().seq(_noise(off, 9), off, ml).end(tail)
    for off in (1791, 1792, 1793, 2048, 2049):
        for ml in (4, 255, 256, 257, 600):
            cases[f"offset {off} match {ml}"] = Lz4Block().seq(_noise(off + ml, 2100), off, ml).end(tail)
    big = _noise(7, 65_535)
    cases["offset 65535"] = Lz4Block().seq(big, 65_535, 300).seq(b"x", 65_535, 70).end(tail)
    cases["empty block"] = (bytes([0]), b"")
    return cases


# --------------------------------------------------------------------------- pglz streams by hand
class Pglz:
    """a pglz stream (PostgreSQL pg_lzcompress.c): control byte = 8 items LSB first, bit set = tag
    [(off >> 8) << 4 | len - 3][off & 0xff] (+ one byte len - 18 when the nibble is 15), bit clear = one literal; behind
    the 8-byte ColumnarCompressHeader {vl_len_ = total << 2 | 2, rawsize}"""

    def __init__(self):
        self.items, self.out = [], bytearray()        # items: (is_tag, bytes)

    def lits(self, data):
        for b in bytes(data):
            self.items.append((False, bytes([b])))
            self.out.append(b)
        return self

    def match(self, off, n, produce=None):
        """a tag of length n at offset off; `produce` bytes of it land in the output (a match clamped at rawsize)"""
        assert 1 <= off <= 4095 and 3 <= n <= 273
        if n < 18:
            tag = bytes([((off >> 8) << 4) | (n - 3), off & 0xff])
        else:
            tag = bytes([((off >> 8) << 4) | 0x0f, off & 0xff, n - 18])
        self.items.append((True, tag))
        for _ in range(n if produce is None else produce):
            self.out.append(self.out[-off])
        return self

    def stream(self, rawsize=None, last_ctrl_fill=0, header_len=None):
        """last_ctrl_fill: bits set in the last control byte past its last item"""
        body = bytearray()
        for g in range(0, len(self.items), 8):
            group = self.items[g:g + 8]
            ctrl = sum(1 << i for i, (is_tag, _) in enumerate(group) if is_tag)
            if len(group) < 8:
                ctrl |= last_ctrl_fill & ~((1 << len(group)) - 1) & 0xff
            body.append(ctrl)
            for _, b in group:
                body += b
        total = len(body) + 8
        raw = len(self.out) if rawsize is None else rawsize
        return struct.pack("<II", ((total if header_len is None else header_len) << 2) | 2, raw) + bytes(body)


def _hand_pglz():
    cases = {}
    p = Pglz().lits(b"0123456789").match(10, 273).lits(b"end")
    cases["length 18 + 255 = 273"] = (p.stream(), bytes(p.out))
    p = Pglz().lits(b"abc").match(3, 18).match(2, 17).match(1, 3).lits(b"!")
    cases["lengths 18, 17, 3"] = (p.stream(), bytes(p.out))
    p = Pglz().lits(_noise(4095, 4100)).match(4095, 273).match(4095, 3).lits(b"z")
    cases["offset 4095"] = (p.stream(), bytes(p.out))
    for off in (1793, 1900, 2000, 2047, 2048):
        p = Pglz().lits(_noise(off, 2100)).match(off, 273).match(off, 18).match(off - 1, 200).lits(b"q")
        cases[f"offset {off}"] = (p.stream(), bytes(p.out))
    p = Pglz().lits(b"xyz").match(3, 273, produce=100)
    cases["last match clamped at rawsize"] = (p.stream(rawsize=103), bytes(p.out))
    p = Pglz().lits(b"abcdefgh").lits(b"i")
    cases["unused control bits set"] = (p.stream(last_ctrl_fill=0xff), bytes(p.out))
    return cases


# --------------------------------------------------------------------------- zstd frames by hand
_P1, _P2, _P3, _P4, _P5 = 11400714785074694791, 14029467366897019727, 1609587929392839161, 9650029242287828579, 2870177450012600261
_M = (1 << 64) - 1


def _rotl(x, r):
    return ((x << r) | (x >> (64 - r))) & _M


def _round(acc, lane):
    return (_rotl((acc + lane * _P2) & _M, 31) * _P1) & _M


def xxh64(data, seed=0):
    """XXH64 (the frame's content checksum is its low 32 bits)"""
    n, i = len(data), 0
    if n >= 32:
        v = [(seed + _P1 + _P2) & _M, (seed + _P2) & _M, seed, (seed - _P1) & _M]
        while i + 32 <= n:
            for j in range(4):
                v[j] = _round(v[j], int.from_bytes(data[i + 8 * j: i + 8 * j + 8], "little"))
            i += 32
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & _M
        for x in v:
            h = ((h ^ _round(0, x)) * _P1 + _P4) & _M
    else:
        h = (seed + _P5) & _M
    h = (h + n) & _M
    while i + 8 <= n:
        h = (_rotl(h ^ _round(0, int.from_bytes(data[i:i + 8], "little")), 27) * _P1 + _P4) & _M
        i += 8
    if i + 4 <= n:
        h = (_rotl(h ^ (int.from_bytes(data[i:i + 4], "little") * _P1 & _M), 23) * _P2 + _P3) & _M
        i += 4
    while i < n:
        h = (_rotl(h ^ (data[i] * _P5 & _M), 11) * _P1) & _M
        i += 1
    h ^= h >> 33
    h = (h * _P2) & _M
    h ^= h >> 29
    h = (h * _P3) & _M
    return h ^ (h >> 32)


def zstd_frame(blocks, content_size=None, fcs_bytes=1, checksum=False, content=None):
    """a frame of raw (0) / RLE (1) / reserved (3) blocks, RFC 8878: single segment with a 1 / 2 / 4 / 8-byte content
    size, or (fcs_bytes 0) a window descriptor and no content size"""
    flag = {0: 0, 1: 0, 2: 1, 4: 2, 8: 3}[fcs_bytes]
    fhd = (flag << 6) | ((1 if fcs_bytes else 0) << 5) | ((1 if checksum else 0) << 2)
    out = bytes([0x28, 0xB5, 0x2F, 0xFD, fhd])
    if fcs_bytes == 0:
        out += bytes([7 << 3])                          # window 2^17 = 128 KB
    else:
        out += (content_size - (256 if fcs_bytes == 2 else 0)).to_bytes(fcs_bytes, "little")
    for i, (btype, size, payload) in enumerate(blocks):
        out += ((size << 3) | (btype << 1) | (1 if i == len(blocks) - 1 else 0)).to_bytes(3, "little") + payload
    if checksum:
        out += struct.pack("<I", xxh64(content) & 0xffffffff)
    return out


def _hand_zstd():
    cases = {}
    cases["raw block"] = (zstd_frame([(0, 5, b"hello")], 5), b"hello")
    cases["RLE block"] = (zstd_frame([(1, 7, b"z")], 7), b"z" * 7)
    cases["raw + RLE"] = (zstd_frame([(0, 3, b"abc"), (1, 4, b"!")], 7), b"abc!!!!")
    data = _noise(5, 300) + b"\x07" * 1000
    blocks = [(0, 300, data[:300]), (1, 1000, b"\x07")]
    for fcs in (1, 2, 4, 8):
        size = len(data) if fcs != 1 else 255
        want = data[:size]
        blks = blocks if fcs != 1 else [(0, 255, want)]
        cases[f"content size in {fcs} bytes"] = (zstd_frame(blks, size, fcs_bytes=fcs), want)
    cases["no content size, window descriptor"] = (zstd_frame(blocks, fcs_bytes=0), data)
    cases["checksum"] = (zstd_frame(blocks, len(data), fcs_bytes=2, checksum=True, content=data), data)
    cases["checksum, short"] = (zstd_frame([(0, 5, b"hello")], 5, checksum=True, content=b"hello"), b"hello")
    return cases


def _hand_zstd_large():
    """whole-block frames, in a relation of its own read as int4 (131072 one-byte rows would not fit one chunk)"""
    big = _noise(128, 131_072)
    return {
        "raw block of 128 KB": (zstd_frame([(0, len(big), big)], len(big), fcs_bytes=4), big),
        "RLE block of 128 KB + raw": (zstd_frame([(1, 131_072, b"\xA5"), (0, 8, b"tailtail")], 131_080, fcs_bytes=4),
                                      b"\xA5" * 131_072 + b"tailtail"),
    }


HAND_LZ4 = _hand_lz4()
HAND_PGLZ = _hand_pglz()
HAND_ZSTD = _hand_zstd()
HAND_ZSTD_LARGE = _hand_zstd_large()
# (relation name, attlen the streams are read as, codec, {case name: (stream, decoded bytes)})
HAND_RELATIONS = [("lz4", 1, COMP_LZ4, HAND_LZ4), ("pglz", 1, COMP_PGLZ, HAND_PGLZ), ("zstd", 1, COMP_ZSTD, HAND_ZSTD),
                  ("zstd 128 KB", 4, COMP_ZSTD, HAND_ZSTD_LARGE)]


def hand_relation_chunks(codec, cases):
    """[(kind, stream, raw_len)] of one hand relation, with raw streams (no codec) between every few codec streams, so
    that one decode launch routes items of two kinds"""
    chunks = []
    for i, (stream, want) in enumerate(cases.values()):
        chunks.append((codec, stream, len(want)))
        if i % 4 == 3:
            chunks.append((COMP_NONE, want, len(want)))
    return chunks


# --------------------------------------------------------------------------- malformed streams
# (codec, stream, raw_len, the bounds check that refuses it)
def _malformed():
    ok_lz4, ok_raw = Lz4Block().seq(b"abcdefgh", 8, 8).end(b"0123456789ab")
    lz4_zero = bytearray(ok_lz4)
    lz4_zero[9:11] = b"\0\0"                                          # the first sequence's offset
    lz4_far = bytearray(ok_lz4)
    lz4_far[9:11] = struct.pack("<H", 9)                              # one byte further back than the output
    pg = Pglz().lits(b"abcdefgh").match(8, 30).lits(b"!")
    pg_raw = bytes(pg.out)
    zs_ok = zstd_frame([(0, 5, b"hello")], 5)
    return [
        ("lz4 offset 0", COMP_LZ4, bytes(lz4_zero), len(ok_raw), "cg_decompress.cu lz4_block: off == 0"),
        ("lz4 offset beyond the output", COMP_LZ4, bytes(lz4_far), len(ok_raw), "lz4_block: off > o.op"),
        ("lz4 literals past the end", COMP_LZ4, bytes([0x50]) + b"abc", 5, "lz4_block: lit > clen - ip"),
        ("lz4 match past raw_len", COMP_LZ4, ok_lz4, len(ok_raw) - 13, "lz4_block: ml > rawlen - o.op"),
        ("pglz header length differs", COMP_PGLZ, pg.stream(header_len=len(pg.stream()) + 1), len(pg_raw),
         "pglz_stream: VARSIZE != buffer length"),
        ("pglz rawsize mismatch", COMP_PGLZ, pg.stream(rawsize=len(pg_raw) + 1), len(pg_raw), "pglz_stream: raw != rawlen"),
        ("zstd reserved block type", COMP_ZSTD, zstd_frame([(3, 5, b"hello")], 5), 5, "zstd_frame_coop: block type 3"),
        ("zstd content size mismatch", COMP_ZSTD, zstd_frame([(0, 5, b"hello")], 6), 6, "zstd_frame_coop: fcs != op"),
        ("zstd frame shorter than raw_len", COMP_ZSTD, zs_ok, 6, "cg_zstd_kernel: decoded size != raw_len"),
    ]


MALFORMED = _malformed()


# --------------------------------------------------------------------------- the readback query
def readback_aggs(cg, attlens):
    """GROUP BY column 0 (rowid), one aggregate per other column: bit_or for integers (one row per group, so the
    value itself, sign-extended), sum for varlena numeric columns; each aggregate's count is the column's non-NULL count"""
    return [cg.sum_(c) if attlens[c] < 0 else cg.bit_or(c) for c in range(1, len(attlens))]


def readback_desc(cg, attlens):
    return cg.make_desc([], [0], readback_aggs(cg, attlens))
