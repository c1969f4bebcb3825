"""Plain reference of the map side of a hash repartition, written from PostgreSQL's and Citus's definitions.

  hash_uint32 / hashint4 / hashint8    src/common/hashfn.c hash_bytes_uint32 (lookup3's final mix of a one-word
                                       key) and src/backend/access/hash/hashfunc.c hashint4 / hashint8
  synthetic_intervals                  GenerateSyntheticShardIntervalArray: P uniform int4 token ranges, the
                                       last one widened to INT32_MAX
  uniform_index                        CalculateUniformHashRangeIndex: the shortcut for those ranges
  find_interval                        SearchCachedShardInterval: the interval holding a value, -1 in a gap
  route                                PartitionedResultDestReceiverReceive: NULL key -> 0, else the interval
  stable_scatter                       rows grouped by partition, input order inside a partition
  copy_files                           the COPY text / binary file of every partition (commands/copy*.c)

Every function works on Python ints or on numpy arrays with explicit widths; none calls the library or the
oracle.  The scalar forms follow the C source line by line; the numpy forms are checked against them.
"""
from __future__ import annotations

import struct

import numpy as np

INT32_MIN, INT32_MAX = -(1 << 31), (1 << 31) - 1
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
HASH_TOKEN_COUNT = 1 << 32
_M32 = 0xFFFFFFFF
_INIT = (0x9E3779B9 + 4 + 3923095) & _M32       # a = b = c = 0x9e3779b9 + len + 3923095, len = sizeof(uint32)

COPY_SIGNATURE = b"PGCOPY\n\377\r\n\0"
COPY_HEADER = COPY_SIGNATURE + struct.pack(">ii", 0, 0)      # flags 0, header extension length 0
COPY_TRAILER = struct.pack(">h", -1)


# ----------------------------------------------------------------------------------------------- hashing
def _rot(x, k):
    return ((x << k) | (x >> (32 - k))) & _M32


def hash_uint32(k: int) -> int:
    """hash_bytes_uint32(k) as an unsigned 32-bit int"""
    a = b = c = _INIT
    a = (a + (k & _M32)) & _M32
    # final(a, b, c)
    c ^= b; c = (c - _rot(b, 14)) & _M32
    a ^= c; a = (a - _rot(c, 11)) & _M32
    b ^= a; b = (b - _rot(a, 25)) & _M32
    c ^= b; c = (c - _rot(b, 16)) & _M32
    a ^= c; a = (a - _rot(c, 4)) & _M32
    b ^= a; b = (b - _rot(a, 14)) & _M32
    c ^= b; c = (c - _rot(b, 24)) & _M32
    return c


def _signed32(u: int) -> int:
    return u - (1 << 32) if u & 0x80000000 else u


def hashint4(v: int) -> int:
    """hashint4: the int4 value's 32 bits through hash_uint32, returned as int4"""
    return _signed32(hash_uint32(v & _M32))


def hashint8(v: int) -> int:
    """hashint8: the high word is folded into the low one (inverted for negative values), so that an int8 holding
    an int4 value hashes like that int4"""
    lo, hi = v & _M32, (v >> 32) & _M32
    lo ^= hi if v >= 0 else (~hi & _M32)
    return _signed32(hash_uint32(lo))


def _rot_np(x, k):
    return (x << np.uint32(k)) | (x >> np.uint32(32 - k))


def hash_uint32_np(k) -> np.ndarray:
    """hash_uint32 of a uint32 array (uint32 arithmetic wraps like C's)"""
    k = np.asarray(k, np.uint32)
    b = np.full(k.shape, _INIT, np.uint32)
    c = b.copy()
    a = b + k
    c ^= b; c -= _rot_np(b, 14)
    a ^= c; a -= _rot_np(c, 11)
    b ^= a; b -= _rot_np(a, 25)
    c ^= b; c -= _rot_np(b, 16)
    a ^= c; a -= _rot_np(c, 4)
    b ^= a; b -= _rot_np(a, 14)
    c ^= b; c -= _rot_np(b, 24)
    return c


def hashint4_np(v) -> np.ndarray:
    """int32 hashes of int4 values (an int64 array is taken modulo 2^32, like a Datum's int4 read)"""
    u = np.asarray(v, np.int64).astype(np.uint64) & np.uint64(_M32)
    return hash_uint32_np(u.astype(np.uint32)).view(np.int32)


def hashint8_np(v) -> np.ndarray:
    v = np.asarray(v, np.int64)
    u = v.astype(np.uint64)
    lo = (u & np.uint64(_M32)).astype(np.uint32)
    hi = (u >> np.uint64(32)).astype(np.uint32)
    lo ^= np.where(v >= 0, hi, ~hi)
    return hash_uint32_np(lo).view(np.int32)


# ----------------------------------------------------------------------------------------------- intervals
def synthetic_intervals(P: int):
    """(mins, maxs) as lists of Python ints"""
    inc = HASH_TOKEN_COUNT // P
    mins = [INT32_MIN + i * inc for i in range(P)]
    maxs = [m + inc - 1 for m in mins]
    maxs[-1] = INT32_MAX
    return mins, maxs


def uniform_index(h, P: int):
    """interval of hash h (int or int array) among the synthetic intervals of P partitions"""
    inc = HASH_TOKEN_COUNT // P
    if isinstance(h, (int, np.integer)):
        i = (int(h) - INT32_MIN) // inc
        return P - 1 if i == P else i          # the last interval also holds the 2^32 mod P values past P * inc
    i = (np.asarray(h, np.int64) - INT32_MIN) // inc
    return np.where(i == P, P - 1, i)


def find_interval(v, mins, maxs):
    """index of the interval [mins[i], maxs[i]] holding v (sorted, non-overlapping bounds), -1 in a gap"""
    mins = np.asarray(mins, np.int64)
    maxs = np.asarray(maxs, np.int64)
    scalar = isinstance(v, (int, np.integer))
    v = np.atleast_1d(np.asarray(v, np.int64))
    i = np.searchsorted(mins, v, side="right") - 1
    ok = (i >= 0) & (v <= maxs[np.maximum(i, 0)])
    out = np.where(ok, i, -1)
    return int(out[0]) if scalar else out


def route(keys, nulls, key_len: int, method: str, mins, maxs):
    """(index[n] int64, counts[P] int64, unroutable rows).  method 'hash' searches hashint4 / hashint8 of the key;
    'range' searches the key itself (an int4 key is the low 32 bits).  NULL keys go to partition 0; a row that
    lies in no interval gets index -1 and is not counted ("could not find shard for partition column value")."""
    keys = np.asarray(keys, np.int64)
    if method == "hash":
        v = hashint4_np(keys) if key_len == 4 else hashint8_np(keys)
    elif method == "range":
        v = keys.astype(np.int32) if key_len == 4 else keys
    else:
        raise ValueError(method)
    idx = find_interval(v.astype(np.int64), mins, maxs)
    if nulls is not None:
        idx = np.where(np.asarray(nulls).astype(bool), 0, idx)
    P = len(mins)
    counts = np.bincount(idx[idx >= 0], minlength=P).astype(np.int64)
    return idx.astype(np.int64), counts, int((idx < 0).sum())


def stable_scatter(index, cols, P: int, order=None):
    """(columns, offsets[P + 1]): rows grouped by output position order[p] (p itself without an order), input order
    inside a partition; offsets[i]..offsets[i + 1] delimit the partition at position i"""
    pos = np.asarray(index, np.int64)
    if order is not None:
        pos = np.asarray(order, np.int64)[pos]
    perm = np.argsort(pos, kind="stable")
    counts = np.bincount(pos, minlength=P)
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    return [np.asarray(c)[perm] for c in cols], offsets


# ----------------------------------------------------------------------------------------------- COPY files
_POW10 = [10 ** k for k in range(20)]


def _decimal_digits(mag: np.ndarray) -> np.ndarray:
    d = np.ones(mag.shape, np.int64)
    for k in range(1, 20):
        d += mag >= np.uint64(_POW10[k])
    return d


def copy_files(index, cols, col_lens, P: int, binary: bool, nulls=None, generate_empty_results=False):
    """the P partition files, rows of a partition in input order.
    text    every field as str(int) or \\N, fields separated by TAB, every row ended by LF
    binary  PGCOPY\\n\\377\\r\\n\\0, int32 flags 0, int32 extension length 0; per row int16 field count, per field int32
            length (-1 for NULL) and the value's col_len bytes big-endian; int16 -1 at the end
    A partition without rows has no file (b"") unless generate_empty_results (then a binary file holds header and
    trailer).  Vectorised over rows: every byte is placed by arithmetic on the row's field lengths."""
    index = np.asarray(index, np.int64)
    n, ncols = len(index), len(cols)
    perm = np.argsort(index, kind="stable")
    vals = [np.asarray(c, np.int64)[perm] for c in cols]
    isnull = [np.zeros(n, bool) if nulls is None or nulls[c] is None else np.asarray(nulls[c]).astype(bool)[perm]
              for c in range(ncols)]
    if binary:
        for c in range(ncols):
            lim = 1 << (8 * col_lens[c] - 1)
            v = vals[c][~isnull[c]]
            assert v.size == 0 or (int(v.min()) >= -lim and int(v.max()) < lim), "value does not fit its binary width"
    # field lengths
    flen, mags, digits = [], [], []
    for c in range(ncols):
        if binary:
            flen.append(4 + np.where(isnull[c], 0, col_lens[c]))
            mags.append(None); digits.append(None)
        else:
            v = vals[c]
            mag = np.where(v < 0, ~v.astype(np.uint64) + np.uint64(1), v.astype(np.uint64))
            d = _decimal_digits(mag)
            mags.append(mag); digits.append(d)
            flen.append(1 + np.where(isnull[c], 2, d + (v < 0)))
    row_len = np.full(n, 2 if binary else 0, np.int64)
    for f in flen:
        row_len += f
    row_start = np.concatenate([[0], np.cumsum(row_len)]).astype(np.int64)
    buf = np.zeros(int(row_start[-1]), np.uint8)
    pos = row_start[:-1].copy()

    def put_be(at, v, nbytes, sel):
        u = np.asarray(v).astype(np.int64).astype(np.uint64)
        for i in range(nbytes):
            buf[at[sel] + i] = ((u[sel] >> np.uint64(8 * (nbytes - 1 - i))) & np.uint64(0xFF)).astype(np.uint8)

    allrows = np.ones(n, bool)
    if binary:
        put_be(pos, np.full(n, ncols), 2, allrows)
        pos += 2
        for c in range(ncols):
            put_be(pos, np.where(isnull[c], -1, col_lens[c]), 4, allrows)
            pos += 4
            put_be(pos, vals[c], col_lens[c], ~isnull[c])
            pos += np.where(isnull[c], 0, col_lens[c])
    else:
        for c in range(ncols):
            nul, v, d, mag = isnull[c], vals[c], digits[c], mags[c]
            buf[pos[nul]] = ord("\\")
            buf[pos[nul] + 1] = ord("N")
            neg = ~nul & (v < 0)
            buf[pos[neg]] = ord("-")
            first = pos + neg                         # first digit
            val = ~nul
            for k in range(20):                       # digit k counted from the right
                sel = val & (d > k)
                if not sel.any():
                    break
                buf[first[sel] + d[sel] - 1 - k] = (ord("0") + (mag[sel] // np.uint64(_POW10[k])) % np.uint64(10)).astype(np.uint8)
            pos += flen[c] - 1
            buf[pos] = ord("\t") if c + 1 < ncols else ord("\n")
            pos += 1
    assert np.array_equal(pos, row_start[1:])
    counts = np.bincount(index, minlength=P) if n else np.zeros(P, np.int64)
    first_row = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    files = []
    for p in range(P):
        body = buf[row_start[first_row[p]]:row_start[first_row[p + 1]]].tobytes()
        if binary and (counts[p] > 0 or generate_empty_results):
            body = COPY_HEADER + body + COPY_TRAILER
        files.append(body)
    return files


def copy_files_rowwise(index, cols, col_lens, P: int, binary: bool, nulls=None, generate_empty_results=False):
    """copy_files one row at a time with str() and struct, as a receiver appends rows to its file; for small inputs"""
    files = [bytearray() for _ in range(P)]
    started = [False] * P
    for r in range(len(index)):
        p = int(index[r])
        f = files[p]
        if binary and not started[p]:
            f += COPY_HEADER
        started[p] = True
        null = [nulls is not None and nulls[c] is not None and bool(nulls[c][r]) for c in range(len(cols))]
        if binary:
            f += struct.pack(">h", len(cols))
            for c, col in enumerate(cols):
                if null[c]:
                    f += struct.pack(">i", -1)
                else:
                    f += struct.pack(">i", col_lens[c]) + int(col[r]).to_bytes(col_lens[c], "big", signed=True)
        else:
            f += ("\t".join("\\N" if null[c] else str(int(col[r])) for c, col in enumerate(cols)) + "\n").encode()
    for p in range(P):
        if binary and (started[p] or generate_empty_results):
            if not started[p]:
                files[p] += COPY_HEADER
            files[p] += COPY_TRAILER
    return [bytes(f) for f in files]
