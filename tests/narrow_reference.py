"""An exact, independent restatement of the narrow images cg_shard_stage keeps next to the plain arena, in plain Python
integers and numpy.  It shares no code with cg_narrow.cu.

    pack(values, rows)  ->  (base, width, words)
        base = min, width = bit_length(max - min) (Python integers: no wrap), field r = value - base at bits
        [r * width, r * width + width) of little-endian uint64 words; ceil(rows / 64) * width words, the bits past the
        last row zero.
    narrow_layout(cols, nulls, layout, staged, candidate)  ->  NarrowLayout
        which staged columns get images, and every chunk column's width, base, stream offset and size, as cg_narrow_plan
        lays them out; cg_shard_narrow_bytes; and the bytes_scanned a scan reports, narrow or plain.

A staged column gets images when it is a candidate (an 8-byte integer column) and every NULL-free chunk column of it spans
max - min < 2^32; then each of its NULL-free chunk columns has one, in chunk group order and, within a chunk group, staged
slot order, each stream padded to 16 bytes.  A shard none of whose candidate chunk columns is NULL-free, or none of whose
columns qualifies, has no images at all.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

NONE = 255                     # CG_NARROW_NONE
MAX_WIDTH = 32
DEVPACKCOL_BYTES = 24          # sizeof(DevPackCol): off, base, width, pad
MASK64 = (1 << 64) - 1


def words_of(rows: int, width: int) -> int:
    return (rows + 63) // 64 * width


def pack(values, rows=None):
    """(base, width, words) of values[:rows]; each 64-row block is its own width-word run of the stream"""
    vals = [int(v) for v in (values.tolist() if hasattr(values, "tolist") else values)]
    rows = len(vals) if rows is None else rows
    vals = vals[:rows]
    base = min(vals)
    width = (max(vals) - base).bit_length()
    words = []
    for b0 in range(0, rows, 64):
        block = 0
        for i, v in enumerate(vals[b0:b0 + 64]):
            block |= (v - base) << (i * width)
        words += [(block >> (64 * k)) & MASK64 for k in range(width)]
    assert len(words) == words_of(rows, width)
    return base, width, np.array(words, np.uint64)


@dataclass
class NarrowLayout:
    groups: list                          # [(first row, rows)] per chunk group, in shard order
    staged: list                          # attribute per staged slot
    col_narrow: dict                      # attribute -> the column has images
    image: dict = field(default_factory=dict)      # (chunk group, attribute) -> (base, width) or None
    offs: dict = field(default_factory=dict)       # (chunk group, attribute) -> byte offset of its stream
    nullfree: dict = field(default_factory=dict)   # (chunk group, attribute) -> no NULLs in the chunk column
    values: dict = field(default_factory=dict)     # (chunk group, attribute) -> non-NULL values of the chunk column
    total: int = 0                                  # bytes of all streams
    any_images: bool = False

    @property
    def narrow_bytes(self) -> int:
        """cg_shard_narrow_bytes"""
        return self.total + len(self.groups) * len(self.staged) * DEVPACKCOL_BYTES if self.any_images else 0

    def stream_bytes(self, g: int, att: int) -> int:
        """bytes of the chunk column's stream, what the fast kernel reads of it (0: no image)"""
        im = self.image.get((g, att))
        return 0 if im is None else words_of(self.groups[g][1], im[1]) * 8

    def plain_bytes(self, g: int, att: int) -> int:
        """bytes of the chunk column in the plain arena a kernel reads: the values and the exists bitmap"""
        return len(self.values[(g, att)]) * 8 + (self.groups[g][1] + 7) // 8

    def scan_bytes(self, plan_atts, selected, narrow: bool) -> int:
        """bytes_scanned of one scan over the selected chunk groups (a list of flags, one per chunk group): with narrow, the
        fast kernel reads the streams of the chunk groups whose plan columns have no NULLs; everything else is plain"""
        total = 0
        for g, kept in enumerate(selected):
            if not kept:
                continue
            fast = narrow and all(self.nullfree[(g, a)] for a in plan_atts)
            total += sum(self.stream_bytes(g, a) if fast else self.plain_bytes(g, a) for a in plan_atts)
        return total

    def narrow_plan(self, plan_atts) -> bool:
        """the fast kernel reads the images: one to three plan columns, each with images"""
        return self.any_images and 1 <= len(plan_atts) <= 3 and all(self.col_narrow[a] for a in plan_atts)


def narrow_layout(cols, nulls, layout, staged, candidate=None) -> NarrowLayout:
    """cols / nulls: per attribute, the values and NULL flags (None: no NULLs) of the relation's rows; layout:
    reference.chunk_layout of the relation; staged: attributes in slot order; candidate: attribute -> 8-byte integer
    column (default: every one)"""
    groups = [g for stripe in layout for g in stripe]
    nulls = list(nulls or []) + [None] * (len(cols) - len(nulls or []))
    out = NarrowLayout(groups, list(staged), {})
    for g, (first, rows) in enumerate(groups):
        for a in staged:
            v = [int(x) for x in cols[a][first:first + rows]]
            if nulls[a] is not None:
                v = [x for x, n in zip(v, nulls[a][first:first + rows]) if not n]
            out.values[(g, a)] = v
            out.nullfree[(g, a)] = len(v) == rows and rows > 0
    is_cand = {a: candidate is None or bool(candidate[a]) for a in staged}
    fits = {}
    for a in staged:
        spans = [max(out.values[(g, a)]) - min(out.values[(g, a)]) for g in range(len(groups)) if out.nullfree[(g, a)]]
        fits[a] = is_cand[a] and all(s < (1 << MAX_WIDTH) for s in spans)
    out.any_images = any(fits.values()) and \
        any(is_cand[a] and out.nullfree[(g, a)] for g in range(len(groups)) for a in staged)
    out.col_narrow = {a: out.any_images and fits[a] for a in staged}
    off = 0
    for g, (first, rows) in enumerate(groups):
        for a in staged:
            out.image[(g, a)] = None
            if not (out.any_images and out.col_narrow[a] and out.nullfree[(g, a)]):
                continue
            v = out.values[(g, a)]
            out.image[(g, a)] = (min(v), (max(v) - min(v)).bit_length())
            out.offs[(g, a)] = off
            off += (words_of(rows, out.image[(g, a)][1]) * 8 + 15) // 16 * 16
    out.total = off if out.any_images else 0
    return out
