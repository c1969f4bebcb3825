"""A plain model of the fused scan's group table, in Python integers: what cg_partial_create chooses (table kind,
capacity, stride, packing shift), what the table's words hold, the packed word (sum << C) + n and its decoding, the drain
schedule that bounds how many rows a packed word takes between drains (and so exactly when a read must report
CG_ERETRY_UNPACKED), the generated small-domain kernel's narrow per-lane cells and launch cutting, and linear probing in
the hash table.  Row semantics (WHERE, terms, NULLs) are tests/reference.py's; this module only says where the rows go.
"""
from __future__ import annotations

from dataclasses import dataclass, field

MASK64 = (1 << 64) - 1
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
DENSE_LIMIT = 1 << 26            # key_max - key_min below this: a direct-indexed table
HASH_EMPTY = I64_MIN             # the hash table's empty-slot key; that key itself has an entry of its own
GOLDEN = 0x9E3779B97F4A7C15      # home slot = (key * GOLDEN mod 2^64) >> (64 - log2 capacity)
GOLDEN_INV = pow(GOLDEN, -1, 1 << 64)
PROBE_LIMIT = 8192               # slots a lookup examines before it reports the table full
DRAIN_DIVISOR = 32               # drain when rows since the last drain exceed capacity * 2^C / 32
NARROW_ROWS_CAP = 160            # rows a lane may see per launch when two 32-bit sums share a 64-bit cell
LANE_ROWS_CAP = 1 << 22          # the same for the 64-bit cells
JIT_THREADS, JIT_R = 256, 2      # the generated kernel: threads per CTA, rows per thread and step
SMALL_MAX_ENTRIES, SMALL_MAX_BYTES, MIN_BLOCKS4_BYTES = 4096, 200 * 1024, 55 * 1024


def s64(x):
    x &= MASK64
    return x - (1 << 64) if x >> 63 else x


def s32(x):
    x &= 0xFFFFFFFF
    return x - (1 << 32) if x >> 31 else x


def pow2_at_least(n):
    c = 1
    while c < n:
        c <<= 1
    return c


# --------------------------------------------------------------------------- table shape
@dataclass
class Shape:
    mode: str                    # "global" | "dense" | "hash"
    capacity: int                # addressable slots
    entries: int                 # + the NULL entry (dense, hash) and the HASH_EMPTY key's entry (hash)
    stride: int                  # words per entry, a power of two


def table_shape(ngroup_cols, key_min, key_max, expected_groups, nwords):
    """cg_partial_shape for one group column (or a composite code) and for two group columns, whose key_min / key_max
    carry the two columns' bounds packed like the key (low 32 bits: the first column)"""
    stride = pow2_at_least(nwords)
    if ngroup_cols == 0:
        return Shape("global", 1, 1, nwords)
    if ngroup_cols == 2:
        lo0, hi0 = s32(key_min), s32(key_max)
        lo1, hi1 = s32(key_min >> 32), s32(key_max >> 32)
        if lo0 <= hi0 and lo1 <= hi1 and (hi0 - lo0 + 1) * (hi1 - lo1 + 1) < DENSE_LIMIT:
            cap = (hi0 - lo0 + 1) * (hi1 - lo1 + 1)
            return Shape("dense", cap, cap + 1, stride)
    elif key_min <= key_max and key_max - key_min < DENSE_LIMIT:
        cap = key_max - key_min + 1
        return Shape("dense", cap, cap + 1, stride)
    cap = pow2_at_least(max(1024, 4 * expected_groups) if expected_groups > 0 else 1 << 22)
    return Shape("hash", cap, cap + 2, stride)


def dense_slot(key, key_min, key_min1=None, range1=None):
    """entry of a key in a direct-indexed table; two columns: (k0 - min0) * range1 + (k1 - min1)"""
    if key_min1 is None:
        return key - key_min
    return (s32(key) - key_min) * range1 + (s32(key >> 32) - key_min1)


# --------------------------------------------------------------------------- packing
def pack_shift(bound):
    """C of cg_partial_create for the first bounded one-word integer sum: R = bound's bit length (at most 62),
    C = (63 - R) // 2 clamped to 24; None (no packing) when C < 12 or there is no bound"""
    if bound <= 0:
        return None
    c = (63 - min(bound.bit_length(), 62)) // 2
    return None if c < 12 else min(c, 24)


def bound_for_shift(c):
    """the largest term bound that gives shift c (c < 24), or the largest that gives 24"""
    r = 63 - 2 * c if c < 24 else 15
    return (1 << r) - 1


def pack(s, n, c):
    return ((s << c) + n) & MASK64


def unpack(w, c):
    """(n, sum) of a packed word whose row count is below 2^C"""
    n = w & ((1 << c) - 1)
    return n, s64(w - n) >> c


@dataclass
class PackedTable:
    """The packed words of one partial and their drains, launch by launch.  A launch adds, per slot, its rows and the sum
    of their terms; `rows_scanned` is what the host counts for the launch (every row of its chunk groups, filtered or
    not).  Reads drain (or decode) and compare the rows added with the rows that came out again."""
    capacity: int
    c: int
    words: dict = field(default_factory=dict)
    wide: dict = field(default_factory=dict)      # slot -> [n, sum] drained so far
    window: dict = field(default_factory=dict)    # slot -> rows since the last drain
    added: int = 0
    drained: int = 0
    rows_since_drain: int = 0
    read_direct: bool = False
    overflowed: bool = False                      # some slot took >= 2^C rows between two drains

    def drain_due(self):
        return self.rows_since_drain * DRAIN_DIVISOR > self.capacity << self.c

    def launch(self, rows_scanned, per_slot):
        """per_slot: slot -> (rows, sum of terms)"""
        if self.read_direct:            # before_scan: a partial read straight from its packed words drains first
            self.drain()
        for slot, (n, s) in per_slot.items():
            self.words[slot] = (self.words.get(slot, 0) + pack(s, n, self.c)) & MASK64
            self.window[slot] = self.window.get(slot, 0) + n
            self.overflowed |= self.window[slot] >= 1 << self.c
            self.added += n
        self.rows_since_drain += rows_scanned
        if self.drain_due():
            self.drain()

    def drain(self):
        for slot, w in self.words.items():
            n, s = unpack(w, self.c)
            acc = self.wide.setdefault(slot, [0, 0])
            acc[0] += n
            acc[1] = s64(acc[1] + s)
            self.drained += n
        self.words, self.window, self.rows_since_drain, self.read_direct = {}, {}, 0, False

    def read(self):
        """the groups {slot: (n, sum)} a read returns, or None for CG_ERETRY_UNPACKED"""
        self.drain()
        if self.added != self.drained:
            return None
        return {k: tuple(v) for k, v in self.wide.items() if v[0]}


@dataclass
class PartialFlags:
    """packed_dirty, wide_dirty and read_packed_direct of a partial with packed words, as the host code moves them, for
    programs that stay below the drain limit (no drain after a launch)"""
    packing: bool = True         # cg_partial_set_packing
    packed: bool = False         # packed words were added since the last drain or reset
    wide: bool = False           # the wide words were written since the last reset
    direct: bool = False         # a read decoded result rows straight from the packed words

    def drain(self):
        if self.packed:
            self.packed, self.wide, self.direct = False, True, False

    def scan(self, packs, packed_only):
        """packs: the kernel that takes the rows writes packed words when packing is on; packed_only: nothing else"""
        if self.direct:          # a partial read straight from its packed words is drained before it is scanned again
            self.drain()
        if self.packing and packs:
            self.packed = True
            self.wide |= not packed_only
        else:
            self.wide = True

    def read(self, direct_form):
        """direct_form: a direct-indexed table of one key column, whose rows can be decoded from the packed words"""
        if direct_form and self.packed and not self.wide:
            self.direct = True
        else:
            self.drain()

    def merge(self):             # merged rows go to the wide words; the merge then checks the partial, which drains
        self.wide = True
        self.drain()

    def reset(self):
        self.packed = self.wide = self.direct = False

    def set_packing(self, on):
        """False: CG_EINVAL (packed words are pending)"""
        if self.packed:
            return False
        self.packing = on
        return True


# --------------------------------------------------------------------------- the generated small-domain kernel
@dataclass
class NarrowShape:
    kind: str                    # "small" | "table"
    candidates: list             # sums that may hold 32-bit halves: tbound * 160 < 2^31
    rows_partner: int            # the candidate in the high half of cell 0 (the row count is its low half), -1 = none
    pairs: list                  # (low-half sum, high-half sum): the low half holds sum(term + tbound)
    nhot: int                    # 64-bit cells per group
    smem: int
    lane_rows_cap: int
    min_blocks: int


def narrow_shape(capacity, sums):
    """choose_shape of a direct-indexed plan of count(*) and integer sums without FILTERs.  sums: [(tbound, nlimbs) or
    (tbound, nlimbs, nullable input)] in aggregate order (the count(*) is not listed); indexes in the result count sums
    from 0.  A sum whose input may be NULL never takes a low (biased) half: its bias would need its own row count"""
    sums = [tuple(s) + (False,) * (3 - len(s)) for s in sums]
    cand = [i for i, (t, _, _) in enumerate(sums) if t > 0 and t * NARROW_ROWS_CAP < 1 << 31]
    pairs, taken = [], set(cand[:1])
    for x in cand[1:]:
        if x in taken or sums[x][2]:
            continue
        y = next((j for j in cand[1:] if j != x and j not in taken), None)
        if y is None:
            break
        pairs.append((x, y))
        taken |= {x, y}
    nhot = 1 + len(pairs)
    for i, (t, nlimbs, _) in enumerate(sums):
        if i not in taken:
            nhot += 1 if nlimbs == 1 or (t > 0 and t * LANE_ROWS_CAP < 1 << 63) else 2
    smem = capacity * nhot * 8 * JIT_THREADS
    if capacity <= SMALL_MAX_ENTRIES and smem <= SMALL_MAX_BYTES:
        return NarrowShape("small", cand, cand[0] if cand else -1, pairs, nhot, smem,
                           NARROW_ROWS_CAP if cand else LANE_ROWS_CAP, 4 if smem + 4096 <= MIN_BLOCKS4_BYTES else 0)
    return NarrowShape("table", cand, -1, [], nhot, 0, LANE_ROWS_CAP, 0)


def interp_small_eligible(capacity, hot_words):
    """cg_small_eligible: the ahead-of-time shared-memory kernel keeps a per-lane table of every hot word (the row count,
    each aggregate's value words) in 200 KB"""
    return capacity * hot_words * 8 * JIT_THREADS <= SMALL_MAX_BYTES


def rows_per_cg_lane(cg_rows):
    step = JIT_THREADS * JIT_R
    return -(-cg_rows // step) * JIT_R


def cgs_per_cta(cg_rows, lane_rows_cap=NARROW_ROWS_CAP):
    """chunk groups one CTA may take per launch (0: the generated kernel declines the chunk groups)"""
    return lane_rows_cap // rows_per_cg_lane(cg_rows)


def jit_small_launches(nselected, cg_rows, grid_full, lane_rows_cap=NARROW_ROWS_CAP):
    per = cgs_per_cta(cg_rows, lane_rows_cap)
    return -(-nselected // (per * grid_full)) if per else 0


# --------------------------------------------------------------------------- hash addressing
def hash_shift(capacity):
    return 64 - (capacity.bit_length() - 1)


def home_slot(key, capacity):
    return ((key * GOLDEN) & MASK64) >> hash_shift(capacity)


def key_with_home(slot, j, capacity):
    """the j-th key (j < 2^(64 - log2 capacity)) whose home slot is `slot`: its product with GOLDEN is slot's prefix
    followed by j"""
    return s64(((slot << hash_shift(capacity)) + j) * GOLDEN_INV)


def probe(keys, capacity, limit=PROBE_LIMIT):
    """linear probing in the given order: (key -> slot, longest probe sequence); a key that finds neither itself nor an
    empty slot within `limit` slots maps to None.  The NULL key and HASH_EMPTY have entries of their own: not here."""
    table, where, longest = {}, {}, 0
    for k in keys:
        if k is None or k == HASH_EMPTY or k in where:
            continue
        h = home_slot(k, capacity)
        for p in range(min(limit, capacity)):
            s = (h + p) % capacity
            if s not in table:
                table[s] = k
                where[k] = s
                longest = max(longest, p + 1)
                break
        else:
            where[k] = None
    return where, longest


def occupied_runs(slots, capacity):
    """lengths of the maximal runs of occupied slots, a run that wraps from capacity - 1 to 0 counted once"""
    occ = set(slots)
    if len(occ) == capacity:
        return [capacity]
    start = next(s for s in range(capacity) if s not in occ)
    runs, cur = [], 0
    for i in range(1, capacity + 1):
        s = (start + i) % capacity
        if s in occ:
            cur += 1
        elif cur:
            runs.append(cur)
            cur = 0
    return runs


def hash_verdict(keys, capacity):
    """what a scan of these keys into a hash table may answer: "exact" (every run of occupied slots is shorter than the
    probe limit and every key has a slot), "full" (more distinct keys than slots: CG_ETABLEFULL) or "either".  The set of
    occupied slots does not depend on the order the keys arrive in, and a key's slot lies in the run that holds its home
    slot, so the claim holds for every interleaving of the kernel's threads."""
    distinct = {k for k in keys if k is not None and k != HASH_EMPTY}
    if len(distinct) > capacity:
        return "full"
    where, _ = probe(sorted(distinct), capacity, limit=capacity)
    runs = occupied_runs(where.values(), capacity)
    return "exact" if max(runs, default=0) < PROBE_LIMIT else "either"


# --------------------------------------------------------------------------- the wide table
def dense_words(groups, shape, key_min, nwords):
    """the [entry][stride] words of a drained direct-indexed table of ADD words: groups {key or None: [nwords word
    values]}; every other word, padding included, is 0 (the identity of ADD); the NULL group's entry is at `capacity`"""
    out = [0] * (shape.entries * shape.stride)
    for key, words in groups.items():
        e = shape.capacity if key is None else dense_slot(key, key_min)
        for w in range(nwords):
            out[e * shape.stride + w] = words[w] & MASK64
    return out
