"""Host-side handles over the C-ABI, named after the reference interfaces they stand for.

  Relation           a columnar relation image: pages + columnar.stripe / columnar.chunk rows
  ScanDesc helpers   ColumnarBeginRead's projectedColumnList / qualConditions + the worker
                     half of the aggregates (columnar.h:251-258, multi_logical_optimizer.c:3160)
  GpuColumnarAgg     the  Agg <- ColumnarScan  subtree of one worker task (SURVEY.md 3.3),
                     executed by the fused kernel; also the coordinator-side combine
  worker_partition_query_result   executor/partitioned_intermediate_results.c:115-298 (map side)

Everything computes on the GPU through libcitus_gpu.so; nothing here has a CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import capi
from .capi import (CG_AGG_COUNT, CG_AGG_COUNT_STAR, CG_AGG_MAX, CG_AGG_MIN, CG_AGG_SUM, CG_TYPE_FLOAT,
                   CG_TYPE_INT, CgAggSpec, CgColumnDesc, CgGenColumn, CgQual, CgRelation, CgScanDesc,
                   CgScanStats, CgSkipNode, CgStripe, check, lib)

_initialised = False
_on_torch_stream = None      # handle of the torch stream the library was put on (use_torch_stream)


def init(device: int = 0):
    global _initialised
    check(lib().cg_init(device))
    _initialised = True


def set_option(name: str, value: int):
    """cg_set_option: "jit" 0/1/2, "force_general" 0/1, "narrow_images" 0/1, ... (include/citus_gpu.h)"""
    check(lib().cg_set_option(name.encode(), value))


def numa_bind() -> int:
    """pin this thread (and the staging/generator threads created after it) to the CPUs of the
    device's NUMA node; returns the node or -1"""
    node = C.c_int32(-1)
    check(lib().cg_numa_bind(C.byref(node)))
    return node.value


def numa_unbind():
    check(lib().cg_numa_unbind())


def use_torch_stream():
    """run the library's kernels on torch's current stream, so that torch ops, NCCL collectives and
    the library's kernels are ordered in one queue (torch's default stream is CUDA's legacy default
    stream, whose handle is 0: it is passed as cudaStreamLegacy = 1)"""
    import torch
    global _on_torch_stream
    h = torch.cuda.current_stream().cuda_stream
    check(lib().cg_set_stream(C.c_void_p(h if h else 1)))
    _on_torch_stream = h


class Relation:
    """Owns (or borrows) a relation image and exposes it as a CgRelation."""

    def __init__(self):
        self._gen = None
        self._keep = []
        self.view = CgRelation()

    # -- constructors -------------------------------------------------------
    @classmethod
    def generate(cls, columns, nrows, seed, first_row=0, stripe_row_limit=150000, chunk_row_limit=10000,
                 nthreads=8):
        """columns: [(attlen, kind, lo, hi, null_ppm)] -- splitmix64 counter-based synthetic data"""
        self = cls()
        arr = (CgGenColumn * len(columns))()
        for i, (attlen, kind, lo, hi, null_ppm) in enumerate(columns):
            arr[i].attlen, arr[i].kind, arr[i].lo, arr[i].hi, arr[i].null_ppm = attlen, kind, lo, hi, null_ppm
        h = C.c_void_p()
        check(lib().cg_gen_relation(arr, len(columns), nrows, first_row, seed, stripe_row_limit,
                                    chunk_row_limit, nthreads, C.byref(h)))
        self._gen = h
        check(lib().cg_gen_relation_view(h, C.byref(self.view)))
        return self

    @classmethod
    def write(cls, attlens, values, nulls=None, type_classes=None, stripe_row_limit=150000, chunk_row_limit=10000):
        """encode caller-supplied columns (int64 arrays; float64 arrays for float columns)"""
        self = cls()
        natts = len(attlens)
        type_classes = type_classes or [CG_TYPE_INT] * natts
        cols = (CgColumnDesc * natts)()
        for i in range(natts):
            cols[i].attlen, cols[i].type_class = attlens[i], type_classes[i]
        vals = []
        for i, v in enumerate(values):
            if type_classes[i] == CG_TYPE_FLOAT:
                vals.append(np.ascontiguousarray(v, np.float64).view(np.int64))
            else:
                vals.append(np.ascontiguousarray(v, np.int64))
        n = vals[0].shape[0] if vals else 0
        vp = (C.c_void_p * natts)(*[v.ctypes.data for v in vals])
        np_ = None
        nk = []
        if nulls is not None:
            nk = [None if x is None else np.ascontiguousarray(x, np.uint8) for x in nulls]
            np_ = (C.c_void_p * natts)(*[None if x is None else x.ctypes.data for x in nk])
        h = C.c_void_p()
        check(lib().cg_write_relation(cols, natts, vp, np_, n, stripe_row_limit, chunk_row_limit, C.byref(h)))
        self._gen = h
        check(lib().cg_gen_relation_view(h, C.byref(self.view)))
        return self

    @classmethod
    def from_image(cls, pages: np.ndarray, stripes_bytes: np.ndarray, nodes_bytes: np.ndarray, attlens,
                   type_classes=None):
        """borrow an image produced elsewhere (e.g. by the oracle's writer in tests)"""
        self = cls()
        natts = len(attlens)
        type_classes = type_classes or [CG_TYPE_INT] * natts
        cols = (CgColumnDesc * natts)()
        for i in range(natts):
            cols[i].attlen, cols[i].type_class = attlens[i], type_classes[i]
        pages = np.ascontiguousarray(pages, np.uint8)
        stripes_bytes = np.ascontiguousarray(stripes_bytes, np.uint8)
        nodes_bytes = np.ascontiguousarray(nodes_bytes, np.uint8)
        self._keep = [pages, stripes_bytes, nodes_bytes, cols]
        v = self.view
        v.pages = pages.ctypes.data
        v.nblocks = pages.shape[0] // 8192
        v.stripes = C.cast(stripes_bytes.ctypes.data, C.POINTER(CgStripe))
        v.nstripes = stripes_bytes.shape[0] // C.sizeof(CgStripe)
        v.nodes = C.cast(nodes_bytes.ctypes.data, C.POINTER(CgSkipNode))
        v.nnodes = nodes_bytes.shape[0] // C.sizeof(CgSkipNode)
        v.columns = cols
        v.natts = natts
        return self

    def prefix(self, nstripes: int) -> "Relation":
        """the first `nstripes` stripes of this relation as a relation of its own (shares the image)"""
        r = Relation()
        r._keep = [self]
        C.memmove(C.byref(r.view), C.byref(self.view), C.sizeof(CgRelation))
        r.view.nstripes = max(0, min(nstripes, self.view.nstripes))
        return r

    def register(self):
        """pin the page image (cudaHostRegister): cg_scan_relation then uses DMA staging"""
        check(lib().cg_relation_register(C.byref(self.view)))
        self._registered = True

    def unregister(self):
        if getattr(self, "_registered", False):
            lib().cg_relation_unregister(C.byref(self.view))
            self._registered = False

    def __del__(self):
        try:
            self.unregister()
            if getattr(self, "_gen", None):
                lib().cg_gen_relation_free(self._gen)
                self._gen = None
        except TypeError:           # interpreter shutdown: module globals are already gone
            pass

    # -- accessors ----------------------------------------------------------
    @property
    def natts(self):
        return self.view.natts

    @property
    def rows(self):
        return sum(self.view.stripes[i].row_count for i in range(self.view.nstripes))

    def pages(self) -> np.ndarray:
        n = self.view.nblocks * 8192
        return np.ctypeslib.as_array(C.cast(self.view.pages, C.POINTER(C.c_uint8)), shape=(n,))

    def stripes_bytes(self) -> np.ndarray:
        n = self.view.nstripes * C.sizeof(CgStripe)
        return np.frombuffer(C.string_at(self.view.stripes, n), np.uint8).copy()

    def nodes_bytes(self) -> np.ndarray:
        n = self.view.nnodes * C.sizeof(CgSkipNode)
        return np.frombuffer(C.string_at(self.view.nodes, n), np.uint8).copy()

    def column_descs(self):
        return [(self.view.columns[i].attlen, self.view.columns[i].type_class) for i in range(self.view.natts)]


# ---------------------------------------------------------------------------
# query description helpers
# ---------------------------------------------------------------------------
@dataclass
class Agg:
    kind: int
    factors: list = field(default_factory=list)    # [(column, a, b)]
    is_float: bool = False
    term_abs_bound: int = 0
    filter: object = None        # FILTER (WHERE ...): a WHERE-style tree of (column, op, constant) atoms, None = none
    arg: object = None           # bool_and / bool_or: the predicate argument, a tree in the same form as `filter`
    case: object = None          # a Case argument (then factors is empty), None = none


@dataclass(frozen=True)
class Const:
    """a constant CASE result: an integer (pre-scaled to the aggregate's scale), or a float for a float aggregate"""
    value: object


_NO_ELSE = object()


@dataclass
class Case:
    """CASE WHEN tree THEN result ... [ELSE result] END as an aggregate argument: arms = [(tree, result), ...] with trees in
    the FILTER form (they share the FILTER atom pool); a result is None (NULL), Const(k), a column index, or a factor list
    [(column, a, b), ...] (a product of at most three affine factors).  Without else_ the value of a row no tree accepts
    is NULL."""
    arms: list
    else_: object = _NO_ELSE


def _arg(kind, col, is_float=False, filter=None):
    if isinstance(col, Case):
        return Agg(kind, [], is_float, filter=filter, case=col)
    return Agg(kind, [(col, 0, 1)], is_float, filter=filter)


def count_star(filter=None):
    return Agg(CG_AGG_COUNT_STAR, filter=filter)


def count(col, filter=None, is_float=False):
    """count(x); with a Case, is_float says whether its results are float (their NULLs are what count counts)"""
    return _arg(CG_AGG_COUNT, col, is_float, filter)


def sum_(col, is_float=False, filter=None):
    return _arg(CG_AGG_SUM, col, is_float, filter)


def min_(col, is_float=False, filter=None):
    return _arg(CG_AGG_MIN, col, is_float, filter)


def max_(col, is_float=False, filter=None):
    return _arg(CG_AGG_MAX, col, is_float, filter)


def bit_and(col, filter=None):
    """bit_and(col) over an int2 / int4 / int8 column: the value comes back sign-extended in minmax"""
    return Agg(capi.CG_AGG_BIT_AND, [(col, 0, 1)], filter=filter)


def bit_or(col, filter=None):
    return Agg(capi.CG_AGG_BIT_OR, [(col, 0, 1)], filter=filter)


def bool_and(tree, filter=None):
    """bool_and(p) (and every(p)) of a predicate tree in the WHERE form: minmax 0 / 1, count = rows whose p is known"""
    return Agg(capi.CG_AGG_BOOL_AND, filter=filter, arg=tree)


def bool_or(tree, filter=None):
    return Agg(capi.CG_AGG_BOOL_OR, filter=filter, arg=tree)


def variance(col, filter=None):
    """the state of var_pop / var_samp / variance / stddev_pop / stddev_samp / stddev over an integer column: fetch()
    gives N in count, sum(x) in sum and sum(x^2) in sumsq; numeric_var_out() makes the SQL value"""
    return _arg(capi.CG_AGG_VARIANCE, col, filter=filter)


def _f8(x):
    return int(np.float64(x).view(np.int64))


def _case_arm(tokens, result, is_float):
    """one arm as (nwhen tokens, form, columns, a, b): the descriptor's CgCaseArm fields"""
    if result is None:
        return (tuple(tokens), capi.CG_CASE_NULL, (), (0,), ())
    if isinstance(result, Const):
        return (tuple(tokens), capi.CG_CASE_CONST, (), (_f8(result.value) if is_float else int(result.value),), ())
    factors = [(result, 0, 1)] if isinstance(result, (int, np.integer)) else list(result)
    if not 1 <= len(factors) <= 3:
        raise ValueError("a CASE product has 1 to 3 factors")
    conv = _f8 if is_float else int
    return (tuple(tokens), capi.CG_CASE_PRODUCT, tuple(int(c) for c, _, _ in factors), tuple(conv(a) for _, a, _ in factors),
            tuple(conv(b) for _, _, b in factors))


def flatten_where(where):
    """WHERE as a nested tuple tree -- ("and" | "or", arm, arm, ...) over atoms (column, op, constant), (column, op,
    Col(other)), (column, "in" |
    "not in", (value, ...)) and (column, "is null" | "is not null"); a plain list of atoms is their AND -- to (atoms, postfix
    tokens).  The tokens are empty for a plain AND-list."""
    if not (isinstance(where, tuple) and where and where[0] in ("and", "or")):
        return list(where), []
    atoms, tokens = [], []

    def walk(node):
        if isinstance(node, tuple) and node and node[0] in ("and", "or"):
            if len(node) < 2:
                raise ValueError("empty boolean node")
            walk(node[1])
            for arm in node[2:]:
                walk(arm)
                tokens.append(capi.CG_QX_AND if node[0] == "and" else capi.CG_QX_OR)
        else:
            tokens.append(len(atoms))
            atoms.append(tuple(node))

    walk(where)
    return atoms, tokens


def _filter_tokens(tree, pool):
    """one aggregate's FILTER tree -> postfix tokens over the shared filter atom pool (new atoms are appended to it; an
    atom already in the pool, e.g. the same filter on several aggregates, is reused).  A list of atoms is their AND; a
    bare atom is a tree of one atom."""
    if isinstance(tree, list):
        tree = ("and", *tree) if len(tree) > 1 else tree[0]
    if isinstance(tree, tuple) and tree and tree[0] in ("and", "or"):
        atoms, tokens = flatten_where(tree)
    else:
        atoms, tokens = [tuple(tree)], [0]
    index = []
    for atom in atoms:
        if atom not in pool:
            pool.append(atom)
        index.append(pool.index(atom))
    return [index[t] if t >= 0 else t for t in tokens]


def _konst(k, col, float_cols):
    return int(np.float64(k).view(np.int64)) if col in float_cols else int(k)


@dataclass(frozen=True)
class Col:
    """the right-hand side of a column-to-column atom: (0, "<", Col(3)) is "column 0 < column 3" of the same row"""
    index: int


def _set_atom(q, atom, float_cols, lists):
    """one atom: (column, op, constant); (column, op, Col(other)); (column, "in" | "not in", (v, ...)) with None for a NULL
    element -- the list goes to `lists`, [(elements, float?)], and konst is its index; (column, "is null" | "is not null")"""
    col, op = atom[0], atom[1]
    q.column = col
    if len(atom) == 3 and isinstance(atom[2], Col):
        q.op = capi.CG_OP["col " + op]
        q.konst = atom[2].index
        return
    q.op = capi.CG_OP[op]
    if op in ("is null", "is not null"):
        if len(atom) != 2:
            raise ValueError(f"{op} takes no constant")
        q.konst = 0
    elif op in ("in", "not in"):
        key = (tuple(atom[2]), col in float_cols)
        if not key[0]:
            raise capi.CitusGpuError(capi.CG_EUNSUPPORTED, "an empty IN list")
        if key not in lists:
            lists.append(key)
        q.konst = lists.index(key)
    else:
        q.konst = _konst(atom[2], col, float_cols)


def _set_lists(d, lists):
    """the list table of a descriptor: every list's non-NULL elements back to back, in konst's convention (NULL elements
    are only counted, so they take no room in in_values)"""
    if len(lists) > capi.CG_MAX_IN_LISTS or sum(sum(v is not None for v in vals) for vals, _ in lists) > capi.CG_MAX_IN_VALUES:
        raise capi.CitusGpuError(capi.CG_EUNSUPPORTED, "IN lists too large")
    d.nin_lists = len(lists)
    n = 0
    for i, (values, is_float) in enumerate(lists):
        vals = [v for v in values if v is not None]
        d.in_lists[i].first, d.in_lists[i].nvalues, d.in_lists[i].nnulls = n, len(vals), len(values) - len(vals)
        for v in vals:
            d.in_values[n] = int(np.float64(v).view(np.int64)) if is_float else int(v)
            n += 1
    d.nin_values = n


def make_desc(quals=(), group_cols=(), aggs=(), qual_pushdown=True, expected_groups=0, float_cols=(), composite=False,
              key_bounds=None):
    """composite=True: the GROUP BY key is the exact mixed-radix code over group_cols (1..4 columns, NULLs included);
    key_bounds = [(min, max)] per group column (relation_key_bounds; min > max = the column is always NULL)"""
    d = CgScanDesc()
    if composite:
        d.composite_key = 1
        if key_bounds is None or len(key_bounds) != len(group_cols):
            raise ValueError("a composite key needs one (min, max) per group column")
        for i, (lo, hi) in enumerate(key_bounds):
            d.key_col_min[i], d.key_col_max[i] = lo, hi
    quals, tokens = flatten_where(quals)
    if len(quals) > capi.CG_MAX_QUALS or len(tokens) > capi.CG_MAX_QEXPR:
        raise capi.CitusGpuError(capi.CG_EUNSUPPORTED, "WHERE tree too large")
    d.nqual_expr = len(tokens)
    for i, t in enumerate(tokens):
        d.qual_expr[i] = t
    d.nquals = len(quals)
    lists = []                   # IN / NOT IN lists of WHERE and the pool: (elements, float column?)
    for i, atom in enumerate(quals):
        _set_atom(d.quals[i], atom, float_cols, lists)
    pool = []                    # FILTERs and bool_and / bool_or arguments share one atom pool
    for i, a in enumerate(aggs):
        for tree, n, expr, what in ((a.filter, d.nfilter_expr, d.filter_expr, "FILTER"),
                                    (getattr(a, "arg", None), d.narg_expr, d.arg_expr, "bool_and / bool_or argument")):
            if tree is None:
                continue
            tok = _filter_tokens(tree, pool)
            if len(pool) > capi.CG_MAX_FILTER_QUALS or len(tok) > capi.CG_MAX_QEXPR:
                raise capi.CitusGpuError(capi.CG_EUNSUPPORTED, f"{what} trees too large")
            n[i] = len(tok)
            for j, t in enumerate(tok):
                expr[i][j] = t
    # CASE arms: WHEN trees over the same pool; identical arm lists (avg's sum and count) share one range
    arms, ranges = [], {}
    for i, a in enumerate(aggs):
        if a.case is None:
            continue
        lst = [_case_arm(_filter_tokens(tree, pool), res, a.is_float) for tree, res in a.case.arms]
        if a.case.else_ is not _NO_ELSE:
            lst.append(_case_arm((), a.case.else_, a.is_float))
        if len(pool) > capi.CG_MAX_FILTER_QUALS or any(len(arm[0]) > capi.CG_MAX_QEXPR for arm in lst):
            raise capi.CitusGpuError(capi.CG_EUNSUPPORTED, "CASE WHEN trees too large")
        key = tuple(lst)
        if key not in ranges:
            ranges[key] = len(arms)
            arms.extend(lst)
        d.case_first[i], d.case_narms[i] = ranges[key], len(lst)
    if len(arms) > capi.CG_MAX_CASE_ARMS:
        raise capi.CitusGpuError(capi.CG_EINVAL, "too many CASE arms")        # the library's code for ncase_arms > CG_MAX_CASE_ARMS
    d.ncase_arms = len(arms)
    for k, (tokens, form, cols, aa, bb) in enumerate(arms):
        A = d.case_arms[k]
        A.nwhen, A.form, A.nfactors = len(tokens), form, len(cols)
        for j, t in enumerate(tokens):
            A.when[j] = t
        for f, c in enumerate(cols):
            A.column[f] = c
        for f, x in enumerate(aa):
            A.a[f] = x
        for f, x in enumerate(bb):
            A.b[f] = x
    d.nfilter_quals = len(pool)
    for i, atom in enumerate(pool):
        _set_atom(d.filter_quals[i], atom, float_cols, lists)
    _set_lists(d, lists)
    d.enable_qual_pushdown = 1 if qual_pushdown else 0
    d.ngroup_cols = len(group_cols)
    for i, c in enumerate(group_cols):
        d.group_cols[i] = c
    d.naggs = len(aggs)
    for i, a in enumerate(aggs):
        s = d.aggs[i]
        s.kind = a.kind
        s.nfactors = len(a.factors)
        s.is_float = 1 if a.is_float else 0
        s.term_abs_bound = a.term_abs_bound
        for f, (col, aa, bb) in enumerate(a.factors):
            s.column[f] = col
            if a.is_float:
                s.a[f] = int(np.float64(aa).view(np.int64))
                s.b[f] = int(np.float64(bb).view(np.int64))
            else:
                s.a[f], s.b[f] = aa, bb
    d.expected_groups = expected_groups
    return d


def relation_bounds(rel: Relation, desc: CgScanDesc):
    """exact key range / |sum argument| bounds / row count from the skip lists"""
    kmin, kmax, rows = C.c_int64(), C.c_int64(), C.c_int64()
    bounds = (C.c_int64 * capi.CG_MAX_AGGS)()
    check(lib().cg_relation_bounds(C.byref(rel.view), C.byref(desc), C.byref(kmin), C.byref(kmax), bounds, C.byref(rows)))
    return kmin.value, kmax.value, [bounds[i] for i in range(desc.naggs)], rows.value


def relation_key_bounds(rel: Relation, desc: CgScanDesc):
    """[(min, max)] of every group column over the chunk groups that survive skipping (min > max: no value)"""
    k = desc.ngroup_cols
    lo, hi = (C.c_int64 * capi.CG_MAX_GROUP_COLS)(), (C.c_int64 * capi.CG_MAX_GROUP_COLS)()
    check(lib().cg_relation_key_bounds(C.byref(rel.view), C.byref(desc), lo, hi))
    return [(lo[i], hi[i]) for i in range(k)]


def group_key_decode(desc: CgScanDesc, codes):
    """composite codes -> list of key tuples (None = NULL)"""
    codes = np.ascontiguousarray(codes, np.int64)
    n, k = codes.shape[0], desc.ngroup_cols
    values, nulls = np.zeros(n * k, np.int64), np.zeros(n * k, np.uint8)
    check(lib().cg_group_key_decode(C.byref(desc), n, codes.ctypes.data, values.ctypes.data, nulls.ctypes.data))
    return [tuple(None if nulls[i * k + c] else int(values[i * k + c]) for c in range(k)) for i in range(n)]


def group_key_encode(desc: CgScanDesc, keys):
    """key tuples (None = NULL) -> composite codes (int64 array)"""
    n, k = len(keys), desc.ngroup_cols
    values, nulls = np.zeros(n * k, np.int64), np.zeros(n * k, np.uint8)
    for i, key in enumerate(keys):
        for c, v in enumerate(key):
            if v is None:
                nulls[i * k + c] = 1
            else:
                values[i * k + c] = v
    codes = np.zeros(n, np.int64)
    check(lib().cg_group_key_encode(C.byref(desc), n, values.ctypes.data, nulls.ctypes.data, codes.ctypes.data))
    return codes


class Shard:
    """A relation's projected columns staged in HBM (cg_shard_stage)."""

    def __init__(self, rel: Relation, columns=None):
        self.rel = rel
        h = C.c_void_p()
        if columns is None:
            check(lib().cg_shard_stage(C.byref(rel.view), None, 0, C.byref(h)))
        else:
            arr = (C.c_int32 * len(columns))(*columns)
            check(lib().cg_shard_stage(C.byref(rel.view), arr, len(columns), C.byref(h)))
        self.h = h

    def free(self):
        if getattr(self, "h", None):
            lib().cg_shard_free(self.h)
            self.h = None

    __del__ = free

    @property
    def device_bytes(self):
        return lib().cg_shard_device_bytes(self.h)

    @property
    def rows(self):
        return lib().cg_shard_rows(self.h)

    def scan_rows(self, desc: CgScanDesc, atts, d_col_ptrs=None, d_null_ptrs=None, capacity=0, want_stats=True):
        """cg_scan_shard_rows: SELECT atts FROM shard WHERE <desc's WHERE tree> in the shard's row order, into the caller's
        device arrays (int64 values; a null list holds None or a device byte array per column, as join_aggregate takes
        them).  capacity 0 only counts.  Returns (passing rows, stats)."""
        atts_arr = (C.c_int32 * len(atts))(*atts)
        cols = None if d_col_ptrs is None else (C.c_void_p * len(d_col_ptrs))(*d_col_ptrs)
        nulls = None if d_null_ptrs is None else (C.c_void_p * len(d_null_ptrs))(*d_null_ptrs)
        n = C.c_int64()
        st = CgScanStats()
        check(lib().cg_scan_shard_rows(self.h, C.byref(desc), atts_arr, len(atts), capacity, cols, nulls, C.byref(n),
                                       C.byref(st) if want_stats else None))
        return n.value, st

    def narrow_image(self, cg: int, att: int):
        """(base, width, words: uint64 array) of the narrow image of attribute att in chunk group cg; width 255 = none"""
        base, width, n = C.c_int64(), C.c_uint32(), C.c_uint64()
        check(lib().cg_shard_narrow_image(self.h, cg, att, C.byref(base), C.byref(width), None, 0, C.byref(n)))
        words = np.zeros(n.value // 8, np.uint64)
        if n.value:
            check(lib().cg_shard_narrow_image(self.h, cg, att, C.byref(base), C.byref(width), words.ctypes.data, n.value,
                                              C.byref(n)))
        return base.value, width.value, words


class GpuColumnarAgg:
    """Partial aggregate of one worker task (or of all the tasks of one GPU), and the combine."""

    def __init__(self, desc: CgScanDesc, column_descs, key_min=0, key_max=-1, max_rows=0):
        self.desc = desc
        natts = len(column_descs)
        self.cols = (CgColumnDesc * natts)()
        for i, (l, t) in enumerate(column_descs):
            self.cols[i].attlen, self.cols[i].type_class = l, t
        h = C.c_void_p()
        check(lib().cg_partial_create(C.byref(desc), self.cols, natts, key_min, key_max, max_rows, C.byref(h)))
        self.h = h
        self.naggs = desc.naggs

    def free(self):
        if getattr(self, "h", None):
            lib().cg_partial_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except TypeError:           # interpreter shutdown
            pass

    def reset(self):
        check(lib().cg_partial_reset(self.h))

    def set_packing(self, enable: bool):
        check(lib().cg_partial_set_packing(self.h, 1 if enable else 0))

    def scan_shard(self, shard: Shard, want_stats=True):
        st = CgScanStats()
        check(lib().cg_scan_shard(shard.h, C.byref(self.desc), self.h, C.byref(st) if want_stats else None))
        return st

    def scan_relation(self, rel: Relation, want_stats=True):
        st = CgScanStats()
        check(lib().cg_scan_relation(C.byref(rel.view), C.byref(self.desc), self.h, C.byref(st) if want_stats else None))
        return st

    def join_aggregate(self, build_ptrs, build_key, nbuild, probe_ptrs, probe_key, nprobe, build_null_ptrs=None,
                       probe_null_ptrs=None, want_stats=True, columns=None):
        """cg_join_aggregate: this partial's query over the equi-join of two device-resident sides (device pointers of
        int64 columns, as join_rows takes them; a null list holds None or a device byte array per column).  The joined
        row's attributes are the build columns, then the probe columns; the partial's column descriptors describe them
        (columns = other descriptors [(attlen, type_class)] for this call only)"""
        keep = []

        def side(ptrs, nulls, key, n):
            cols = (C.c_void_p * len(ptrs))(*ptrs)
            nul = None if nulls is None else (C.c_void_p * len(ptrs))(*nulls)
            keep.extend([cols, nul])
            s = capi.CgJoinSide()
            s.d_cols = C.cast(cols, C.POINTER(C.c_void_p))
            s.d_nulls = None if nul is None else C.cast(nul, C.POINTER(C.c_void_p))
            s.ncols, s.key, s.nrows = len(ptrs), key, n
            return s

        b = side(build_ptrs, build_null_ptrs, build_key, nbuild)
        p = side(probe_ptrs, probe_null_ptrs, probe_key, nprobe)
        cols = self.cols
        if columns is not None:
            cols = (CgColumnDesc * len(columns))()
            for i, (l, t) in enumerate(columns):
                cols[i].attlen, cols[i].type_class = l, t
        st = CgScanStats()
        check(lib().cg_join_aggregate(C.byref(b), C.byref(p), cols, C.byref(self.desc), self.h,
                                      C.byref(st) if want_stats else None))
        return st

    def ngroups(self):
        n = C.c_int64()
        check(lib().cg_partial_ngroups(self.h, C.byref(n)))
        return n.value

    def layout(self):
        nw, dense, cap = C.c_int32(), C.c_int32(), C.c_int64()
        ops = (C.c_int32 * 32)()
        check(lib().cg_partial_layout(self.h, C.byref(nw), ops, C.byref(dense), C.byref(cap)))
        return nw.value, [ops[i] for i in range(nw.value)], bool(dense.value), cap.value

    def fetch(self, reuse=False):
        """dict: keys, key_nulls, sum (python ints [ngroups][naggs]), count, minmax, fsum.
        reuse=True returns views of buffers owned by this object (overwritten by the next fetch):
        what a caller with its own result memory -- a tuplestore -- does"""
        na = max(self.naggs, 1)
        bufs = getattr(self, "_fetch_bufs", None) if reuse else None
        cap = bufs[0].shape[0] if bufs else 0
        if not bufs:
            cap = max(self.ngroups(), 1)
        while True:
            if not bufs or bufs[0].shape[0] < cap:
                bufs = (np.zeros(cap, np.int64), np.zeros(cap, np.uint8), np.zeros(cap * na, np.int64),
                        np.zeros(cap * na, np.uint64), np.zeros(cap * na, np.int64), np.zeros(cap * na, np.int64),
                        np.zeros(cap * na, np.float64), np.zeros(cap * na * 3, np.uint64))
            keys, kn, hi, lo, cnt, mm, fs, sq = bufs
            got = C.c_int64()
            rc = lib().cg_partial_fetch_ex(self.h, keys.shape[0], keys.ctypes.data, kn.ctypes.data, hi.ctypes.data,
                                           lo.ctypes.data, cnt.ctypes.data, mm.ctypes.data, fs.ctypes.data, sq.ctypes.data,
                                           C.byref(got))
            if rc != 0 and reuse and got.value > keys.shape[0]:      # cached buffers too small for this result: grow once
                cap, bufs = got.value, None
                continue
            check(rc)
            break
        if reuse:
            self._fetch_bufs = bufs
        n = got.value
        return dict(n=n, keys=keys[:n], key_nulls=kn[:n], sum_hi=hi[:n * na].reshape(n, na),
                    sum_lo=lo[:n * na].reshape(n, na), count=cnt[:n * na].reshape(n, na),
                    minmax=mm[:n * na].reshape(n, na), fsum=fs[:n * na].reshape(n, na),
                    sumsq=sq[:n * na * 3].reshape(n, na, 3))

    def groups(self):
        """same shape as oracle.Result.groups(): key (None = NULL group) -> per-aggregate dicts.  A composite partial's
        keys are tuples with None for NULL (the shape tests/reference.py produces)"""
        f = self.fetch()
        keys = group_key_decode(self.desc, f["keys"]) if self.desc.composite_key else None
        out = {}
        for i in range(f["n"]):
            per = []
            for a in range(self.naggs):
                s = (int(f["sum_hi"][i, a]) << 64) + int(f["sum_lo"][i, a])
                d = dict(sum=s, count=int(f["count"][i, a]), minmax=int(f["minmax"][i, a]), fsum=float(f["fsum"][i, a]))
                if self.desc.aggs[a].kind == capi.CG_AGG_VARIANCE:
                    q = f["sumsq"][i, a]
                    d["sumsq"] = int(q[0]) | (int(q[1]) << 64) | (int(q[2]) << 128)
                per.append(d)
            if keys is not None:
                out[keys[i]] = per
            else:
                out[None if f["key_nulls"][i] else int(f["keys"][i])] = per
        return out

    def merge_values(self, keys, key_nulls, sum_hi, sum_lo, count, minmax, fsum):
        """cg_partial_merge_values over host rows laid out like fetch()'s.  For a composite partial, keys may be a list of
        key tuples (None = NULL): they are encoded to codes and key_nulls is ignored"""
        if self.desc.composite_key and len(keys) and isinstance(keys[0], tuple):
            keys, key_nulls = group_key_encode(self.desc, keys), None
        keys = np.ascontiguousarray(keys, np.int64)
        arrs = [None if x is None else np.ascontiguousarray(x, t) for x, t in
                ((key_nulls, np.uint8), (sum_hi, np.int64), (sum_lo, np.uint64), (count, np.int64), (minmax, np.int64),
                 (fsum, np.float64))]
        check(lib().cg_partial_merge_values(self.h, keys.shape[0], keys.ctypes.data,
                                            *[None if x is None else x.ctypes.data for x in arrs]))

    # -- combine (device arrays are torch tensors or any object with data_ptr()) ---------
    def export_device(self, d_keys_ptr, d_nulls_ptr, d_words_ptr, capacity):
        n = C.c_int64()
        check(lib().cg_partial_export_device(self.h, capacity, d_keys_ptr, d_nulls_ptr, d_words_ptr, C.byref(n)))
        return n.value

    def merge_rows(self, d_keys_ptr, d_nulls_ptr, d_words_ptr, nrows):
        check(lib().cg_partial_merge_rows(self.h, d_keys_ptr, d_nulls_ptr, d_words_ptr, nrows))

    def dense_words_enqueue(self):
        """like dense_words, but only enqueues the table maintenance (no host sync, no error check)"""
        p, total, stride = C.c_void_p(), C.c_int64(), C.c_int32()
        check(lib().cg_partial_dense_words_enqueue(self.h, C.byref(p), C.byref(total), C.byref(stride)))
        return p.value, total.value, stride.value

    def check(self):
        """wait for the partial's pending work and raise what its kernels flagged"""
        check(lib().cg_partial_check(self.h))

    def packed_state(self):
        """(pack_shift C, pack_word, state bits capi.CG_PSTATE_*, packed words: uint64 array, one per entry; empty when
        the partial has no packed words) -- a read that changes nothing"""
        shift, word, state, n = C.c_int32(), C.c_int32(), C.c_uint32(), C.c_uint64()
        check(lib().cg_partial_packed_state(self.h, None, 0, C.byref(shift), C.byref(word), C.byref(state), C.byref(n)))
        words = np.zeros(n.value, np.uint64)
        check(lib().cg_partial_packed_state(self.h, words.ctypes.data, n.value, None, None, None, C.byref(n)))
        return shift.value, word.value, state.value, words

    def dense_words(self):
        p, total, stride = C.c_void_p(), C.c_int64(), C.c_int32()
        check(lib().cg_partial_dense_words(self.h, C.byref(p), C.byref(total), C.byref(stride)))
        return p.value, total.value, stride.value


def numeric_out(value: int, scale: int) -> str:
    buf = C.create_string_buffer(128)
    check(lib().cg_numeric_out((value >> 64), value & ((1 << 64) - 1), scale, buf, 128))
    return buf.value.decode()


def numeric_div_out(value: int, scale: int, count: int) -> str:
    buf = C.create_string_buffer(160)
    check(lib().cg_numeric_div_out((value >> 64), value & ((1 << 64) - 1), scale, count, buf, 160))
    return buf.value.decode()


def worker_partition_query_result(d_keys_ptr, d_nulls_ptr, n, key_len, method, mins, maxs, d_index_ptr, d_counts_ptr):
    """partition index of every row (device arrays).  method 'hash' | 'range'."""
    if method not in ("hash", "range"):
        raise capi.CitusGpuError(capi.CG_EINVAL, "only hash and range partitiong schemes are supported")
    mins = np.ascontiguousarray(mins, np.int32)
    maxs = np.ascontiguousarray(maxs, np.int32)
    if len(mins) != len(maxs):
        raise capi.CitusGpuError(capi.CG_EINVAL, "min values and max values must have the same number of elements")
    check(lib().cg_partition_index(d_keys_ptr, d_nulls_ptr, n, key_len, 1 if method == "hash" else 0,
                                   mins.ctypes.data, maxs.ctypes.data, len(mins), d_index_ptr, d_counts_ptr))


def join_count_sum(d_build_keys, d_build_payload, nbuild, d_probe_keys, d_probe_payload, nprobe, d_build_nulls=None,
                   d_probe_nulls=None):
    """(joined rows, exact sum(b.payload + p.payload)) of the equi-join of two device-resident partitions"""
    rows, hi, lo = C.c_int64(), C.c_int64(), C.c_uint64()
    check(lib().cg_join_count_sum(d_build_keys, d_build_nulls, d_build_payload, nbuild, d_probe_keys, d_probe_nulls,
                                  d_probe_payload, nprobe, C.byref(rows), C.byref(hi), C.byref(lo)))
    return rows.value, (hi.value << 64) + lo.value


def join_rows(d_build_keys, d_build_payload, nbuild, d_probe_keys, d_probe_payload, nprobe, capacity=0, d_out=(None, None, None),
              d_build_nulls=None, d_probe_nulls=None):
    """rows of the equi-join into the caller's device arrays (key, build payload, probe payload); returns the row count
    (capacity 0: count only)"""
    n = C.c_int64()
    check(lib().cg_join_rows(d_build_keys, d_build_nulls, d_build_payload, nbuild, d_probe_keys, d_probe_nulls, d_probe_payload, nprobe,
                             capacity, d_out[0], d_out[1], d_out[2], C.byref(n)))
    return n.value


def set_writer_compression(name: str):
    """columnar.compression for Relation.generate / Relation.write: "none", "lz4" or "zstd" (level 3)"""
    check(lib().cg_gen_set_compression({"none": 0, "lz4": 2, "zstd": 3}[name]))


def partition_copy_bytes(d_index_ptr, n, P, d_col_ptrs, col_lens, binary, d_null_ptrs=None, generate_empty_results=False):
    """(rows_written[P], bytes_written[P]) of worker_partition_query_result's return rows"""
    cols = (C.c_void_p * len(d_col_ptrs))(*d_col_ptrs)
    nulls = (C.c_void_p * len(d_col_ptrs))(*(d_null_ptrs or [None] * len(d_col_ptrs)))
    lens = (C.c_int32 * len(d_col_ptrs))(*col_lens)
    rows = np.zeros(P, np.int64)
    nbytes = np.zeros(P, np.int64)
    check(lib().cg_partition_copy_bytes(d_index_ptr, n, P, cols, nulls, lens, len(d_col_ptrs), 1 if binary else 0,
                                        1 if generate_empty_results else 0, rows.ctypes.data, nbytes.ctypes.data))
    return rows, nbytes


def partition_copy_serialize(d_index_ptr, n, P, d_col_ptrs, col_lens, binary, d_out_ptr, out_capacity, d_null_ptrs=None,
                             generate_empty_results=False):
    """the P partition files (COPY text / binary) back to back in the device buffer; returns file offsets [P + 1]"""
    cols = (C.c_void_p * len(d_col_ptrs))(*d_col_ptrs)
    nulls = (C.c_void_p * len(d_col_ptrs))(*(d_null_ptrs or [None] * len(d_col_ptrs)))
    lens = (C.c_int32 * len(d_col_ptrs))(*col_lens)
    offs = np.zeros(P + 1, np.int64)
    check(lib().cg_partition_copy_serialize(d_index_ptr, n, P, cols, nulls, lens, len(d_col_ptrs), 1 if binary else 0,
                                            1 if generate_empty_results else 0, d_out_ptr, out_capacity, offs.ctypes.data))
    return offs


def partition_scatter(d_index_ptr, n, P, d_col_ptrs, d_out_ptrs, order=None):
    """stable scatter into partition-contiguous order; order[p] = output position of partition p"""
    cols = (C.c_void_p * len(d_col_ptrs))(*d_col_ptrs)
    outs = (C.c_void_p * len(d_out_ptrs))(*d_out_ptrs)
    offs = np.zeros(P + 1, np.int64)
    if order is None:
        check(lib().cg_partition_scatter(d_index_ptr, n, P, cols, len(d_col_ptrs), outs, offs.ctypes.data))
    else:
        order = np.ascontiguousarray(order, np.int32)
        check(lib().cg_partition_scatter_ordered(d_index_ptr, n, P, order.ctypes.data, cols, len(d_col_ptrs), outs,
                                                 offs.ctypes.data))
    return offs


def numeric_var_out(final: int, n: int, s: int, q: int, scale: int, buflen: int = 1100):
    """PostgreSQL's text of var_pop / var_samp / stddev_pop / stddev_samp (final = capi.CG_VAR_* / CG_STDDEV_*) from the
    exact state N = n, sum(x) = s, sum(x^2) = q in units of 10^-scale; None for SQL NULL"""
    buf = C.create_string_buffer(buflen)
    isnull = C.c_int32()
    qs = np.array([(q >> (64 * i)) & ((1 << 64) - 1) for i in range(3)], np.uint64)
    check(lib().cg_numeric_var_out(final, n, s >> 64, s & ((1 << 64) - 1), qs.ctypes.data, scale, buf, buflen, C.byref(isnull)))
    return None if isnull.value else buf.value.decode()
