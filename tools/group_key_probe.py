#!/usr/bin/env python
"""Cost of composite GROUP BY keys against today's one-column key, on HBM-resident synthetic shards (32 shards):

    c2        the C2 shape (WHERE f < 50, sum(v), count(*)) grouped by its 1 M-value int8 key: one-column dense path
    c2_k16    the same grouped by (key, k16), k16 an int4 of 16 values: composite, direct-indexed (16 M groups)
    c2_16m    its one-column twin: GROUP BY key * 16 + k16, the same 16 M groups, today's direct-indexed path
    c2_wide   the same grouped by (wkey, k16), wkey = key * 1048573 (the same 1 M values spread over 2^40): composite
              hash table
    c2_16m_h  its one-column twin: GROUP BY wkey * 16 + k16, the same 16 M groups, today's hash path
    q1        TPC-H Q1 over the synthetic lineitem: GROUP BY l_returnflag, l_linestatus (packed two-column key)
    q1_mode   Q1 with l_shipmode (int1, 7 codes) as a third key: composite (42 groups)
    q1_42     its one-column twin: Q1 grouped by an int1 column of 42 values, today's path

A composite query is compared with its one-column twin, which has the same group count and table kind: the group count
decides where the table lives (shared memory, L2 or HBM) and so dominates the cost of a grouped scan.

Each query's scans are timed alternately in one process after a warm-up: median ms per query (all shards, ending in a
device synchronise), the fused kernels' summed device time (CUDA events), algorithmic bytes (the scanned chunk groups'
value and exists bytes of the projected columns, from CgScanStats) per kernel second and its share of 3.35 TB/s.  The
card and its power limit are printed with the numbers.  Every query is checked exactly against tests/reference.py on the
first stripes of shard 0.

    python tools/group_key_probe.py [--rows 320000000] [--reps 7] [--sample-rows 150000] [--json FILE]
"""
import argparse
import ctypes as C
import dataclasses
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402
from citus_b200 import build  # noqa: E402

build.build()
from citus_b200 import capi  # noqa: E402
from citus_b200 import columnar as cg  # noqa: E402

import reference as ref  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
NSHARDS = 32
SPREAD = 1048573                     # 1 M keys * SPREAD < 2^40


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


def splitmix_columns(columns, first_row, nrows, seed):
    """cg_gen_relation's values (include/citus_gpu.h: lo + splitmix64(seed ^ col << 56 ^ row) % (hi - lo)), int64 arrays"""
    rows = np.arange(first_row, first_row + nrows, dtype=np.uint64)
    out = []
    with np.errstate(over="ignore"):
        for c, (_, _, lo, hi, _) in enumerate(columns):
            x = (np.uint64(seed) ^ np.uint64(c << 56) ^ rows) + np.uint64(0x9E3779B97F4A7C15)
            x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
            x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
            x = x ^ (x >> np.uint64(31))
            out.append(lo + (x % np.uint64(hi - lo)).astype(np.int64))
    return out


# C2 plus k16 (int4, 16 values), wkey (the key spread over 2^40) and the one-column twins key * 16 + k16 and wkey * 16 + k16;
# written from numpy, so that the derived columns can be computed from the key
C2X = bench.C2_COLUMNS[:3] + [(4, 0, 0, 16, 0)]
C2X_ATTLENS = [8, 8, 8, 4, 8, 8, 8]
LINEITEM_MODE = bench.LINEITEM + [(1, 0, 0, 7, 0), (1, 0, 0, 42, 0)]          # 8 l_shipmode, 9 a 42-value key


def c2x_shard(s, per):
    cols = splitmix_columns(C2X, s * per, per, bench.SEED)
    wkey = cols[0] * SPREAD
    return cols + [wkey, cols[0] * 16 + cols[3], wkey * 16 + cols[3]]


def queries():
    c2 = dict(table="c2x", quals=bench.C2_QUALS, aggs=[cg.sum_(2), cg.count_star()], expected_groups=1 << 24)
    q1 = bench.tpch_queries(cg)["q1"]
    q1 = dict(table="lineitem", quals=q1["quals"], aggs=q1["aggs"], expected_groups=64)
    return {"c2": dict(c2, group=[0], composite=False), "c2_k16": dict(c2, group=[0, 3], composite=True),
            "c2_16m": dict(c2, group=[5], composite=False), "c2_wide": dict(c2, group=[4, 3], composite=True),
            "c2_16m_h": dict(c2, group=[6], composite=False), "q1": dict(q1, group=[4, 5], composite=False),
            "q1_mode": dict(q1, group=[4, 5, 8], composite=True), "q1_42": dict(q1, group=[9], composite=False)}


def make_partial(rels, q, total_rows):
    aggs = [dataclasses.replace(a) for a in q["aggs"]]
    d = cg.make_desc(q["quals"], q["group"], aggs)
    kmin = kmax = None
    kb, proven = None, [0] * len(aggs)
    for rel in rels:
        a, b, pr, _ = cg.relation_bounds(rel, d)
        proven = [max(x, y) for x, y in zip(proven, pr)]
        if q["composite"]:
            k = cg.relation_key_bounds(rel, d)
            kb = k if kb is None else [(min(x[0], y[0]), max(x[1], y[1])) for x, y in zip(kb, k)]
        elif len(q["group"]) == 2:
            lo, hi = [bench._s32(a), bench._s32(a >> 32)], [bench._s32(b), bench._s32(b >> 32)]
            kmin = lo if kmin is None else [min(x, y) for x, y in zip(kmin, lo)]
            kmax = hi if kmax is None else [max(x, y) for x, y in zip(kmax, hi)]
        else:
            kmin = a if kmin is None else min(kmin, a)
            kmax = b if kmax is None else max(kmax, b)
    for a, b in zip(aggs, proven):
        a.term_abs_bound = b
    d = cg.make_desc(q["quals"], q["group"], aggs, expected_groups=q["expected_groups"], composite=q["composite"], key_bounds=kb)
    if q["composite"]:
        kmin, kmax = 0, -1
    elif len(q["group"]) == 2:
        kmin = bench._s64((kmin[0] & 0xffffffff) | ((kmin[1] & 0xffffffff) << 32))
        kmax = bench._s64((kmax[0] & 0xffffffff) | ((kmax[1] & 0xffffffff) << 32))
    return cg.GpuColumnarAgg(d, rels[0].column_descs(), kmin, kmax, total_rows), aggs


def keyed(q, got):
    """groups() keys -> the reference's key tuples"""
    if q["composite"]:
        return got
    if len(q["group"]) == 2:
        return {ref.unpack_two_column_key(k): v for k, v in got.items()}
    return {(k,): v for k, v in got.items()}


def exact(got, want):
    if set(got) != set(want.groups):
        return False
    for key, per in want.groups.items():
        for g, w in zip(got[key], per):
            if g["count"] != w.count or (w.count and w.sum is not None and g["sum"] != w.sum):
                return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=320_000_000)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--sample-rows", type=int, default=150_000)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    cg.init(0)
    per = args.rows // NSHARDS
    threads = max(4, min(64, os.cpu_count() or 8))
    t0 = time.time()
    tables = {"c2x": {}, "lineitem": {}}
    for s in range(NSHARDS):
        tables["c2x"][s] = cg.Relation.write(C2X_ATTLENS, c2x_shard(s, per), stripe_row_limit=bench.STRIPE_ROWS, chunk_row_limit=bench.CHUNK_ROWS)
        tables["lineitem"][s] = cg.Relation.generate(LINEITEM_MODE, per, seed=100, first_row=s * per, stripe_row_limit=bench.STRIPE_ROWS,
                                                     chunk_row_limit=bench.CHUNK_ROWS, nthreads=threads)
    print(f"generated 2 x {NSHARDS} shards x {per} rows in {time.time() - t0:.0f} s", flush=True)
    shards = {t: {s: cg.Shard(r) for s, r in rels.items()} for t, rels in tables.items()}
    qs = queries()
    parts = {n: make_partial(list(tables[q["table"]].values()), q, per * NSHARDS)[0] for n, q in qs.items()}
    algo = {}

    def run(name, stats=False):
        p = parts[name]
        p.reset()
        total = 0
        for sh in shards[qs[name]["table"]].values():
            st = p.scan_shard(sh, want_stats=stats)
            total += st.bytes_scanned if stats else 0
        n = p.ngroups()
        if stats:
            algo[name] = total
        return n

    for name in qs:                                         # warm-up: NVRTC compiles, module loads
        run(name, stats=True)
        run(name)
    times = {n: [] for n in qs}
    kern = {n: [] for n in qs}
    for _ in range(args.reps):
        for name in qs:
            capi.check(capi.lib().cg_profile_begin())
            torch.cuda.synchronize()
            t = time.perf_counter()
            run(name)
            capi.check(capi.lib().cg_synchronize())
            times[name].append((time.perf_counter() - t) * 1e3)
            n, tot, mx = C.c_int32(), C.c_double(), C.c_double()
            capi.check(capi.lib().cg_profile_collect(C.byref(n), C.byref(tot), C.byref(mx)))
            kern[name].append(tot.value)
    groups = {n: parts[n].ngroups() for n in qs}
    kinds = {n: ("dense" if parts[n].layout()[2] else "hash") for n in qs}
    # exact check on the first stripes of shard 0
    nstripes = max(1, args.sample_rows // bench.STRIPE_ROWS)
    checks = {}
    for name, q in qs.items():
        sample = tables[q["table"]][0].prefix(nstripes)
        n = sample.rows
        cols = c2x_shard(0, per) if q["table"] == "c2x" else splitmix_columns(LINEITEM_MODE, 0, per, 100)
        cols = [c[:n] for c in cols]
        p, aggs = make_partial([sample], q, n)
        p.scan_shard(cg.Shard(sample), want_stats=False)
        got = keyed(q, p.groups())
        p.free()
        want = ref.aggregate(cols, None, q["quals"], q["group"], aggs)
        checks[name] = dict(ok=exact(got, want), rows=int(n), groups=len(got))
    out = {"card": card(), "rows": per * NSHARDS, "reps": args.reps, "queries": {}}
    for name in qs:
        kms = float(np.median(kern[name]))
        bps = algo[name] / (kms / 1e3) if kms > 0 else 0.0
        out["queries"][name] = dict(ms_per_query=float(np.median(times[name])), ms_spread=[float(min(times[name])), float(max(times[name]))],
                                    kernel_ms=kms, algorithmic_bytes=int(algo[name]), bytes_per_s=bps, hbm_share=bps / HBM_BYTES_PER_S,
                                    groups=int(groups[name]), table=kinds[name], check=checks[name])
    print(f"card: {out['card']}")
    print(f"{'query':<8} {'ms/query':>9} {'kernel ms':>10} {'GB/s':>8} {'of 3.35 TB/s':>13} {'groups':>9} {'table':>6}  exact")
    for name, r in out["queries"].items():
        print(f"{name:<8} {r['ms_per_query']:9.2f} {r['kernel_ms']:10.2f} {r['bytes_per_s'] / 1e9:8.0f} {r['hbm_share']:13.1%} "
              f"{r['groups']:9d} {r['table']:>6}  {r['check']['ok']} ({r['check']['rows']} rows)")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    for p in parts.values():
        p.free()
    for t in shards.values():
        for sh in t.values():
            sh.free()
    if not all(c["ok"] for c in checks.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
