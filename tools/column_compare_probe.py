#!/usr/bin/env python
"""Cost of column-to-column atoms in the fused scan, on a synthetic lineitem-like relation with three int4 date columns
(600 M rows, 32 shards, HBM resident) and on bench.py's C2 relation:

    q12        count(*), sum(l_extendedprice) WHERE l_commitdate < l_receiptdate AND l_shipdate < l_commitdate
               AND l_receiptdate >= lo AND l_receiptdate < lo + 365 GROUP BY l_returnflag      (TPC-H Q12's predicates)
    q12_const  the same with the two column atoms replaced by l_commitdate < k AND l_shipdate < k, k = 1993-10-06
               (SAME_ROWS): on this data the two forms pass the same share of rows (within 1 % on the checked sample)
    c2         C2: sum(v), count(*) WHERE f < 50 GROUP BY key
    c2_col     C2 with one more atom, v > f

timed alternately in one process.  Prints per query the median ms per query over the runs, the fused kernels' device
time, the kernel family that ran (generated kernels launched per query; none = an ahead-of-time kernel) and the card with
its power limit, and checks every query's groups against the exact reference (tests/reference.py) on a
sample.

    python tools/column_compare_probe.py [--rows 600000000] [--c2-rows 200000000] [--reps 10] [--sample-rows 150000] [--json FILE]
"""
import argparse
import ctypes as C
import dataclasses
import json
import os
import sys
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
from citus_b200 import build  # noqa: E402

build.build()
from citus_b200 import capi  # noqa: E402
from citus_b200 import columnar as cg  # noqa: E402
from filter_probe import _Env, card, synth_columns  # noqa: E402

import reference as ref  # noqa: E402

DATE_LO, DATE_HI = -2922, -366                     # 1992-01-01 .. 1998-12-31 as days since 2000-01-01
DATES = [(4, 0, DATE_LO, DATE_HI, 0)] * 3         # 0 l_shipdate, 1 l_commitdate, 2 l_receiptdate
LINEITEM_DATES = DATES + [(8, 0, 90000, 10500000, 0),     # 3 l_extendedprice
                          (1, 0, 65, 68, 0)]               # 4 l_returnflag
YEAR = -2191                                       # 1994-01-01
SAME_ROWS = -2278                                  # 1993-10-06


def queries():
    Col = cg.Col
    aggs = lambda: [cg.count_star(), cg.sum_(3)]
    window = [(2, ">=", YEAR), (2, "<", YEAR + 365)]
    return {"q12": ("lineitem", dict(quals=[(1, "<", Col(2)), (0, "<", Col(1))] + window, group=[4], aggs=aggs())),
            "q12_const": ("lineitem", dict(quals=[(1, "<", SAME_ROWS), (0, "<", SAME_ROWS)] + window, group=[4], aggs=aggs())),
            "c2": ("c2", dict(quals=bench.C2_QUALS, group=bench.C2_GROUP, aggs=[cg.sum_(2), cg.count_star()])),
            "c2_col": ("c2", dict(quals=bench.C2_QUALS + [(2, ">", Col(1))], group=bench.C2_GROUP, aggs=[cg.sum_(2), cg.count_star()]))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=600_000_000)
    ap.add_argument("--c2-rows", type=int, default=200_000_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--sample-rows", type=int, default=150_000)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    cg.init(0)
    nshards = bench.NSHARDS
    env = types.SimpleNamespace(cg=cg, args=types.SimpleNamespace(gen_threads=0), ncpu=os.cpu_count() or 8, world=1, rank=0)
    tables = {}                                  # name -> (relations, shards, seed, columns, rows per shard)
    per = args.rows // nshards
    rels = bench.generate_shards(env, LINEITEM_DATES, range(nshards), per, 101)
    tables["lineitem"] = (rels, {s: cg.Shard(rels[s]) for s in rels}, 101, LINEITEM_DATES, per)
    per2 = args.c2_rows // nshards
    rels2 = bench.generate_shards(env, bench.C2_COLUMNS, range(nshards), per2, bench.SEED)
    tables["c2"] = (rels2, {s: cg.Shard(rels2[s], [0, 1, 2]) for s in rels2}, bench.SEED, bench.C2_COLUMNS, per2)
    qs = queries()
    parts = {}
    for name, (t, q) in qs.items():
        aggs = [dataclasses.replace(a) for a in q["aggs"]]
        rels_t, _, _, _, per_t = tables[t]
        parts[name] = bench.make_partial(_Env(), rels_t, q["quals"], q["group"], aggs, per_t * nshards, expected_groups=16)[0]

    def run(name):
        p = parts[name]
        p.reset()
        shards = tables[qs[name][0]][1]
        for s in shards:
            p.scan_shard(shards[s], want_stats=False)
        return p.ngroups()

    for name in qs:                                         # warm-up: NVRTC compiles, module loads
        for _ in range(3):
            run(name)
    times = {n: [] for n in qs}
    kern = {n: [] for n in qs}
    jit = {n: [] for n in qs}
    for _ in range(args.reps):
        for name in qs:
            capi.check(capi.lib().cg_profile_begin())
            capi.check(capi.lib().cg_synchronize())
            j0 = capi.lib().cg_jit_launches()
            t0 = time.perf_counter()
            run(name)
            capi.check(capi.lib().cg_synchronize())
            times[name].append((time.perf_counter() - t0) * 1e3)
            jit[name].append(capi.lib().cg_jit_launches() - j0)
            n, tot, mx = C.c_int32(), C.c_double(), C.c_double()
            capi.check(capi.lib().cg_profile_collect(C.byref(n), C.byref(tot), C.byref(mx)))
            kern[name].append(tot.value)
    # exact check on the first sample_rows rows of shard 0 (its first stripes)
    checks = {}
    for name, (t, q) in qs.items():
        rels_t, _, seed, columns, _ = tables[t]
        sample = rels_t[0].prefix(max(1, args.sample_rows // bench.STRIPE_ROWS))
        cols = synth_columns(columns, 0, sample.rows, seed)
        aggs = [dataclasses.replace(a) for a in q["aggs"]]
        part = bench.make_partial(_Env(), {0: sample}, q["quals"], q["group"], aggs, sample.rows, expected_groups=16)[0]
        sh = cg.Shard(sample)
        st = part.scan_shard(sh)
        sh.free()
        got = part.groups()
        part.free()
        want = ref.aggregate(cols, None, q["quals"], q["group"], aggs)
        ok = st.rows_passed == want.rows_passed and {(k,) for k in got} == set(want.groups)
        for k, per_got in got.items():
            for a, (g, w) in enumerate(zip(per_got, want.groups.get((k,), []))):
                ok &= g["count"] == w.count and (aggs[a].kind != 2 or w.count == 0 or g["sum"] == w.sum)
        checks[name] = dict(ok=bool(ok), rows=int(sample.rows), groups=len(got), rows_passed=int(st.rows_passed))
    out = {"card": card(), "lineitem_rows": per * nshards, "c2_rows": per2 * nshards, "reps": args.reps, "queries": {}}
    for name in qs:
        out["queries"][name] = dict(ms_per_query=float(np.median(times[name])), kernel_ms=float(np.median(kern[name])),
                                    ms_spread=[float(min(times[name])), float(max(times[name]))],
                                    generated_kernel_launches=int(np.median(jit[name])),
                                    family="generated" if np.median(jit[name]) > 0 else "ahead-of-time", check=checks[name])
    r = out["queries"]
    out["q12_over_q12_const"] = r["q12"]["ms_per_query"] / r["q12_const"]["ms_per_query"]
    out["c2_col_over_c2"] = r["c2_col"]["ms_per_query"] / r["c2"]["ms_per_query"]
    print(f"card: {out['card']}")
    print(f"{'query':<10} {'ms/query':>9} {'kernel ms':>10} {'spread':>17} {'family':>14}  exact")
    for name, x in r.items():
        print(f"{name:<10} {x['ms_per_query']:9.2f} {x['kernel_ms']:10.2f} {x['ms_spread'][0]:8.2f}-{x['ms_spread'][1]:<8.2f} {x['family']:>14}  {x['check']['ok']}")
    print(f"q12 / q12_const: {out['q12_over_q12_const']:.3f}   c2_col / c2: {out['c2_col_over_c2']:.3f}")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    for p in parts.values():
        p.free()
    for t in tables.values():
        for sh in t[1].values():
            sh.free()
    if not all(c["ok"] for c in checks.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
