#!/usr/bin/env python
"""Cost of stddev_samp / var_pop next to a Q1-style grouped aggregate: the synthetic lineitem of bench.py's C5 leg
(SF100, 32 shards, HBM resident), Q1's WHERE and GROUP BY l_returnflag, l_linestatus with

    A: count(*), sum(l_quantity), sum(l_extendedprice)
    B: A + stddev_samp(l_quantity), var_pop(l_extendedprice)

timed alternately in one process.  Both variance aggregates are one CG_AGG_VARIANCE state each (N, sum(x), sum(x^2));
with the skip lists' bounds their sum(x^2) is one word (l_quantity) and two 32-bit limbs (l_extendedprice).  Prints per
query the median ms per query and the fused kernel's device time, with the card and its power limit, and checks both
queries' groups exactly against tests/reference.py on a sample, the final texts included.

    python tools/variance_probe.py [--rows 600000000] [--reps 10] [--sample-rows 150000] [--json FILE]
"""
import argparse
import ctypes as C
import dataclasses
import json
import os
import subprocess
import sys
import time
import types

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



def queries():
    q1 = bench.tpch_queries(cg)["q1"]
    a = [cg.count_star(), cg.sum_(0), cg.sum_(1)]
    b = a + [cg.variance(0), cg.variance(1)]                 # stddev_samp(l_quantity), var_pop(l_extendedprice)
    return {"A": dict(q1, aggs=a), "B": dict(q1, aggs=b)}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


def synth_columns(columns, first_row, nrows, seed):
    """the values cg_gen_relation writes (its splitmix64 formula), as int64 arrays"""
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


FINAL = {3: ref.STDDEV_SAMP, 4: ref.VAR_POP}               # aggregate number in B -> its SQL final function


def exact(g, w, kind, a):
    """one fetched aggregate against the reference's (decimal(15,2) columns: scale 2)"""
    if g["count"] != w.count:
        return False
    if w.count == 0 or kind in (0, 1):
        return True
    if g["sum"] != w.sum:
        return False
    if kind == ref.VARIANCE:
        return g["sumsq"] == w.sumsq and cg.numeric_var_out(FINAL[a], g["count"], g["sum"], g["sumsq"], 2) == \
            ref.var_out(FINAL[a], w.count, w.sum, w.sumsq, 2)
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=600_000_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--sample-rows", type=int, default=150_000)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    cg.init(0)
    nshards = bench.NSHARDS
    per = args.rows // nshards
    env = types.SimpleNamespace(cg=cg, args=types.SimpleNamespace(gen_threads=0), ncpu=os.cpu_count() or 8, world=1, rank=0)
    rels = bench.generate_shards(env, bench.LINEITEM, range(nshards), per, 100)
    shards = {s: cg.Shard(rels[s], [0, 1, 2, 3, 4, 5, 6, 7]) for s in rels}
    qs = queries()
    parts = {}
    for name, q in qs.items():
        aggs = [dataclasses.replace(a) for a in q["aggs"]]
        parts[name] = bench.make_partial(_Env(), rels, q["quals"], q["group"], aggs, per * nshards, expected_groups=16)[0]
    part_words = {name: p.layout()[0] for name, p in parts.items()}

    def run(name):
        p = parts[name]
        p.reset()
        for s in shards:
            p.scan_shard(shards[s], want_stats=False)
        return p.ngroups()

    for name in qs:                                         # warm-up: NVRTC compiles, module loads
        for _ in range(3):
            run(name)
    times = {n: [] for n in qs}
    kern = {n: [] for n in qs}
    for _ in range(args.reps):
        for name in qs:
            capi.check(capi.lib().cg_profile_begin())
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(name)
            capi.check(capi.lib().cg_synchronize())
            times[name].append((time.perf_counter() - t0) * 1e3)
            n, tot, mx = C.c_int32(), C.c_double(), C.c_double()
            capi.check(capi.lib().cg_profile_collect(C.byref(n), C.byref(tot), C.byref(mx)))
            kern[name].append(tot.value)
    # exact check on the first sample_rows rows of shard 0 (its first stripes)
    nstripes = max(1, args.sample_rows // bench.STRIPE_ROWS)
    sample = rels[0].prefix(nstripes)
    cols = synth_columns(bench.LINEITEM, 0, sample.rows, 100)
    checks = {}
    for name, q in qs.items():
        aggs = [dataclasses.replace(a) for a in q["aggs"]]
        part = bench.make_partial(_Env(), {0: sample}, q["quals"], q["group"], aggs, sample.rows, expected_groups=16)[0]
        part.scan_shard(cg.Shard(sample), want_stats=False)
        got = part.groups()
        part.free()
        want = ref.aggregate(cols, None, q["quals"], q["group"], aggs)
        ok = len(got) == len(want.groups)
        for k, per_got in got.items():
            key = ref.unpack_two_column_key(k)
            if key not in want.groups:
                ok = False
                continue
            for a, (g, w) in enumerate(zip(per_got, want.groups[key])):
                ok &= exact(g, w, aggs[a].kind, a)
        checks[name] = dict(ok=bool(ok), rows=int(sample.rows), groups=len(got), layout_words=part_words[name])
    out = {"card": card(), "rows": per * nshards, "reps": args.reps, "queries": {}}
    for name in qs:
        out["queries"][name] = dict(ms_per_query=float(np.median(times[name])), kernel_ms=float(np.median(kern[name])),
                                    ms_spread=[float(min(times[name])), float(max(times[name]))], check=checks[name])
    out["ratio_b_over_a"] = out["queries"]["B"]["ms_per_query"] / out["queries"]["A"]["ms_per_query"]
    print(f"card: {out['card']}")
    print(f"{'query':<6} {'ms/query':>9} {'kernel ms':>10}  exact on {checks['A']['rows']} rows")
    for name, r in out["queries"].items():
        print(f"{name:<6} {r['ms_per_query']:9.2f} {r['kernel_ms']:10.2f}  {r['check']['ok']}")
    print(f"B / A: {out['ratio_b_over_a']:.3f}")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    for p in parts.values():
        p.free()
    for sh in shards.values():
        sh.free()
    if not all(c["ok"] for c in checks.values()):
        sys.exit(1)


class _Env:
    """a single-GPU view for bench.make_partial (plan constants are not agreed across ranks)"""
    world = 1
    cg = cg
    cgd = None


if __name__ == "__main__":
    main()
