#!/usr/bin/env python
"""Cost of aggregate FILTER (WHERE ...) on TPC-H Q1: the synthetic lineitem of bench.py's C5 leg (SF100, 32 shards,
HBM resident), Q1 as bench.py runs it and Q1 without sum(l_discount) (eight aggregates at most) plus

    count(*) FILTER (WHERE l_discount > 5), sum(l_extendedprice) FILTER (WHERE l_shipdate >= -1000),
    sum(l_quantity) FILTER (WHERE l_returnflag = 65 OR l_tax < 3)

(every column already staged for Q1), timed alternately in one process.  Prints per query the ms per query, the
fused kernel's device time, bytes per row and the fraction of 3.35 TB/s, with the card and its power limit, and
checks both queries' groups against the exact reference (tests/reference.py) on a sample.

    python tools/filter_probe.py [--rows 600000000] [--reps 10] [--sample-rows 150000] [--json FILE]
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

HBM_GBS = 3350.0            # NVIDIA's data sheet for the H100 SXM: a bound, not a measured rate
BYTES_PER_ROW = 38.75       # Q1's projected columns: 4 x 8 + 2 x 1 + 4 bytes + 7 exists bits


def queries():
    q1 = bench.tpch_queries(cg)["q1"]
    # CG_MAX_AGGS = 8: the filtered query drops Q1's sum(l_discount) (aggregate 4) to make room for the three filters
    filt = q1["aggs"][:4] + q1["aggs"][5:] + [cg.count_star(filter=(2, ">", 5)), cg.sum_(1, filter=(6, ">=", -1000)),
                         cg.sum_(0, filter=("or", (4, "=", 65), (3, "<", 3)))]
    return {"q1": q1, "q1_filter": dict(q1, aggs=filt)}


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
    shards = {s: cg.Shard(rels[s], [0, 1, 2, 3, 4, 5, 6]) for s in rels}
    qs = queries()
    parts = {}
    for name, q in qs.items():
        aggs = [dataclasses.replace(a) for a in q["aggs"]]
        parts[name] = bench.make_partial(_Env(), rels, q["quals"], q["group"], aggs, per * nshards, expected_groups=16)[0]

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
                ok &= g["count"] == w.count and (aggs[a].kind != 2 or w.count == 0 or g["sum"] == w.sum)
        checks[name] = dict(ok=bool(ok), rows=int(sample.rows), groups=len(got))
    out = {"card": card(), "rows": per * nshards, "reps": args.reps, "queries": {}}
    for name in qs:
        ms = float(np.median(times[name]))
        kms = float(np.median(kern[name]))
        out["queries"][name] = dict(ms_per_query=ms, kernel_ms=kms, bytes_per_row=BYTES_PER_ROW,
                                    hbm_frac=BYTES_PER_ROW * per * nshards / (kms / 1e3) / 1e9 / HBM_GBS if kms > 0 else None,
                                    ms_spread=[float(min(times[name])), float(max(times[name]))], check=checks[name])
    out["ratio_filter_over_plain"] = out["queries"]["q1_filter"]["ms_per_query"] / out["queries"]["q1"]["ms_per_query"]
    print(f"card: {out['card']}")
    print(f"{'query':<10} {'ms/query':>9} {'kernel ms':>10} {'B/row':>6} {'of 3.35 TB/s':>13}  exact on {checks['q1']['rows']} rows")
    for name, r in out["queries"].items():
        print(f"{name:<10} {r['ms_per_query']:9.2f} {r['kernel_ms']:10.2f} {r['bytes_per_row']:6.2f} {r['hbm_frac']:13.3f}  {r['check']['ok']}")
    print(f"filtered / plain: {out['ratio_filter_over_plain']:.3f}")
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
