#!/usr/bin/env python
"""Cost of IN lists and IS NULL in the fused scan, on the synthetic lineitem of bench.py's C5 leg (SF100, 32 shards, HBM
resident) and on C2 with 5 % NULLs in v:

    in8      sum(l_extendedprice * l_discount) WHERE l_quantity IN (8 values)        (Q6's aggregate)
    or8      the same WHERE as an OR of eight "=" atoms (the form the library ran before lists existed; with Q6's other
             four conjuncts it would need 12 atoms, more than CG_MAX_QUALS, so both forms carry the list alone)
    in8_alt  in8 with a different 8-value list on every other shard scan: the list codes are copied to the device again
             before each scan (a scan whose list equals the last one copies nothing)
    in64     the same with 64 values
    in1024   the same with 1024 values
    c2null   C2-NULL: sum(v), count(*) WHERE f < 50 GROUP BY key
    c2null_f the same plus count(*) FILTER (WHERE v IS NULL)

timed alternately in one process.  Prints per query the ms per query and the fused kernel's device time with the card and
its power limit, and checks every query's groups against the exact reference (tests/reference.py) on a sample.

    python tools/in_list_probe.py [--rows 600000000] [--c2-rows 200000000] [--reps 10] [--sample-rows 150000] [--json FILE]
"""
import argparse
import ctypes as C
import dataclasses
import json
import os
import sys
import time

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

C2_NULL = list(bench.C2_COLUMNS)
C2_NULL[2] = (8, 0, -10**9, 10**9, 50000)           # 5 % NULLs in v, as bench.py's C2-NULL leg


def lineitem_queries(rng):
    q = [int(x) for x in rng.choice(np.arange(100, 5100), 1024, replace=False)]
    agg = lambda: [cg.Agg(2, [(1, 0, 1), (2, 0, 1)])]
    return {"in8": dict(quals=[(0, "in", tuple(q[:8]))], group=[], aggs=agg()),
            "or8": dict(quals=("or",) + tuple((0, "=", v) for v in q[:8]), group=[], aggs=agg()),
            "in8_alt": dict(quals=[(0, "in", tuple(q[:8]))], alt=[(0, "in", tuple(q[8:16]))], group=[], aggs=agg()),
            "in64": dict(quals=[(0, "in", tuple(q[:64]))], group=[], aggs=agg()),
            "in1024": dict(quals=[(0, "in", tuple(q))], group=[], aggs=agg())}


def c2_queries():
    base = [cg.sum_(2), cg.count_star()]
    return {"c2null": dict(quals=bench.C2_QUALS, group=bench.C2_GROUP, aggs=base),
            "c2null_f": dict(quals=bench.C2_QUALS, group=bench.C2_GROUP, aggs=base + [cg.count_star(filter=(2, "is null"))])}


def synth_nulls(columns, first_row, nrows, seed):
    """the NULL flags cg_gen_relation writes: splitmix64(~seed ^ col << 56 ^ row) % 10^6 < null_ppm"""
    rows = np.arange(first_row, first_row + nrows, dtype=np.uint64)
    out = []
    with np.errstate(over="ignore"):
        for c, (_, _, _, _, ppm) in enumerate(columns):
            x = (np.uint64(~seed & (2**64 - 1)) ^ np.uint64(c << 56) ^ rows) + np.uint64(0x9E3779B97F4A7C15)
            x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
            x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
            x = x ^ (x >> np.uint64(31))
            out.append((x % np.uint64(1000000) < np.uint64(ppm)).astype(np.uint8) if ppm else None)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=600_000_000)
    ap.add_argument("--c2-rows", type=int, default=200_000_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--sample-rows", type=int, default=150_000)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import types
    cg.init(0)
    nshards = bench.NSHARDS
    env = types.SimpleNamespace(cg=cg, args=types.SimpleNamespace(gen_threads=0), ncpu=os.cpu_count() or 8, world=1, rank=0)
    rng = np.random.default_rng(6)
    tables = {}                                  # name -> (relations, shards, seed, columns, rows per shard, staged columns)
    per = args.rows // nshards
    rels = bench.generate_shards(env, bench.LINEITEM, range(nshards), per, 100)
    tables["lineitem"] = (rels, {s: cg.Shard(rels[s], [0, 1, 2]) for s in rels}, 100, bench.LINEITEM, per)
    per2 = args.c2_rows // nshards
    rels2 = bench.generate_shards(env, C2_NULL, range(nshards), per2, bench.SEED)
    tables["c2"] = (rels2, {s: cg.Shard(rels2[s], [0, 1, 2]) for s in rels2}, bench.SEED, C2_NULL, per2)
    qs = {**{k: ("lineitem", q) for k, q in lineitem_queries(rng).items()}, **{k: ("c2", q) for k, q in c2_queries().items()}}
    parts = {}
    for name, (t, q) in qs.items():
        aggs = [dataclasses.replace(a) for a in q["aggs"]]
        rels_t, _, _, _, per_t = tables[t]
        parts[name] = bench.make_partial(_Env(), rels_t, q["quals"], q["group"], aggs, per_t * nshards, expected_groups=16)[0]
    # in8_alt: the second list's descriptor, with the aggregate (and its term bound) of the partial
    alt = {}
    for name, (t, q) in qs.items():
        if "alt" in q:
            d = cg.make_desc(q["alt"], q["group"], [dataclasses.replace(a) for a in q["aggs"]])
            C.memmove(C.byref(d, capi.CgScanDesc.aggs.offset), C.byref(parts[name].desc, capi.CgScanDesc.aggs.offset),
                      C.sizeof(capi.CgAggSpec) * capi.CG_MAX_AGGS)
            alt[name] = (parts[name].desc, d)

    def run(name):
        p = parts[name]
        p.reset()
        shards = tables[qs[name][0]][1]
        for i, s in enumerate(shards):
            if name in alt:
                p.desc = alt[name][i % 2]
            p.scan_shard(shards[s], want_stats=False)
        if name in alt:
            p.desc = alt[name][0]
        return p.ngroups()

    for name in qs:                                         # warm-up: NVRTC compiles, module loads
        for _ in range(3):
            run(name)
    times = {n: [] for n in qs}
    kern = {n: [] for n in qs}
    for _ in range(args.reps):
        for name in qs:
            capi.check(capi.lib().cg_profile_begin())
            capi.check(capi.lib().cg_synchronize())
            t0 = time.perf_counter()
            run(name)
            capi.check(capi.lib().cg_synchronize())
            times[name].append((time.perf_counter() - t0) * 1e3)
            n, tot, mx = C.c_int32(), C.c_double(), C.c_double()
            capi.check(capi.lib().cg_profile_collect(C.byref(n), C.byref(tot), C.byref(mx)))
            kern[name].append(tot.value)
    # exact check on the first sample_rows rows of shard 0 (its first stripes)
    checks = {}
    for name, (t, q) in qs.items():
        rels_t, _, seed, columns, _ = tables[t]
        sample = rels_t[0].prefix(max(1, args.sample_rows // bench.STRIPE_ROWS))
        cols = synth_columns(columns, 0, sample.rows, seed)
        nulls = synth_nulls(columns, 0, sample.rows, seed)
        aggs = [dataclasses.replace(a) for a in q["aggs"]]
        part = bench.make_partial(_Env(), {0: sample}, q["quals"], q["group"], aggs, sample.rows, expected_groups=16)[0]
        sh = cg.Shard(sample)
        st = part.scan_shard(sh)
        sh.free()
        got = part.groups()
        part.free()
        want = ref.aggregate(cols, nulls, q["quals"], q["group"], aggs)
        ok = st.rows_passed == want.rows_passed
        if q["group"]:
            ok &= {(k,) for k in got} == set(want.groups)
        for k, per_got in got.items():
            key = (k,) if q["group"] else ()
            if key not in want.groups:                      # a plain aggregate over no row: one row of NULLs
                ok &= not q["group"] and all(g["count"] == 0 for g in per_got)
                continue
            for a, (g, w) in enumerate(zip(per_got, want.groups[key])):
                ok &= g["count"] == w.count and (aggs[a].kind != 2 or w.count == 0 or g["sum"] == w.sum)
        checks[name] = dict(ok=bool(ok), rows=int(sample.rows), groups=len(got))
    out = {"card": card(), "lineitem_rows": per * nshards, "c2_rows": per2 * nshards, "reps": args.reps, "queries": {}}
    for name in qs:
        out["queries"][name] = dict(ms_per_query=float(np.median(times[name])), kernel_ms=float(np.median(kern[name])),
                                    ms_spread=[float(min(times[name])), float(max(times[name]))], check=checks[name])
    r = out["queries"]
    out["in8_over_or8"] = r["in8"]["ms_per_query"] / r["or8"]["ms_per_query"]
    out["in8_alt_over_in8"] = r["in8_alt"]["ms_per_query"] / r["in8"]["ms_per_query"]
    out["is_null_filter_over_plain"] = r["c2null_f"]["ms_per_query"] / r["c2null"]["ms_per_query"]
    print(f"card: {out['card']}")
    print(f"{'query':<10} {'ms/query':>9} {'kernel ms':>10} {'spread':>17}  exact")
    for name, x in r.items():
        print(f"{name:<10} {x['ms_per_query']:9.2f} {x['kernel_ms']:10.2f} {x['ms_spread'][0]:8.2f}-{x['ms_spread'][1]:<8.2f} {x['check']['ok']}")
    print(f"in8 / or8: {out['in8_over_or8']:.3f}   in8_alt / in8: {out['in8_alt_over_in8']:.3f}   c2null with IS NULL filter / without: {out['is_null_filter_over_plain']:.3f}")
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
