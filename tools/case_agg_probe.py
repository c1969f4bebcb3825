#!/usr/bin/env python
"""Cost of CASE aggregate arguments, one process, builds alternated within every repetition:

    pivot     C2-shaped relation r(key, m, v): key ~ U[0, 2^20) (dense 1 M groups), m ~ U[0, 8), v ~ U[0, 1000); --rows rows
              (default 200 M) in 32 HBM-resident shards, GROUP BY key with
                P_case    8 x sum(CASE WHEN m = i THEN v ELSE 0 END)
                P_filter  8 x sum(v) FILTER (WHERE m = i)          the same totals (NULL where the CASE gives 0)
                P_plain   count(*), sum(v)
    ch_q12    a CH-Q12-shaped single-table query over l(mode, prio, ship, commit, receipt), mode ~ U[0, 7) (a small-domain
              key), prio ~ U[1, 6): WHERE mode IN (2, 5) AND commit < receipt AND ship < commit AND receipt in one year,
              GROUP BY mode, sum(CASE WHEN prio = 1 OR prio = 2 THEN 1 ELSE 0 END) and the complementary CASE
    join_q12  the TPC-H Q12 shape through cg_join_aggregate: orders(k, prio) JOIN lineitem(k, mode, ship, commit,
              receipt), --join-rows rows per side (default 256 M), k ~ U[0, 2^28), next to J2 of
              tools/join_aggregate_probe.py (count(*), sum(r.x), sum(s.y) GROUP BY r.g) on the same keys

Prints per query the median over --reps warm runs (host clock around the launches and a device synchronise), with the
card, its power limit and SM clock read in the same run.  Each query is checked against tests/reference.py on a
sample (the scans: the first stripe of one shard, 150 000 rows; the join: --sample-rows rows per side); the run fails
when a check does.

    python tools/case_agg_probe.py [--rows 200000000] [--join-rows 268435456] [--reps 10] [--sample-rows 20000] [--json FILE]
"""
import argparse
import dataclasses
import json
import os
import statistics
import sys
import time


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from citus_b200 import build  # noqa: E402

build.build()
from citus_b200 import capi  # noqa: E402
from citus_b200 import columnar as cg  # noqa: E402
from filter_probe import card, synth_columns  # noqa: E402

import reference as ref  # noqa: E402
import join_agg_reference as jref  # noqa: E402

NSHARDS = 32
KEYS = 1 << 20
PIVOT_COLS = [(8, 0, 0, KEYS, 0), (8, 0, 0, 8, 0), (8, 0, 0, 1000, 0)]                           # key, m, v
Q12_COLS = [(8, 0, 0, 7, 0), (8, 0, 1, 6, 0), (8, 0, 0, 2000, 0), (8, 0, 0, 2000, 0), (8, 0, 0, 2000, 0)]   # mode prio ship commit receipt


def pivot_queries():
    Case, Const = cg.Case, cg.Const
    return {"P_case": dict(where=[], group=[0], aggs=[cg.sum_(Case([((1, "=", i), 2)], else_=Const(0))) for i in range(8)]),
            "P_filter": dict(where=[], group=[0], aggs=[cg.sum_(2, filter=(1, "=", i)) for i in range(8)]),
            "P_plain": dict(where=[], group=[0], aggs=[cg.count_star(), cg.sum_(2)])}


def q12_aggs(prio):
    Case, Const = cg.Case, cg.Const
    high = Case([(("or", (prio, "=", 1), (prio, "=", 2)), Const(1))], else_=Const(0))
    low = Case([(("and", (prio, "<>", 1), (prio, "<>", 2)), Const(1))], else_=Const(0))
    return [cg.sum_(high), cg.sum_(low)]


def q12_where(mode, ship, commit, receipt):
    return [(mode, "in", (2, 5)), (commit, "<", cg.Col(receipt)), (ship, "<", cg.Col(commit)), (receipt, ">=", 500), (receipt, "<", 865)]


def ch_queries():
    return {"ch_q12": dict(where=q12_where(0, 2, 3, 4), group=[0], aggs=q12_aggs(1))}


def partial_for(rels, q, rows):
    d = cg.make_desc(q["where"], q["group"], q["aggs"])
    kmin = min(cg.relation_bounds(r, d)[0] for r in rels)
    kmax = max(cg.relation_bounds(r, d)[1] for r in rels)
    bounds = [max(b) for b in zip(*[cg.relation_bounds(r, d)[2] for r in rels])]
    aggs = [dataclasses.replace(a, term_abs_bound=b) for a, b in zip(q["aggs"], bounds)]
    d = cg.make_desc(q["where"], q["group"], aggs)
    return cg.GpuColumnarAgg(d, rels[0].column_descs(), kmin, kmax, rows), aggs


def scan_all(agg, shards):
    agg.reset()
    for sh in shards:
        agg.scan_shard(sh, want_stats=False)
    capi.check(capi.lib().cg_synchronize())


def timed(run, names, reps):
    for name in names:                                     # warm-up: NVRTC compiles, module loads
        run(name)
        run(name)
    ms = {n: [] for n in names}
    for _ in range(reps):
        for name in names:                                 # alternated
            t0 = time.perf_counter()
            run(name)
            ms[name].append((time.perf_counter() - t0) * 1e3)
    return {n: dict(median_ms=statistics.median(v), ms=v) for n, v in ms.items()}


def scan_leg(cols_spec, queries, nrows, reps, seed, out):
    per = nrows // NSHARDS
    rels = [cg.Relation.generate(cols_spec, per, seed=seed, first_row=s * per, stripe_row_limit=150000, chunk_row_limit=10000,
                                 nthreads=max(4, os.cpu_count() or 8)) for s in range(NSHARDS)]
    shards = [cg.Shard(r) for r in rels]
    parts = {n: partial_for(rels, q, per * NSHARDS)[0] for n, q in queries.items()}
    try:
        res = timed(lambda n: scan_all(parts[n], shards), list(queries), reps)
        for n, q in queries.items():
            res[n]["groups"] = parts[n].ngroups()
            res[n]["rows"] = per * NSHARDS
            # the sample: the first stripe of shard 0 (150 000 rows)
            sample = rels[0].prefix(1)
            agg, aggs = partial_for([sample], q, sample.rows)
            try:
                sh = cg.Shard(sample)
                agg.scan_shard(sh, want_stats=False)
                sh.free()
                got = agg.groups()
            finally:
                agg.free()
            cols = synth_columns(cols_spec, 0, sample.rows, seed)
            want = ref.aggregate(cols, None, q["where"], q["group"], aggs)
            ok = set(got) == {k[0] for k in want.groups}
            for (k,), pw in want.groups.items():
                for a, w in enumerate(pw):
                    g = got.get(k)
                    ok &= g is not None and g[a]["count"] == w.count and (aggs[a].kind != 2 or w.count == 0 or g[a]["sum"] == w.sum)
            res[n]["check"] = dict(ok=bool(ok), rows=int(sample.rows))
            print(n, round(res[n]["median_ms"], 3), "ms,", res[n]["groups"], "groups, sample exact:", bool(ok), flush=True)
        out["queries"].update(res)
    finally:
        for p in parts.values():
            p.free()
        for sh in shards:
            sh.free()


def join_tables(n, nkeys, seed):
    import torch
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    ri = lambda lo, hi: torch.randint(lo, hi, (n,), generator=g, device="cuda")     # noqa: E731
    orders = [ri(0, nkeys), ri(1, 6), ri(-2**31, 2**31), ri(0, 1000)]                # k, prio, x, g
    line = [ri(0, nkeys), ri(0, 7), ri(0, 2000), ri(0, 2000), ri(0, 2000), ri(-2**31, 2**31)]   # k, mode, ship, commit, receipt, y
    torch.cuda.synchronize()
    return orders, line


# attributes: 0 o.k, 1 o.prio, 2 o.x, 3 o.g | 4 l.k, 5 l.mode, 6 l.ship, 7 l.commit, 8 l.receipt, 9 l.y
JOIN_COLS = [(8, 0)] * 10


def join_queries():
    return {"join_q12": dict(where=q12_where(5, 6, 7, 8), group=[5], aggs=q12_aggs(1), kmin=0, kmax=6),
            "join_J2": dict(where=[], group=[3], aggs=[cg.count_star(), cg.sum_(2), cg.sum_(9)], kmin=0, kmax=999)}


def join_call(agg, o, li, want_stats=False):
    return agg.join_aggregate([t.data_ptr() for t in o], 0, o[0].numel(), [t.data_ptr() for t in li], 0, li[0].numel(),
                              want_stats=want_stats)


def join_leg(nrows, reps, sample_rows, out):
    qs = join_queries()
    # the sample: every query against the CASE reference over numpy's equi-join
    o, li = join_tables(sample_rows, sample_rows, 7)
    jc, jn = jref.join([t.cpu().numpy() for t in o], [None] * 4, 0, [t.cpu().numpy() for t in li], [None] * 6, 0)
    checks = {}
    for n, q in qs.items():
        agg = cg.GpuColumnarAgg(cg.make_desc(q["where"], q["group"], q["aggs"]), JOIN_COLS, q["kmin"], q["kmax"], len(jc[0]) + 1)
        try:
            join_call(agg, o, li)
            got = agg.groups()
        finally:
            agg.free()
        want = ref.aggregate(jc, jn, q["where"], q["group"], q["aggs"])
        ok = set(got) == {k[0] for k in want.groups}
        for (k,), pw in want.groups.items():
            for a, w in enumerate(pw):
                ok &= k in got and got[k][a]["count"] == w.count and (q["aggs"][a].kind != 2 or w.count == 0 or got[k][a]["sum"] == w.sum)
        checks[n] = dict(ok=bool(ok), rows_per_side=sample_rows, joined_rows=len(jc[0]))
    del o, li
    o, li = join_tables(nrows, 1 << 28, 11)
    parts = {n: cg.GpuColumnarAgg(cg.make_desc(q["where"], q["group"], q["aggs"]), JOIN_COLS, q["kmin"], q["kmax"], 0) for n, q in qs.items()}
    try:
        def run(n):
            parts[n].reset()
            join_call(parts[n], o, li)
            capi.check(capi.lib().cg_synchronize())
        res = timed(run, list(qs), reps)
        for n in qs:
            parts[n].reset()
            st = join_call(parts[n], o, li, want_stats=True)
            res[n].update(rows_per_side=nrows, joined_rows=st.rows_scanned, kernel_ms=st.kernel_ms, groups=parts[n].ngroups(), check=checks[n])
            print(n, round(res[n]["median_ms"], 3), "ms,", st.rows_scanned, "joined rows, sample exact:", checks[n]["ok"], flush=True)
        out["queries"].update(res)
    finally:
        for p in parts.values():
            p.free()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=200_000_000)
    ap.add_argument("--join-rows", type=int, default=1 << 28)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--sample-rows", type=int, default=20_000)
    ap.add_argument("--json")
    a = ap.parse_args()
    cg.init(0)
    out = dict(card=card(), reps=a.reps, queries={})
    print("card:", out["card"], flush=True)
    scan_leg(PIVOT_COLS, pivot_queries(), a.rows, a.reps, 100, out)
    scan_leg(Q12_COLS, ch_queries(), a.rows, a.reps, 200, out)
    join_leg(a.join_rows, a.reps, a.sample_rows, out)
    q = out["queries"]
    out["ratios"] = dict(case_over_filter=q["P_case"]["median_ms"] / q["P_filter"]["median_ms"],
                         case_over_plain=q["P_case"]["median_ms"] / q["P_plain"]["median_ms"],
                         join_q12_over_J2=q["join_q12"]["median_ms"] / q["join_J2"]["median_ms"])
    out["card_after"] = card()
    print(json.dumps(out["ratios"]))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)
    if not all(v["check"]["ok"] for v in q.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
