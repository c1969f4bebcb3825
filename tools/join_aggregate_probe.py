#!/usr/bin/env python
"""Cost of cg_join_aggregate against the fixed cg_join_count_sum on the C4 shape: r(k, x, g) and s(k, y, h), N rows each
(default 256 M), k ~ U[0, 2^28), held in HBM as device arrays (what the repartition exchange delivers):

    J0   cg_join_count_sum(r.k, r.x, s.k, s.y)                       count(*), sum(r.x + s.y), the fixed query
    J1   count(*), sum(r.x), sum(s.y)                                 the join aggregate, no GROUP BY
    J2   J1 GROUP BY r.g, g ~ U[0, 1000)                              dense table
    J3   J1 GROUP BY s.h, h ~ U[0, 2^20)                              hash table
    J4   J2 WHERE r.x < s.y, with sum(s.y) FILTER (WHERE s.h < 2^19)

Prints per query the median over --reps warm runs of the call (host clock around the call and a device synchronise) and,
for J1..J4, of kernel_ms (CUDA events around the table build and the probe-aggregate launch), the card with its power
limit and SM clock read in the same run, and the checks: J1 equals J0 at full size; J2..J4 equal an exact numpy reference
on a sample of --sample-rows rows per side (keys U[0, sample-rows)).

    python tools/join_aggregate_probe.py [--rows 268435456] [--reps 10] [--sample-rows 1000000] [--json FILE]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from citus_b200 import build  # noqa: E402

build.build()
from citus_b200 import capi  # noqa: E402
from citus_b200 import columnar as cg  # noqa: E402
from filter_probe import card  # noqa: E402

import join_agg_reference as jref  # noqa: E402

INT = 0
COLS = [(8, INT), (8, INT), (4, INT), (8, INT), (8, INT), (4, INT)]     # r.k r.x r.g s.k s.y s.h
G, H = 1000, 1 << 20


def queries():
    j1 = lambda filt=None: [cg.count_star(), cg.sum_(1), cg.sum_(4, filter=filt)]     # noqa: E731
    return {"J1": dict(where=[], group=[], aggs=j1(), kw=dict()),
            "J2": dict(where=[], group=[2], aggs=j1(), kw=dict(key_min=0, key_max=G - 1)),
            "J3": dict(where=[], group=[5], aggs=j1(), kw=dict(), expected_groups=H),
            "J4": dict(where=[(1, "<", cg.Col(4))], group=[2], aggs=j1((5, "<", H // 2)), kw=dict(key_min=0, key_max=G - 1))}


def tables(n, nkeys, seed):
    import torch
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    r = [torch.randint(0, nkeys, (n,), generator=g, device="cuda"), torch.randint(-2**31, 2**31, (n,), generator=g, device="cuda"),
         torch.randint(0, G, (n,), generator=g, device="cuda")]
    s = [torch.randint(0, nkeys, (n,), generator=g, device="cuda"), torch.randint(-2**31, 2**31, (n,), generator=g, device="cuda"),
         torch.randint(0, H, (n,), generator=g, device="cuda")]
    torch.cuda.synchronize()
    return r, s


def partial(q):
    d = cg.make_desc(q["where"], q["group"], q["aggs"], expected_groups=q.get("expected_groups", 0))
    return cg.GpuColumnarAgg(d, COLS, q["kw"].get("key_min", 0), q["kw"].get("key_max", -1), 0)


def call(agg, r, s, want_stats=True):
    n = r[0].numel()
    return agg.join_aggregate([t.data_ptr() for t in r], 0, n, [t.data_ptr() for t in s], 0, s[0].numel(), want_stats=want_stats)


def reference(q, r, s):
    """{key: (count(*), sum(x), sum(y) with its FILTER)} of the query, exact"""
    rk, rx, rg = (t.cpu().numpy() for t in r)
    sk, sy, sh = (t.cpu().numpy() for t in s)
    bi, pi = jref.join_indexes(rk, np.ones(len(rk), bool), sk, np.ones(len(sk), bool))
    x, y, gk, hk = rx[bi], sy[pi], rg[bi], sh[pi]
    keep = x < y if q["where"] else np.ones(len(x), bool)
    x, y, gk, hk = x[keep], y[keep], gk[keep], hk[keep]
    key = gk if q["group"] == [2] else hk if q["group"] == [5] else np.zeros(len(x), np.int64)
    yf = y * (hk < H // 2) if q["aggs"][2].filter is not None else y
    uk, inv = np.unique(key, return_inverse=True)
    out = {}
    cnt = np.bincount(inv, minlength=len(uk))
    sums = []
    for v in (x, yf):
        hi, lo = np.zeros(len(uk), np.int64), np.zeros(len(uk), np.int64)
        np.add.at(hi, inv, v >> 32)
        np.add.at(lo, inv, v & 0xffffffff)
        sums.append([int(a) * 2**32 + int(b) for a, b in zip(hi, lo)])
    for i, k in enumerate(uk):
        out[int(k) if q["group"] else None] = (int(cnt[i]), sums[0][i], sums[1][i])
    return out


def got_of(agg, q):
    out = {}
    for k, per in agg.groups().items():
        out[k if q["group"] else None] = (per[0]["count"], per[1]["sum"], per[2]["sum"])
    return out


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 28)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--sample-rows", type=int, default=1_000_000)
    ap.add_argument("--json")
    a = ap.parse_args()
    cg.init(0)
    out = dict(card=card(), rows=a.rows, keys=1 << 28, reps=a.reps, sample_rows=a.sample_rows, queries={}, checks={})

    # checks on the sample: J2..J4 against numpy
    rs, ss = tables(a.sample_rows, a.sample_rows, 7)
    for name, q in queries().items():
        if name == "J1":
            continue
        agg = partial(q)
        try:
            call(agg, rs, ss)
            ok = got_of(agg, q) == reference(q, rs, ss)
        finally:
            agg.free()
        out["checks"][name + "_sample_matches_numpy"] = ok
        print(name, "sample matches numpy:", ok, flush=True)
    del rs, ss

    r, s = tables(a.rows, 1 << 28, 11)
    n = a.rows
    times = []
    for i in range(a.reps + 1):
        t0 = time.perf_counter()
        rows, total = cg.join_count_sum(r[0].data_ptr(), r[1].data_ptr(), n, s[0].data_ptr(), s[1].data_ptr(), n)
        t1 = time.perf_counter()
        if i:
            times.append((t1 - t0) * 1e3)
    out["queries"]["J0"] = dict(median_ms=statistics.median(times), ms=times, joined_rows=rows)
    print("J0", round(statistics.median(times), 3), "ms,", rows, "joined rows", flush=True)
    for name, q in queries().items():
        agg = partial(q)
        try:
            wall, kern = [], []
            for i in range(a.reps + 1):
                agg.reset()
                capi.check(capi.lib().cg_synchronize())
                t0 = time.perf_counter()
                st = call(agg, r, s)
                t1 = time.perf_counter()
                if i:
                    wall.append((t1 - t0) * 1e3)
                    kern.append(st.kernel_ms)
            rec = dict(median_ms=statistics.median(wall), median_kernel_ms=statistics.median(kern), ms=wall, kernel_ms=kern,
                       rows_scanned=st.rows_scanned, rows_passed=st.rows_passed, groups=agg.ngroups())
            if name == "J1":
                (per,) = agg.groups().values()
                ok = per[0]["count"] == rows and per[1]["sum"] + per[2]["sum"] == total
                out["checks"]["J1_equals_J0_full_size"] = ok
                print("J1 equals J0:", ok, flush=True)
        finally:
            agg.free()
        out["queries"][name] = rec
        print(name, round(rec["median_ms"], 3), "ms, kernels", round(rec["median_kernel_ms"], 3), "ms,", rec["rows_scanned"],
              "joined rows,", rec["groups"], "groups", flush=True)
    out["card_after"] = card()
    torch.cuda.synchronize()
    print(json.dumps({k: v for k, v in out.items() if k != "queries"}))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
