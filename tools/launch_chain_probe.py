#!/usr/bin/env python
"""What the ends of the C2 scan launches cost: the 1 B-row C2 query (WHERE f < 50 GROUP BY key, sum(v), count(*),
bench.py's data, its three projected columns only) timed two ways on HBM-resident data, alternately in one process:

    (a) reset + 32 shard scans back to back, as bench.py's headline step runs them (CUDA events around the sequence)
    (b) reset + the same rows staged as ONE shard and scanned in one launch

(a) - (b) is what the drain at the end of each launch and the gap to the next one cost.  Then (c): a torch.profiler
trace of (a), written to --out, and from it each scan kernel's start and end: the gap (or, when launches overlap, the
negative gap) between consecutive scan kernels.  Prints the card and its power limit with the numbers.

    python tools/launch_chain_probe.py [--rows 1000000000] [--reps 5] [--out DIR] [--json FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from citus_b200 import build  # noqa: E402

build.build()
from citus_b200 import columnar as cg  # noqa: E402

NSHARDS = 32
SEED = 20260922                 # bench.py's C2 data
STRIPE_ROWS, CHUNK_ROWS = 150_000, 10_000
NKEYS = 1_000_000
COLUMNS = [(8, 0, 0, NKEYS, 0), (8, 0, 0, 100, 0), (8, 0, -10**9, 10**9, 0)]     # key, f, v
QUALS, GROUP = [(1, "<", 50)], [0]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip()


def stage(rows, first_row, threads):
    rel = cg.Relation.generate(COLUMNS, rows, seed=SEED, first_row=first_row, stripe_row_limit=STRIPE_ROWS,
                               chunk_row_limit=CHUNK_ROWS, nthreads=threads)
    sh = cg.Shard(rel)
    return rel, sh


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="directory for the trace (default: a new temporary directory)")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this probe measures the GPU"
    cg.init(0)
    torch.cuda.set_stream(torch.cuda.Stream())
    cg.use_torch_stream()
    threads = max(4, min(64, os.cpu_count() or 4))
    per = args.rows // NSHARDS
    rows = per * NSHARDS
    t0 = time.time()
    shards, one_shape = [], None
    for s in range(NSHARDS):
        rel, sh = stage(per, s * per, threads)
        shards.append(sh)
        del rel
    # (b): the same rows as one shard; a 1 B-row shard is within the library's limits (uint32 chunk-group ids)
    rel1, one = stage(rows, 0, threads)
    one_shape = f"1 shard x {rows} rows"
    aggs = [cg.sum_(2), cg.count_star()]
    desc = cg.make_desc(QUALS, GROUP, aggs)
    kmin, kmax, bounds, _ = cg.relation_bounds(rel1, desc)
    aggs[0].term_abs_bound = bounds[0]
    desc = cg.make_desc(QUALS, GROUP, aggs)
    coldescs = rel1.column_descs()
    del rel1
    part = cg.GpuColumnarAgg(desc, coldescs, kmin, kmax, rows)
    print(f"staged {NSHARDS} shards + {one_shape} in {time.time() - t0:.1f}s", file=sys.stderr)

    def run_a():
        part.reset()
        for sh in shards:
            part.scan_shard(sh, want_stats=False)

    def run_b():
        part.reset()
        part.scan_shard(one, want_stats=False)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1)

    def result():
        f = part.fetch()
        o = np.argsort(f["keys"], kind="stable")
        return [f[x][o] for x in ("keys", "key_nulls", "sum_hi", "sum_lo", "count")]

    # both forms give the same groups
    run_a()
    ga = result()
    run_b()
    gb = result()
    same = all(np.array_equal(x, y) for x, y in zip(ga, gb))
    for _ in range(args.warmup):
        timed(run_a)
        timed(run_b)
    a, b = [], []
    for _ in range(args.reps):
        a.append(timed(run_a))
        b.append(timed(run_b))
    a, b = np.array(a), np.array(b)

    # (c) the trace of (a)
    from torch.profiler import ProfilerActivity, profile
    out = args.out or tempfile.mkdtemp(prefix="launch_chain_")
    os.makedirs(out, exist_ok=True)
    trace = os.path.join(out, "launch_chain_a.pt.trace.json")
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run_a()
        torch.cuda.synchronize()
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        ev = json.load(f)["traceEvents"]
    k = sorted((e["ts"], e["ts"] + e["dur"]) for e in ev
               if e.get("cat") == "kernel" and e.get("name", "").startswith(("cg_scan_fast_kernel", "cg_jit_scan", "void cg_scan_fast_kernel")))
    gaps = [k[i + 1][0] - k[i][1] for i in range(len(k) - 1)]
    durs = [e - s for s, e in k]

    res = {
        "card": card(),
        "rows": rows,
        "a_ms": {"mean": float(a.mean()), "min": float(a.min()), "max": float(a.max()), "runs": a.tolist()},
        "b_ms": {"mean": float(b.mean()), "min": float(b.min()), "max": float(b.max()), "runs": b.tolist(), "shape": one_shape},
        "a_minus_b_ms": float(a.mean() - b.mean()),
        "a_minus_b_frac_of_a": float((a.mean() - b.mean()) / a.mean()),
        "spread_ms": float(max(a.max() - a.min(), b.max() - b.min())),
        "same_groups": bool(same),
        "trace": {"file": trace, "scan_kernels": len(k),
                  "kernel_us": {"mean": float(np.mean(durs)) if durs else None, "max": float(np.max(durs)) if durs else None},
                  "gap_us": {"mean": float(np.mean(gaps)) if gaps else None, "min": float(np.min(gaps)) if gaps else None,
                             "max": float(np.max(gaps)) if gaps else None},
                  "overlapping_pairs": int(sum(g < 0 for g in gaps)),
                  "first_start_to_last_end_us": float(k[-1][1] - k[0][0]) if k else None},
    }
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
