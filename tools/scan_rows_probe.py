#!/usr/bin/env python
"""Cost of the row-emitting scan (cg_scan_shard_rows): the map query of a repartition join over C2-shaped shards.

    relation  C2's schema: eight int8 columns, c0 ~ U[0, 2000), c1 ~ U[0, 100), c2 ~ U[-1e9, 1e9), c3..c7 ~ U[0, 2^40),
              no NULLs; --rows rows (default 1 B) in 32 shards, c0, c1 and c2 staged in HBM
    query     SELECT c0, c2 FROM shard WHERE c1 < k, k = 1, 10, 50, 100: about 1 %, 10 %, 50 % and 100 % of the rows,
              into one pair of device columns sized for the largest shard (a map task routes a shard's rows before the
              next shard is scanned)
    baseline  SELECT count(*) FROM shard WHERE c1 < k through cg_scan_shard, into one partial

Per selectivity, the median over --reps warm repetitions of the 32 shards:
    select    kernel time of pass 1 + the tile-offset scan (the stats of the count-only call, capacity 0)
    write     kernel time of pass 3 (the stats of the writing call, minus its select part)
    call      host clock around the 32 writing calls and a device synchronise
    count(*)  kernel time of the 32 aggregate scans
with the algorithmic bytes of each pass (select: the WHERE column's 8 bytes per row + its exists bits + one bitmap bit
per row; write: one bitmap bit per row + 8 bytes per passing row and projected column read and written) over its kernel
time, and that rate over the H100 SXM data-sheet bandwidth of 3.35 TB/s.  The card, its power limit and SM clock are read
in the same run.  Shard 0's rows at every selectivity are checked against the generator's formula; the run fails when a
check does.

    python tools/scan_rows_probe.py [--rows 1000000000] [--reps 5] [--json profiles/h100_scan_rows_probe.json]
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

from citus_b200 import build  # noqa: E402

build.build()
from citus_b200 import columnar as cg  # noqa: E402
from filter_probe import card, synth_columns  # noqa: E402

NSHARDS = 32
C2_COLS = [(8, 0, 0, 2000, 0), (8, 0, 0, 100, 0), (8, 0, -10**9, 10**9, 0)] + [(8, 0, 0, 1 << 40, 0)] * 5
STAGED = [0, 1, 2]
ATTS = [0, 2]
SELECTIVITY = {"1%": 1, "10%": 10, "50%": 50, "100%": 100}
PEAK_BYTES_PER_S = 3.35e12
SEED = 20261019


def make_shards(nrows):
    per = nrows // NSHARDS
    shards, firsts = [], []
    for s in range(NSHARDS):
        rel = cg.Relation.generate(C2_COLS, per, seed=SEED, first_row=s * per)
        sh = cg.Shard(rel, columns=STAGED)
        sh.rel = None                                       # the staged shard no longer needs the host pages
        shards.append(sh)
        firsts.append(s * per)
    return shards, firsts, per


def save(out, path):
    """written after every selectivity, so that a run cut short keeps what it measured"""
    if not path:
        return
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "w") as f:
        json.dump(out, f, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json")
    a = ap.parse_args()
    import torch
    cg.init(0)
    out = dict(card=card(), rows=a.rows, shards=NSHARDS, reps=a.reps, peak_bytes_per_s=PEAK_BYTES_PER_S, queries={})
    print("card:", out["card"], flush=True)
    t0 = time.perf_counter()
    shards, firsts, per = make_shards(a.rows)
    print(f"{NSHARDS} shards of {per} rows generated and staged in {time.perf_counter() - t0:.1f} s", flush=True)
    d_cols = [torch.empty(per, dtype=torch.int64, device="cuda") for _ in ATTS]
    ptrs = [c.data_ptr() for c in d_cols]
    ok = True
    for name, k in SELECTIVITY.items():
        desc = cg.make_desc([(1, "<", k)])
        cdesc = cg.make_desc([(1, "<", k)], (), [cg.count_star()])
        sel_ms, write_ms, call_ms, count_ms = [], [], [], []
        passed = 0
        for rep in range(a.reps + 1):                       # the first repetition warms up
            t_sel = t_write = 0.0
            passed = 0
            for sh in shards:
                n, st0 = sh.scan_rows(desc, ATTS)
                _, st = sh.scan_rows(desc, ATTS, ptrs, None, n)
                t_sel += st0.kernel_ms
                t_write += st.kernel_ms - st0.kernel_ms
                passed += n
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for sh in shards:
                n, _ = sh.scan_rows(desc, ATTS, want_stats=False)
                sh.scan_rows(desc, ATTS, ptrs, None, n, want_stats=False)
            torch.cuda.synchronize()
            t_call = (time.perf_counter() - t0) * 1e3
            agg = cg.GpuColumnarAgg(cdesc, [(8, 0)] * 8, 0, -1, per)
            t_count = sum(agg.scan_shard(sh).kernel_ms for sh in shards)
            counted = agg.groups()
            agg.free()
            if rep == 0:
                continue
            sel_ms.append(t_sel)
            write_ms.append(t_write)
            call_ms.append(t_call)
            count_ms.append(t_count)
        want_count = list(counted.values())[0][0]["count"] if counted else 0
        # shard 0 against the generator's formula
        n0, _ = shards[0].scan_rows(desc, ATTS, ptrs, None, per)
        vals = synth_columns(C2_COLS[:3], firsts[0], per, SEED)
        keep = vals[1] < k
        check = (n0 == int(keep.sum()) and np.array_equal(d_cols[0][:n0].cpu().numpy(), vals[0][keep])
                 and np.array_equal(d_cols[1][:n0].cpu().numpy(), vals[2][keep]) and passed == want_count)
        ok &= check
        rows = per * NSHARDS
        sel_bytes = rows * 8 + rows // 8 + rows // 8
        write_bytes = rows // 8 + passed * 8 * len(ATTS) * 2
        m_sel, m_write = statistics.median(sel_ms), statistics.median(write_ms)
        q = dict(k=k, rows=rows, passed=passed, fraction=passed / rows, check=check,
                 select_ms=m_sel, write_ms=m_write, call_ms=statistics.median(call_ms), count_star_ms=statistics.median(count_ms),
                 select_bytes=sel_bytes, write_bytes=write_bytes,
                 select_gb_per_s=sel_bytes / m_sel / 1e6, write_gb_per_s=write_bytes / m_write / 1e6 if m_write > 0 else None,
                 select_share_of_peak=sel_bytes / (m_sel / 1e3) / PEAK_BYTES_PER_S,
                 write_share_of_peak=write_bytes / (m_write / 1e3) / PEAK_BYTES_PER_S if m_write > 0 else None,
                 spread=dict(select_ms=[min(sel_ms), max(sel_ms)], write_ms=[min(write_ms), max(write_ms)],
                             call_ms=[min(call_ms), max(call_ms)]))
        out["queries"][name] = q
        print(name, json.dumps({x: (round(v, 4) if isinstance(v, float) else v) for x, v in q.items() if x != "spread"}), flush=True)
        save(out, a.json)
    out["card_after"] = card()
    for sh in shards:
        sh.free()
    save(out, a.json)
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
