#!/usr/bin/env python
"""Builds the committed fixtures of the CASE-aggregate goldens (TPC-H Q12 and Q14) from the reference's own test inputs
and outputs.

Needs a checkout of citusdata/citus (the commit SURVEY.md names):
    python tests/golden/make_case_golden.py /path/to/citus
Outputs (committed):
    tests/golden/case_golden.npz   orders (o_orderkey, o_orderpriority as its leading digit 1..5), the l_shipmode code of
                                   every lineitem row in lineitem.npz's row order (SHIPMODES index), and part (p_partkey,
                                   p_type LIKE 'PROMO%' as 0 / 1; part.data only: multi_load_more_data appends
                                   part.more.data after the TPC-H query tests have run)
    tests/golden/case_golden.json  the Q12 and Q14 result rows of multi_tpch_query12.out / multi_tpch_query14.out
The tests only read the committed outputs, never the Citus sources.
"""
import json
import os
import re
import sys

import numpy as np

REF = os.path.join(sys.argv[1] if len(sys.argv) > 1 else "citus", "src", "test", "regress")
HERE = os.path.dirname(os.path.abspath(__file__))
SHIPMODES = ["AIR", "FOB", "MAIL", "RAIL", "REG AIR", "SHIP", "TRUCK"]


def rows(name):
    with open(f"{REF}/data/{name}") as f:
        for line in f:
            yield line.rstrip("\n").split("|")


def main():
    okey, oprio = [], []
    for fi in (1, 2):
        for p in rows(f"orders.{fi}.data"):
            okey.append(int(p[0]))
            oprio.append(int(p[5][0]))
    shipmode = [SHIPMODES.index(p[14]) for fi in (1, 2) for p in rows(f"lineitem.{fi}.data")]
    li = np.load(os.path.join(HERE, "lineitem.npz"))
    assert len(shipmode) == len(li["l_orderkey"]), "lineitem.npz must come from the same data files"
    pkey, promo = [], []
    for p in rows("part.data"):
        pkey.append(int(p[0]))
        promo.append(int(p[4].startswith("PROMO")))
    np.savez_compressed(os.path.join(HERE, "case_golden.npz"), o_orderkey=np.asarray(okey, np.int64),
                        o_orderpriority=np.asarray(oprio, np.int64), l_shipmode=np.asarray(shipmode, np.int64),
                        p_partkey=np.asarray(pkey, np.int64), p_promo=np.asarray(promo, np.int64))

    def result_rows(name):
        text = open(f"{REF}/expected/{name}").read()
        body = text.split("-" * 20)[-1]
        return [[c.strip() for c in line.split("|")] for line in body.splitlines()
                if line.strip() and not re.match(r"^\(\d+ rows?\)$", line.strip()) and not line.startswith("-")]
    out = {"shipmodes": SHIPMODES, "q12": result_rows("multi_tpch_query12.out"), "q14": result_rows("multi_tpch_query14.out")}
    with open(os.path.join(HERE, "case_golden.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
