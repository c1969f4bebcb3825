#!/usr/bin/env python
"""Builds tests/golden/variance.json from the reference's regression tests that compute stddev over integers.

Needs a checkout of citusdata/citus (the commit SURVEY.md names):
    python tests/golden/make_variance_golden.py /path/to/citus
Output (committed): tests/golden/variance.json --
    contestant    the ratings of data/contestants.{1,2}.csv and stddev_samp(rating) of
                  expected/columnar_query.out ("SELECT avg(rating), stddev_samp(rating) FROM contestant;")
    aggdata       the rows (id, key, val) of sql/aggregate_support.sql's aggdata and the result of
                  "select id, stddev(val) from aggdata group by id order by 1;" (expected/aggregate_support.out): every
                  group has at most one input, so every stddev is NULL ("" as psql prints it)
The tests only read the committed output.
"""
import json
import os
import re
import sys

REF = os.path.join(sys.argv[1] if len(sys.argv) > 1 else "citus", "src", "test", "regress")
HERE = os.path.dirname(os.path.abspath(__file__))


def table_rows(lines, after_regex):
    """rows of the first psql result table that follows a line matching after_regex"""
    i = next(k for k, l in enumerate(lines) if re.search(after_regex, l))
    while not lines[i].startswith("----"):
        i += 1
    i += 1
    rows = []
    while not re.match(r"^\(\d+ rows?\)", lines[i]):
        rows.append([c.strip() for c in lines[i].split("|")])
        i += 1
    return rows


def main():
    ratings = []
    for fi in (1, 2):
        for line in open(f"{REF}/data/contestants.{fi}.csv"):
            ratings.append(int(line.rstrip("\n").split(",")[2]))
    cq = open(f"{REF}/expected/columnar_query.out").read().split("\n")
    (avg, stddev_samp), = table_rows(cq, r"^SELECT avg\(rating\), stddev_samp\(rating\) FROM contestant;")
    sql = open(f"{REF}/sql/aggregate_support.sql").read()
    ins = re.search(r"insert into aggdata \(id, key, val, valf\) values (.*?);\n", sql).group(1)
    rows = [[None if x.strip() == "NULL" else int(x) for x in t.split(",")[:3]] for t in re.findall(r"\(([^)]*)\)", ins)]
    asup = open(f"{REF}/expected/aggregate_support.out").read().split("\n")
    by_id = table_rows(asup, r"^select id, stddev\(val\) from aggdata group by id order by 1;")
    out = {
        "contestant": {"rating": ratings, "avg": avg, "stddev_samp": stddev_samp},
        "aggdata": {"rows": rows, "stddev_by_id": [[int(i), s] for i, s in by_id]},
    }
    with open(os.path.join(HERE, "variance.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
