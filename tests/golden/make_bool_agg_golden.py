#!/usr/bin/env python
"""Builds tests/golden/bool_agg.json from the reference's bool_agg regression test (expected/bool_agg.out).

Needs a checkout of citusdata/citus (the commit SURVEY.md names):
    python tests/golden/make_bool_agg_golden.py /path/to/citus
Output (committed): tests/golden/bool_agg.json -- the bool_test rows [id, val, flag, kind] and every query's result
table, cells as psql prints them ("t" / "f", integers).  The tests only read the committed output.
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
    text = open(f"{REF}/expected/bool_agg.out").read()
    lines = text.split("\n")
    ins = re.search(r"INSERT INTO bool_test VALUES (.*?);\n", text).group(1)
    rows = [[x.strip() for x in t.split(",")] for t in re.findall(r"\(([^)]*)\)", ins)]
    out = {
        "rows": [[int(r[0]), int(r[1]), r[2] == "true", int(r[3])] for r in rows],
        "queries": [[q, table_rows(lines, "^" + re.escape(q) + "$")] for q in re.findall(r"^(SELECT .*FROM bool_test.*;)$", text, re.M)],
    }
    with open(os.path.join(HERE, "bool_agg.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print("wrote", len(out["rows"]), "rows and", len(out["queries"]), "queries")


if __name__ == "__main__":
    main()
