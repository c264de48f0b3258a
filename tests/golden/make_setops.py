#!/usr/bin/env python
"""Extract the reference's set-operation test data into setops.json.

Run in the build container (needs /root/reference); the JSON is committed so the tests run anywhere.  Raw data only:
  test/sqlite-small/setops.test   the six queries: their SQL and their answer rows (rowsort)
  test/sqlite/select4.test        the rows of t1..t9 (its INSERT statements, in file order; columns a..e, the text column x is never
                                  read by the queries kept) and the SQL and valuesort answer of every 8th compound query (in file order)
                                  in which INTERSECT, if present, is the first operator, so that its meaning does not depend on operator
                                  precedence (SQLite applies compound operators left to right, standard SQL binds INTERSECT tighter).
                                  An answer is either its values, as listed, or "N values hashing to <md5>".
The file holds one table or one query per line.
"""
import json
import os
import re

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))


def records(path):
    """(header, sql lines, answer lines, first line number) of every `query` record"""
    lines = open(path).read().split("\n")
    i = 0
    while i < len(lines):
        if lines[i].startswith("query"):
            start, head = i + 1, lines[i]
            i += 1
            sql = []
            while lines[i].strip() != "----":
                sql.append(lines[i])
                i += 1
            i += 1
            ans = []
            while i < len(lines) and lines[i].strip():
                ans.append(lines[i].strip())
                i += 1
            yield head, sql, ans, start
        i += 1


OPS = re.compile(r"^\s*(UNION ALL|UNION|EXCEPT|INTERSECT)\s*$")
STRIDE = 8  # every 8th qualifying query: their operators, operand shapes and answer forms are those of the whole file


def main():
    out = {"setops_test": [], "select4": {"tables": {}, "queries": []}}
    for head, sql, ans, line in records(os.path.join(REF, "test/sqlite-small/setops.test")):
        out["setops_test"].append({"line": line, "sql": "\n".join(sql), "rows": ans})
    s4 = os.path.join(REF, "test/sqlite/select4.test")
    ins = re.compile(r"^INSERT INTO (t\d) VALUES\((.*)\)$")
    for ln in open(s4):
        m = ins.match(ln.strip())
        if m:
            vals = [v.strip() for v in m.group(2).split(",")]
            row = [None if v == "NULL" else int(v) for v in vals[:5]]
            out["select4"]["tables"].setdefault(m.group(1), []).append(row)
    total = qualifying = 0
    for head, sql, ans, line in records(s4):
        if head.split()[2] != "valuesort":
            continue
        total += 1
        ops = [OPS.match(x).group(1) for x in sql if OPS.match(x)]
        if "INTERSECT" in ops[1:]:
            continue
        qualifying += 1
        if (qualifying - 1) % STRIDE:
            continue
        q = {"line": line, "sql": "\n".join(sql)}
        m = re.match(r"^(\d+) values hashing to ([0-9a-f]{32})$", ans[0]) if ans else None
        if m:
            q["n_values"], q["md5"] = int(m.group(1)), m.group(2)
        else:
            q["values"] = ans
        out["select4"]["queries"].append(q)
    out["select4"]["valuesort_queries_in_file"] = total
    out["select4"]["qualifying_queries_in_file"] = qualifying
    dump = lambda x: json.dumps(x, separators=(",", ":"))
    s4 = out["select4"]
    lines = ['{"setops_test":[', ",\n".join(dump(q) for q in out["setops_test"]), '],"select4":{"valuesort_queries_in_file":%d,"qualifying_queries_in_file":%d,'
             % (total, qualifying), '"tables":{', ",\n".join(dump(k) + ":" + dump(v) for k, v in sorted(s4["tables"].items())), '},"queries":[',
             ",\n".join(dump(q) for q in s4["queries"]), "]}}"]
    with open(os.path.join(HERE, "setops.json"), "w") as fh:
        fh.write("\n".join(lines) + "\n")
    assert json.load(open(os.path.join(HERE, "setops.json"))) == out
    print(len(out["setops_test"]), "setops.test queries;", {k: len(v) for k, v in s4["tables"].items()}, len(s4["queries"]), "of", qualifying, "of", total)


if __name__ == "__main__":
    main()
