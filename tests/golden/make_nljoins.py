#!/usr/bin/env python
"""Extract the reference's inequality-correlated subquery test data into nljoins.json.

Run in the build container (needs the reference checkout); the JSON is committed so the tests run anywhere.  Raw data only:
  test/sqlite/select1.test, select2.test, select3.test   each file's t1 rows (its INSERT statements in file order, columns a..e,
      NULL as null), and the SQL, sort mode and answer of EVERY query whose only subquery is
      (SELECT count(*) FROM t1 AS x WHERE x.b<t1.b) and whose other tokens are the columns a..e of t1, integer literals, + - *,
      parentheses, the comparisons < <= > >= = <> !=, BETWEEN, AND, OR, NOT, IS [NOT] NULL, and a positional ORDER BY.  An answer is
      either its values, as listed, or "N values hashing to <md5>".
  test/sqlite-small/unnesting.test   the rows of `integers` and the inequality-correlated queries at lines 196, 282, 573, 663, 815
                                      and 831 (a record counts when its SQL starts at most two lines before), their SQL and answer rows
  test/sqlite-small/join.test        the query `x=all(... where y<=x)` at line 134, its SQL and answer rows
The file holds one table or one query per line.
"""
import json
import os
import re

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
SUB = "(SELECT count(*) FROM t1 AS x WHERE x.b<t1.b)"
WORDS = {"SELECT", "FROM", "t1", "WHERE", "ORDER", "BY", "AND", "OR", "NOT", "BETWEEN", "IS", "NULL", "a", "b", "c", "d", "e"}
TOKEN = re.compile(r"\s*(?:(__CNT__)|([A-Za-z_][A-Za-z_0-9]*)|(\d+)|(<=|>=|<>|!=|[-+*(),<>=]))")


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


def covered(sql: str) -> bool:
    """the query has the count subquery, no other subquery, and only the tokens the docstring lists"""
    if SUB not in sql:
        return False
    rest = sql.replace(SUB, " __CNT__ ")
    pos = 0
    while pos < len(rest):
        if not rest[pos:].strip():
            return True
        m = TOKEN.match(rest, pos)
        if not m:
            return False
        if m.group(2) and m.group(2) not in WORDS:
            return False
        pos = m.end()
    return rest.count("SELECT") == 1


def main():
    out = {"files": {}}
    ins = re.compile(r"^INSERT INTO t1\(([a-e,]+)\) VALUES\((.*)\)$")
    for f in ("select1", "select2", "select3"):
        path = os.path.join(REF, "test/sqlite", f + ".test")
        rows = []
        for ln in open(path):
            m = ins.match(ln.strip())
            if m:
                cols = m.group(1).split(",")
                vals = [None if v.strip() == "NULL" else int(v) for v in m.group(2).split(",")]
                d = dict(zip(cols, vals))
                rows.append([d[c] for c in "abcde"])
        queries = []
        for head, sql, ans, line in records(path):
            text = "\n".join(sql)
            if not covered(text):
                continue
            q = {"line": line, "sort": head.split()[2], "sql": text}
            m = re.match(r"^(\d+) values hashing to ([0-9a-f]{32})$", ans[0]) if ans else None
            if m:
                q["n_values"], q["md5"] = int(m.group(1)), m.group(2)
            else:
                q["values"] = ans
            queries.append(q)
        out["files"][f] = {"t1": rows, "queries": queries}
    small = []
    for f, lines in (("unnesting", (196, 282, 573, 663, 815, 831)), ("join", (134,))):
        path = os.path.join(REF, "test/sqlite-small", f + ".test")
        for head, sql, ans, line in records(path):
            if any(line <= want <= line + 2 for want in lines):
                small.append({"file": f, "line": line, "sql": "\n".join(sql), "rows": ans})
    text = open(os.path.join(REF, "test/sqlite-small/unnesting.test")).read()
    ints = re.search(r"INSERT INTO integers VALUES (.*);", text).group(1)
    out["small"] = {"integers": [None if v == "NULL" else int(v) for v in re.findall(r"\((\w+)\)", ints)], "queries": small}
    dump = lambda x: json.dumps(x, separators=(",", ":"))
    parts = []
    for f, v in out["files"].items():
        parts.append(dump(f) + ':{"t1":' + dump(v["t1"]) + ',"queries":[\n' + ",\n".join(dump(q) for q in v["queries"]) + "]}")
    with open(os.path.join(HERE, "nljoins.json"), "w") as fh:
        fh.write('{"files":{\n' + ",\n".join(parts) + '},\n"small":{"integers":' + dump(out["small"]["integers"]) + ',"queries":[\n' +
                 ",\n".join(dump(q) for q in out["small"]["queries"]) + "]}}\n")
    assert json.load(open(os.path.join(HERE, "nljoins.json"))) == out
    print({f: (len(v["t1"]), len(v["queries"])) for f, v in out["files"].items()}, [(q["file"], q["line"]) for q in small])


if __name__ == "__main__":
    main()
