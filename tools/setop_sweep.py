"""Set operations (ldb_gpu_table_setop): DISTINCT over one int64 column, over (int64, utf8 of 16-40 bytes) and over 4 columns; UNION,
INTERSECT ALL and EXCEPT of two tables; 2^24 and 2^27 rows per side; 1, 2^10, n/8 and n distinct rows.  For DISTINCT over one int64
column, the same rows through the program hash aggregation (GROUP BY the column, COUNT(*)) as an in-repo yardstick.

  python tools/setop_sweep.py [--sizes 24,27] [--reps 5] [--out result.json]

The tables are DEVICE batches of 2^24 rows built with torch: int64 columns a, b, c (a uniform over the distinct count; b and c functions of a,
so the 4-column rows are as distinct as a) and a utf8 column s of 16-40 bytes, also a function of a.  The right side of the two-table
kinds draws from the same distribution with another seed.  Per configuration, from the context's per-family CUDA-event timers:
  insert_ms   setop_insert (the set build and, for INTERSECT / EXCEPT, the right side's probe)
  scan_ms     setop_count and setop_scan (the counts, their scan and the ids)
  permute_ms  sort_exchange_permute (the result's cells)
  call_ms     the whole call, wall clock (host reads of the output size and string bytes included)
  groupby_ms  (DISTINCT over a alone) the program hash aggregation's "program" kernel and "hashagg_init"; ratio = insert + scan over it
Every number is the median of `reps` runs after a warm-up run, the cases of one size alternating run by run, reported with the card's
name and power limit read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lingodb_b200 import capi, program, runtime  # noqa: E402
from lingodb_b200.datagen import ColumnSpec  # noqa: E402
from markjoin_sweep import card  # noqa: E402

FAMILIES = {"insert": ("setop_insert",), "scan": ("setop_count", "setop_scan"), "permute": ("sort_exchange_permute",)}
CASES = [("distinct_i64", "distinct", ["a"]), ("distinct_i64_utf8", "distinct", ["a", "s"]), ("distinct_4col", "distinct", ["a", "b", "c", "s"]),
         ("union", "union", ["a"]), ("intersect_all", "intersect_all", ["a"]), ("except", "except", ["a"])]


def device_table(ctx, n, distinct, seed, strings=True):
    import torch
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(seed)
    a = torch.randint(0, distinct, (n,), device=dev, generator=g, dtype=torch.int64) if distinct < n else torch.randperm(n, device=dev, generator=g)
    if not strings:  # the right side of the two-table kinds: a alone
        t = runtime.Table(ctx, "r", [ColumnSpec("a", "int64")])
        t.append_device({"a": a}, n)
        torch.cuda.synchronize()
        return t
    t = runtime.Table(ctx, "s", [ColumnSpec("a", "int64"), ColumnSpec("b", "int64"), ColumnSpec("c", "int64"), ColumnSpec("s", "utf8")])
    # batches of 2^24 rows (int32 utf8 offsets); s: 16 + (a % 25) bytes, the decimal digits of a padded with '#'
    for r0 in range(0, n, 1 << 24):
        ab = a[r0:r0 + (1 << 24)].contiguous()
        m = ab.numel()
        offs = torch.zeros(m + 1, dtype=torch.int64, device=dev)
        offs[1:] = torch.cumsum(16 + (ab % 25), 0)
        pos = torch.arange(int(offs[-1]), device=dev, dtype=torch.int64)
        row = torch.searchsorted(offs[1:], pos, right=True)
        k = pos - offs[row]
        digit = (ab[row] // torch.pow(10, torch.clamp(k, max=18))) % 10
        data = torch.where(k < 19, digit + 48, torch.full_like(k, 35)).to(torch.uint8)
        del pos, row, k, digit
        t.append_device({"a": ab, "b": ab * 7 + 3, "c": ab ^ 0x5555, "s": (offs.to(torch.int32), data)}, m)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()  # the string build's temporaries go back to the device
    return t


def timed(ctx, fn, families):
    ctx.synchronize()
    ctx.kernel_time_reset(True)
    t0 = time.perf_counter()
    out = fn()
    ctx.synchronize()
    call = (time.perf_counter() - t0) * 1e3
    r = {k: sum(ctx.kernel_time(f)[0] for f in fs) for k, fs in families.items()}
    r["call"] = call
    ctx.kernel_time_reset(False)
    return out, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="24,27", help="log2 of the row counts per side")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    res = {"card": card(), "reps": a.reps}
    for lg in [int(x) for x in a.sizes.split(",")]:
        n = 1 << lg
        for dname, distinct in (("d1", 1), ("d1024", 1 << 10), ("dn8", n // 8), ("dn", n)):
            # a context per configuration: its pool of scratch buffers is freed with it
            with runtime.Context(0) as ctx:
                L = device_table(ctx, n, distinct, 1)
                R = device_table(ctx, n, distinct, 2, strings=False)
                lr, rr = program.RawTable(ctx, L.h), program.RawTable(ctx, R.h)
                samples = {c[0]: [] for c in CASES}
                samples["groupby"] = []
                rows = {}
                for rep in range(a.reps + 1):  # the first run warms up
                    for name, kind, cols in CASES:
                        if f"n2^{lg}_{dname}_{name}_error" in res:
                            continue
                        fn = (lambda cols=cols: lr.distinct(cols)) if kind == "distinct" else (lambda kind=kind, cols=cols: lr.setop(rr, kind, cols, cols))
                        try:
                            out, r = timed(ctx, fn, FAMILIES)
                        except capi.LdbRuntimeError as e:  # a result utf8 column past 2^31 - 1 bytes (int32 offsets)
                            ctx.kernel_time_reset(False)
                            res[f"n2^{lg}_{dname}_{name}_error"] = str(e)
                            continue
                        rows[name] = out.num_rows
                        out.destroy()
                        if rep:
                            samples[name].append(r)
                    if f"n2^{lg}_{dname}_groupby_error" in res:
                        continue
                    try:
                        st, r = timed(ctx, lambda: program.group_by(ctx, L, [("col", "a")], [("count_star", None)], expected_groups=min(n, distinct)),
                                      {"groupby": ("program", "hashagg_init")})
                    except capi.LdbRuntimeError as e:  # the aggregation table does not fit: no yardstick at this size
                        ctx.kernel_time_reset(False)
                        res[f"n2^{lg}_{dname}_groupby_error"] = str(e)
                        continue
                    ctx.L.ldb_gpu_state_destroy(st)
                    if rep:
                        samples["groupby"].append(r)
                for name, rs in samples.items():
                    if not rs:
                        continue
                    key = f"n2^{lg}_{dname}_{name}"
                    med = {k: float(np.median([x[k] for x in rs])) for k in rs[0]}
                    for k, v in med.items():
                        res[f"{key}_{k}_ms"] = v
                    if name in rows:
                        res[f"{key}_rows"] = rows[name]
                d = f"n2^{lg}_{dname}_"
                if samples["groupby"] and samples["distinct_i64"]:
                    res[d + "distinct_i64_vs_groupby"] = (res[d + "distinct_i64_insert_ms"] + res[d + "distinct_i64_scan_ms"]) / res[d + "groupby_groupby_ms"]
                print(json.dumps({k: v for k, v in res.items() if k.startswith(d)}), flush=True)
                L.clear()
                R.clear()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
