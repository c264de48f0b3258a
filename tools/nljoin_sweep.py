"""Nested-loop joins (ldb_gpu_table_nl_join): COUNT and SEMI of  x < y  at n = m in {2^12, 2^16, 2^20}; INNER of  |x - y| < w  written as
the band x - w < y AND y < x + w at selectivities 10^-6 .. 10^-2 (the band width over a uniform key); a band join of events against
windows; a 2^12 x 2^16 cross product.

  python tools/nljoin_sweep.py [--reps 5] [--out result.json]

The tables are DEVICE batches of int64 columns built with torch (x, and x -/+ w for the band).  Per configuration, from the context's
per-family CUDA-event timers: words_ms (nljoin_words), count_ms (nljoin_count), write_ms (nljoin_rows, nljoin_scan, nljoin_write and the
permute of the carried cells), call_ms the whole call (wall clock), and pairs_per_s = n m / count_ms, the predicate checks per second
of the count pass.  Every number is the median of `reps` runs after a warm-up, with the card's name and power limit read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from lingodb_b200 import program, runtime  # noqa: E402
from lingodb_b200.datagen import ColumnSpec  # noqa: E402
from markjoin_sweep import card  # noqa: E402

FAMILIES = {"words": ("nljoin_words",), "count": ("nljoin_count",), "write": ("nljoin_rows", "nljoin_scan", "nljoin_write", "sort_exchange_permute")}


def table(ctx, cols: dict, name):
    import torch
    n = next(iter(cols.values())).numel()
    t = runtime.Table(ctx, name, [ColumnSpec(k, "int64") for k in cols])
    t.append_device({k: v.contiguous() for k, v in cols.items()}, n)
    torch.cuda.synchronize()
    return program.RawTable(ctx, t.h), t


def measure(ctx, fn, reps):
    fn().destroy()
    res = {k: [] for k in list(FAMILIES) + ["call"]}
    for _ in range(reps):
        ctx.kernel_time_reset(True)
        t0 = time.perf_counter()
        out = fn()
        res["call"].append((time.perf_counter() - t0) * 1e3)
        for k, fams in FAMILIES.items():
            res[k].append(sum(ctx.kernel_time(f)[0] for f in fams))
        rows = out.num_rows
        out.destroy()
    ctx.kernel_time_reset(False)
    return {k + "_ms": float(np.median(v)) for k, v in res.items()}, rows


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(1)
    rows = []
    with runtime.Context(0) as ctx:
        def run(case, n, m, L, R, kind, conds, **kw):
            r, out_rows = measure(ctx, lambda: L.nl_join(R, kind, conds, **kw), a.reps)
            r.update(case=case, n=n, m=m, rows=out_rows, pairs_per_s=n * m / (r["count_ms"] * 1e-3))
            rows.append(r)
            print(json.dumps(r), flush=True)

        for lg in (12, 16, 20):
            n = 1 << lg
            x = torch.randint(0, 1 << 40, (n,), device=dev, generator=g)
            y = torch.randint(0, 1 << 40, (n,), device=dev, generator=g)
            L, lt = table(ctx, {"x": x}, "l")
            R, rt = table(ctx, {"y": y}, "r")
            run("count_lt", n, n, L, R, "count", [("x", "<", "y")], columns=[], value_name="c")
            run("semi_lt", n, n, L, R, "semi", [("x", "<", "y")], columns=["x"])
            lt.clear(), rt.clear()
        n = m = 1 << 16
        span = 1 << 40
        x = torch.randint(0, span, (n,), device=dev, generator=g)
        y = torch.randint(0, span, (m,), device=dev, generator=g)
        for sel in (1e-6, 1e-4, 1e-2):
            w = int(sel * span / 2)
            L, lt = table(ctx, {"x": x, "lo": x - w, "hi": x + w}, "l")
            R, rt = table(ctx, {"y": y}, "r")
            run(f"inner_band_sel_{sel:g}", n, m, L, R, "inner", [("lo", "<", "y"), ("hi", ">", "y")], columns=["x"], other_columns=["y"])
            lt.clear(), rt.clear()
        ev = torch.randint(0, 1 << 30, (1 << 20,), device=dev, generator=g)
        st = torch.randint(0, 1 << 30, (1 << 12,), device=dev, generator=g)
        L, lt = table(ctx, {"ts": ev}, "events")
        R, rt = table(ctx, {"start": st, "stop": st + (1 << 16)}, "windows")
        run("band_events_windows", 1 << 20, 1 << 12, L, R, "inner", [("ts", ">=", "start"), ("ts", "<=", "stop")], columns=["ts"], other_columns=["start"])
        lt.clear(), rt.clear()
        L, lt = table(ctx, {"a": torch.arange(1 << 12, device=dev)}, "a")
        R, rt = table(ctx, {"b": torch.arange(1 << 16, device=dev)}, "b")
        run("cross_2^12x2^16", 1 << 12, 1 << 16, L, R, "inner", [], columns=["a"], other_columns=["b"])
    res = {"card": card(), "rows": rows}
    if a.out:
        json.dump(res, open(a.out, "w"), indent=1)
    print("card:", res["card"])


if __name__ == "__main__":
    main()
