"""The sorted-ranges path of nested-loop joins (csrc/nljoin_sorted.cu): per-stage times and the cases either side of its selection
constants (kNljSortMinPairs, kNljCandidateRatio in csrc/nljoin.cuh).

  python tools/nljoin_sorted_sweep.py [--reps 5] [--out result.json]

Cases: COUNT and SEMI of  x < y  at n = m in {2^11 .. 2^14} (the loop below 2^24 pairs, the sorted ranges from it) and at 2^20, 2^24
and 2^27; a band join of 2^24 events against 2^16 windows with the windows on the left and on the right; COUNT of  k = k AND x < y  at
2^24 (2^12 keys); INNER  |x - y| < w  at 2^16 x 2^16 and selectivities 10^-6 .. 1/16 (a band of selectivity s has s n m candidates: past 1/kNljCandidateRatio the loop runs); a
2^12 x 2^16 cross product (the loop).  The tables are DEVICE batches of int64 columns built with torch.  Per configuration, from the
context's per-family CUDA-event timers: words_ms, sort_ms (nljoin_sort), search_ms (nljoin_search), cover_ms (nljoin_cover),
expand_ms (nljoin_expand), order_ms (nljoin_order), count_ms (the loop's nljoin_count), write_ms (nljoin_rows, nljoin_scan,
nljoin_write and the permute of the carried cells), call_ms the whole call (wall clock), and path.  Every number is the median of
`reps` runs after a warm-up, with the card's name and power limit read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from lingodb_b200 import runtime  # noqa: E402
from markjoin_sweep import card  # noqa: E402
from nljoin_sweep import table  # noqa: E402

FAMILIES = {"words": ("nljoin_words",), "sort": ("nljoin_sort",), "search": ("nljoin_search",), "cover": ("nljoin_cover",),
            "expand": ("nljoin_expand",), "order": ("nljoin_order",), "count": ("nljoin_count",),
            "write": ("nljoin_rows", "nljoin_scan", "nljoin_write", "sort_exchange_permute")}


def measure(ctx, fn, reps):
    fn().destroy()
    res = {k: [] for k in list(FAMILIES) + ["call"]}
    path = None
    for _ in range(reps):
        ctx.kernel_time_reset(True)
        t0 = time.perf_counter()
        out = fn()
        res["call"].append((time.perf_counter() - t0) * 1e3)
        for k, fams in FAMILIES.items():
            res[k].append(sum(ctx.kernel_time(f)[0] for f in fams))
        searched, looped = ctx.kernel_time("nljoin_search")[1], ctx.kernel_time("nljoin_count")[1]
        path = "sort, then loop" if searched and looped else "sort" if searched else "loop"
        rows = out.num_rows
        out.destroy()
    ctx.kernel_time_reset(False)
    return {k + "_ms": round(float(np.median(v)), 4) for k, v in res.items()}, rows, path


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
            r, out_rows, path = measure(ctx, lambda: L.nl_join(R, kind, conds, **kw), a.reps)
            r.update(case=case, n=n, m=m, rows=out_rows, path=path)
            rows.append(r)
            print(json.dumps(r), flush=True)

        for lg in (11, 12, 13, 14, 20, 24, 27):
            n = 1 << lg
            x = torch.randint(0, 1 << 40, (n,), device=dev, generator=g)
            y = torch.randint(0, 1 << 40, (n,), device=dev, generator=g)
            L, lt = table(ctx, {"x": x}, "l")
            R, rt = table(ctx, {"y": y}, "r")
            run("count_lt", n, n, L, R, "count", [("x", "<", "y")], columns=[], value_name="c")
            run("semi_lt", n, n, L, R, "semi", [("x", "<", "y")], columns=[])
            del x, y
            lt.clear(), rt.clear()
        ne, nw = 1 << 24, 1 << 16
        ev = torch.randint(0, 1 << 40, (ne,), device=dev, generator=g)
        st = torch.randint(0, 1 << 40, (nw,), device=dev, generator=g)
        E, et = table(ctx, {"ts": ev}, "events")
        W, wt = table(ctx, {"start": st, "stop": st + (1 << 16)}, "windows")
        run("band_events_windows", ne, nw, E, W, "inner", [("ts", ">=", "start"), ("ts", "<=", "stop")], columns=["ts"], other_columns=["start"])
        run("band_windows_events", nw, ne, W, E, "inner", [("start", "<=", "ts"), ("stop", ">=", "ts")], columns=["start"], other_columns=["ts"])
        et.clear(), wt.clear()
        n = 1 << 24
        L, lt = table(ctx, {"k": torch.randint(0, 1 << 12, (n,), device=dev, generator=g), "x": torch.randint(0, 1 << 40, (n,), device=dev, generator=g)}, "l")
        R, rt = table(ctx, {"k2": torch.randint(0, 1 << 12, (n,), device=dev, generator=g), "y": torch.randint(0, 1 << 40, (n,), device=dev, generator=g)}, "r")
        run("count_eq_lt", n, n, L, R, "count", [("k", "=", "k2"), ("x", "<", "y")], columns=[], value_name="c")
        lt.clear(), rt.clear()
        n = m = 1 << 16
        span = 1 << 40
        x = torch.randint(0, span, (n,), device=dev, generator=g)
        y = torch.randint(0, span, (m,), device=dev, generator=g)
        for sel in (1e-6, 1e-4, 1 / 1024, 1 / 512, 1 / 128, 1e-2, 1 / 48, 1 / 16):
            w = int(sel * span / 2)
            L, lt = table(ctx, {"x": x, "lo": x - w, "hi": x + w}, "l")
            R, rt = table(ctx, {"y": y}, "r")
            run(f"inner_band_sel_{sel:.3g}", n, m, L, R, "inner", [("lo", "<", "y"), ("hi", ">", "y")], columns=["x"], other_columns=["y"])
            lt.clear(), rt.clear()
        L, lt = table(ctx, {"a": torch.arange(1 << 12, device=dev)}, "a")
        R, rt = table(ctx, {"b": torch.arange(1 << 16, device=dev)}, "b")
        run("cross_2^12x2^16", 1 << 12, 1 << 16, L, R, "inner", [], columns=["a"], other_columns=["b"])
        lt.clear(), rt.clear()
    res = {"card": card(), "rows": rows}
    if a.out:
        json.dump(res, open(a.out, "w"), indent=1)
    print("card:", res["card"])


if __name__ == "__main__":
    main()
