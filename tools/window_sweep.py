"""Window functions (ldb_gpu_table_window / _ex): SUM and MAX of an int64 argument over 2^24 and 2^27 rows, 1, 2^10 and n/8 partitions, and a
running frame (UNBOUNDED PRECEDING .. CURRENT ROW), a sliding one (3 PRECEDING .. 3 FOLLOWING) and the whole partition; then the
ranking, offset and RANGE cases over the same tables:
  rank        RANK + DENSE_RANK by o (peer heads, the peer scans and the dense scan)
  lag_first   LAG(a) + FIRST_VALUE(a) over the running ROWS frame (two gathers of int64 cells)
  range_peers a RANGE running SUM(a) by q, 1024 distinct values: many peers per key in the larger partitions
  range_7day  SUM(a) OVER (ORDER BY d RANGE BETWEEN 6 PRECEDING AND CURRENT ROW), d a date over ten years

  python tools/window_sweep.py [--sizes 24,27] [--reps 3] [--out result.json]

The source is one DEVICE batch of int64 columns p (the partition key, uniform over the partition count; one partition has no key), o (the
order key, uniform), a (the argument, uniform) and q (uniform over 1024 values), and a date32 column d (uniform over 3650 days); nothing is
carried.  Per configuration, from the context's per-family CUDA-event timers:
  sort_ms     the radix sort by (p, o) ("radix_sort")
  window_ms   everything after the sort: partition heads, the start / end scans, the SUM scan, the MAX segment tree and the frame kernel
              ("window_partition", "window_scan", "window_tree", "window_frames"), the peer heads and scans ("window_peers"), the RANGE
              bounds ("window_range") and the value functions' gathers ("sort_exchange_permute"), each family also on its own
  call_ms     the whole call, wall clock
  rows_per_s  rows / (sort_ms + window_ms)
Every number is the median of `reps` runs after a warm-up run, reported with the card's name and power limit read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lingodb_b200 import program, runtime  # noqa: E402
from lingodb_b200.datagen import ColumnSpec  # noqa: E402
from markjoin_sweep import card  # noqa: E402

FRAMES = {"running": (None, 0), "sliding3": (-3, 3), "whole": (None, None)}
WINDOW_FAMILIES = ("window_partition", "window_scan", "window_tree", "window_frames", "window_peers", "window_range", "sort_exchange_permute")
# the new functions: name -> (order key, frame, mode, funcs)
CASES = {"rank": ("o", (None, 0), "range", [("sql_rank", None, "r"), ("dense_rank", None, "d")]),
         "lag_first": ("o", (None, 0), "rows", [("lag", "a", "l", 1), ("first_value", "a", "f")]),
         "range_peers": ("q", (None, 0), "range", [("sum", "a", "s")]),
         "range_7day": ("d", (-6, 0), "range", [("sum", "a", "s")])}


def device_table(ctx, n, parts, seed=5):
    import torch
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(seed)
    t = runtime.Table(ctx, "w", [ColumnSpec("p", "int64"), ColumnSpec("o", "int64"), ColumnSpec("a", "int64"), ColumnSpec("q", "int64"),
                                 ColumnSpec("d", "date32")])
    cols = {"p": torch.randint(0, parts, (n,), device=dev, generator=g, dtype=torch.int64),
            "o": torch.randint(-(1 << 62), 1 << 62, (n,), device=dev, generator=g, dtype=torch.int64),
            "a": torch.randint(-(1 << 40), 1 << 40, (n,), device=dev, generator=g, dtype=torch.int64)}
    cols["q"] = torch.randint(0, 1024, (n,), device=dev, generator=g, dtype=torch.int64)
    cols["d"] = torch.randint(8000, 11650, (n,), device=dev, generator=g, dtype=torch.int32)
    t.append_device(cols, n)
    torch.cuda.synchronize()
    return t


def one(ctx, t, n, parts, frame, reps, key="o", mode="rows", funcs=(("sum", "a", "s"), ("max", "a", "m"))):
    raw = program.RawTable(ctx, t.h)
    out = {k: [] for k in ("sort", "call") + WINDOW_FAMILIES}
    for _ in range(reps + 1):  # the first run warms up
        ctx.synchronize()
        ctx.kernel_time_reset(True)
        t0 = time.perf_counter()
        w = raw.window(partition_by=["p"] if parts > 1 else [], order_by=[(key, False)], frame=frame, funcs=list(funcs), columns=[], mode=mode)
        out["call"].append((time.perf_counter() - t0) * 1e3)
        assert w.num_rows == n
        out["sort"].append(ctx.kernel_time("radix_sort")[0])
        for f in WINDOW_FAMILIES:
            out[f].append(ctx.kernel_time(f)[0])
        w.destroy()
    ctx.kernel_time_reset(False)
    med = {f"{k}_ms": float(np.median(v[1:])) for k, v in out.items()}
    med["window_ms"] = sum(med[f"{f}_ms"] for f in WINDOW_FAMILIES)
    med["rows_per_s"] = n / ((med["sort_ms"] + med["window_ms"]) / 1e3)
    return med


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="24,27", help="log2 of the row counts")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    res = {"card": card(), "reps": a.reps}
    with runtime.Context(0) as ctx:
        for lg in [int(x) for x in a.sizes.split(",")]:
            n = 1 << lg
            for pname, parts in (("p1", 1), ("p1024", 1 << 10), ("pn8", n // 8)):
                t = device_table(ctx, n, parts)
                for fname, frame in FRAMES.items():
                    name = f"n2^{lg}_{pname}_{fname}"
                    for k, v in one(ctx, t, n, parts, frame, a.reps).items():
                        res[f"{name}_{k}"] = v
                    print(json.dumps({k: v for k, v in res.items() if k.startswith(name)}), flush=True)
                for cname, (key, frame, mode, funcs) in CASES.items():
                    name = f"n2^{lg}_{pname}_{cname}"
                    for k, v in one(ctx, t, n, parts, frame, a.reps, key, mode, funcs).items():
                        res[f"{name}_{k}"] = v
                    print(json.dumps({k: v for k, v in res.items() if k.startswith(name)}), flush=True)
                t.clear()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
