"""Group-by on string keys through a string dictionary (LDB_OP_STRCODE) against the 8-byte prefix key (LDB_OP_STRKEY8).

  python tools/strcode_sweep.py [--sf 10] [--reps 5] [--out result.json]

1. SF`sf` lineitem's l_shipmode (7 values, dbgen's stream): count(*) group by ("strcode", l_shipmode) and by ("strkey8", l_shipmode),
   the dictionary cold (created per run: every distinct string is inserted once) and warm (reused: every row is a hit).
2. A high-cardinality column: "Customer#%09d" over 1.5 M x sf / 10 customers, each 10 times (Q13/Q18-like c_name keys).
Each case is timed with CUDA events on the context's compute stream after one warm-up run; the median of `reps` runs is reported
with the card's name and power limit, read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lingodb_b200 import dbgen, program as P, runtime  # noqa: E402
from lingodb_b200.datagen import ColumnSpec  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def utf8_table(ctx, name, offs, data, batch_rows=1 << 24):
    t = runtime.Table(ctx, name, [ColumnSpec("s", "utf8")])
    n = len(offs) - 1
    for b in range(0, n, batch_rows):
        m = min(batch_rows, n - b)
        t.append_host({"s": (offs, data)}, m, offset=b)
    return t


def shipmodes(sf):
    from lingodb_b200 import datagen
    import ctypes as C
    s = dbgen.scale_compiled(sf)
    L = datagen.lib()
    L.ldbgen_dbgen_line_counts_host.argtypes = [C.POINTER(datagen.GenScale), C.c_int64, C.c_int64, C.c_void_p]
    counts = np.zeros(s.n_orders, np.int32)
    L.ldbgen_dbgen_line_counts_host(C.byref(s), 0, s.n_orders, counts.ctypes.data)
    idx = dbgen.extra_columns(sf, counts)["l_shipmode"]
    offs, data = dbgen._categorical_utf8(idx, dbgen.SHIP_MODES)
    return offs.astype(np.int32), data


def customers(n_distinct, repeat):
    keys = np.tile(np.arange(1, n_distinct + 1, dtype=np.int64), repeat)
    np.random.default_rng(1).shuffle(keys)
    text = np.zeros((len(keys), 18), np.uint8)
    text[:, :9] = np.frombuffer(b"Customer#", np.uint8)
    v = keys.copy()
    for j in range(17, 8, -1):
        text[:, j] = ord("0") + v % 10
        v //= 10
    return np.arange(0, 18 * len(keys) + 1, 18, dtype=np.int64).astype(np.int32), text.reshape(-1)


def timed(ctx, fn, reps):
    fn()  # warm-up
    ms = []
    for _ in range(reps):
        ctx.synchronize()
        ctx.timer_start()
        fn()
        ms.append(ctx.timer_stop())
    return float(np.median(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=float, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    res = {"card": card(), "sf": a.sf, "reps": a.reps}
    with runtime.Context(0) as ctx:
        cases = {"l_shipmode": (shipmodes(a.sf), 8), "c_name": (customers(int(150_000 * a.sf), 10), int(150_000 * a.sf))}
        for name, ((offs, data), distinct) in cases.items():
            t = utf8_table(ctx, name, offs, data)
            n = len(offs) - 1
            r = {"rows": n, "distinct": distinct}

            def group(key):
                st = P.group_by(ctx, t, [key], [("count_star", None)], expected_groups=max(distinct, 16))
                ctx.L.ldb_gpu_state_destroy(st)

            def cold():
                d = P.dict_state(ctx, distinct, int(distinct * 20))
                group(("strcode", d, "s"))
                ctx.L.ldb_gpu_state_destroy(d)

            warm_dict = P.dict_state(ctx, distinct, int(distinct * 20))
            r["strkey8_ms"] = timed(ctx, lambda: group(("strkey8", "s")), a.reps)
            r["strcode_cold_ms"] = timed(ctx, cold, a.reps)
            r["strcode_warm_ms"] = timed(ctx, lambda: group(("strcode", warm_dict, "s")), a.reps)
            r["dict_strings"] = P.dict_count(ctx, warm_dict)
            ctx.L.ldb_gpu_state_destroy(warm_dict)
            res[name] = r
            t.clear()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
