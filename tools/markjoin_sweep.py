"""Join-table markers (LDB_OP_MARK) in program joins: PROBE_EACH without and with a MARK, the marks scan, and the plain JOIN_BUILD /
PROBE / PROBE_EACH program times of this build against a baseline build of the library, in one process.

  python tools/markjoin_sweep.py [--build-rows 16M] [--probe-rows 128M] [--reps 5] [--baseline-lib other/libldb_gpu.so] [--out result.json]

Build side: `build-rows` distinct int32 keys (a permutation of 0..n-1) with row-id payloads in a plain join table; probe side: `probe-rows`
keys uniform in 0..2n-1 (half hit).  The probe programs keep no row (WHERE payload = -1), so their sink costs nothing:
  each_ms          PROBE_EACH of every probe row
  each_mark_ms     the same program with a MARK of every match (condition TRUE) evaluated in its WHERE
  each_mark_none_ms  PROBE_EACH + MARK with LDB_SINK_NONE
  marks_scan_ms    ldb_gpu_join_table_marks(which = 1) over the marked table, read-back of the count included
  build_ms / probe_ms / probe_each_ms   JOIN_BUILD into a fresh table, PROBE, PROBE_EACH; with --baseline-lib the same three again on a
                   context of the baseline library ("base_" prefix), the two alternating within each repetition
Match and mark counts are checked once outside the timings.  Every number is the median of `reps` runs timed with CUDA events on the
context's compute stream (the host waits for the stream), reported with the card's name and power limit read in the same run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lingodb_b200 import capi, program as P, runtime  # noqa: E402
from lingodb_b200.datagen import ColumnSpec, TableData  # noqa: E402

col, const = (lambda n: ("col", n)), (lambda v: ("const", v))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def rows_arg(s):
    s = s.upper()
    return int(float(s[:-1]) * (1 << 20)) if s.endswith("M") else int(s)


def int32_table(ctx, name, cols, batch_rows=1 << 24):
    n = len(next(iter(cols.values())))
    td = TableData(name, [ColumnSpec(k, "int32") for k in cols])
    for b in range(0, n, batch_rows):
        td.chunks.append({k: np.ascontiguousarray(v[b:b + batch_rows]) for k, v in cols.items()})
        td.chunk_rows.append(min(batch_rows, n - b))
    return ctx.table_from_host(td)


def timed(ctx, fn):
    ctx.synchronize()
    ctx.timer_start()
    fn()
    return ctx.timer_stop()


def context_of(path):
    """a context of another build of the library (the symbols it lacks stay unbound)"""
    L = C.CDLL(path)
    for name, (res, args) in capi.SIGNATURES.items():
        fn = getattr(L, name, None)
        if fn is not None:
            fn.restype, fn.argtypes = res, args
    capi.lib()
    saved, capi._lib = capi._lib, L
    try:
        return runtime.Context(0)
    finally:
        capi._lib = saved


def count_where(ctx, table, where):
    st = P.group_by(ctx, table, [], [("count_star", None)], where=where)
    n = P.decode_groups(P.read_groups(ctx, st, 4), 0, 1)[()][0]
    runtime.state_destroy(ctx, st)
    return n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--build-rows", type=rows_arg, default=16 << 20)
    ap.add_argument("--probe-rows", type=rows_arg, default=128 << 20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--baseline-lib")
    ap.add_argument("--out")
    a = ap.parse_args()
    res = {"card": card(), "build_rows": a.build_rows, "probe_rows": a.probe_rows, "reps": a.reps, "baseline": bool(a.baseline_lib)}
    nb, na = a.build_rows, a.probe_rows
    rng = np.random.default_rng(5)
    k = rng.permutation(nb).astype(np.int32)
    q = rng.integers(0, 2 * nb, na, dtype=np.int64).astype(np.int32)
    ctxs = {"": runtime.Context(0)}
    if a.baseline_lib:
        ctxs["base_"] = context_of(a.baseline_lib)
    data = {p: (int32_table(c, "build", {"k": k}), int32_table(c, "probe", {"k": q})) for p, c in ctxs.items()}
    ctx = ctxs[""]
    B, A = data[""]
    jt = runtime.join_table(ctx, nb)
    P.build_join(ctx, B, jt, col("k"), payload=("rowid",))
    m = ("probe_each", jt, col("k"))
    none = ("cmp", "=", m, const(-1))
    mark = ("mark", m, const(1))
    # correctness once, untimed: every hit marks its entry, and the marked entries are the distinct hit keys
    hits = count_where(ctx, A, ("not", ("isnull", ("probe", jt, col("k")))))
    assert count_where(ctx, A, mark) == hits
    marked = P.join_marks(ctx, jt, P.MARKED)
    res["hits"], res["marked"] = hits, marked.num_rows
    assert marked.num_rows == len(np.unique(q[q < nb]))
    marked.destroy()
    del k, q
    times = {n: [] for n in ("each_ms", "each_mark_ms", "each_mark_none_ms", "marks_scan_ms")}
    times.update({f"{p}{n}": [] for p in ctxs for n in ("build_ms", "probe_ms", "probe_each_ms")})
    for _ in range(a.reps):
        times["each_ms"].append(timed(ctx, lambda: count_where(ctx, A, none)))
        times["each_mark_ms"].append(timed(ctx, lambda: count_where(ctx, A, ("and", mark, none))))
        times["each_mark_none_ms"].append(timed(ctx, lambda: P.run_effects(ctx, A, [mark])))
        times["marks_scan_ms"].append(timed(ctx, lambda: P.join_marks(ctx, jt, P.MARKED).destroy()))
        for p, c in ctxs.items():
            b_, a_ = data[p]
            fresh = runtime.join_table(c, nb)
            times[f"{p}build_ms"].append(timed(c, lambda: P.build_join(c, b_, fresh, col("k"), payload=("rowid",))))
            times[f"{p}probe_ms"].append(timed(c, lambda: count_where(c, a_, ("cmp", "=", ("probe", fresh, col("k")), const(-1)))))
            times[f"{p}probe_each_ms"].append(timed(c, lambda: count_where(c, a_, ("cmp", "=", ("probe_each", fresh, col("k")), const(-1)))))
            runtime.state_destroy(c, fresh)
    res.update({n: float(np.median(v)) for n, v in times.items()})
    runtime.state_destroy(ctx, jt)
    for p, c in ctxs.items():
        for t in data[p]:
            t.clear()
        c.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
