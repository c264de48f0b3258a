"""Exchange of program hash aggregations across ranks (ldb_gpu_hashagg_exchange): the send and merge kernels for `groups` distinct keys
split over 2 and 4 ranks, and the single-GPU program aggregation the interpreter's lookup-or-insert serves, against a baseline build.

  python tools/hashagg_exchange_sweep.py [--groups 16M] [--reps 5] [--baseline-lib other/libldb_gpu.so] [--out result.json]

Exchange: every rank is a context of this process on device 0 (parallel.Comm.local_group), so these are ONE-GPU figures: the "peer"
stores land in the same HBM, and NVLink throughput between separate GPUs is not measured here.  Rank r holds the keys
r, r + W, r + 2W, … (groups / W of them) in a local state with COUNT(*) and SUM; each repetition exchanges into fresh owned states.
  send_ms_W    the send kernel with its cursor reset and count publication (family "hashagg_send"), the largest over the ranks
  merge_ms_W   the merge kernel (family "hashagg_merge"), the largest over the ranks
  call_ms_W    the whole collective call, wall clock of the slowest rank (barriers and the host read of the counts included)
Aggregation: GROUP BY key → COUNT(*), SUM over `groups` rows with 16 and with `groups` distinct keys (agg16_ms, aggN_ms; "base_" the
same on a context of the baseline library, the two alternating within each repetition), CUDA events on the compute stream.
Every number is the median of `reps` runs, reported with the card's name and power limit read in the same run."""
import argparse
import ctypes as C
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lingodb_b200 import capi, parallel, program as P, runtime  # noqa: E402
from lingodb_b200.datagen import ColumnSpec, TableData  # noqa: E402
from markjoin_sweep import card, context_of, rows_arg, timed  # noqa: E402

col = lambda n: ("col", n)  # noqa: E731
AGGS = [("count_star", None), ("sum", col("v"))]


def table(ctx, name, keys):
    td = TableData(name, [ColumnSpec("key", "int64"), ColumnSpec("v", "int64")])
    td.chunks.append({"key": keys, "v": keys * 3 + 1})
    td.chunk_rows.append(len(keys))
    return ctx.table_from_host(td)


def exchange_times(n, world, reps):
    ctxs = [runtime.Context(0) for _ in range(world)]
    entry = 48 + 16 * len(AGGS)
    per = n // world
    cap = per // world + per // (4 * world) + 4096  # owner shares are uniform: 1/W of each source's groups, plus slack
    comms = parallel.Comm.local_group(ctxs, user_bytes=world * cap * entry + 4096)
    tabs = [table(c, f"r{r}", np.arange(r, n, world, dtype=np.int64)) for r, c in enumerate(ctxs)]
    locals_ = [P.group_by(c, t, [col("key")], AGGS, expected_groups=per) for c, t in zip(ctxs, tabs)]
    out = {"send": [], "merge": [], "call": []}
    for _ in range(reps):
        owned = [P.hashagg_state(c, 1, [k for k, _ in AGGS], n // world) for c in ctxs]
        for c in ctxs:
            c.synchronize()
            c.kernel_time_reset(True)

        def one(r):
            t0 = time.perf_counter()
            comms[r].hashagg_exchange(locals_[r], owned[r], capacity=cap)
            ctxs[r].synchronize()
            return (time.perf_counter() - t0) * 1e3
        with ThreadPoolExecutor(world) as ex:
            walls = list(ex.map(one, range(world)))
        out["call"].append(max(walls))
        out["send"].append(max(c.kernel_time("hashagg_send")[0] for c in ctxs))
        out["merge"].append(max(c.kernel_time("hashagg_merge")[0] for c in ctxs))
        got = 0
        for c, o in zip(ctxs, owned):
            n_, e = C.c_int64(), capi.Error()
            capi.check(c.L.ldb_gpu_hashagg_count(o, C.byref(n_), C.byref(e)), e)
            got += n_.value
            runtime.state_destroy(c, o)
        assert got == world * per, (got, n)
    for c in ctxs:
        c.kernel_time_reset(False)
    for cm in comms:
        cm.close()
    for c, s, t in zip(ctxs, locals_, tabs):
        runtime.state_destroy(c, s)
        t.clear()
        c.close()
    return {k: float(np.median(v)) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=rows_arg, default=16 << 20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--baseline-lib")
    ap.add_argument("--out")
    a = ap.parse_args()
    n = a.groups
    res = {"card": card(), "groups": n, "reps": a.reps, "baseline": bool(a.baseline_lib), "exchange_on_one_gpu": True}
    for w in (2, 4):
        for k, v in exchange_times(n, w, a.reps).items():
            res[f"{k}_ms_{w}"] = v
    ctxs = {"": runtime.Context(0)}
    if a.baseline_lib:
        ctxs["base_"] = context_of(a.baseline_lib)
    keys = np.random.default_rng(3).permutation(n).astype(np.int64)
    data = {p: (table(c, "few", keys % 16), table(c, "many", keys)) for p, c in ctxs.items()}
    times = {f"{p}{m}": [] for p in ctxs for m in ("agg16_ms", "aggN_ms")}
    for _ in range(a.reps):
        for p, c in ctxs.items():
            few, many = data[p]
            for m, t, g in (("agg16_ms", few, 16), ("aggN_ms", many, n)):
                st = P.hashagg_state(c, 1, [k for k, _ in AGGS], g)
                times[f"{p}{m}"].append(timed(c, lambda: P.group_by(c, t, [col("key")], AGGS, state=st)))
                runtime.state_destroy(c, st)
    res.update({m: float(np.median(v)) for m, v in times.items()})
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
