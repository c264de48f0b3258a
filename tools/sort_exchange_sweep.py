"""ORDER BY across ranks (ldb_gpu_table_sort_exchange, no LIMIT): `rows` rows per rank of an int64 key with an int64 and a decimal128
payload (and, with --strings, a utf8 payload of 16-64 random bytes), uniform or skewed keys, over 1, 2 and 4 ranks.

  python tools/sort_exchange_sweep.py [--rows 32M] [--reps 3] [--strings] [--out result.json]

Every rank is a context of this process on device 0 (parallel.Comm.local_group), so these are ONE-GPU, HBM-bound figures: the "peer"
stores land in the same HBM, and NVLink throughput between separate GPUs is not measured here.  The source batches are DEVICE tensors.
  count_ms    samples and range-owner count (families "sort_exchange_sample" + "table_exchange_count"), the largest over the ranks
  send_ms     the send kernels ("table_exchange_send"), the largest over the ranks
  sort_ms     the receiver's radix sort ("radix_sort"), the largest over the ranks
  permute_ms  the permute into the new table ("sort_exchange_permute"), the largest over the ranks
  call_ms     the whole collective call, wall clock of the slowest rank (all-gathers, barriers and host reads included)
  max_over_mean   the largest received row count over the mean
The baseline runs ldb_gpu_table_order_by_keys over world x rows rows on one rank (its radix-sort kernels, "obk_sort_ms") and the
same rows through a one-rank sort exchange ("one_rank_call_ms": a local ORDER BY into a new table, its permute "one_rank_permute_ms").
Every number is the median of `reps` runs after a warm-up run, reported with the card's name and power limit read in the same run."""
import argparse
import ctypes as C
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lingodb_b200 import capi, parallel, runtime  # noqa: E402
from lingodb_b200.datagen import ColumnSpec  # noqa: E402
from markjoin_sweep import card, rows_arg  # noqa: E402

COLUMNS = [ColumnSpec("key", "int64"), ColumnSpec("a", "int64"), ColumnSpec("b", "decimal128", 38, 2), ColumnSpec("s", "utf8")]


def device_table(ctx, name, seed, n, skewed, strings):
    """n rows in batches of 8 M; skewed keys: u^8 scaled to 2^20 values, so a few small keys hold most rows"""
    import torch
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(seed)
    t = runtime.Table(ctx, name, COLUMNS if strings else COLUMNS[:3])
    for lo in range(0, n, 8 << 20):
        m = min(8 << 20, n - lo)
        if skewed:
            key = (torch.rand(m, device=dev, generator=g, dtype=torch.float64) ** 8 * (1 << 20)).to(torch.int64)
        else:
            key = torch.randint(-(1 << 62), 1 << 62, (m,), device=dev, generator=g, dtype=torch.int64)
        cols = {"key": key, "a": key * 3 + 1, "b": torch.stack([key, key >> 63], 1).contiguous()}
        if strings:
            lens = torch.randint(16, 65, (m,), device=dev, generator=g, dtype=torch.int32)
            offs = torch.zeros(m + 1, dtype=torch.int32, device=dev)
            offs[1:] = torch.cumsum(lens, 0, dtype=torch.int32)
            cols["s"] = (offs, torch.randint(0, 256, (int(offs[-1]),), device=dev, generator=g, dtype=torch.uint8))
        t.append_device(cols, m)
    torch.cuda.synchronize()
    return t


def sweep(world, n, skewed, strings, reps):
    ctxs = [runtime.Context(0) for _ in range(world)]
    tabs = [device_table(c, f"r{r}", 1000 + r, n, skewed, strings) for r, c in enumerate(ctxs)]
    per = n * 5 // 4 + (1 << 16)  # a receiver's rows stay within 1.25 x the mean
    recv = per * (8 + 8 + 16 + 3 + (5 + 64 if strings else 0)) + (1 << 24)
    comms = parallel.Comm.local_group(ctxs, user_bytes=recv)
    fams = {"count": ("sort_exchange_sample", "table_exchange_count"), "send": ("table_exchange_send",), "sort": ("radix_sort",),
            "permute": ("sort_exchange_permute",)}
    out = {k: [] for k in list(fams) + ["call", "max_over_mean"]}
    for _ in range(reps + 1):  # the first run warms up
        for c in ctxs:
            c.synchronize()
            c.kernel_time_reset(True)

        def one(r):
            t0 = time.perf_counter()
            t, _, _ = comms[r].sort_exchange(tabs[r], [("key", False)], recv_bytes=recv)
            return (time.perf_counter() - t0) * 1e3, t
        with ThreadPoolExecutor(world) as ex:
            res = list(ex.map(one, range(world)))
        counts = [t.num_rows for _, t in res]
        assert sum(counts) == world * n, counts
        out["call"].append(max(w for w, _ in res))
        out["max_over_mean"].append(max(counts) / (sum(counts) / world))
        for k, fs in fams.items():
            out[k].append(max(sum(c.kernel_time(f)[0] for f in fs) for c in ctxs))
        for _, t in res:
            t.destroy()
    for c in ctxs:
        c.kernel_time_reset(False)
    for cm in comms:
        cm.close()
    for c, t in zip(ctxs, tabs):
        t.clear()
        c.close()
    med = {f"{k}_ms" if k != "max_over_mean" else k: float(np.median(v[1:])) for k, v in out.items()}
    med["rows_per_rank"] = n
    return med


def baseline(total, skewed, reps):
    """order_by_keys over `total` rows on one rank (its radix-sort kernels), and the same rows through a one-rank sort exchange"""
    ctx = runtime.Context(0)
    # one batch: order_by_keys takes single-batch tables
    import torch
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(7)
    key = (torch.rand(total, device=dev, generator=g, dtype=torch.float64) ** 8 * (1 << 20)).to(torch.int64) if skewed else \
        torch.randint(-(1 << 62), 1 << 62, (total,), device=dev, generator=g, dtype=torch.int64)
    t = runtime.Table(ctx, "all", COLUMNS[:3])
    t.append_device({"key": key, "a": key * 3 + 1, "b": torch.stack([key, key >> 63], 1).contiguous()}, total)
    torch.cuda.synchronize()
    ids = (C.c_int64 * 1)()
    cols, desc = (C.c_char_p * 1)(b"key"), (C.c_int32 * 1)(0)
    sort_ms = []
    for _ in range(reps + 1):
        ctx.synchronize()
        ctx.kernel_time_reset(True)
        m, e = C.c_int64(), capi.Error()
        capi.check(ctx.L.ldb_gpu_table_order_by_keys(t.h, 1, cols, desc, 1, ids, C.byref(m), C.byref(e)), e)  # limit 1: no id read-back
        sort_ms.append(ctx.kernel_time("radix_sort")[0])
    ctx.kernel_time_reset(False)
    t.clear()
    ctx.close()
    one = sweep(1, total, skewed, False, reps)  # one receiver of every string would pass the 2^31 - 1 bytes of a utf8 column
    return {"obk_sort_ms": float(np.median(sort_ms[1:])), "one_rank_call_ms": one["call_ms"], "one_rank_permute_ms": one["permute_ms"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=rows_arg, default=32 << 20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--strings", action="store_true", help="a utf8 payload of 16-64 bytes as well")
    ap.add_argument("--baseline", action="store_true", help="also order_by_keys and a one-rank sort exchange over world x rows rows")
    ap.add_argument("--out")
    a = ap.parse_args()
    res = {"card": card(), "reps": a.reps, "exchange_on_one_gpu": True, "strings": a.strings}
    for skewed in (False, True):
        for w in (1, 2, 4):
            name = f"{'skewed' if skewed else 'uniform'}_{w}"
            for k, v in sweep(w, a.rows, skewed, a.strings, a.reps).items():
                res[f"{name}_{k}"] = v
            if a.baseline and w > 1:
                for k, v in baseline(w * a.rows, skewed, a.reps).items():
                    res[f"{name}_{k}"] = v
            print(json.dumps({k: v for k, v in res.items() if k.startswith(name)}), flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
