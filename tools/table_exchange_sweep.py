"""Repartition of table rows across ranks (ldb_gpu_table_exchange): the count, send and copy-out kernels for `rows` rows per rank of one
int64 key and three 8- and 16-byte columns (int64, decimal128, float64), over 2 and 4 ranks, partitioned by the key and broadcast.

  python tools/table_exchange_sweep.py [--rows 64M] [--broadcast-rows-4 16M] [--reps 5] [--out result.json]

Every rank is a context of this process on device 0 (parallel.Comm.local_group), so these are ONE-GPU, HBM-bound figures: the "peer"
stores land in the same HBM, and NVLink throughput between separate GPUs is not measured here.  The source batches are DEVICE
tensors.  Broadcast over 4 ranks gives every rank 4 x rows rows: with 64 M rows per rank the four receive regions and the four
received tables would not fit one 80 GB card, so that case runs --broadcast-rows-4 rows per rank.
  count_ms    count + scan kernels (family "table_exchange_count"), the largest over the ranks (partitioned only)
  send_ms     the send kernels (family "table_exchange_send"), the largest over the ranks
  copy_ms     the copy-out of the own region (family "table_exchange_copy"), the largest over the ranks
  call_ms     the whole collective call, wall clock of the slowest rank (all-gather, barriers and host reads included)
  send_GBps   bytes the ranks store into receive regions (rows received x 44 bytes: 40 of cells, 4 validity bytes), summed over the
              ranks, over the largest send time
Every number is the median of `reps` runs, reported with the card's name and power limit read in the same run."""
import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lingodb_b200 import parallel, runtime  # noqa: E402
from lingodb_b200.datagen import ColumnSpec  # noqa: E402
from markjoin_sweep import card, rows_arg  # noqa: E402

COLUMNS = [ColumnSpec("key", "int64"), ColumnSpec("a", "int64"), ColumnSpec("b", "decimal128", 38, 2), ColumnSpec("c", "float64")]
WIDTHS = [8, 8, 16, 8]
ROW_BYTES = sum(WIDTHS) + len(WIDTHS)


def region_bytes(n: int) -> int:
    a16 = lambda x: (x + 15) // 16 * 16  # noqa: E731
    return sum(a16(n * w) for w in WIDTHS) + len(WIDTHS) * a16(n)


def device_table(ctx, name, rank, n):
    import torch
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(1000 + rank)
    key = torch.randint(-(1 << 62), 1 << 62, (n,), device=dev, generator=g, dtype=torch.int64)
    cols = {"key": key, "a": key * 3 + 1, "b": torch.stack([key, key >> 63], 1).contiguous(), "c": key.to(torch.float64)}
    t = runtime.Table(ctx, name, COLUMNS)
    t.append_device(cols, n)
    torch.cuda.synchronize()
    return t


def sweep(world, n, broadcast, reps):
    ctxs = [runtime.Context(0) for _ in range(world)]
    per = n * world if broadcast else n + n // 50 + 65536  # owner shares are uniform: n rows per receiver, plus slack
    recv = region_bytes(per)
    comms = parallel.Comm.local_group(ctxs, user_bytes=recv)
    tabs = [device_table(c, f"r{r}", r, n) for r, c in enumerate(ctxs)]
    keys = [] if broadcast else ["key"]
    out = {"count": [], "send": [], "copy": [], "call": [], "rows": []}
    for _ in range(reps + 1):  # the first run warms up
        for c in ctxs:
            c.synchronize()
            c.kernel_time_reset(True)

        def one(r):
            t0 = time.perf_counter()
            t = comms[r].table_exchange(tabs[r], keys, recv_bytes=recv)
            return (time.perf_counter() - t0) * 1e3, t
        with ThreadPoolExecutor(world) as ex:
            res = list(ex.map(one, range(world)))
        rows = sum(t.num_rows for _, t in res)
        assert rows == (world * world * n if broadcast else world * n), rows
        out["call"].append(max(w for w, _ in res))
        out["rows"].append(rows)
        for fam in ("count", "send", "copy"):
            out[fam].append(0.0 if broadcast and fam == "count" else max(c.kernel_time(f"table_exchange_{fam}")[0] for c in ctxs))
        for _, t in res:
            t.destroy()
    for c in ctxs:
        c.kernel_time_reset(False)
    for cm in comms:
        cm.close()
    for c, t in zip(ctxs, tabs):
        t.clear()
        c.close()
    med = {f"{k}_ms": float(np.median(v[1:])) for k, v in out.items() if k != "rows"}
    med["send_GBps"] = out["rows"][-1] * ROW_BYTES / (med["send_ms"] * 1e-3) / 1e9
    med["rows_per_rank"] = n
    return med


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=rows_arg, default=64 << 20)
    ap.add_argument("--broadcast-rows-4", type=rows_arg, default=16 << 20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    res = {"card": card(), "reps": a.reps, "exchange_on_one_gpu": True, "row_bytes": ROW_BYTES}
    for w in (2, 4):
        for mode in ("partitioned", "broadcast"):
            n = a.broadcast_rows_4 if (mode == "broadcast" and w == 4) else a.rows
            for k, v in sweep(w, n, mode == "broadcast", a.reps).items():
                res[f"{mode}_{w}_{k}"] = v
            print(json.dumps({k: v for k, v in res.items() if k.startswith(f"{mode}_{w}_")}), flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
