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
Every number is the median of `reps` runs, reported with the card's name and power limit read in the same run.

--strings runs the utf8 cases of ldb_gpu_table_exchange_varlen instead: --string-rows rows per rank (32 M: a receiver's bytes of one utf8
column must stay below 2^31) of an int64 key and one utf8 column of 16-64 random bytes (mean 40), partitioned over 2 and 4 ranks, and
half as many broadcast over 2; the same rows without the string column; and --distinct
distinct strings per rank (the count of the dictionary unification sweep) partitioned over 2 and 4 ranks.  There send_GBps counts every
byte stored into receive regions: 8 key bytes, 4 offset bytes and 2 validity bytes per row plus the strings' bytes."""
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


STRING_COLUMNS = [ColumnSpec("key", "int64"), ColumnSpec("s", "utf8")]


def string_table(ctx, name, rank, n, with_strings):
    """n rows of a random int64 key and (with_strings) a utf8 column of 16-64 random bytes; returns the table and its string bytes"""
    import torch
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(2000 + rank)
    t, nbytes = runtime.Table(ctx, name, STRING_COLUMNS if with_strings else STRING_COLUMNS[:1]), 0
    for lo in range(0, n, 8 << 20):  # batches of 8 M rows: a batch's strings must fit int32 offsets
        m = min(8 << 20, n - lo)
        cols = {"key": torch.randint(-(1 << 62), 1 << 62, (m,), device=dev, generator=g, dtype=torch.int64)}
        if with_strings:
            lens = torch.randint(16, 65, (m,), device=dev, generator=g, dtype=torch.int32)
            offs = torch.zeros(m + 1, dtype=torch.int32, device=dev)
            offs[1:] = torch.cumsum(lens, 0, dtype=torch.int32)
            cols["s"] = (offs, torch.randint(0, 256, (int(offs[-1]),), device=dev, generator=g, dtype=torch.uint8))
            nbytes += int(offs[-1])
        t.append_device(cols, m)
    torch.cuda.synchronize()
    return t, nbytes


def sweep_strings(world, n, broadcast, reps, with_strings):
    ctxs = [runtime.Context(0) for _ in range(world)]
    made = [string_table(c, f"r{r}", r, n, with_strings) for r, c in enumerate(ctxs)]
    tabs, total_bytes = [t for t, _ in made], sum(b for _, b in made)
    per = n * world if broadcast else n + n // 50 + 65536
    recv = per * 15 + (total_bytes if broadcast else total_bytes // world + total_bytes // 50) + (1 << 24)
    comms = parallel.Comm.local_group(ctxs, user_bytes=recv)
    keys = [] if broadcast else ["key"]
    out = {"count": [], "send": [], "copy": [], "call": []}
    for _ in range(reps + 1):  # the first run warms up
        for c in ctxs:
            c.synchronize()
            c.kernel_time_reset(True)

        def one(r):
            t0 = time.perf_counter()
            t = comms[r].table_exchange_varlen(tabs[r], keys, recv_bytes=recv)
            return (time.perf_counter() - t0) * 1e3, t
        with ThreadPoolExecutor(world) as ex:
            res = list(ex.map(one, range(world)))
        rows = sum(t.num_rows for _, t in res)
        assert rows == (world * world * n if broadcast else world * n), rows
        out["call"].append(max(w for w, _ in res))
        for fam in ("count", "send", "copy"):
            out[fam].append(0.0 if broadcast and fam == "count" and not with_strings else max(c.kernel_time(f"table_exchange_{fam}")[0] for c in ctxs))
        for _, t in res:
            t.destroy()
    for c in ctxs:
        c.kernel_time_reset(False)
    for cm in comms:
        cm.close()
    for c, t in zip(ctxs, tabs):
        t.clear()
        c.close()
    med = {f"{k}_ms": float(np.median(v[1:])) for k, v in out.items()}
    stored = rows * (8 + 1 + (4 + 1 if with_strings else 0)) + total_bytes * (world if broadcast else 1)
    med["send_GBps"] = stored / (med["send_ms"] * 1e-3) / 1e9
    med["rows_per_rank"] = n
    med["string_bytes_per_rank"] = total_bytes // world
    return med


def main_strings(a):
    res = {"card": card(), "reps": a.reps, "exchange_on_one_gpu": True}
    # a receiver's bytes of one utf8 column must fit int32 offsets: 32 M rows per rank partitioned, 16 M broadcast to 2 ranks
    cases = [(w, "partitioned", s, a.string_rows) for w in (2, 4) for s in (True, False)]
    cases += [(2, "broadcast", s, a.string_rows // 2) for s in (True, False)]
    cases += [(w, "distinct", True, a.distinct) for w in (2, 4)]
    for w, mode, s, n in cases:
        name = f"{mode}_{w}_{'utf8' if s else 'key_only'}"
        for k, v in sweep_strings(w, n, mode == "broadcast", a.reps, s).items():
            res[f"{name}_{k}"] = v
        print(json.dumps({k: v for k, v in res.items() if k.startswith(name)}), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=rows_arg, default=64 << 20)
    ap.add_argument("--broadcast-rows-4", type=rows_arg, default=16 << 20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    ap.add_argument("--strings", action="store_true", help="the utf8 cases of ldb_gpu_table_exchange_varlen instead")
    ap.add_argument("--string-rows", type=rows_arg, default=32 << 20)
    ap.add_argument("--distinct", type=rows_arg, default=10 << 20)
    a = ap.parse_args()
    if a.strings:
        res = main_strings(a)
        line = json.dumps(res)
        print(line)
        if a.out:
            with open(a.out, "w") as fh:
                fh.write(line + "\n")
        return
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
