"""Union of string dictionaries across ranks (ldb_gpu_dict_unify): `n` distinct strings of 8-64 bytes per rank, half of them shared by
every rank and half the rank's own, unified over 1, 2, 4 and 8 ranks.

  python tools/dict_unify_sweep.py [--strings 1M,10M] [--worlds 1,2,4,8] [--reps 3] [--out result.json]

In-process ranks are contexts of this process on device 0 (parallel.Comm.local_group): ONE-GPU figures, the "peer" stores land in the
same HBM and the ranks' sorts share one card.  Where several GPUs are visible the sweep also runs one process per GPU (--processes,
default: the visible GPUs, up to 8), which measures the stores over NVLink.  The strings are generated on the device and inserted into
each rank's local dictionary before the timed calls.
  call_ms       the whole collective call, wall clock of the slowest rank, each call between two device synchronisations
  sort_share    the union's radix sort (family "radix_sort") over call_ms, on the slowest rank
  bytes_moved   string bytes stored into receive regions: every rank's bytes to every rank (offsets not counted)
Every number is the median of `reps` calls after one warm-up call, reported with the card's name and power limit read in the same run."""
import argparse
import json
import os

# up to 8 in-process ranks share one GPU: with the default 8 hardware work queues their streams would share queues, and a collective
# kernel could wait behind a peer's kernel that waits for it (set before CUDA starts)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from lingodb_b200 import parallel, program as P, runtime  # noqa: E402
from lingodb_b200.datagen import ColumnSpec  # noqa: E402
from markjoin_sweep import card, rows_arg  # noqa: E402


def strings(seed: int, n: int, dev):
    """n random strings of 8-64 letters as device utf8 buffers (int32 offsets, bytes); total bytes"""
    import torch
    g = torch.Generator(device=dev).manual_seed(seed)
    lens = torch.randint(8, 65, (n,), device=dev, generator=g, dtype=torch.int32)
    offs = torch.zeros(n + 1, dtype=torch.int32, device=dev)
    offs[1:] = torch.cumsum(lens, 0, dtype=torch.int32)
    total = int(offs[-1])
    data = torch.randint(97, 123, (total,), device=dev, generator=g, dtype=torch.uint8)
    return offs, data, total


def local_dict(ctx, rank: int, n: int):
    """rank's dictionary: n // 2 strings every rank shares, n - n // 2 of its own; and its string bytes"""
    import torch
    dev = torch.device("cuda", ctx.device)
    d = P.dict_state(ctx, n, n * 64)
    total = 0
    for seed, m in ((7, n // 2), (1000 + rank, n - n // 2)):
        offs, data, b = strings(seed, m, dev)
        t = runtime.Table(ctx, "s", [ColumnSpec("s", "utf8")])
        t.append_device({"s": (offs, data)}, m)
        torch.cuda.synchronize(dev)
        P.run_effects(ctx, t, [("strcode", d, "s")])
        t.clear()
        total += b
    return d, total


def region_bytes(n: int, b: int) -> int:
    return (n + 1) * 4 + b + 32


def timed(ctxs, call):
    for c in ctxs:
        c.synchronize()
        c.kernel_time_reset(True)
    t0 = time.perf_counter()
    u = call()
    for c in ctxs:
        c.synchronize()
    return (time.perf_counter() - t0) * 1e3, u


def sweep_in_process(world: int, n: int, reps: int):
    ctxs = [runtime.Context(0) for _ in range(world)]
    locs = [local_dict(c, r, n) for r, c in enumerate(ctxs)]
    bytes_total = sum(b for _, b in locs)
    comms = parallel.Comm.local_group(ctxs, user_bytes=world * region_bytes(n, max(b for _, b in locs)))
    calls, sorts = [], []
    for rep in range(reps + 1):
        def one(r):
            return timed([ctxs[r]], lambda: comms[r].dict_unify(locs[r][0]))
        with ThreadPoolExecutor(world) as ex:
            res = list(ex.map(one, range(world)))
        slow = max(range(world), key=lambda r: res[r][0])
        if rep:
            calls.append(res[slow][0])
            sorts.append(ctxs[slow].kernel_time("radix_sort")[0])
        n_union = P.dict_count(ctxs[0], res[0][1])
        for c, (_, u) in zip(ctxs, res):
            c.L.ldb_gpu_state_destroy(u)
    for cm in comms:
        cm.close()
    for c, (d, _) in zip(ctxs, locs):
        c.L.ldb_gpu_state_destroy(d)
        c.close()
    call = float(np.median(calls))
    return {"call_ms": call, "sort_share": float(np.median(sorts)) / call, "bytes_moved": bytes_total * world, "union_strings": n_union}


def _rank_main(rank: int, world: int, n: int, reps: int, rendezvous: str):
    """one rank of the cross-process sweep: its timings as JSON under `rendezvous`"""
    def swap(handle: bytes):
        with open(os.path.join(rendezvous, f"h{rank}.tmp"), "wb") as f:
            f.write(handle)
        os.replace(os.path.join(rendezvous, f"h{rank}.tmp"), os.path.join(rendezvous, f"h{rank}"))
        paths = [os.path.join(rendezvous, f"h{r}") for r in range(world)]
        deadline = time.monotonic() + 300
        while not all(os.path.exists(x) for x in paths):
            if time.monotonic() > deadline:
                sys.exit(f"rank {rank}: the peers' handles did not arrive within 300 s")
            time.sleep(0.05)
        return [open(x, "rb").read() for x in paths]
    ctx = runtime.Context(rank)
    d, b = local_dict(ctx, rank, n)
    comm = parallel.Comm(ctx, rank, world, user_bytes=world * region_bytes(n, b + (1 << 20)), exchange=swap)
    calls, sorts = [], []
    for rep in range(reps + 1):
        ms, u = timed([ctx], lambda: comm.dict_unify(d))
        if rep:
            calls.append(ms)
            sorts.append(ctx.kernel_time("radix_sort")[0])
        ctx.L.ldb_gpu_state_destroy(u)
    with open(os.path.join(rendezvous, f"out{rank}.json"), "w") as f:
        json.dump({"calls": calls, "sorts": sorts, "bytes": b}, f)
    comm.close()
    ctx.L.ldb_gpu_state_destroy(d)
    ctx.close()


def sweep_processes(world: int, n: int, reps: int):
    with tempfile.TemporaryDirectory() as tmp:
        procs = []
        try:
            for r in range(world):
                procs.append(subprocess.Popen([sys.executable, os.path.abspath(__file__), "--rank", str(r), "--world", str(world), "--n", str(n), "--reps", str(reps),
                                               "--rendezvous", tmp]))
            codes = [p.wait(timeout=1800) for p in procs]
        finally:  # no rank outlives the sweep
            for p in procs:
                if p.poll() is None:
                    p.kill()
                p.wait()
        if codes != [0] * world:
            raise RuntimeError(f"a rank failed: exit codes {codes}")
        outs = [json.load(open(os.path.join(tmp, f"out{r}.json"))) for r in range(world)]
    calls = [max(o["calls"][i] for o in outs) for i in range(reps)]
    sorts = [max(o["sorts"][i] for o in outs) for i in range(reps)]
    call = float(np.median(calls))
    return {"call_ms": call, "sort_share": float(np.median(sorts)) / call, "bytes_moved": sum(o["bytes"] for o in outs) * world}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--strings", default="1M,10M")
    ap.add_argument("--worlds", default="1,2,4,8")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--processes", type=int, default=None, help="ranks of the cross-process sweep (default: the visible GPUs, up to 8; < 2 skips it)")
    ap.add_argument("--out")
    ap.add_argument("--rank", type=int, help=argparse.SUPPRESS)
    ap.add_argument("--world", type=int, help=argparse.SUPPRESS)
    ap.add_argument("--n", type=int, help=argparse.SUPPRESS)
    ap.add_argument("--rendezvous", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.rank is not None:
        return _rank_main(a.rank, a.world, a.n, a.reps, a.rendezvous)
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: the sweep measures on the GPU only")
    procs = a.processes if a.processes is not None else min(torch.cuda.device_count(), 8)
    res = {"card": card(), "reps": a.reps}
    for n in [rows_arg(x) for x in a.strings.split(",")]:
        for w in [int(x) for x in a.worlds.split(",")]:
            r = sweep_in_process(w, n, a.reps)
            res.update({f"in_process_{w}_{n}_{k}": v for k, v in r.items()})
            print(json.dumps({"world": w, "strings_per_rank": n, "in_process": True, **r}), flush=True)
        if procs >= 2:
            r = sweep_processes(procs, n, a.reps)
            res.update({f"processes_{procs}_{n}_{k}": v for k, v in r.items()})
            print(json.dumps({"world": procs, "strings_per_rank": n, "in_process": False, **r}), flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
