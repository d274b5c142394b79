"""What running a GEMM chain and the element-wise tasks around it in one window changes (development aid, not the bench).

1. the card: name, power limit and maximum SM clock (read-only nvidia-smi query);
2. --ab LIB: the mixed DTD pool of tests/mixed_pool.py (per C tile: FILL, the GEMM k-chain, CHECK, and an AXPY on tiles
   of its own) through the stand-alone runtime at NT = 8 and NT = 16 (T x T bf16 tiles, --tile), on library LIB (a build
   whose windows hold one body kind, e.g. the parent commit's: three windows per pool) and on this tree's (one window),
   in child processes with PB2_LIB_PATH set, alternated: --rounds children per library, each --warmup and --runs
   steps.  A step inserts the pool and waits for it (the tiles stay resident between steps); windows per step are
   reported with it;
3. wide HBM bodies next to one 128^3 GEMM, on resident tiles: 256 SCALE_I32 on 2 MiB tiles (every SM has units),
   4 SCALE_I32 on 8 MiB tiles and a lone CHECK_I32 of 2 MiB (most SMs idle without parts).  Each as a GEMM window whose
   HBM units run as one part (part_bytes -1) and cut by the part rule (default part_bytes), and as an HBM window of the
   same HBM tasks, the three alternated run by run.
Each row: median / min / max / spread.

    python tools/ab_mixed_windows.py --ab /path/to/parent/parsec_b200/libparsec_b200.so [--runs 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
from parsec_b200 import _lib as L
from parsec_b200 import runtime as R
from parsec_b200.engine import Engine
from ab_read_groups import card, summary
import mixed_pool as P


def pool_steps(NT, T, warmup, runs):
    """Steps of the mixed pool on this process's library: (ms per step, windows per step)."""
    data = P.Data(NT, T, seed=3)
    ms, wins = [], []
    # host tiles come in through the kernels' stage-in on both libraries (no copy-engine prefetch runs)
    with R.Context(cuda_devices=(0,), mca={"device_engine_dma_prefetch_min_bytes": 0}) as ctx:
        dev = ctx.devices[0]
        dcs = P.collections(ctx, data)
        for i in range(warmup + runs):
            w0 = ctx.stats(dev)["windows_launched"]
            t0 = time.perf_counter()
            tp, _ = P.insert(ctx, data, dcs)
            ctx.wait()
            t1 = time.perf_counter()
            ctx.l.pb2_taskpool_free(tp)
            if i >= warmup:
                ms.append((t1 - t0) * 1e3)
                wins.append(ctx.stats(dev)["windows_launched"] - w0)
    return ms, wins


def ab_pool(args, NT):
    libs = {"split_lib_a": os.path.abspath(args.ab), "one_window_lib_b": L.LIB_PATH}
    ms = {k: [] for k in libs}
    wins = {k: set() for k in libs}
    for _ in range(args.rounds):
        for k, lib in libs.items():
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--NT", str(NT), "--tile", str(args.tile),
                                "--runs", str(args.runs), "--warmup", str(args.warmup)],
                               env=dict(os.environ, PB2_LIB_PATH=lib), capture_output=True, text=True)
            if p.returncode != 0:
                raise RuntimeError("child on %s failed (rc %d): %s" % (lib, p.returncode, p.stderr[-2000:]))
            got = json.loads([l for l in p.stdout.splitlines() if l.startswith("{")][-1])
            ms[k] += got["ms"]
            wins[k] |= set(got["windows"])
    res = {k: dict(summary(v), lib=libs[k], windows_per_step=sorted(wins[k])) for k, v in ms.items()}
    res["one_over_split_median"] = res["one_window_lib_b"]["median_ms"] / res["split_lib_a"]["median_ms"]
    return {"NT": NT, "tile": args.tile, "tasks": P.ntasks(NT), **res}


def wide(args, n, tb, body):
    """One engine, three resident windows of the same n HBM tasks on tiles of tb bytes, run alternately."""
    with Engine(0) as e:
        slab = e.malloc(n * tb + 3 * 128 * 128 * 2)
        e.h2d(slab, np.zeros((n * tb + 3 * 128 * 128 * 2) // 4, np.int32))
        tiles = np.zeros(n + 3, L.TILE_DTYPE)
        tiles["dev_ptr"] = slab + np.concatenate([np.arange(n) * tb, n * tb + np.arange(3) * 128 * 128 * 2]).astype(np.uint64)
        tiles["bytes"] = [tb] * n + [128 * 128 * 2] * 3
        tiles["state"] = L.TILE_VALID
        t = np.zeros(n + 1, L.TASK_DTYPE)
        t["tile"][:] = -1
        t["body"][:n], t["nb_flows"][:n] = body, 1
        t["iparam"][:n, 0] = 0 if body == L.BODY_CHECK_I32 else 3           # the CHECK finds what it expects
        t["tile"][:n, 0] = np.arange(n)
        t["access"][:n, 0] = L.ACCESS_READ if body == L.BODY_CHECK_I32 else L.ACCESS_RW
        t["body"][n], t["nb_flows"][n], t["iparam"][n] = L.BODY_GEMM_BF16, 3, (128, 128, 128)
        t["tile"][n, :3], t["access"][n, :3] = (n, n + 1, n + 2), (L.ACCESS_READ, L.ACCESS_READ, L.ACCESS_RW)
        none = np.zeros(0, np.uint32)
        wins = {}
        e.set_part_bytes(-1)
        wins["gemm_window_one_part"] = e.window(1, t, none, tiles, np.arange(n + 1, dtype=np.int32))
        e.set_part_bytes(0)
        wins["gemm_window_part_rule"] = e.window(1, t, none, tiles, np.arange(n + 1, dtype=np.int32))
        wins["hbm_window_part_rule"] = e.window(0, t[:n], none, tiles, np.arange(n, dtype=np.int32))
        ms = {k: [] for k in wins}
        for i in range(args.warmup + args.runs):
            for k, w in wins.items():
                st = w.run()
                if i >= args.warmup:
                    ms[k].append(st["reset_ms"] + st["kernel_ms"])
        for w in wins.values():
            w.close()
    res = {k: summary(v) for k, v in ms.items()}
    res["part_rule_over_one_part_median"] = res["gemm_window_part_rule"]["median_ms"] / res["gemm_window_one_part"]["median_ms"]
    return {"tasks": n, "body": "CHECK_I32" if body == L.BODY_CHECK_I32 else "SCALE_I32", "tile_bytes": tb, **res}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tile", type=int, default=512, help="T: C tiles of T x T bf16")
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3, help="--ab: child processes per library and NT")
    ap.add_argument("--ab", metavar="LIB", help="alternate the mixed pool on library LIB (split windows) and on this tree's")
    ap.add_argument("--NT", type=int, default=8, help=argparse.SUPPRESS)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        ms, wins = pool_steps(args.NT, args.tile, args.warmup, args.runs)
        print(json.dumps({"ms": ms, "windows": wins}), flush=True)
        return
    print(json.dumps({"card": card()}), flush=True)
    for n, tb, body in ((256, 2 << 20, L.BODY_SCALE_I32), (4, 8 << 20, L.BODY_SCALE_I32), (1, 2 << 20, L.BODY_CHECK_I32)):
        print(json.dumps({"wide": wide(args, n, tb, body)}), flush=True)
    if args.ab:
        for NT in (8, 16):
            print(json.dumps({"pool": ab_pool(args, NT)}), flush=True)


if __name__ == "__main__":
    main()
