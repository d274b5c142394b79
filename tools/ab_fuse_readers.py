"""Where the resident Ex05 window spends its time, and what fusing each producer with its read group changes
(development aid, not the bench).

1. the card: name, power limit and maximum SM clock (read-only nvidia-smi query);
2. tools/l2_probe (compiled into a temporary directory): the L2 read rate and the DRAM rates of this GPU;
3. a FILL-only window (the K producers of the Ex05 window, no readers): the write floor of the fused window;
4. the resident Ex05 window (dags.ex05_broadcast(K, 14, 262144), tiles VALID) with fusion off and on;
5. --ab LIB [LIB ...]: the fused window on each library LIB (other builds of libparsec_b200.so, e.g. the parent
   commit's) and on this tree's library, alternated: --rounds child processes per build, each with PB2_LIB_PATH set,
   --warmup and --runs runs each; besides the sum, the medians of reset_ms and kernel_ms of each build.
Each row: median / min / max / spread of reset_ms + kernel_ms.

    python tools/ab_fuse_readers.py [--runs 30] [--ab /path/to/parent/libparsec_b200.so ...]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from parsec_b200 import _lib as L
from oracle import orc_dags as dags
from parsec_b200.engine import Engine
from ab_read_groups import TB, card, l2_probe, summary


class Window:
    """One engine and one resident window of the Ex05 DAG (or of its producers alone) on it."""

    def __init__(self, K, fuse_readers=0, fill_only=False, part_bytes=0, workers_per_sm=0, ipc=False):
        self.e = Engine(0, workers_per_sm=workers_per_sm, fuse_readers=fuse_readers, part_bytes=part_bytes)
        dag = dags.ex05_broadcast(K, 14, TB)
        tasks, succ = dag.tasks, dag.succ
        if fill_only:
            tasks = tasks[:K].copy()
            tasks["succ_begin"], tasks["succ_count"] = 0, 0
            succ = np.zeros(0, np.uint32)
        self.ntasks = len(tasks)
        self.slab = self.e.malloc(K * TB, ipc=ipc)       # ipc=True: plain cudaMalloc memory, never compressible
        self.e.h2d(self.slab, np.zeros(K * TB // 4, np.int32))
        tiles = np.zeros(K, L.TILE_DTYPE)
        tiles["dev_ptr"] = self.slab + np.arange(K, dtype=np.uint64) * np.uint64(TB)
        tiles["bytes"] = TB
        tiles["state"] = L.TILE_VALID
        self.w = self.e.window(0, tasks, succ, tiles, dag.ready)
        self.split = []                    # (reset_ms, kernel_ms) of every run

    def run(self):
        st = self.w.run()
        assert st["body_errors"] == 0 and st["tasks_retired"] == self.ntasks
        self.split.append((st["reset_ms"], st["kernel_ms"]))
        return st["reset_ms"] + st["kernel_ms"]

    def close(self):
        self.w.close()
        self.e.close()


def runs_of(x, warmup, runs):
    for _ in range(warmup):
        x.run()
    x.split.clear()
    ms = [x.run() for _ in range(runs)]
    x.close()
    return ms


def measure(x, warmup, runs):
    return summary(runs_of(x, warmup, runs))


def ab_libraries(args):
    """The fused window on the --ab library builds (lib_a, lib_a2, ...) and this tree's (lib_b), one child process at a
    time, alternated."""
    libs = {("lib_a%d" % i if i else "lib_a"): os.path.abspath(p) for i, p in enumerate(args.ab)}
    libs["lib_b"] = L.LIB_PATH
    got = {k: {"child_ms": [], "reset_ms": [], "kernel_ms": []} for k in libs}
    medians = {k: [] for k in libs}
    for _ in range(args.rounds):
        for k, lib in libs.items():
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--K", str(args.K),
                                  "--runs", str(args.runs), "--warmup", str(args.warmup)],
                                 env=dict(os.environ, PB2_LIB_PATH=lib), capture_output=True, text=True, check=True).stdout
            child = json.loads([l for l in out.splitlines() if l.startswith("{")][-1])
            for key in got[k]:
                got[k][key] += child[key]
            medians[k].append(summary(child["child_ms"])["median_ms"])
    res = {k: dict(summary(v["child_ms"]), lib=libs[k], round_medians_ms=medians[k],
                   reset_median_ms=float(np.median(v["reset_ms"])), kernel_median_ms=float(np.median(v["kernel_ms"])))
           for k, v in got.items()}
    for k in libs:
        if k != "lib_b":
            res["b_over_%s_median" % k[4:]] = res["lib_b"]["median_ms"] / res[k]["median_ms"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--K", type=int, default=4096)
    ap.add_argument("--runs", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ab", metavar="LIB", nargs="+", help="alternate the fused window on libraries LIB (lib_a, lib_a1, ...) and on this tree's (lib_b)")
    ap.add_argument("--rounds", type=int, default=4, help="--ab: child processes per library")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        x = Window(args.K, 0)
        ms = runs_of(x, args.warmup, args.runs)
        print(json.dumps({"child_ms": ms, "reset_ms": [r for r, _ in x.split], "kernel_ms": [k for _, k in x.split]}), flush=True)
        return
    print(json.dumps({"card": card()}), flush=True)
    print(json.dumps({"l2_probe": l2_probe()}), flush=True)
    print(json.dumps({"fill_only": measure(Window(args.K, fill_only=True), args.warmup, args.runs)}), flush=True)
    print(json.dumps({"sweep": "fusion_off", **measure(Window(args.K, -1), args.warmup, args.runs)}), flush=True)
    print(json.dumps({"sweep": "fusion_on", **measure(Window(args.K, 0), args.warmup, args.runs)}), flush=True)
    if args.ab:
        print(json.dumps({"ab": ab_libraries(args)}), flush=True)


if __name__ == "__main__":
    main()
