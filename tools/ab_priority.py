"""FIFO (queue_policy 0) against priority lanes (queue_policy 1) on resident windows, alternated run by run in one
process (development aid, not the bench).

1. the card: name, power limit, SM clock now and at most (read-only nvidia-smi query), before and after;
2. the Cholesky shape with the classes and priorities of pb2_ptg_cholesky_shape_new (POTRF 4(NT-k) > TRSM 3(NT-k) >
   SYRK 2(NT-k) > GEMM NT-k; multigpu.cholesky_global on one GPU), nb = 1024 bf16, NT in --nts, tiles resident in HBM
   with seeded values;
3. the DTD GEMM DAG of bench configs[2] (dtd_gemm(32, 1024), priorities NT^3 - i*NT + j);
4. Ex05 at K = 4096 (dags.ex05_broadcast(4096, 14, 262144)): every priority is 0, so this is the cost of the lane scan.

For each window, one engine per policy; after --warmup runs each, --runs runs of each policy, alternating; reported:
median and min / max of reset_ms + kernel_ms.  The first run of policy 1 must leave the tiles exactly as the first run
of policy 0 does (both start from the same seeded bytes).

    python tools/ab_priority.py [--runs 20] [--warmup 3] [--nts 8,16,32,64]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200 import multigpu as M
from parsec_b200.engine import Engine


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=" + q, "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:
        return "nvidia-smi failed: %r" % (exc,)


def cholesky_dag(NT, nb):
    """The Cholesky shape with the classes and priorities of pb2_ptg_cholesky_shape_new, as one window."""
    tasks, succ, tiles, ready, _, _ = M.cholesky_global(NT, nb, 1, 1)
    return dags.Dag(tasks, succ, ready, ntiles=len(tiles), tile_bytes=nb * nb * 2, kind=1, name="cholesky_shape_NT%d" % NT)


class Resident:
    """One engine (policy `pol`) and one window of `dag` whose tiles live in a slab that holds `init` before the first
    run (later runs keep accumulating into C: the time of a bf16 GEMM does not depend on the values)."""

    def __init__(self, dag, pol, init):
        self.e = Engine(0, queue_policy=pol)
        self.dag = dag
        self.slab = self.e.malloc(dag.ntiles * dag.tile_bytes)
        tiles = np.zeros(dag.ntiles, L.TILE_DTYPE)
        tiles["dev_ptr"] = self.slab + np.arange(dag.ntiles, dtype=np.uint64) * np.uint64(dag.tile_bytes)
        tiles["bytes"] = dag.tile_bytes
        tiles["state"] = L.TILE_VALID
        self.e.h2d(self.slab, init)
        self.w = self.e.window(dag.kind, dag.tasks, dag.succ, tiles, dag.ready)

    def run(self):
        st = self.w.run()
        assert st["tasks_retired"] == self.dag.ntasks and st["body_errors"] == 0
        return st["reset_ms"] + st["kernel_ms"]

    def tiles(self):
        return self.e.d2h(np.empty(self.dag.ntiles * self.dag.tile_bytes, np.uint8), self.slab)

    def close(self):
        self.w.close()
        self.e.close()


def seeded(nbytes, rng):
    """bf16 values in [2^-7, 2^-6): the sums of a trailing update stay finite for a while; a 64 MiB seeded pattern
    repeated over the slab."""
    pat = (rng.integers(0, 1 << 32, 16 << 20, dtype=np.uint32) & np.uint32(0x007F007F)) | np.uint32(0x3C003C00)
    return np.resize(pat.view(np.uint8), nbytes)


def summary(ms):
    ms = sorted(ms)
    return {"median_ms": ms[len(ms) // 2], "min_ms": ms[0], "max_ms": ms[-1], "runs": len(ms)}


def ab(name, dag, init, runs, warmup):
    xs = [Resident(dag, 0, init), Resident(dag, 1, init)]
    for x in xs:
        x.run()
    same = bool(np.array_equal(xs[0].tiles(), xs[1].tiles()))
    for _ in range(warmup):
        for x in xs:
            x.run()
    ms = [[], []]
    for _ in range(runs):
        for i, x in enumerate(xs):
            ms[i].append(x.run())
    for x in xs:
        x.close()
    res = {"window": name, "ntasks": dag.ntasks, "policy0": summary(ms[0]), "policy1": summary(ms[1]),
           "policy1_over_policy0_median": summary(ms[1])["median_ms"] / summary(ms[0])["median_ms"], "tiles_equal": same}
    print(json.dumps(res), flush=True)
    assert same, "policy 1 left different tiles than policy 0"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--nts", default="8,16,32,64")
    args = ap.parse_args()
    print(json.dumps({"card_before": card()}), flush=True)
    nb = 1024
    rng = np.random.default_rng(1)
    for NT in [int(x) for x in args.nts.split(",") if x]:
        dag = cholesky_dag(NT, nb)
        init = seeded(dag.ntiles * dag.tile_bytes, rng)
        ab("cholesky_shape NT=%d nb=%d bf16" % (NT, nb), dag, init, args.runs, args.warmup)
    dag = dags.dtd_gemm(32, 1024)
    dag.tasks["access"] &= ~np.uint8(L.FLOW_PUSHOUT)
    init = seeded(dag.ntiles * dag.tile_bytes, rng)
    ab("dtd_gemm NT=32 T=1024 bf16 (configs[2])", dag, init, args.runs, args.warmup)
    dag = dags.ex05_broadcast(4096, 14, 262144)
    ab("ex05 K=4096 NB=14 256 KiB tiles (all priorities 0)", dag, np.zeros(dag.ntiles * dag.tile_bytes, np.uint8), args.runs, args.warmup)
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
