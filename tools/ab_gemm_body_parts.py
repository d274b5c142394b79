"""What cutting GEMM-worker tasks into parts (pb2_engine_set_gemm_body_parts) buys the fp64 DTD GEMM (development aid,
not the bench).

The DTD GEMM of tests/fp64_gemm.py (C(i,j) += A(i,k) B(k,j)^T over NT x NT x NT tasks) in one GEMM window with every
tile resident in HBM and C never pushed out, through the parted DGEMM of tests/cuda/gemm_part_bodies.cu (linked with
PB2_LINK_GEMM_BODY_ENTRY), at three shapes:
  - NT = 4, 1024 x 1024 tiles: 16 C chains, so at most 16 of 132 SMs busy with one part per task;
  - NT = 8, 512 x 512: 64 chains;
  - NT = 32, 512 x 512: 1024 chains, wider than the machine.
For each shape, one window per part count (1, 2, 4, 8, and 16 for the narrow shapes) on one engine and one slab.  Each
window runs once from the same seeded tiles, and its C is compared bit for bit with nparts = 1's; then the windows run
alternately, run by run, after warm-up.

Prints JSON lines: the card (name, power limit, maximum SM clock), then per shape and part count the median / min /
max / spread of kernel_ms (CUDA events around the window kernel), TFLOP/s and its fraction of the H100 SXM data-sheet
FP64 tensor-core figure, 67 TFLOP/s (a data-sheet number, not one reached), and whether C matched nparts = 1; the card
again, with the current SM clock, at the end.

    python tools/ab_gemm_body_parts.py [--runs 10 --warmup 2] [--shapes 4x1024,8x512,32x512]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
from parsec_b200 import _lib as L
from parsec_b200.engine import Engine
from ab_read_groups import card, summary
from ab_gemm_worker_bodies import DATASHEET_FP64_TENSOR_TFLOPS, resident
import fp64_gemm as F


def sm_clock():
    try:
        return subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=clocks.sm,power.draw", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:
        return "nvidia-smi failed: %r" % (exc,)


def shape(e, NT, T, counts, runs, warmup):
    dag, sizes = F.dag(NT, T, T, T)
    dag.tasks["access"][:, 2] &= ~np.uint8(L.FLOW_PUSHOUT)      # C stays resident
    slab, tiles = resident(e, dag, sizes)
    nt = NT * NT
    rng = np.random.default_rng(7)
    c0 = {}
    for tid in range(dag.ntiles):
        x = rng.uniform(-1, 1, (T, T))
        e.h2d(int(tiles["dev_ptr"][tid]), x)
        if tid >= 2 * nt:
            c0[tid] = x
    e.synchronize()
    wins, cs = {}, {}
    try:
        for n in counts:
            e.set_gemm_body_parts(F.DGEMM, n)
            wins[n] = e.window(1, dag.tasks, dag.succ, tiles, dag.ready)
        e.set_gemm_body_parts(F.DGEMM, 1)
        # one run of each from the same C, then C compared with nparts = 1's
        for n, w in wins.items():
            for tid, x in c0.items():
                e.h2d(int(tiles["dev_ptr"][tid]), x)
            e.synchronize()
            assert w.run()["tasks_retired"] == dag.ntasks
            got = [e.d2h(np.empty((T, T), np.float64), int(tiles["dev_ptr"][tid])) for tid in sorted(c0)]
            e.synchronize()
            cs[n] = np.concatenate([x.reshape(-1) for x in got])
        same = {n: bool(np.array_equal(cs[n].view(np.uint64), cs[counts[0]].view(np.uint64))) for n in counts}
        for _ in range(warmup):
            for w in wins.values():
                w.run()
        ms = {n: [] for n in counts}
        for _ in range(runs):
            for n, w in wins.items():
                st = w.run()
                assert st["tasks_retired"] == dag.ntasks
                ms[n].append(st["kernel_ms"])
    finally:
        for w in wins.values():
            w.close()
        e.free(slab)
    flop = 2.0 * (NT * T) ** 3
    for n in counts:
        s = summary(ms[n])
        tf = flop / (s["median_ms"] * 1e-3) / 1e12
        print(json.dumps({"window": "fp64_dtd_gemm", "NT": NT, "T": T, "nparts": n, "flop": flop, "kernel_ms": s,
                          "tflops_median": tf, "fraction_of_datasheet_fp64_tensor_67": tf / DATASHEET_FP64_TENSOR_TFLOPS,
                          "c_same_bits_as_nparts_1": same[n],
                          "median_over_nparts_1": s["median_ms"] / summary(ms[counts[0]])["median_ms"]}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--shapes", default="4x1024,8x512,32x512")
    a = ap.parse_args()
    print(json.dumps({"card": card(), "sm_clock_power": sm_clock()}), flush=True)
    e = Engine(0, timeout_ms=120000)
    try:
        with open(os.path.join(ROOT, "tests", "cuda", "gemm_part_bodies.cubin"), "rb") as f:
            e.link_bodies(f.read(), L.IMAGE_CUBIN, 0, gemm_windows=True, gemm_bodies=F.GEMM_BODIES, gemm_body_entry=True)
        print(json.dumps({"linked_gemm_info": e.linked_gemm_info()}), flush=True)
        for sh in a.shapes.split(","):
            NT, T = map(int, sh.split("x"))
            counts = [1, 2, 4, 8] + ([16] if NT * NT < 132 else [])
            shape(e, NT, T, counts, a.runs, a.warmup)
            print(json.dumps({"after": sh, "sm_clock_power": sm_clock()}), flush=True)
    finally:
        e.close()
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
