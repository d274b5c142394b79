"""What the GEMM-worker entry point (PB2_LINK_GEMM_BODY_ENTRY) buys the fp64 DTD GEMM (development aid, not the bench).

The reference program's DTD GEMM (dtd_test_simple_gemm.c) at NT = 32 with 512 x 512 fp64 tiles, 8.8e12 flop, in one
GEMM window with C resident in HBM, on the reference's LCG data, on two engines:
  - worker: tests/cuda/gemm_worker_bodies.cu through pb2_linked_body, compiled for the HBM kernels' 80 registers
    (12 warps of 32 x 16 C);
  - entry: tests/cuda/gemm_entry_bodies.cu through pb2_linked_gemm_body, at the GEMM kernels' 168 (12 warps of 32 x 32).
After one run of each, a few C tiles are checked against NumPy and compared bit for bit between the engines; then the
two windows run alternately, run by run.

Prints JSON lines: the card (name, power limit, maximum SM clock), each engine's pb2_engine_linked_gemm_info, and per
engine the median / min / max / spread of kernel_ms (CUDA events around the window kernel) with TFLOP/s and its fraction
of the H100 SXM data-sheet FP64 tensor-core figure, 67 TFLOP/s.

    python tools/ab_gemm_body_entry.py [--runs 30 --warmup 3]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
from parsec_b200 import _lib as L
from parsec_b200.engine import Engine
from ab_read_groups import card, summary
from ab_gemm_worker_bodies import DATASHEET_FP64_TENSOR_TFLOPS, NT, T, resident
import fp64_gemm as F


def engines():
    worker = Engine(0, timeout_ms=60000)
    worker.link_bodies(F.image(), L.IMAGE_CUBIN, 0, gemm_windows=True, gemm_bodies=F.GEMM_BODIES)
    entry = Engine(0, timeout_ms=60000)
    with open(os.path.join(ROOT, "tests", "cuda", "gemm_entry_bodies.cubin"), "rb") as f:
        entry.link_bodies(f.read(), L.IMAGE_CUBIN, 0, gemm_windows=True, gemm_bodies=F.GEMM_BODIES, gemm_body_entry=True)
    return {"worker": worker, "entry": entry}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    dag, sizes = F.dag(NT, T, T, T)
    dag.tasks["access"][:, 2] &= ~np.uint8(L.FLOW_PUSHOUT)      # C stays resident
    nt = NT * NT
    sample = [(0, 0), (NT // 2, 3), (NT - 1, NT - 1)]
    keep = {i * NT + k for i, _ in sample for k in range(NT)} | {nt + k * NT + j for _, j in sample for k in range(NT)} | \
           {2 * nt + i * NT + j for i, j in sample}
    es = engines()
    placed, wins, gen = {}, {}, {}
    try:
        for name, e in es.items():
            print(json.dumps({"engine": name, "linked_gemm_info": e.linked_gemm_info()}), flush=True)
            placed[name] = resident(e, dag, sizes)
        for tid in range(dag.ntiles):
            w, r = divmod(tid, nt)
            m, n = divmod(r, NT)
            mat = "ABC"[w]
            r0, c0 = (m * T, n * T) if mat != "B" else (n * T, m * T)
            x = F.lcg_tile(mat, r0, c0, T, T, NT * T)
            for name, e in es.items():
                e.h2d(int(placed[name][1]["dev_ptr"][tid]), x)
            if tid in keep:
                gen[tid] = x
        for name, e in es.items():
            wins[name] = e.window(1, dag.tasks, dag.succ, placed[name][1], dag.ready)
        # one run each, then the sampled C tiles: within the float64 bound of NumPy's, and the same bits on both
        checked, cs = [], {}
        for name, w in wins.items():
            assert w.run()["tasks_retired"] == dag.ntasks
        rng = np.random.default_rng(3)
        tiles_cmp = sorted({2 * nt + i * NT + j for i, j in sample} | set((2 * nt + rng.choice(nt, 16, replace=False)).tolist()))
        for name, e in es.items():
            cs[name] = {}
            for tid in tiles_cmp:
                cs[name][tid] = e.d2h(np.empty((T, T), np.float64), int(placed[name][1]["dev_ptr"][tid]))
            e.synchronize()
        for i, j in sample:
            want, bound = F.reference([gen.get(x) for x in range(3 * nt)], NT, i, j)
            err = np.abs(cs["entry"][2 * nt + i * NT + j] - want)
            assert np.all(err <= bound), (i, j, float(err.max()))
            checked.append({"tile": [i, j], "max_abs_err": float(err.max()), "min_bound": float(bound.min())})
        same = all(np.array_equal(cs["entry"][t].view(np.uint64), cs["worker"][t].view(np.uint64)) for t in tiles_cmp)
        print(json.dumps({"checked_tiles": checked, "c_tiles_compared": len(tiles_cmp), "same_bits": same}), flush=True)
        for _ in range(a.warmup):
            for w in wins.values():
                w.run()
        ms = {name: [] for name in wins}
        for _ in range(a.runs):
            for name, w in wins.items():
                st = w.run()
                assert st["tasks_retired"] == dag.ntasks
                ms[name].append(st["kernel_ms"])
    finally:
        for w in wins.values():
            w.close()
        for name, (slab, _) in placed.items():
            es[name].free(slab)
        for e in es.values():
            e.close()
    flop = 2.0 * (NT * T) ** 3
    out = {"window": "fp64_dtd_gemm", "NT": NT, "T": T, "flop": flop, "runs": a.runs}
    for name, v in ms.items():
        s = summary(v)
        tf = flop / (s["median_ms"] * 1e-3) / 1e12
        out[name] = {"kernel_ms": s, "tflops_median": tf, "fraction_of_datasheet_fp64_tensor_67": tf / DATASHEET_FP64_TENSOR_TFLOPS}
    out["entry_over_worker_median"] = out["entry"]["kernel_ms"]["median_ms"] / out["worker"]["kernel_ms"]["median_ms"]
    print(json.dumps(out), flush=True)
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
