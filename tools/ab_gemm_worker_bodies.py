"""What GEMM-worker bodies (PB2_LINK_GEMM_BODIES) reach and cost (development aid, not the bench).

  - fp64: the reference program's DTD GEMM (dtd_test_simple_gemm.c) at NT = 32 with 512 x 512 fp64 tiles, 8.8e12 flop,
    through the DGEMM body of tests/cuda/gemm_worker_bodies.cu (mma.m16n8k8 fp64 on the operand ring) in one GEMM window,
    C resident in HBM; the reference's LCG data.  A few sampled C tiles are checked against NumPy after the first run.
  - probes: bench.py's config2_gemm window (dags.dtd_gemm(32, 512), bf16, C resident) alone and with a ring probe
    released by every chain's last task, on one linked engine, alternated run by run; both from the same data, and the
    tool asserts that the bf16 C of both windows is the same after one run.
  - link: pb2_engine_link_bodies_ex with the fixture and the GEMM-worker mask, on fresh engines.

Prints JSON lines: the card (name, power limit, maximum SM clock), pb2_engine_linked_gemm_info, and per window the
median / min / max / spread of kernel_ms (CUDA events around the window kernel), with TFLOP/s for the fp64 window and its
fraction of the H100 SXM data-sheet FP64 tensor-core figure, 67 TFLOP/s.

    python tools/ab_gemm_worker_bodies.py [--runs 30 --warmup 3]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200.engine import Engine
from ab_read_groups import card, summary
import fp64_gemm as F

NT, T = 32, 512
DATASHEET_FP64_TENSOR_TFLOPS = 67.0


def linked_engine():
    e = Engine(0, timeout_ms=60000)
    e.link_bodies(F.image(), L.IMAGE_CUBIN, 0, gemm_windows=True, gemm_bodies=F.GEMM_BODIES)
    return e


def resident(e, dag, sizes):
    """One slab for the window's tiles, every tile VALID in it; returns (slab, tile table)."""
    off = np.concatenate([[0], np.cumsum((sizes + 511) // 512 * 512)[:-1]]).astype(np.uint64)
    slab = e.malloc(int(off[-1]) + int(sizes[-1]))
    tiles = np.zeros(dag.ntiles, L.TILE_DTYPE)
    tiles["dev_ptr"] = np.uint64(slab) + off
    tiles["bytes"], tiles["state"] = sizes, L.TILE_VALID
    return slab, tiles


def fp64_window(e, runs, warmup):
    dag, sizes = F.dag(NT, T, T, T)
    dag.tasks["access"][:, 2] &= ~np.uint8(L.FLOW_PUSHOUT)      # C stays resident
    slab, tiles = resident(e, dag, sizes)
    nt = NT * NT
    gen = {}                                   # tile id -> its initial values (kept only for the sampled tiles' inputs)
    sample = [(0, 0), (NT // 2, 3), (NT - 1, NT - 1)]
    keep = {i * NT + k for i, _ in sample for k in range(NT)} | {nt + k * NT + j for _, j in sample for k in range(NT)} | \
           {2 * nt + i * NT + j for i, j in sample}
    for tid in range(dag.ntiles):
        w, r = divmod(tid, nt)
        m, n = divmod(r, NT)
        name, rows = "ABC"[w], NT * T
        # A(i,k): rows i*T.., cols k*T..; B(k,j) is N x K: rows j*T.., cols k*T..; C(i,j): rows i*T.., cols j*T..
        r0, c0 = (m * T, n * T) if name != "B" else (n * T, m * T)
        x = F.lcg_tile(name, r0, c0, T, T, rows)
        e.h2d(int(tiles["dev_ptr"][tid]), x)
        if tid in keep:
            gen[tid] = x
    e.synchronize()
    win = e.window(1, dag.tasks, dag.succ, tiles, dag.ready)
    try:
        st = win.run()
        assert st["tasks_retired"] == dag.ntasks
        checked = []
        for i, j in sample:
            t = [gen.get(x) for x in range(3 * nt)]
            want, bound = F.reference(t, NT, i, j)
            got = np.empty((T, T), np.float64)
            e.d2h(got, int(tiles["dev_ptr"][2 * nt + i * NT + j]))
            e.synchronize()
            err = np.abs(got - want)
            assert np.all(err <= bound), (i, j, float(err.max()))
            checked.append({"tile": [i, j], "max_abs_err": float(err.max()), "min_bound": float(bound.min())})
        for _ in range(warmup):
            win.run()
        ms = [win.run()["kernel_ms"] for _ in range(runs)]
    finally:
        win.close()
        e.free(slab)
    flop = 2.0 * (NT * T) ** 3
    s = summary(ms)
    tf = flop / (s["median_ms"] * 1e-3) / 1e12
    return {"window": "fp64_dtd_gemm", "NT": NT, "T": T, "flop": flop, "kernel_ms": s, "tflops_median": tf,
            "fraction_of_datasheet_fp64_tensor_67": tf / DATASHEET_FP64_TENSOR_TFLOPS, "checked_tiles": checked}


def with_probes(g):
    """g with a ring probe (nb_flows 0) released by the last task of every chain."""
    nc = NT * NT
    t = np.concatenate([g.tasks, dags._new_tasks(nc)])
    p = t[g.ntasks:]
    p["body"], p["dep_goal"], p["iparam"][:, 0] = F.PROBE, 1, np.arange(nc)
    src, dst, flow = g.edges()
    tails = np.arange(nc) * NT + NT - 1
    src = np.concatenate([src, tails])
    dst = np.concatenate([dst, g.ntasks + np.arange(nc)])
    flow = np.concatenate([flow, np.zeros(nc, np.int64)])
    begin, count, succ = dags._csr_from_edges(len(t), src, dst, flow)
    t["succ_begin"], t["succ_count"] = begin, count
    return dags.Dag(t, succ, g.ready, ntiles=g.ntiles, tile_bytes=g.tile_bytes, kind=1)


def probe_windows(e, runs, warmup):
    g = dags.dtd_gemm(NT, T)
    g.tasks["access"][:, 2] &= ~np.uint8(L.FLOW_PUSHOUT)
    tb = T * T * 2
    rng = np.random.default_rng(7)
    data = rng.integers(0, 1 << 16, g.ntiles * tb // 2, dtype=np.uint32).astype(np.uint16) & 0xBFFF
    wins, slabs = {}, []
    for name, dag in (("config2_gemm", g), ("config2_gemm_with_probes", with_probes(g))):
        slab, tiles = resident(e, dag, np.full(dag.ntiles, tb, np.int64))
        e.h2d(slab, data)
        slabs.append((slab, tiles))
        wins[name] = (dag, e.window(1, dag.tasks, dag.succ, tiles, dag.ready))
    try:
        for _, w in wins.values():
            w.run()
        cs = []
        for slab, tiles in slabs:
            c = np.empty(NT * NT * tb // 2, np.uint16)
            e.d2h(c, int(tiles["dev_ptr"][2 * NT * NT]))
            e.synchronize()
            cs.append(c)
        same_c = bool(np.array_equal(cs[0], cs[1]))
        probe_results = wins["config2_gemm_with_probes"][1].results()["result"][g.ntasks:]
        for _ in range(warmup):
            for _, w in wins.values():
                w.run()
        ms = {k: [] for k in wins}
        for _ in range(runs):
            for k, (dag, w) in wins.items():
                st = w.run()
                assert st["tasks_retired"] == dag.ntasks
                ms[k].append(st["kernel_ms"])
    finally:
        for _, w in wins.values():
            w.close()
        for slab, _ in slabs:
            e.free(slab)
    out = {"window": "probes", "same_bf16_c": same_c, "probe_results_nonzero": int(np.count_nonzero(probe_results))}
    flop = 2.0 * (NT * T) ** 3
    for k, v in ms.items():
        out[k] = summary(v)
        out[k]["tflops_median"] = flop / (out[k]["median_ms"] * 1e-3) / 1e12
    out["probe_cost_ms_median"] = out["config2_gemm_with_probes"]["median_ms"] - out["config2_gemm"]["median_ms"]
    return out


def link_ms(mask):
    e = Engine(0)
    try:
        t0 = time.perf_counter()
        e.link_bodies(F.image(), L.IMAGE_CUBIN, 0, gemm_windows=True, gemm_bodies=mask)
        return (time.perf_counter() - t0) * 1e3
    finally:
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    links = {"link_ms_gemm_windows": [link_ms(0) for _ in range(3)],
             "link_ms_gemm_windows_and_gemm_bodies": [link_ms(F.GEMM_BODIES) for _ in range(3)]}
    print(json.dumps({k: [round(x, 1) for x in v] for k, v in links.items()}), flush=True)
    e = linked_engine()
    try:
        print(json.dumps({"linked_gemm_info": e.linked_gemm_info()}), flush=True)
        print(json.dumps(fp64_window(e, a.runs, a.warmup)), flush=True)
        print(json.dumps(probe_windows(e, a.runs, a.warmup)), flush=True)
    finally:
        e.close()
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
