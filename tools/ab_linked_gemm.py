"""What linking the GEMM window kernel costs (development aid, not the bench).

The DTD GEMM window of bench.py's config2_gemm (dags.dtd_gemm(32, 512), C resident in HBM), with every C(i,j) filled
with zeros before its k-chain and checked against zero after it, runs on two engines, alternated run by run:
  - builtin: FILL_I32 and CHECK_I32 on the built-in GEMM window kernel;
  - linked: the FILL of tests/cuda/linked_bodies.cu (PB2_BODY_LINKED_0 + 3, sliceable) on the linked GEMM window kernel
    (pb2_engine_link_bodies_ex with PB2_LINK_GEMM_WINDOWS).  The fixture has no CHECK, so the CHECK tasks stay built-in.
Both compute the same C (and so the same CHECK results); the tool asserts it.  It also times pb2_engine_link_bodies_ex
with and without the flag, on fresh engines.

Prints one JSON line: the card (name, power limit, maximum SM clock), pb2_engine_linked_gemm_info, the step-time
median / min / max / spread of each window (reset + kernel CUDA-event time) with its median TFLOP/s, and the link times.

    python tools/ab_linked_gemm.py [--runs 30]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200.engine import Engine
from ab_read_groups import card, summary

NT, T = 32, 512
TB = T * T * 2
LINKED_FILL = L.BODY_LINKED_0 + 3


def image():
    with open(os.path.join(ROOT, "tests", "cuda", "linked_bodies.cubin"), "rb") as f:
        return f.read()


def gemm_with_fill_and_check(fill_body):
    """dtd_gemm(NT, T) without pushout; task c (c < NT^2) fills C(c) with 0, then the chain of C(c), then a CHECK."""
    g = dags.dtd_gemm(NT, T)
    nc, ng = NT * NT, g.ntasks
    t = np.concatenate([dags._new_tasks(nc), g.tasks, dags._new_tasks(nc)])
    t["access"][nc:nc + ng, 2] &= ~np.uint8(L.FLOW_PUSHOUT)
    c_tile = 2 * nc + np.arange(nc)
    for sl, body, acc in ((slice(0, nc), fill_body, L.ACCESS_WRITE), (slice(nc + ng, None), L.BODY_CHECK_I32, L.ACCESS_READ)):
        x = t[sl]
        x["body"], x["nb_flows"], x["tile"][:, 0], x["access"][:, 0] = body, 1, c_tile, acc
    gsrc, gdst, gflow = g.edges()
    heads, tails = nc + np.arange(nc) * NT, nc + np.arange(nc) * NT + NT - 1
    src = np.concatenate([np.arange(nc), gsrc + nc, tails])
    dst = np.concatenate([heads, gdst + nc, nc + ng + np.arange(nc)])
    flow = np.concatenate([np.full(nc, 2), gflow, np.zeros(nc, np.int64)])
    begin, count, succ = dags._csr_from_edges(len(t), src, dst, flow)
    t["succ_begin"], t["succ_count"] = begin, count
    t["dep_goal"] = np.bincount(dst, minlength=len(t))
    return dags.Dag(t, succ, np.arange(nc, dtype=np.int32), ntiles=g.ntiles, tile_bytes=TB, kind=1)


class GemmWindow:
    def __init__(self, linked):
        self.e = Engine(0)
        self.info = None
        if linked:
            self.e.link_bodies(image(), L.IMAGE_CUBIN, 1 << 3, gemm_windows=True)
            self.info = self.e.linked_gemm_info()
        self.dag = gemm_with_fill_and_check(LINKED_FILL if linked else L.BODY_FILL_I32)
        rng = np.random.default_rng(7)
        self.slab = self.e.malloc(self.dag.ntiles * TB)
        self.e.h2d(self.slab, rng.integers(0, 1 << 16, self.dag.ntiles * TB // 2, dtype=np.uint32).astype(np.uint16) & 0xBFFF)
        tiles = np.zeros(self.dag.ntiles, L.TILE_DTYPE)
        tiles["dev_ptr"] = self.slab + np.arange(self.dag.ntiles, dtype=np.uint64) * np.uint64(TB)
        tiles["bytes"], tiles["state"] = TB, L.TILE_VALID
        self.w = self.e.window(1, self.dag.tasks, self.dag.succ, tiles, self.dag.ready)

    def run(self):
        st = self.w.run()
        assert st["tasks_retired"] == self.dag.ntasks
        return st["reset_ms"] + st["kernel_ms"]

    def c_tiles(self):
        out = np.empty(NT * NT * TB // 2, np.uint16)
        self.e.d2h(out, self.slab + 2 * NT * NT * TB)
        return out

    def close(self):
        self.w.close()
        self.e.close()


def link_ms(gemm_windows):
    e = Engine(0)
    try:
        t0 = time.perf_counter()
        e.link_bodies(image(), L.IMAGE_CUBIN, 1 << 3, gemm_windows=gemm_windows)
        return (time.perf_counter() - t0) * 1e3
    finally:
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    links = {"link_ms_hbm_only": [], "link_ms_with_gemm_windows": []}
    for _ in range(3):
        links["link_ms_hbm_only"].append(link_ms(False))
        links["link_ms_with_gemm_windows"].append(link_ms(True))
    wins = {"builtin": GemmWindow(False), "linked": GemmWindow(True)}
    ms = {k: [] for k in wins}
    try:
        for _ in range(a.warmup):
            for w in wins.values():
                w.run()
        for _ in range(a.runs):
            for k, w in wins.items():
                ms[k].append(w.run())
        same_c = bool(np.array_equal(wins["builtin"].c_tiles(), wins["linked"].c_tiles()))
        rb, rl = (w.w.results() for w in wins.values())
        same_results = bool(np.array_equal(rb["result"], rl["result"]) and np.array_equal(rb["seen_version"], rl["seen_version"]))
    finally:
        for w in wins.values():
            w.close()
    flop = 2.0 * NT ** 3 * T ** 3
    out = {"card": card(), "NT": NT, "T": T, "linked_gemm_info": wins["linked"].info, "same_c": same_c,
           "same_results_and_versions": same_results}
    for k, v in ms.items():
        out[k] = summary(v)
        out[k]["tflops_median"] = flop / (float(np.median(v)) * 1e-3) / 1e12
    out.update({k: [round(x, 1) for x in v] for k, v in links.items()})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
