"""What compressible tile memory changes (development aid, not the bench).

1. the card: name, power limit and maximum SM clock (read-only nvidia-smi query), whether the device offers compressible
   memory (pb2_engine_info's compression_supported) and whether a 1 GiB pb2_engine_malloc was granted it;
2. tools/l2_probe --compressible (compiled into a temporary directory): 1 GiB written with a constant and with random
   words, on cudaMalloc memory and on compressible memory;
3. three resident windows, each on a plain slab (Engine.malloc(ipc=True), cudaMalloc memory) and on a compressible one
   (Engine.malloc), all six alternated run by run after --warmup runs each:
   - fill_only: the K producers of the Ex05 window alone (one broadcast constant per 256 KiB tile);
   - fused: the resident Ex05 window (dags.ex05_broadcast(K, 14, 262144), producers fused with their read groups);
   - config2_gemm: bench.py's DTD GEMM window (NT = 32, 512 x 512 bf16 tiles of the reference's LCG data, which does
     not compress; C resident);
   each row: median / min / max / spread of reset_ms + kernel_ms, and the compressible median over the plain one;
4. whether the plain and the compressible slab of each window end with the same results, versions and tile bytes
   (the tool fails otherwise).

    python tools/ab_compressible.py [--runs 30]
"""
import argparse
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
from oracle import orc, orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200.bf16 import f32_to_bf16_bits
from parsec_b200.engine import Engine
from ab_fuse_readers import Window
from ab_read_groups import card, l2_probe, summary

NT, T = 32, 512
GEMM_TB = T * T * 2


def lcg_operands():
    """bench.py's config2_gemm data: the reference's LCG tiles (seeds 1789, 1805, 1901) as bf16 bits."""
    O = orc.lib()
    host = np.empty(3 * NT * NT * T * T, np.uint16)
    tmp = np.empty(T * T, np.float32)
    for which, seed in enumerate((1789, 1805, 1901)):
        for i in range(NT):
            for j in range(NT):
                O.orc_lcg_tile(tmp.ctypes.data_as(C.c_void_p), i * T, j * T, T, T, NT * T, T, seed)
                host[((which * NT + i) * NT + j) * T * T:][:T * T] = f32_to_bf16_bits(tmp)
    return host


class Gemm:
    """One engine and bench.py's config2_gemm window on it."""

    def __init__(self, host, ipc):
        self.e = Engine(0)
        dag = dags.dtd_gemm(NT, T)
        dag.tasks["access"][:, 2] &= ~np.uint8(L.FLOW_PUSHOUT)
        self.ntasks = dag.ntasks
        self.slab = self.e.malloc(dag.ntiles * GEMM_TB, ipc=ipc)
        self.e.h2d(self.slab, host)
        tiles = np.zeros(dag.ntiles, L.TILE_DTYPE)
        tiles["dev_ptr"] = self.slab + np.arange(dag.ntiles, dtype=np.uint64) * np.uint64(GEMM_TB)
        tiles["bytes"], tiles["state"] = GEMM_TB, L.TILE_VALID
        self.slab_bytes = dag.ntiles * GEMM_TB
        self.w = self.e.window(1, dag.tasks, dag.succ, tiles, dag.ready)

    def run(self):
        st = self.w.run()
        assert st["tasks_retired"] == self.ntasks
        return st["reset_ms"] + st["kernel_ms"]

    def close(self):
        self.w.close()
        self.e.close()


def outputs(x, slab_bytes):
    """What a window leaves: its results, versions and the slab's bytes."""
    res = x.w.results()
    tiles = np.empty(slab_bytes // 4, np.int32)
    x.e.d2h(tiles, x.slab)
    return {"result": res["result"], "seen_version": res["seen_version"], "tiles": tiles}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--K", type=int, default=4096)
    ap.add_argument("--runs", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    probe = Engine(0)
    ptr = probe.malloc(1 << 30)
    info = probe.info()
    probe.free(ptr)
    probe.close()
    print(json.dumps({"card": card(), "compression_supported": info["compression_supported"],
                      "granted_1gib": info["slab_compressible"]}), flush=True)
    print(json.dumps({"l2_probe": l2_probe("--compressible")}), flush=True)
    host = lcg_operands()
    wins = {}
    for ipc, mem in ((True, "plain"), (False, "compressible")):
        wins[("fill_only", mem)] = Window(args.K, fill_only=True, ipc=ipc)
        wins[("fused", mem)] = Window(args.K, ipc=ipc)
        wins[("config2_gemm", mem)] = Gemm(host, ipc)
    granted = {"%s/%s" % key: x.e.info()["slab_compressible"] for key, x in wins.items()}
    print(json.dumps({"slab_compressible": granted}), flush=True)
    for x in wins.values():
        for _ in range(args.warmup):
            x.run()
    ms = {key: [] for key in wins}
    for _ in range(args.runs):
        for key, x in wins.items():
            ms[key].append(x.run())
    rows = {key: summary(v) for key, v in ms.items()}
    for (kind, mem), row in rows.items():
        print(json.dumps({"window": kind, "memory": mem, **row}), flush=True)
    same = {}
    for kind in ("fill_only", "fused", "config2_gemm"):
        a, b = wins[(kind, "plain")], wins[(kind, "compressible")]
        nbytes = a.slab_bytes if kind == "config2_gemm" else args.K * 256 * 1024
        oa, ob = outputs(a, nbytes), outputs(b, nbytes)
        same[kind] = {k: bool(np.array_equal(oa[k], ob[k])) for k in oa}
        plain, comp = rows[(kind, "plain")], rows[(kind, "compressible")]
        print(json.dumps({"window": kind, "compressible_over_plain_median": comp["median_ms"] / plain["median_ms"],
                          "ranges_overlap": comp["max_ms"] >= plain["min_ms"] and plain["max_ms"] >= comp["min_ms"],
                          "same_outputs": same[kind]}), flush=True)
    for x in wins.values():
        x.close()
    assert all(all(v.values()) for v in same.values()), same


if __name__ == "__main__":
    main()
