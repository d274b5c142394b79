"""What the linking point costs (development aid, not the bench): the resident Ex05 window (dags.ex05_broadcast(K, 14,
256 KiB), tiles VALID) with TaskBcast's FILL as the built-in FILL_I32 body, and with the same FILL as a linked body
(PB2_BODY_LINKED_0 + 3 of tests/cuda/linked_bodies.cu, sliceable, linked from the cubin the Makefile builds), alternated
run by run on engines of their own.  That linked FILL has no checked form, so its tile's read group runs after it instead
of with it (no fused unit).  So a third window, the built-in FILL with fusion off (fuse_readers=-1), separates the two:
linked against unfused built-in is the cost of the call across the link (a stack frame in the linked kernel).  A fourth
window runs the checked FILL of tests/cuda/checked_bodies.cu (PB2_BODY_LINKED_0, linked with its checked bit set), which
runs fused with its read group as the built-in FILL does, but stores without the built-ins' L2 evict-first hint.

Prints one JSON line: the card (name, power limit, maximum SM clock), the linked kernel's pb2_engine_linked_info, and
the step-time median / min / max / spread of each window (reset + kernel CUDA-event time).

    python tools/ab_linked.py [--K 4096] [--runs 30]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200.engine import Engine
from ab_read_groups import card, summary

TB = 256 * 1024
LINKED_FILL = L.BODY_LINKED_0 + 3
CHECKED_FILL = L.BODY_LINKED_0


class Ex05:
    """One engine and one resident Ex05 window on it; linked: its FILL tasks run the linked FILL ("plain") or the
    checked linked FILL ("checked")."""

    def __init__(self, K, linked=None, fuse_readers=0):
        self.e = Engine(0, fuse_readers=fuse_readers)
        self.dag = dags.ex05_broadcast(K, 14, TB)
        tasks = self.dag.tasks.copy()
        self.info = None
        if linked:
            image, body, mask = (("checked_bodies.cubin", CHECKED_FILL, 1) if linked == "checked"
                                 else ("linked_bodies.cubin", LINKED_FILL, 1 << 3))
            with open(os.path.join(ROOT, "tests", "cuda", image), "rb") as f:
                self.e.link_bodies(f.read(), L.IMAGE_CUBIN, mask, mask if linked == "checked" else 0)
            self.info = self.e.linked_info()
            tasks["body"][tasks["body"] == L.BODY_FILL_I32] = body
        self.slab = self.e.malloc(K * TB)
        self.e.h2d(self.slab, np.zeros(K * TB // 4, np.int32))
        tiles = np.zeros(K, L.TILE_DTYPE)
        tiles["dev_ptr"] = self.slab + np.arange(K, dtype=np.uint64) * np.uint64(TB)
        tiles["bytes"] = TB
        tiles["state"] = L.TILE_VALID
        self.w = self.e.window(0, tasks, self.dag.succ, tiles, self.dag.ready)

    def run(self):
        st = self.w.run()
        assert st["body_errors"] == 0 and st["tasks_retired"] == self.dag.ntasks
        return st["reset_ms"] + st["kernel_ms"]

    def outputs(self):
        r = self.w.results()
        return r["result"], r["seen_version"]

    def close(self):
        self.w.close()
        self.e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--K", type=int, default=4096)
    ap.add_argument("--runs", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    wins = {"builtin_fill": Ex05(a.K), "builtin_fill_unfused": Ex05(a.K, None, -1), "linked_fill": Ex05(a.K, "plain"),
            "linked_checked_fill": Ex05(a.K, "checked")}
    ms = {k: [] for k in wins}
    try:
        for _ in range(a.warmup):
            for w in wins.values():
                w.run()
        for _ in range(a.runs):
            for k, w in wins.items():
                ms[k].append(w.run())
        ref = wins["builtin_fill"].outputs()
        same = all(np.array_equal(x, y) for w in wins.values() for x, y in zip(ref, w.outputs()))
    finally:
        for w in wins.values():
            w.close()
    linked = wins["linked_fill"]
    out = {"card": card(), "K": a.K, "linked_info": linked.info, "same_results_and_versions": same}
    out.update({k: summary(v) for k, v in ms.items()})
    out["linked_over_builtin"] = out["linked_fill"]["median_ms"] / out["builtin_fill"]["median_ms"]
    out["linked_over_builtin_unfused"] = out["linked_fill"]["median_ms"] / out["builtin_fill_unfused"]["median_ms"]
    out["checked_over_builtin"] = out["linked_checked_fill"]["median_ms"] / out["builtin_fill"]["median_ms"]
    out["checked_over_linked"] = out["linked_checked_fill"]["median_ms"] / out["linked_fill"]["median_ms"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
