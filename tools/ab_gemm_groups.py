"""What read groups and fused producers do for a GEMM window (development aid, not the bench).

Three resident windows over the Ex05 DAG (K = 4096 tiles of 256 KiB, F = 8 readers each, dags.ex05_broadcast):
  - gemm: Ex05 beside one small GEMM chain (two 128^3 GEMMs and four CHECK readers of their C) as one kind-1 window,
    the way the stand-alone runtime's take_closure builds a window whose closure holds a GEMM task;
  - linked_gemm: the same window with TaskBcast's FILL as the checked linked FILL of tests/cuda/checked_bodies.cubin,
    on an engine linked with PB2_LINK_GEMM_WINDOWS;
  - hbm: the Ex05 DAG alone as an HBM window (the reference point; in the child of this tree's library only).
With --ab LIB, child processes alternate between library LIB (e.g. the parent commit's libparsec_b200.so, through
PB2_LIB_PATH) and this tree's, --rounds each, every child timing --runs launches of each window after a warm-up.
Prints one JSON line: the card (name, power limit, maximum SM clock), per library and window the median and
min ... max of kernel_ms over all its runs, and whether every library computed the same results and versions.

    python tools/ab_gemm_groups.py --ab /path/to/parent/parsec_b200/libparsec_b200.so [--rounds 3 --runs 10]
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

K, TB = 4096, 256 * 1024


def windows(hbm):
    """{name: (engine, window, slab)} of the resident windows; hbm: also the HBM window."""
    from oracle import orc_dags as dags
    from parsec_b200 import _lib as L
    from parsec_b200.engine import Engine
    from gemm_chain_dags import ex05_beside_gemm
    dag, ex, sizes, host = ex05_beside_gemm(K, TB)
    linked = dag.tasks.copy()
    linked["body"][linked["body"] == L.BODY_FILL_I32] = L.BODY_LINKED_0
    ldag = dags.Dag(linked, dag.succ, dag.ready, ntiles=dag.ntiles, tile_bytes=TB, kind=1)
    with open(os.path.join(ROOT, "tests", "cuda", "checked_bodies.cubin"), "rb") as f:
        image = f.read()
    out = {}
    cases = [("gemm", dag, False), ("linked_gemm", ldag, True)] + ([("hbm", ex, False)] if hbm else [])
    for name, d, link in cases:
        e = Engine(0)
        if link:
            e.link_bodies(image, L.IMAGE_CUBIN, 0b11, 0b11, gemm_windows=True)
        # every tile resident, in 512-byte slots back to back, holding its bytes of the host image
        nb = np.array(sizes[:d.ntiles], np.int64)
        off = np.concatenate([[0], np.cumsum(nb)[:-1]])
        slot = np.concatenate([[0], np.cumsum((nb + 511) // 512 * 512)[:-1]])
        image_dev = np.zeros(int(slot[-1] + nb[-1]), np.uint8)
        for i in range(d.ntiles):
            image_dev[slot[i]:slot[i] + nb[i]] = host[off[i]:off[i] + nb[i]]
        slab = e.malloc(len(image_dev))
        e.h2d(slab, image_dev)
        tiles = np.zeros(d.ntiles, L.TILE_DTYPE)
        tiles["dev_ptr"] = np.uint64(slab) + slot.astype(np.uint64)
        tiles["bytes"], tiles["state"] = nb, L.TILE_VALID
        out[name] = (e, e.window(d.kind, d.tasks, d.succ, tiles, d.ready), slab)
    return out


def child(args):
    wins = windows(args.hbm)
    ms = {k: [] for k in wins}
    try:
        for _ in range(args.warmup):
            for e, w, _ in wins.values():
                w.run()
        for _ in range(args.runs):
            for k, (e, w, _) in wins.items():
                st = w.run()
                ms[k].append(st["kernel_ms"])
        res = {k: w.results() for k, (e, w, _) in wins.items()}
        digest = {k: [int(np.bitwise_xor.reduce(r["result"])), int(r["seen_version"].astype(np.int64).sum())]
                  for k, r in res.items()}
    finally:
        for e, w, slab in wins.values():
            w.close()
            e.free(slab)
            e.close()
    print(json.dumps({"ms": ms, "digest": digest}))


def summary(v):
    return {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v)), "n": len(v)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ab", metavar="LIB", help="alternate with library LIB (lib_a); this tree's is lib_b")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--child", action="store_true")
    ap.add_argument("--hbm", action="store_true")
    args = ap.parse_args()
    if args.child:
        return child(args)
    from ab_read_groups import card
    libs = {"lib_b": os.path.join(ROOT, "parsec_b200", "libparsec_b200.so")}
    if args.ab:
        libs = {"lib_a": os.path.abspath(args.ab), **libs}
    ms, digests = {k: {} for k in libs}, {}
    for _ in range(args.rounds):
        for k, lib in libs.items():
            cmd = [sys.executable, os.path.abspath(__file__), "--child", "--runs", str(args.runs), "--warmup", str(args.warmup)]
            out = json.loads(subprocess.run(cmd + (["--hbm"] if k == "lib_b" else []), env=dict(os.environ, PB2_LIB_PATH=lib),
                                            capture_output=True, text=True, check=True).stdout.strip().splitlines()[-1])
            for w, v in out["ms"].items():
                ms[k].setdefault(w, []).extend(v)
            digests[k] = out["digest"]
    same = all(digests[k][w] == digests["lib_b"][w] for k in digests for w in digests[k])
    print(json.dumps({"card": card(), "K": K, "tile_bytes": TB, "kernel_ms": {k: {w: summary(v) for w, v in m.items()} for k, m in ms.items()},
                      "same_results_and_versions": same}))


if __name__ == "__main__":
    main()
