"""What read groups and fused units do for linked readers (development aid, not the bench).

The resident Ex05 window (K = 4096 tiles of 256 KiB, F = 8 readers each, dags.ex05_broadcast) with TaskRecv as the linked
reader COUNT_NE of tests/cuda/reader_bodies.cubin, which does CHECK's work (it counts the elements that differ from its
constant), in these windows of one process, alternated run by run:
  - builtin_fused: the built-in CHECK readers, fused with the built-in FILL (the reference point);
  - builtin_ungrouped: the same with read_groups = -1;
  - linked_ungrouped: linked readers with read_groups = -1 (what an application got before linked readers);
  - linked_grouped: linked readers in read groups, fuse_readers = -1;
  - linked_fused_builtin: linked readers grouped and fused with the built-in FILL;
  - linked_fused_linked: linked readers grouped and fused with the linked FILL;
  - gemm: linked_fused_builtin's DAG beside one small GEMM chain whose C tile four linked readers read, as one GEMM
    window on an engine linked with PB2_LINK_GEMM_WINDOWS (as tools/ab_gemm_groups.py builds it; the chain adds into C
    on every run, so only the Ex05 tasks' results are compared);
  - gemm_ungrouped: the same GEMM window with read_groups = -1;
  - group_grouped, group_fused_builtin, group_fused_linked, group_gemm: linked_grouped, linked_fused_builtin,
    linked_fused_linked and gemm on engines linked with tests/cuda/reader_group_bodies.cubin and its readers declared
    with the group form (PB2_LINK_READER_GROUPS): each read group calls pb2_linked_reader_group once per chunk.
Each window runs --runs times after --warmup runs.  Prints one JSON line: the card (name, power limit, maximum SM
clock), per window the median and min ... max of kernel_ms, the linked kernels' resources (pb2_engine_linked_info and,
for the GEMM windows, pb2_engine_linked_gemm_info), and whether every window computed the same results (a
CHECK reader's mismatch count is the high word of its result) and versions; it fails if they did not.

    python tools/ab_linked_readers.py [--runs 30 --warmup 3]
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

K, TB = 4096, 256 * 1024
COUNT_NE, FILL = 20, 24               # tests/cuda/reader_bodies.cu
READERS, SLICEABLE = 0b1000111, 0x7F


def windows():
    """{name: (engine, window, slab, dag)} of the resident windows."""
    from oracle import orc_dags as dags
    from parsec_b200 import _lib as L
    from parsec_b200.engine import Engine
    from gemm_chain_dags import ex05_beside_gemm
    images = {}
    for fixture in ("reader_bodies", "reader_group_bodies"):
        with open(os.path.join(ROOT, "tests", "cuda", fixture + ".cubin"), "rb") as f:
            images[fixture] = f.read()
    ex = dags.ex05_broadcast(K, 14, TB)

    def bodies(dag, producer, reader):
        t = dag.tasks.copy()
        t["body"][t["body"] == L.BODY_CHECK_I32] = reader
        t["body"][t["body"] == L.BODY_FILL_I32] = producer
        return dags.Dag(t, dag.succ, dag.ready, ntiles=dag.ntiles, tile_bytes=TB, kind=dag.kind)

    gdag, _, gsizes, ghost = ex05_beside_gemm(K, TB)
    gdag = bodies(gdag, L.BODY_FILL_I32, COUNT_NE)
    # (name, dag, engine parameters, the fixture linked or None, its group mask)
    cases = [
        ("builtin_fused", ex, {}, None, 0),
        ("builtin_ungrouped", ex, dict(read_groups=-1), None, 0),
        ("linked_ungrouped", bodies(ex, L.BODY_FILL_I32, COUNT_NE), dict(read_groups=-1), "reader_bodies", 0),
        ("linked_grouped", bodies(ex, L.BODY_FILL_I32, COUNT_NE), dict(fuse_readers=-1), "reader_bodies", 0),
        ("linked_fused_builtin", bodies(ex, L.BODY_FILL_I32, COUNT_NE), {}, "reader_bodies", 0),
        ("linked_fused_linked", bodies(ex, FILL, COUNT_NE), {}, "reader_bodies", 0),
        ("gemm", gdag, {}, "reader_bodies", 0),
        ("gemm_ungrouped", gdag, dict(read_groups=-1), "reader_bodies", 0),
        ("group_grouped", bodies(ex, L.BODY_FILL_I32, COUNT_NE), dict(fuse_readers=-1), "reader_group_bodies", READERS),
        ("group_fused_builtin", bodies(ex, L.BODY_FILL_I32, COUNT_NE), {}, "reader_group_bodies", READERS),
        ("group_fused_linked", bodies(ex, FILL, COUNT_NE), {}, "reader_group_bodies", READERS),
        ("group_gemm", gdag, {}, "reader_group_bodies", READERS),
    ]
    out = {}
    for name, d, kw, fixture, groups in cases:
        e = Engine(0, **kw)
        if fixture:
            e.link_bodies(images[fixture], L.IMAGE_CUBIN, SLICEABLE, 0, gemm_windows=d.kind == 1, readers=READERS,
                          reader_groups=groups)
        # every tile resident, in 512-byte slots back to back: the Ex05 tiles all -1, the chain's as ex05_beside_gemm
        nb = np.array(gsizes[:d.ntiles], np.int64)
        off = np.concatenate([[0], np.cumsum(nb)[:-1]])
        slot = np.concatenate([[0], np.cumsum((nb + 511) // 512 * 512)[:-1]])
        image_dev = np.zeros(int(slot[-1] + nb[-1]), np.uint8)
        for i in range(d.ntiles):
            image_dev[slot[i]:slot[i] + nb[i]] = ghost[off[i]:off[i] + nb[i]]
        slab = e.malloc(len(image_dev))
        e.h2d(slab, image_dev)
        tiles = np.zeros(d.ntiles, L.TILE_DTYPE)
        tiles["dev_ptr"] = np.uint64(slab) + slot.astype(np.uint64)
        tiles["bytes"], tiles["state"] = nb, L.TILE_VALID
        out[name] = (e, e.window(d.kind, d.tasks, d.succ, tiles, d.ready), slab, d)
    return out


def summary(v):
    return {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v)), "n": len(v)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    from ab_read_groups import card
    wins = windows()
    ms = {k: [] for k in wins}
    try:
        for _ in range(args.warmup):
            for e, w, _, _ in wins.values():
                w.run()
        for _ in range(args.runs):
            for k, (e, w, _, _) in wins.items():
                ms[k].append(w.run()["kernel_ms"])
        res = {k: w.results() for k, (e, w, _, _) in wins.items()}
        infos = {k: e.linked_info() for k, (e, w, _, d) in wins.items() if not k.startswith("builtin")}
        infos.update({k + "_gemm_kernel": e.linked_gemm_info() for k, (e, w, _, d) in wins.items() if d.kind == 1})
    finally:
        for e, w, slab, _ in wins.values():
            w.close()
            e.free(slab)
            e.close()
    # the Ex05 tasks' results: a reader's mismatch count (CHECK keeps it in the high word), versions
    n = K + K * 8
    norm = {}
    for k, r in res.items():
        v = r["result"][:n].copy()
        if k.startswith("builtin"):
            v[K:] >>= np.uint64(32)
        norm[k] = (v, r["seen_version"][:n], r["tiles"]["version"][:K])
    ref = norm["builtin_fused"]
    same = {k: all(np.array_equal(a, b) for a, b in zip(v, ref)) for k, v in norm.items()}
    print(json.dumps({"card": card(), "K": K, "F": 8, "tile_bytes": TB,
                      "kernel_ms": {k: summary(v) for k, v in ms.items()},
                      "linked_info": infos, "same_results_and_versions": same}))
    assert all(same.values()), same


if __name__ == "__main__":
    main()
