"""How the resident Ex05 step responds to the number of workers per SM of HBM windows (development aid, not the bench).

1. the card: name, power limit and maximum SM clock (read-only nvidia-smi query);
2. Engine(workers_per_sm=n) for n in --counts, each with three resident windows of K producers of 256 KiB tiles:
   the fused Ex05 window, the Ex05 window with fusion off (fuse_readers=-1: the read-group path of shared windows), and
   the FILL-only window (the producers alone, no readers); all fifteen run alternated run by run, after --warmup runs
   each.  Each row: median / min / max / spread of reset_ms + kernel_ms;
3. the comparison against 12 workers per SM: for each n, the fused and fusion-off medians over 12's, and how much
   slower the fusion-off median is than at 12 next to its own min ... max spread at n.

    python tools/ab_workers.py [--runs 30] [--counts 3,4,6,8,12]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ab_fuse_readers import Window
from ab_read_groups import card, summary

KINDS = {"fused": dict(fuse_readers=0), "fusion_off": dict(fuse_readers=-1), "fill_only": dict(fill_only=True)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--K", type=int, default=4096)
    ap.add_argument("--runs", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--counts", default="3,4,6,8,12")
    args = ap.parse_args()
    counts = [int(c) for c in args.counts.split(",")]
    print(json.dumps({"card": card()}), flush=True)
    wins = {(kind, n): Window(args.K, workers_per_sm=n, **kw) for n in counts for kind, kw in KINDS.items()}
    for w in wins.values():
        for _ in range(args.warmup):
            w.run()
    ms = {key: [] for key in wins}
    for _ in range(args.runs):
        for key, w in wins.items():
            ms[key].append(w.run())
    for w in wins.values():
        w.close()
    rows = {key: summary(v) for key, v in ms.items()}
    for (kind, n), row in rows.items():
        print(json.dumps({"window": kind, "workers_per_sm": n, **row}), flush=True)
    if 12 in counts:
        ref_fused, ref_off = rows[("fused", 12)], rows[("fusion_off", 12)]
        for n in counts:
            fused, off = rows[("fused", n)], rows[("fusion_off", n)]
            print(json.dumps({"workers_per_sm": n,
                              "fused_over_12": fused["median_ms"] / ref_fused["median_ms"],
                              "fusion_off_over_12": off["median_ms"] / ref_off["median_ms"],
                              "fusion_off_slower_than_12_by_ms": off["median_ms"] - ref_off["median_ms"],
                              "fusion_off_spread_ms": off["max_ms"] - off["min_ms"]}), flush=True)


if __name__ == "__main__":
    main()
