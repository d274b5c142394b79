"""How the resident Ex05 window's time depends on the number of fused units per worker, and on the parts they are cut
into (development aid, not the bench).

1. the card: name, power limit and maximum SM clock (read-only nvidia-smi query), and the engine's worker count n;
2. staircase: the resident Ex05 window (dags.ex05_broadcast(K, 14, 262144), tiles VALID, every producer fused with its
   8-reader CHECK group) at the default part size for K = n, n + 1, 3n/2, 2n, 2n + 1, 4096 and 3n.  A time that steps
   at multiples of n and is flat in between is a tail of idle workers; a time linear in K is the DRAM write rate;
3. part sweep at K = --K: the default cut, then explicit part_bytes of 256 KiB, 128 KiB, 87 392 B (3 parts), 64 KiB,
   43 696 B (6 parts) and 32 KiB, alternated run by run;
4. fits: the staircase rows against ms = a + b * K (DRAM-bound: b is the time to write one tile) and against
   ms = a + t_wave * waves (tail-bound, waves = ceil(K / n)); the kernel time of the part sweep (median of the sum less
   median reset_ms) against ms = a + t_entry * K * p, p the parts per unit the window chose (pb2_window_task_entries):
   a part costs t_part = n * t_entry on each worker, and c = t_part / t_unit = t_entry / b is that cost in units of a
   whole unit at the DRAM rate.
Each row: median / min / max / spread of reset_ms + kernel_ms, and the median reset_ms alone.

    python tools/ab_balance.py [--runs 30]
"""
import argparse
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from ab_fuse_readers import Window
from ab_read_groups import card, summary

SWEEP = (("default", 0), ("256KiB", 262144), ("128KiB", 131072), ("3_parts", 87392), ("64KiB", 65536),
         ("6_parts", 43696), ("32KiB", 32768))


def unit_parts(x):
    """Parts of the first producer of the window (task 0 of dags.ex05_broadcast)."""
    return int((int(x.w.task_entries()[0]) & 0xFFFFFFFF) >> 22) + 1


def warm(x, warmup):
    for _ in range(warmup):
        x.run()


def run(x, reset_ms):
    """One run of window x: reset_ms + kernel_ms; appends reset_ms alone to the list reset_ms."""
    ms = x.run()
    reset_ms.append(x.w.stats["reset_ms"])
    return ms


def lstsq(cols, y):
    A = np.stack([np.ones_like(y)] + cols, axis=1)
    coef, *_ = np.linalg.lstsq(A, y, rcond=None)
    return coef, float(np.max(np.abs(A @ coef - y)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--K", type=int, default=4096)
    ap.add_argument("--runs", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    probe = Window(64)
    n = probe.e.info()["nworkers"]
    probe.close()
    print(json.dumps({"card": card(), "nworkers": n}), flush=True)

    stairs = []
    for K in (n, n + 1, 3 * n // 2, 2 * n, 2 * n + 1, 4096, 3 * n):
        x = Window(K)
        p = unit_parts(x)
        warm(x, args.warmup)
        reset = []
        s = summary([run(x, reset) for _ in range(args.runs)])
        x.close()
        s.update(K=K, parts=p, waves=math.ceil(K * p / n), units_per_worker=K / n, reset_median_ms=float(np.median(reset)))
        stairs.append(s)
        print(json.dumps({"staircase": s}), flush=True)
    K = np.array([r["K"] for r in stairs], np.float64)
    y = np.array([r["median_ms"] for r in stairs], np.float64)
    (a, b), res_lin = lstsq([K], y)
    (aw, t_wave), res_wave = lstsq([np.array([r["waves"] for r in stairs], np.float64)], y)
    print(json.dumps({"fit": "staircase", "linear_a_ms": a, "linear_us_per_unit": b * 1e3, "linear_write_tbs": 262144 / (b * 1e-3) / 1e12,
                      "linear_max_residual_ms": res_lin, "waves_a_ms": aw, "waves_ms_per_wave": t_wave, "waves_max_residual_ms": res_wave}),
          flush=True)

    xs = [(label, Window(args.K, part_bytes=pb)) for label, pb in SWEEP]
    for _, x in xs:
        warm(x, args.warmup)
    ms = {label: [] for label, _ in xs}
    reset = {label: [] for label, _ in xs}
    for _ in range(args.runs):
        for label, x in xs:
            ms[label].append(run(x, reset[label]))
    sweep = []
    for label, x in xs:
        p = unit_parts(x)
        s = dict(summary(ms[label]), K=args.K, parts=p, waves=math.ceil(args.K * p / n), part_bytes=dict(SWEEP)[label],
                 reset_median_ms=float(np.median(reset[label])))
        sweep.append(s)
        print(json.dumps({"sweep": label, **s}), flush=True)
        x.close()
    explicit = [r for r in sweep if r["part_bytes"]]
    entries = np.array([r["K"] * r["parts"] for r in explicit], np.float64)
    y = np.array([r["median_ms"] - r["reset_median_ms"] for r in explicit], np.float64)
    (a_k, t_entry), res = lstsq([entries], y)
    print(json.dumps({"fit": "sweep: kernel ms = a + t_entry * K * p", "a_ms": a_k, "t_entry_ns": t_entry * 1e6,
                      "t_part_us_per_worker": t_entry * n * 1e3, "c": t_entry / b, "max_residual_ms": res}), flush=True)


if __name__ == "__main__":
    main()
