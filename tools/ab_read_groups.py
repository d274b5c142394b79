"""Where the resident Ex05 window spends its time, and what read groups change (development aid, not the bench).

1. the card: name, power limit and maximum SM clock (read-only nvidia-smi query);
2. tools/l2_probe (compiled into a temporary directory): the L2 read rate and the DRAM rates of this GPU;
3. the resident Ex05 window (dags.ex05_broadcast(K, NB, 262144), tiles VALID) at NB = 0, 2, 6, 14, i.e. F = 1, 2, 4, 8
   readers per tile, with read groups off and on: median / min / max of reset_ms + kernel_ms, and the fit ms = a + b*F;
4. --ab: the NB = 14 window with read groups off and on, alternated run by run.

    python tools/ab_read_groups.py [--runs 30] [--ab]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from parsec_b200 import _lib as L
from oracle import orc_dags as dags
from parsec_b200.engine import Engine

TB = 256 * 256 * 4
HERE = os.path.dirname(os.path.abspath(__file__))


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=" + q, "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:
        out = "nvidia-smi failed: %r" % (exc,)
    return out


def l2_probe(*args):
    """tools/l2_probe's last JSON line, run with args."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "l2_probe")
        subprocess.check_call([nvcc, "-O3", "-gencode", "arch=compute_90a,code=sm_90a", os.path.join(HERE, "l2_probe.cu"), "-o", exe])
        out = subprocess.run([exe, *args], capture_output=True, text=True, timeout=120).stdout
    lines = [l for l in out.splitlines() if l.startswith("{")]
    return json.loads(lines[-1]) if lines else {"error": out[-400:]}


class Ex05:
    """One engine (read groups on or off) and one resident Ex05 window on it."""

    def __init__(self, K, NB, read_groups):
        self.e = Engine(0, read_groups=read_groups)
        self.dag = dags.ex05_broadcast(K, NB, TB)
        self.slab = self.e.malloc(K * TB)
        self.e.h2d(self.slab, np.zeros(K * TB // 4, np.int32))
        tiles = np.zeros(K, L.TILE_DTYPE)
        tiles["dev_ptr"] = self.slab + np.arange(K, dtype=np.uint64) * np.uint64(TB)
        tiles["bytes"] = TB
        tiles["state"] = L.TILE_VALID
        self.w = self.e.window(0, self.dag.tasks, self.dag.succ, tiles, self.dag.ready)

    def run(self):
        st = self.w.run()
        assert st["body_errors"] == 0 and st["tasks_retired"] == self.dag.ntasks
        return st["reset_ms"] + st["kernel_ms"]

    def close(self):
        self.w.close()
        self.e.close()


def summary(ms):
    ms = sorted(ms)
    return {"median_ms": ms[len(ms) // 2], "min_ms": ms[0], "max_ms": ms[-1], "runs": len(ms),
            "spread_pct": (ms[-1] - ms[0]) / ms[len(ms) // 2] * 100.0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--K", type=int, default=4096)
    ap.add_argument("--runs", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ab", action="store_true", help="also alternate read groups off / on on the NB = 14 window")
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    print(json.dumps({"l2_probe": l2_probe()}), flush=True)

    for label, rg in (("groups_off", -1), ("groups_on", 0)):
        rows = []
        for NB in (0, 2, 6, 14):
            x = Ex05(args.K, NB, rg)
            for _ in range(args.warmup):
                x.run()
            s = summary([x.run() for _ in range(args.runs)])
            x.close()
            s.update(NB=NB, F=NB // 2 + 1)
            rows.append(s)
            print(json.dumps({"sweep": label, **s}), flush=True)
        F = np.array([r["F"] for r in rows], np.float64)
        y = np.array([r["median_ms"] for r in rows], np.float64)
        b, a = np.polyfit(F, y, 1)
        print(json.dumps({"fit": label, "a_ms": a, "b_ms_per_reader": b, "F1_ms": rows[0]["median_ms"], "F8_ms": rows[-1]["median_ms"],
                          "F8_over_F1": rows[-1]["median_ms"] / rows[0]["median_ms"]}), flush=True)

    if args.ab:
        xs = {"groups_off": Ex05(args.K, 14, -1), "groups_on": Ex05(args.K, 14, 0)}
        for x in xs.values():
            for _ in range(args.warmup):
                x.run()
        ms = {k: [] for k in xs}
        for _ in range(args.runs):
            for k, x in xs.items():
                ms[k].append(x.run())
        res = {k: summary(v) for k, v in ms.items()}
        res["speedup_median"] = res["groups_off"]["median_ms"] / res["groups_on"]["median_ms"]
        print(json.dumps({"ab": res}), flush=True)
        for x in xs.values():
            x.close()


if __name__ == "__main__":
    main()
