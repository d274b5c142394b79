"""Where the resident Ex05 step's time goes: one traced run of the window bench.py times, as a Chrome trace.

The window is built the way bench.py builds its device-resident value: the stand-alone runtime's Ex05 task pool
(K groups, fan-out NB // 2 + 1), the window its device module would build for it (export_window), tiles VALID in HBM.
The same tasks then run as two windows of one engine, one created with window trace off and one with it on
(pb2_engine_set_window_trace); both are warmed up and then alternated run by run, and the medians of their steps
(reset_ms + kernel_ms, the quantity bench.py sums) are printed side by side: the difference is the cost of tracing.

From the last traced run it prints
  - span: the first pop to the last entity's end (device clock);
  - tail: the last pop to the last entity's end;
  - per SM, the busy fraction of the span: the union of the intervals that SM retired.  A task's interval is its
    scheduling entity's (a fused producer with its read group here), from the earliest pop of any of its parts to the
    latest end of their pushouts, so an entity cut into parts counts on the SM that retired it;
and writes the trace (one row per SM) to --out.  The card's name and power limit are read in the same run.

    python tools/trace_window.py --runs 30 --out trace_ex05.json
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

TILE = 256 * 256 * 4
NB = 14
F = NB // 2 + 1
CLASS_NAMES = {0: "TaskBcast", 1: "TaskRecv"}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=" + q, "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:
        return "nvidia-smi failed: %r" % (exc,)


def busy_fractions(t0, t1, sm, span0, span1):
    """Per SM: the union of its intervals [t0, t1] over the span [span0, span1]."""
    out = {}
    for s in np.unique(sm):
        sel = np.nonzero(sm == s)[0]
        order = sel[np.argsort(t0[sel], kind="stable")]
        busy, cur0, cur1 = 0, None, None
        for i in order:
            a, b = int(t0[i]), int(t1[i])
            if cur1 is None or a > cur1:
                if cur1 is not None:
                    busy += cur1 - cur0
                cur0, cur1 = a, b
            else:
                cur1 = max(cur1, b)
        if cur1 is not None:
            busy += cur1 - cur0
        out[int(s)] = busy / max(1, span1 - span0)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=4096, help="broadcast groups (bench.py's K)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=30, help="timed runs of each window, alternated")
    ap.add_argument("--out", default="trace_ex05.json", help="Chrome trace of the last traced run")
    args = ap.parse_args()

    from parsec_b200 import _lib as L
    from parsec_b200 import runtime as R
    from parsec_b200.engine import Engine, chrome_trace

    print("card:", card(), flush=True)
    K = args.groups
    host = np.zeros(K * TILE // 4, np.int32)
    ctx = R.Context(nb_cores=os.cpu_count() or 1, cuda_devices=(0,))
    dev = ctx.devices[0]
    dc = ctx.block_cyclic(4, TILE // 4, 1, K * TILE // 4, 1, mat=host)
    assert ctx.l.pb2_dc_register_memory(dc, dev) == 0
    tp = C.c_void_p(ctx.l.pb2_ptg_ex05_broadcast_new(ctx.h, dc, K, NB))
    win = ctx.export_window(tp, dev)
    assert len(win["tasks"]) == K * (1 + F)

    with Engine(0) as eng:
        slab = eng.malloc(K * TILE)
        eng.h2d(slab, host)
        tiles = win["tiles"].copy()
        order = np.argsort(tiles["src_ptr"])
        tiles["dev_ptr"][order] = slab + np.arange(K, dtype=np.uint64) * np.uint64(TILE)
        tiles["state"] = L.TILE_VALID
        plain = eng.window(0, win["tasks"], win["succ"], tiles, win["ready"])
        eng.set_window_trace(True)
        traced = eng.window(0, win["tasks"], win["succ"], tiles, win["ready"])
        eng.set_window_trace(False)
        for w in (plain, traced):
            for _ in range(args.warmup):
                w.run()
        steps = {"untraced": [], "traced": []}
        for _ in range(args.runs):
            for name, w in (("untraced", plain), ("traced", traced)):
                st = w.run()
                assert st["body_errors"] == 0 and st["tasks_retired"] == len(win["tasks"])
                steps[name].append(st["reset_ms"] + st["kernel_ms"])
        tr = traced.trace()
        info = eng.info()
        for w in (plain, traced):
            w.close()

    t0, t1, sm = tr["t_start_ns"], tr["t_end_ns"], tr["smid"]
    assert np.all(t0 > 0) and np.all(t1 >= t0)
    span0, span1 = int(t0.min()), int(t1.max())
    busy = busy_fractions(t0, t1, sm, span0, span1)
    fr = np.array(sorted(busy.values()))
    doc = chrome_trace(t0, t1, sm, class_id=win["tasks"]["class_id"], locals=win["tasks"]["locals"],
                       class_names=CLASS_NAMES, unit=tr["unit"], process_name="cuda:0 Ex05 window (K=%d)" % K)
    with open(args.out, "w") as f:
        json.dump(doc, f)
    med = {k: float(np.median(v)) for k, v in steps.items()}
    summary = {
        "card": card(), "groups": K, "tasks": int(len(t0)), "entities": int(len(np.unique(tr["unit"]))),
        "workers": info["nworkers"], "sms_used": int(len(busy)), "sm_count": info["sm_count"],
        "step_ms_median": med, "step_ms_min_max": {k: [float(min(v)), float(max(v))] for k, v in steps.items()},
        "trace_cost_pct": 100.0 * (med["traced"] / med["untraced"] - 1.0),
        "span_us": (span1 - span0) / 1e3, "tail_us": (span1 - int(t0.max())) / 1e3,
        "busy_fraction": {"min": float(fr.min()), "median": float(np.median(fr)), "max": float(fr.max())},
        "busy_fraction_per_sm": {str(k): round(v, 4) for k, v in sorted(busy.items())},
        "trace": args.out,
    }
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
