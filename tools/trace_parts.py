"""Where the SMs' time goes inside a window: part records (pb2_window_part_trace) of three windows.

  ex05_resident   the resident Ex05 window bench.py times (the stand-alone runtime's Ex05 pool, K groups, fan-out
                  NB // 2 + 1, as its device module would build the window; tiles VALID in HBM), as tools/trace_window.py
                  builds it;
  ex05_host_fed   the same window with every tile INVALID and its home in pinned host memory: each run stages the
                  tiles in over PCIe inside the kernel;
  gemm            the configs[2] GEMM window of bench.py (DTD tile GEMM, NT = 32, 512 x 512 bf16 tiles, C resident).
                  Its operands are small random bf16 values, not bench.py's LCG data: the run is timed, not checked.

Each window is created twice on one engine, with window trace off and on; both are warmed up and then alternated run by
run, and the medians of their steps (reset_ms + kernel_ms) are printed side by side: the difference is the cost of
tracing.  From the last traced run, per SM, over the span from the first pop to the last retirement:
  - movein / exec / moveout: the SM's worker time in each phase of the part records (t_pop..t_in, t_in..t_exec,
    t_exec..t_out) over its worker time, the span times the window's workers per SM; idle is the rest;
  - entity_busy: what tools/trace_window.py reports from the window trace, the union of the intervals of the entities
    the SM retired, over the span.  It gives every part of an entity to the SM that retired it.
The summary line of each window gives min / median / max over the SMs; --out gets the per-SM figures and, with
--chrome, Chrome traces of the part records.  The card's name, power limit and SM clock are read in the same run.

    python tools/trace_parts.py --runs 20 --out trace_parts.json
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from trace_window import busy_fractions  # noqa: E402

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


def phase_shares(rec, span0, span1, workers_per_sm):
    """Per SM: {movein, exec, moveout, idle} as shares of its worker time over [span0, span1]."""
    t = [rec[k].astype(np.int64) for k in ("t_pop_ns", "t_in_ns", "t_exec_ns", "t_out_ns")]
    out = {}
    denom = max(1, span1 - span0) * workers_per_sm
    for s in np.unique(rec["smid"]):
        sel = rec["smid"] == s
        sh = {name: float((t[i + 1][sel] - t[i][sel]).sum()) / denom
              for i, name in enumerate(("movein", "exec", "moveout"))}
        sh["idle"] = 1.0 - sum(sh.values())
        out[int(s)] = sh
    return out


def stats(values):
    v = np.array(sorted(values))
    return {"min": round(float(v.min()), 4), "median": round(float(np.median(v)), 4), "max": round(float(v.max()), 4)}


def measure(eng, name, kind, tasks, succ, tiles, ready, args, class_id=None):
    """Alternated untraced / traced runs of one window; the summary of the last traced run."""
    from parsec_b200.engine import chrome_trace_parts
    plain = eng.window(kind, tasks, succ, tiles, ready)
    eng.set_window_trace(True)
    traced = eng.window(kind, tasks, succ, tiles, ready)
    eng.set_window_trace(False)
    for w in (plain, traced):
        for _ in range(args.warmup):
            w.run()
    steps = {"untraced": [], "traced": []}
    for _ in range(args.runs):
        for which, w in (("untraced", plain), ("traced", traced)):
            st = w.run()
            assert st["tasks_retired"] == len(tasks)
            steps[which].append(st["reset_ms"] + st["kernel_ms"])
    tr, rec, st = traced.trace(), traced.part_trace(), traced.stats
    for w in (plain, traced):
        w.close()
    info = eng.info()
    assert np.all(rec["t_pop_ns"] > 0)
    assert int(rec["in_bytes"].sum()) == st["bytes_h2d"] + st["bytes_d2d"]
    span0, span1 = int(tr["t_start_ns"].min()), int(tr["t_end_ns"].max())
    nworkers = info["nworkers_gemm"] if kind == 1 else info["nworkers"]
    per_sm = nworkers / info["sm_count"]
    shares = phase_shares(rec, span0, span1, per_sm)
    busy = busy_fractions(tr["t_start_ns"], tr["t_end_ns"], tr["smid"], span0, span1)
    med = {k: float(np.median(v)) for k, v in steps.items()}
    summary = {
        "window": name, "tasks": int(len(tasks)), "entities": int(len(np.unique(tr["unit"]))), "parts": int(len(rec)),
        "workers": nworkers, "workers_per_sm": per_sm, "sms_used": int(len(shares)),
        "step_ms_median": med, "step_ms_min_max": {k: [float(min(v)), float(max(v))] for k, v in steps.items()},
        "trace_cost_pct": 100.0 * (med["traced"] / med["untraced"] - 1.0),
        "span_us": (span1 - span0) / 1e3, "bytes_in": int(rec["in_bytes"].sum()), "bytes_out": int(rec["out_bytes"].sum()),
        "parts_waited_input": int(np.sum((rec["flags"] & 1) != 0)),
        "per_sm_share": {k: stats([s[k] for s in shares.values()]) for k in ("movein", "exec", "moveout", "idle")},
        "per_sm_entity_busy": stats(busy.values()),
    }
    detail = {"per_sm": {str(s): dict({k: round(v, 4) for k, v in shares[s].items()}, entity_busy=round(busy.get(s, 0.0), 4))
                         for s in sorted(shares)}}
    if args.chrome:
        path = "%s_%s.json" % (os.path.splitext(args.out)[0], name)
        with open(path, "w") as f:
            json.dump(chrome_trace_parts(rec, class_id=class_id, class_names=CLASS_NAMES if class_id is not None else None,
                                         process_name="cuda:0 %s" % name), f)
        summary["chrome"] = path
    return summary, detail


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=4096, help="Ex05 broadcast groups (bench.py's K)")
    ap.add_argument("--gemm-nt", type=int, default=32, help="tiles per side of the GEMM window (bench.py's NT)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=20, help="timed runs of each window, alternated")
    ap.add_argument("--out", default="trace_parts.json", help="per-SM figures of every window")
    ap.add_argument("--chrome", action="store_true", help="also write a Chrome trace of each window's part records")
    ap.add_argument("--only", default="", help="comma-separated subset of ex05_resident, ex05_host_fed, gemm")
    args = ap.parse_args()
    only = set(args.only.split(",")) if args.only else {"ex05_resident", "ex05_host_fed", "gemm"}

    from oracle import orc_dags as dags
    from parsec_b200 import _lib as L
    from parsec_b200 import runtime as R
    from parsec_b200.engine import Engine

    print("card:", card(), flush=True)
    out = {"card": card(), "windows": {}}
    K = args.groups
    if only & {"ex05_resident", "ex05_host_fed"}:
        host = np.zeros(K * TILE // 4, np.int32)
        ctx = R.Context(nb_cores=os.cpu_count() or 1, cuda_devices=(0,))
        dc = ctx.block_cyclic(4, TILE // 4, 1, K * TILE // 4, 1, mat=host)
        assert ctx.l.pb2_dc_register_memory(dc, ctx.devices[0]) == 0
        tp = C.c_void_p(ctx.l.pb2_ptg_ex05_broadcast_new(ctx.h, dc, K, NB))
        win = ctx.export_window(tp, ctx.devices[0])
        assert len(win["tasks"]) == K * (1 + F)
        with Engine(0) as eng:
            slab = eng.malloc(K * TILE)
            eng.h2d(slab, host)
            tiles = win["tiles"].copy()
            order = np.argsort(tiles["src_ptr"])
            tiles["dev_ptr"][order] = slab + np.arange(K, dtype=np.uint64) * np.uint64(TILE)
            cases = []
            if "ex05_resident" in only:
                t = tiles.copy()
                t["state"] = L.TILE_VALID
                cases.append(("ex05_resident", t))
            if "ex05_host_fed" in only:
                pinned = np.zeros(K * TILE // 4, np.int32)
                alias = eng.host_register(pinned)
                t = tiles.copy()
                t["src_ptr"][order] = alias + np.arange(K, dtype=np.uint64) * np.uint64(TILE)
                t["state"] = L.TILE_INVALID
                cases.append(("ex05_host_fed", t))
            for name, t in cases:
                s, d = measure(eng, name, 0, win["tasks"], win["succ"], t, win["ready"], args, win["tasks"]["class_id"])
                print(json.dumps(s), flush=True)
                out["windows"][name] = dict(s, **d)
            if "ex05_host_fed" in only:
                eng.host_unregister(pinned)
            eng.free(slab)
    if "gemm" in only:
        NT, T = args.gemm_nt, 512
        tb = T * T * 2
        dag = dags.dtd_gemm(NT, T)
        dag.tasks["access"][:, 2] &= ~np.uint8(L.FLOW_PUSHOUT)             # device-resident: C stays in HBM
        rng = np.random.default_rng(0)
        bits = (rng.integers(-64, 64, dag.ntiles * tb // 2) * 0x10 + 0x3C00).astype(np.uint16)   # small bf16 values
        with Engine(0) as eng:
            slab = eng.malloc(dag.ntiles * tb)
            eng.h2d(slab, bits)
            tiles = np.zeros(dag.ntiles, L.TILE_DTYPE)
            tiles["dev_ptr"] = slab + np.arange(dag.ntiles, dtype=np.uint64) * np.uint64(tb)
            tiles["bytes"], tiles["state"] = tb, L.TILE_VALID
            s, d = measure(eng, "gemm", 1, dag.tasks, dag.succ, tiles, dag.ready, args)
            print(json.dumps(s), flush=True)
            out["windows"]["gemm"] = dict(s, **d)
            eng.free(slab)
    with open(args.out, "w") as f:
        json.dump(out, f)


if __name__ == "__main__":
    main()
