"""Reference of the priority ready order (the engine's queue_policy 1), for the tests.

The order is what the reference's device module does with its pending list (parsec_list_push_sorted,
device_gpu.c:2169-2174): the ready task with the highest priority first, FIFO among equal priorities.  With `lanes` > 0
the priorities are first quantised the way the engine's windows do it (include/pb2_engine.h, queue_policy): the distinct
priorities of the window ranked highest first, rank r -> lane r when there are at most `lanes` of them, else
floor(r * lanes / ndistinct); then the lowest lane first, FIFO within a lane.  The engine's host code implements the
same rule a second time (task_priority_lanes in pb2_window_plan.cpp); this one is what the tests compare it against.

`replay` executes a given order with the sequential oracle (oracle/orc.py, one single-task window per task, tiles and
their bytes carried from one to the next), so bodies, stage-in, versions and pushout follow the oracle's rules."""
import numpy as np

from oracle import orc

LANES = 16


def lane_of(priority, lanes=LANES):
    """Key of every task, smaller first: its priority's rank among the distinct priorities (highest first), quantised
    into `lanes` lanes when there are more distinct priorities than lanes; lanes = 0: the exact rank."""
    priority = np.asarray(priority)
    values = np.unique(priority)[::-1]
    rank = np.searchsorted(-values, -priority)
    return rank if lanes == 0 or len(values) <= lanes else rank * lanes // len(values)


def priority_order(dag, lanes=0):
    """Retire order of one worker that always takes the first-ready task of the smallest key (lane_of).  Dependency
    words follow the oracle: counter mode counts down to 0, mask mode ORs the destination flow bits up to the goal."""
    t = dag.tasks
    key = lane_of(t["priority"], lanes)
    mask = (t["flags"] & orc.TASK_DEPS_MASK) != 0
    dep = np.where(mask, 0, t["dep_goal"]).astype(np.int64)
    goal = t["dep_goal"].astype(np.int64)
    ready = [int(i) for i in dag.ready]
    order = []
    while ready:
        best = min(range(len(ready)), key=lambda j: (key[ready[j]], j))
        tid = ready.pop(best)
        order.append(tid)
        b, c = int(t["succ_begin"][tid]), int(t["succ_count"][tid])
        for s in dag.succ[b:b + c]:
            sid, flow = int(s & 0x07FFFFFF), int(s >> 27)
            if mask[sid]:
                old = dep[sid]
                dep[sid] = old | (1 << flow)
                now = (dep[sid] & goal[sid]) == goal[sid] and (old & goal[sid]) != goal[sid]
            else:
                dep[sid] -= 1
                now = dep[sid] == 0
            if now:
                ready.append(sid)
    assert len(order) == len(t), "the DAG deadlocks"
    return np.array(order, np.int32)


def replay(dag, order, tiles_spec, host=None):
    """Run the tasks one after the other in `order` through the oracle.  tiles_spec as orc.run_window takes it
    (src_ptr: byte offset of the tile's home in `host`, modified in place by pushout).  Returns the outputs of
    orc.run_window for the whole window: retire_order, start_seq / end_seq (two events per task), seen_version,
    result, stats, tiles (final descriptors) and device (final tile bytes)."""
    tiles = np.array(tiles_spec, dtype=orc.TILE_DTYPE, copy=True)
    dev = [np.zeros(max(int(b), 1), np.uint8) for b in tiles["bytes"]]
    host_u8 = host.view(np.uint8).reshape(-1) if host is not None else None
    for i in range(len(tiles)):
        off = int(tiles["src_ptr"][i])
        tiles["dev_ptr"][i] = dev[i].ctypes.data
        tiles["src_ptr"][i] = (host_u8.ctypes.data + off) if host_u8 is not None else 0
    n = dag.ntasks
    out = {"retire_order": np.asarray(order, np.int32), "start_seq": np.zeros(n, np.uint32), "end_seq": np.zeros(n, np.uint32),
           "seen_version": np.zeros((n, 4), np.uint32), "result": np.zeros(n, np.uint64)}
    stats = {}
    for step, tid in enumerate(order):
        one = dag.tasks[tid:tid + 1].copy()
        one["succ_begin"], one["succ_count"], one["dep_goal"], one["flags"] = 0, 0, 0, 0
        r = orc.run_window_raw(one, np.zeros(0, np.uint32), tiles, np.zeros(1, np.int32))
        assert r["rc"] == 0
        tiles = r["tiles"]
        out["start_seq"][tid], out["end_seq"][tid] = 2 * step, 2 * step + 1
        out["seen_version"][tid] = r["seen_version"][0]
        out["result"][tid] = r["result"][0]
        for k, v in r["stats"].items():
            stats[k] = stats.get(k, 0) + v
    out.update(stats=stats, tiles=tiles, device=dev, rc=0)
    return out
