"""Priority ready order (queue_policy 1 of the engine) on the CPU: the reference order of priority_order.py on a
hand-built DAG, its equivalence with the oracle's FIFO order when every priority is equal, the 16-lane quantisation of
the engine, and the replay of an order through the sequential oracle."""
import numpy as np
import pytest

from oracle import orc, orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200.engine import Engine
from priority_order import LANES, lane_of, priority_order, replay


def random_dag(n, seed, nprio, tile_bytes=64, ntiles=6, body_mix=(L.BODY_INCR_I32, L.BODY_SCALE_I32, L.BODY_ADD_IOTA_I32)):
    """A random DAG of HBM bodies: task j has up to three predecessors among the earlier tasks (counter mode), runs a
    read-modify-write body on one of `ntiles` tiles, and has one of `nprio` distinct priorities (spread out, negatives
    included)."""
    rng = np.random.default_rng(seed)
    t = dags._new_tasks(n)
    src, dst = [], []
    for j in range(1, n):
        for i in sorted(set(rng.integers(0, j, size=int(rng.integers(0, 4))).tolist())):
            src.append(i); dst.append(j)
    src, dst = np.array(src, np.int64), np.array(dst, np.int64)
    begin, count, succ = dags._csr_from_edges(n, src, dst, np.zeros(len(src), np.int64))
    t["succ_begin"], t["succ_count"] = begin, count
    t["dep_goal"] = np.bincount(dst, minlength=n)
    t["body"] = rng.choice(np.array(body_mix), n)
    t["nb_flows"] = 1
    t["tile"][:, 0] = rng.integers(0, ntiles, n)
    t["access"][:, 0] = L.ACCESS_RW
    t["iparam"][:, 0] = rng.integers(-5, 6, n)
    values = np.sort(rng.choice(np.arange(-1000, 1000), nprio, replace=False))
    t["priority"] = rng.choice(values, n)
    ready = np.flatnonzero(t["dep_goal"] == 0).astype(np.int32)
    rng.shuffle(ready)
    return dags.Dag(t, succ, ready, ntiles=ntiles, tile_bytes=tile_bytes, name="random")


def tiles_of(dag, state=orc.TILE_VALID):
    tiles = np.zeros(dag.ntiles, orc.TILE_DTYPE)
    tiles["bytes"] = dag.tile_bytes
    tiles["state"] = state
    tiles["src_ptr"] = np.arange(dag.ntiles, dtype=np.uint64) * np.uint64(dag.tile_bytes)
    return tiles


def fifo(dag, host=None, state=orc.TILE_VALID):
    """The oracle's own run, FIFO ready order (the engine's order with one worker and queue_policy 0)."""
    if host is None:
        host = np.zeros(max(dag.ntiles * dag.tile_bytes, 1), np.uint8)      # pushout flows write home
    out = orc.run_window(dag.tasks, dag.succ, tiles_of(dag, state), dag.ready, host)
    assert out["rc"] == 0
    return out


def walk(dag, retire_order):
    """Yield (picked task, tasks ready at that moment in readiness order) along a retire order, checking that it is a
    linear extension of the DAG (counter-mode dependencies)."""
    dep = dag.tasks["dep_goal"].astype(np.int64).copy()
    ready = list(dag.ready)
    for tid in retire_order:
        assert tid in ready, "task %d retired before it was ready" % tid
        yield tid, list(ready)
        ready.remove(tid)
        t = dag.tasks[tid]
        for s in dag.succ[t["succ_begin"]:t["succ_begin"] + t["succ_count"]]:
            sid = int(s & 0x07FFFFFF)
            dep[sid] -= 1
            if dep[sid] == 0:
                ready.append(sid)
    assert not ready


def test_exact_priority_order_on_a_hand_built_dag():
    """Higher priority first, FIFO among equal priorities: 1 (5) before 0 (1); its successors 4 and 5 (5, 5) in
    release order before 0; then 2 (9) before 3 (1)."""
    t = dags._new_tasks(6)
    t["priority"] = [1, 5, 9, 1, 5, 5]
    t["dep_goal"] = [0, 0, 1, 1, 1, 1]
    begin, count, succ = dags._csr_from_edges(6, [0, 0, 1, 1], [2, 3, 4, 5], [0, 0, 0, 0])
    t["succ_begin"], t["succ_count"] = begin, count
    dag = dags.Dag(t, succ, np.array([0, 1], np.int32), ntiles=0, tile_bytes=0)
    assert fifo(dag)["retire_order"].tolist() == [0, 1, 2, 3, 4, 5]
    assert priority_order(dag).tolist() == [1, 4, 5, 0, 2, 3]
    assert priority_order(dag, LANES).tolist() == [1, 4, 5, 0, 2, 3]


def test_lane_rule():
    assert lane_of([7, 3, 7, -2]).tolist() == [0, 1, 0, 2]                          # <= 16 distinct: the rank
    assert lane_of(np.arange(32)).tolist() == [15 - r // 2 for r in range(32)]       # 32 distinct: two per lane
    assert lane_of(np.arange(32), 0).tolist() == list(range(31, -1, -1))             # exact: the rank


@pytest.mark.parametrize("make", [lambda: dags.ex05_broadcast(32, 14, 64), lambda: dags.dtd_gemm(3, 16),
                                  lambda: random_dag(300, 1, 1), lambda: random_dag(500, 2, 1)])
def test_equal_priorities_give_the_fifo_order(make):
    """Also checks the readiness bookkeeping of priority_order (counter and mask modes) against the oracle's."""
    dag = make()
    dag.tasks["priority"] = 7
    order = fifo(dag)["retire_order"]
    assert np.array_equal(priority_order(dag), order)
    assert np.array_equal(priority_order(dag, LANES), order)


@pytest.mark.parametrize("seed,nprio", [(3, 2), (4, 9), (5, 16)])
def test_up_to_16_distinct_priorities_keep_the_exact_order(seed, nprio):
    dag = random_dag(400, seed, nprio)
    exact = priority_order(dag)
    assert np.array_equal(priority_order(dag, LANES), exact)
    assert not np.array_equal(exact, fifo(dag)["retire_order"])      # the policy changes the order at all


@pytest.mark.parametrize("seed,nprio", [(6, 17), (7, 40), (8, 300)])
def test_more_than_16_distinct_priorities_are_quantised_into_lanes(seed, nprio):
    """Every picked task is in the lowest lane among the ready tasks, and the first of that lane to become ready."""
    dag = random_dag(600, seed, nprio)
    lane = lane_of(dag.tasks["priority"])
    assert lane.max() == LANES - 1
    for tid, ready in walk(dag, priority_order(dag, LANES)):
        low = min(lane[r] for r in ready)
        assert lane[tid] == low and tid == next(r for r in ready if lane[r] == low)


def test_exact_order_is_a_linear_extension_by_priority():
    dag = random_dag(400, 9, 300)
    prio = dag.tasks["priority"]
    for tid, ready in walk(dag, priority_order(dag)):
        assert prio[tid] == max(prio[r] for r in ready)


@pytest.mark.parametrize("make", [lambda: random_dag(300, 10, 5, tile_bytes=256), lambda: dags.dtd_gemm(3, 16)])
def test_replay_of_the_fifo_order_is_the_oracle_run(make):
    """replay() runs an order task by task through the oracle: on the FIFO order it gives what one oracle run gives,
    stage-ins from host memory and pushouts included."""
    dag = make()
    host = np.random.default_rng(3).integers(0, 255, max(dag.ntiles * dag.tile_bytes, 1), dtype=np.uint8)
    h1, h2 = host.copy(), host.copy()
    ref = fifo(dag, h1, orc.TILE_INVALID)
    got = replay(dag, ref["retire_order"], tiles_of(dag, orc.TILE_INVALID), h2)
    for k in ("start_seq", "end_seq", "seen_version", "result"):
        assert np.array_equal(got[k], ref[k]), k
    assert got["stats"] == ref["stats"]
    assert np.array_equal(got["tiles"]["version"], ref["tiles"]["version"])
    assert np.array_equal(np.concatenate(got["device"]), np.concatenate(ref["device"]))
    assert np.array_equal(h1, h2)


def test_unknown_queue_policy_is_refused():
    """Only 0 (FIFO) and 1 (priority) exist; the check comes before any device work."""
    with pytest.raises(L.Pb2Error) as ei:
        Engine(0, queue_policy=2)
    assert ei.value.rc == L.PB2_ERR_BAD_PARAM
