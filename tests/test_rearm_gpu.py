"""One window launched many times.  Consecutive runs of a non-shared HBM window alternate between two copies of its
per-run state, and while a run runs the reset kernel arms the other copy for the next run on a stream of its own, so
from the third launch on no reset kernel runs in front of a run.  A GEMM window keeps one copy, unit words included,
and re-arms it in front of every run.  Every run must compute exactly what a fresh window's first run computes, and
what the sequential oracle computes: retire log, start / end events, seen versions, results, tile table and
statistics."""
import numpy as np
import pytest

from parsec_b200 import _lib as L
from oracle import orc
from oracle import orc_dags as dags
from parsec_b200.engine import Engine
from window_harness import Layout, assert_like_oracle, assert_same_run, placed, run_oracle

pytestmark = pytest.mark.gpu

RUNS = 6


def counter_mode(dag):
    """The same DAG with counter dependency words (every task has one in-edge or none, and no other flag)."""
    t = dag.tasks.copy()
    t["flags"] = 0
    t["dep_goal"] = np.where(t["dep_goal"] != 0, 1, 0)
    return dags.Dag(t, dag.succ, dag.ready, ntiles=dag.ntiles, tile_bytes=dag.tile_bytes, name=dag.name + "_counter")


def wide_group_dag(tb=1 << 20):
    """A NOP root releases eight CHECK readers of one tile, one of which fails: a read group of wide, multi-part CHECKs."""
    t = np.zeros(9, L.TASK_DTYPE)
    t["tile"][:] = -1
    t["nb_flows"][1:] = 1
    t["tile"][1:, 0] = 0
    t["body"][1:] = L.BODY_CHECK_I32
    t["access"][1:, 0] = L.ACCESS_READ
    t["iparam"][1:, 0] = [4, 4, 4, 3, 4, 4, 4, 4]
    t["dep_goal"][1:] = 1
    t["succ_begin"][0], t["succ_count"][0] = 0, 8
    t["succ_begin"][1:] = 8
    return dags.Dag(t, np.arange(1, 9, dtype=np.uint32), np.array([0], np.int32), ntiles=1, tile_bytes=tb, name="wide")


def gemm_chains_dag():
    """A GEMM window over tiles of 256 x 256 bf16: two k-chains C0 = A0 B0 + A1 B1 and C1 = A0 B1 + A1 B0 (units of two
    parts), CHECKs of C0 and C1, and INCR, COPY, SCALE and CHECKs of two integer tiles X and Y around them.  A holds
    1.0 and B 1 / 256, so every GEMM adds exactly 1.0 to each element of C.  DTD dependency words; tiles A0 A1 B0 B1 C0
    C1 X Y."""
    T = 256
    A0, A1, B0, B1, C0, C1, X, Y = range(8)
    R, W = L.ACCESS_READ, L.ACCESS_RW
    gemm = lambda a, b, c: (L.BODY_GEMM_BF16, [(a, R), (b, R), (c, W)], (T, T, T))
    rows = [(L.BODY_INCR_I32, [(X, W)], (1, 0, 0)), gemm(A0, B0, C0), gemm(A1, B1, C0), gemm(A0, B1, C1),
            gemm(A1, B0, C1), (L.BODY_CHECK_I32, [(C0, R)], (0x40004000, 0, 0)),
            (L.BODY_CHECK_I32, [(C1, R)], (0x40004000, 0, 0)), (L.BODY_COPY, [(X, R), (Y, W)], (0, 0, 0)),
            (L.BODY_CHECK_I32, [(X, R)], (5, 0, 0)), (L.BODY_SCALE_I32, [(Y, W)], (3, 0, 0)),
            (L.BODY_CHECK_I32, [(Y, R)], (15, 0, 0))]
    n = len(rows)
    t = np.zeros(n, L.TASK_DTYPE)
    t["tile"][:] = -1
    ft, fo = np.full((n, 4), -1, np.int32), np.zeros((n, 4), np.int32)
    for i, (body, flows, ip) in enumerate(rows):
        t["body"][i], t["nb_flows"][i], t["iparam"][i] = body, len(flows), ip
        for f, (tile, acc) in enumerate(flows):
            t["tile"][i, f], t["access"][i, f] = tile, acc
            ft[i, f], fo[i, f] = tile, orc.DTD_INPUT if acc == R else orc.DTD_INOUT
    t["priority"] = [2, 0, 0, 3, 3, 1, 1, 2, 0, 1, 0]
    src, dst, flow, dep = orc.dtd_build(t["nb_flows"].astype(np.int32), ft, fo, 8)
    begin, count, succ = dags._csr_from_edges(n, src, dst, flow)
    t["succ_begin"], t["succ_count"], t["dep_goal"] = begin, count, dep
    tb = T * T * 2
    host = np.zeros((8, tb // 4), np.uint32)
    host[[A0, A1]] = 0x3F803F80                                  # bf16 1.0
    host[[B0, B1]] = 0x3B803B80                                  # bf16 1 / 256
    host[[X, Y]] = 4
    host[X:].reshape(-1)[::977] = 0
    return dags.Dag(t, succ, np.nonzero(dep == 0)[0].astype(np.int32), ntiles=8, tile_bytes=tb, kind=1,
                    name="gemm_chains", meta={"host": host.view(np.int32).reshape(-1)})


TB = 256 * 1024
# (id, engine keywords, dag, tiles staged in from host memory every run)
CASES = [
    ("ex05_fused_resident", {}, lambda: dags.ex05_broadcast(64, 14, TB), False),
    ("ex05_fused_staged", {}, lambda: dags.ex05_broadcast(64, 14, TB), True),
    ("ex05_groups_unfused", {"fuse_readers": -1}, lambda: dags.ex05_broadcast(64, 14, TB), True),
    ("ex05_queue_policy_1", {"queue_policy": 1}, lambda: dags.ex05_broadcast(64, 14, TB), True),
    ("ex05_counter_words", {}, lambda: counter_mode(dags.ex05_broadcast(64, 14, TB)), True),
    ("wide_check_parts", {"part_bytes": 64 * 1024}, wide_group_dag, True),
    ("chain_one_worker", {"max_workers": 1}, lambda: dags.ex02_chain(40), False),
    ("gemm_chains_wide_parts", {"part_bytes": 32 * 1024}, gemm_chains_dag, True),
    ("gemm_chains_wide_parts_queue_policy_1", {"part_bytes": 32 * 1024, "queue_policy": 1}, gemm_chains_dag, True),
]


@pytest.mark.parametrize("wait_between", [True, False], ids=["wait_each", "queued"])
@pytest.mark.parametrize("name,engine_kw,make_dag,staged", CASES, ids=[c[0] for c in CASES])
def test_every_run_matches_a_fresh_window(name, engine_kw, make_dag, staged, wait_between):
    dag = make_dag()
    if "host" in dag.meta:
        host = dag.meta["host"]
    else:
        host = np.full(dag.ntiles * dag.tile_bytes // 4, 4, np.int32)
        host[::977] = 0
    layout = Layout.packed(dag, host, valid=not staged)
    with Engine(0, **engine_kw) as e, placed(e, layout) as p:
        fresh = e.window(dag.kind, dag.tasks, dag.succ, p.tiles, dag.ready)
        try:
            runs = [p.run(fresh.run(), fresh.results())]
        finally:
            fresh.close()
        w = e.window(dag.kind, dag.tasks, dag.succ, p.tiles, dag.ready)
        try:
            if wait_between:
                for _ in range(RUNS):
                    runs.append(p.run(w.run(), w.results()))
            else:
                # launches queued back to back: each run starts from the copy the run before it armed
                for _ in range(RUNS):
                    w.launch()
                runs.append(p.run(w.wait(), w.results()))
        finally:
            w.close()
    ref = run_oracle(dag, layout)
    for run in runs:
        assert_same_run(run, runs[0])
        assert_like_oracle(run, ref, dag)
        if engine_kw.get("max_workers") == 1:
            for key in ("retire_order", "start_seq", "end_seq", "worker"):
                assert np.array_equal(run.res[key], runs[0].res[key]), key
            assert np.array_equal(run.res["retire_order"], ref.res["retire_order"])
