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

pytestmark = pytest.mark.gpu

RUNS = 6
STATS = ("tasks_retired", "bytes_h2d", "bytes_d2d", "bytes_d2h", "stage_ins", "body_errors")


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


def host_data(dag):
    if "host" in dag.meta:
        return dag.meta["host"].copy()
    host = np.full(dag.ntiles * dag.tile_bytes // 4, 4, np.int32)
    host[::977] = 0
    return host


def tile_table(e, dag, host, staged):
    tb = dag.tile_bytes
    slot = (tb + 511) // 512 * 512
    slab = e.malloc(max(dag.ntiles * slot, 16))
    tiles = np.zeros(dag.ntiles, L.TILE_DTYPE)
    tiles["dev_ptr"] = slab + np.arange(dag.ntiles, dtype=np.uint64) * np.uint64(slot)
    tiles["src_ptr"] = e.host_register(host) + np.arange(dag.ntiles, dtype=np.uint64) * np.uint64(tb)
    tiles["bytes"] = tb
    tiles["state"] = L.TILE_INVALID if staged else L.TILE_VALID
    if not staged:
        for i in range(dag.ntiles):
            e.h2d(int(tiles["dev_ptr"][i]), host.view(np.uint8)[i * tb:(i + 1) * tb])
    return tiles, slab


def oracle(dag, host, staged):
    spec = np.zeros(dag.ntiles, orc.TILE_DTYPE)
    spec["bytes"] = dag.tile_bytes
    spec["src_ptr"] = np.arange(dag.ntiles, dtype=np.uint64) * np.uint64(dag.tile_bytes)
    spec["state"] = orc.TILE_INVALID if staged else orc.TILE_VALID
    ref = orc.run_window(dag.tasks, dag.succ, spec, dag.ready, host.copy())
    assert ref["rc"] == 0
    return ref


def assert_run_matches(dag, st, res, first, ref, exact_order):
    st0, res0 = first
    for k in STATS:
        assert st[k] == st0[k], k
    assert st["tasks_retired"] == dag.ntasks
    assert st["bytes_h2d"] == ref["stats"]["bytes_h2d"] and st["body_errors"] == ref["stats"]["body_errors"]
    assert np.array_equal(res["result"], res0["result"]) and np.array_equal(res["result"], ref["result"])
    assert np.array_equal(res["seen_version"], res0["seen_version"]) and np.array_equal(res["seen_version"], ref["seen_version"])
    assert res["tiles"].tobytes() == res0["tiles"].tobytes()
    assert np.array_equal(res["tiles"]["version"], ref["tiles"]["version"])
    assert np.array_equal(res["tiles"]["state"], ref["tiles"]["state"])
    assert all(v == 0 for v in dags.check_execution(dag, res).values())
    if exact_order:
        for key in ("retire_order", "start_seq", "end_seq", "worker"):
            assert np.array_equal(res[key], res0[key]), key
        assert np.array_equal(res["retire_order"], ref["retire_order"])


@pytest.mark.parametrize("wait_between", [True, False], ids=["wait_each", "queued"])
@pytest.mark.parametrize("name,engine_kw,make_dag,staged", CASES, ids=[c[0] for c in CASES])
def test_every_run_matches_a_fresh_window(name, engine_kw, make_dag, staged, wait_between):
    dag = make_dag()
    host = host_data(dag)
    ref = oracle(dag, host, staged)
    with Engine(0, **engine_kw) as e:
        tiles, slab = tile_table(e, dag, host, staged)
        fresh = e.window(dag.kind, dag.tasks, dag.succ, tiles, dag.ready)
        first = (fresh.run(), fresh.results())
        fresh.close()
        exact = engine_kw.get("max_workers") == 1
        assert_run_matches(dag, *first, first, ref, exact)
        w = e.window(dag.kind, dag.tasks, dag.succ, tiles, dag.ready)
        if wait_between:
            for _ in range(RUNS):
                st = w.run()
                assert_run_matches(dag, st, w.results(), first, ref, exact)
        else:
            # launches queued back to back: each run starts from the copy the run before it armed
            for _ in range(RUNS):
                w.launch()
            assert_run_matches(dag, w.wait(), w.results(), first, ref, exact)
        w.close()
        e.host_unregister(host)
        e.free(slab)
