"""Read groups of HBM windows: consecutive CHECK readers of one tile version run as one task that streams the tile once.
Every per-task output must be what the same window computes with groups off, and what the sequential oracle computes."""
import numpy as np
import pytest

from parsec_b200 import _lib as L
from oracle import orc_dags as dags
from parsec_b200.engine import Engine
from window_harness import KS, Layout, assert_like_oracle, assert_same_run, readers_dag, run_engine, run_oracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engines():
    with Engine(0) as on, Engine(0, read_groups=-1) as off:
        yield on, off


@pytest.mark.parametrize("valid", [False, True], ids=["staged", "resident"])
@pytest.mark.parametrize("K,NB,tile_bytes", [(8, 6, 4), (64, 14, 256 * 256 * 4), (33, 4, 1000), (1, 0, 16), (512, 14, 256 * 256 * 4)])
def test_ex05_groups_on_off_identical(engines, K, NB, tile_bytes, valid):
    on, off = engines
    dag = dags.ex05_broadcast(K, NB, tile_bytes)
    F = dag.meta["F"]
    layout = Layout.packed(dag, np.full(K * tile_bytes // 4, -7, np.int32), valid)
    a = run_engine(on, dag, layout)
    assert_same_run(a, run_engine(off, dag, layout))
    st, res = a.stats, a.res
    assert st["tasks_retired"] == dag.ntasks and st["body_errors"] == 0
    assert all(v == 0 for v in dags.check_execution(dag, res).values())
    if not valid:
        assert st["bytes_h2d"] == K * tile_bytes and st["stage_ins"] == K
    assert np.array_equal(res["result"][K:], np.repeat(np.arange(K, dtype=np.uint64), F))   # 0 mismatches, first element k
    if F >= 2:                                  # one group per k: one worker, consecutive start events
        wk = res["worker"][K:].reshape(K, F)
        ss = res["start_seq"][K:].reshape(K, F).astype(np.int64)
        assert np.all(wk == wk[:, :1])
        assert np.all(np.diff(ss, axis=1) == 1)


@pytest.mark.parametrize("producer", ["fill5", "iota"])
@pytest.mark.parametrize("tile_bytes,part_bytes", [(4096 + 12, 0), (1 << 20, 64 * 1024)])
def test_mismatches_inside_a_group(producer, tile_bytes, part_bytes):
    """Members with different constants, some of which fail: per-member results and body_errors are the oracle's."""
    body, k = (L.BODY_FILL_I32, 5) if producer == "fill5" else (L.BODY_IOTA_I32, 0)
    dag = readers_dag(body, k, KS, tile_bytes)
    layout = Layout.packed(dag, np.zeros(tile_bytes // 4, np.int32))
    ref = run_oracle(dag, layout)
    with Engine(0, part_bytes=part_bytes) as e:
        run = run_engine(e, dag, layout)
    assert_like_oracle(run, ref, dag)
    assert run.stats["body_errors"] > 0
    assert len(set(run.res["worker"][1:].tolist())) == 1              # the eight readers ran as one group


def broken_runs_dag(mask):
    """P fills tile 0; its out-edges are [R1, R2, X, R3, R4] with X a NOP (not a reader): groups {R1, R2}, {R3, R4}.
    R2 has a successor of its own, S (INCR on tile 1).  Counter or mask dependency words."""
    P, R1, R2, X, R3, R4, S = range(7)
    t = np.zeros(7, L.TASK_DTYPE)
    t["tile"][:] = -1
    t["nb_flows"] = 1
    t["tile"][:, 0] = 0
    t["body"][P], t["iparam"][P, 0], t["access"][P, 0] = L.BODY_FILL_I32, 9, L.ACCESS_WRITE
    for r, k in ((R1, 9), (R2, 9), (R3, 9), (R4, 8)):
        t["body"][r], t["iparam"][r, 0], t["access"][r, 0] = L.BODY_CHECK_I32, k, L.ACCESS_READ
    t["body"][X], t["nb_flows"][X], t["tile"][X, 0] = L.BODY_NOP, 0, -1
    t["body"][S], t["iparam"][S, 0], t["tile"][S, 0], t["access"][S, 0] = L.BODY_INCR_I32, 3, 1, L.ACCESS_RW
    src = [P, P, P, P, P, R2]
    dst = [R1, R2, X, R3, R4, S]
    begin, count, succ = dags._csr_from_edges(7, src, dst, np.zeros(6, np.int64))
    t["succ_begin"], t["succ_count"] = begin, count
    if mask:
        t["flags"] = L.TASK_DEPS_MASK
        t["dep_goal"] = 0x1
    else:
        t["dep_goal"] = 1
    t["dep_goal"][P] = 0
    return dags.Dag(t, succ, np.array([P], np.int32), ntiles=2, tile_bytes=1024, name="broken_runs")


@pytest.mark.parametrize("mask", [False, True], ids=["counter", "mask"])
def test_runs_broken_by_other_successors(mask):
    dag = broken_runs_dag(mask)
    layout = Layout.packed(dag, np.arange(2 * 256, dtype=np.int32))
    ref = run_oracle(dag, layout)
    for workers in (0, 1):
        with Engine(0, max_workers=workers) as e:
            run = run_engine(e, dag, layout)
        assert_like_oracle(run, ref, dag)
        assert run.stats["body_errors"] == 256
        res = run.res
        if workers == 1:
            assert np.array_equal(res["retire_order"], ref.res["retire_order"])
        ss = res["start_seq"].astype(np.int64)
        assert res["worker"][1] == res["worker"][2] and ss[2] == ss[1] + 1            # {R1, R2}
        assert res["worker"][4] == res["worker"][5] and ss[5] == ss[4] + 1            # {R3, R4}


def test_wide_invalid_tile_staged_once_for_a_group():
    """A 1 MiB INVALID tile read by a group of 8 in 64 KiB parts: staged once, slice by slice; results exact."""
    tb = 1 << 20
    t = np.zeros(8, L.TASK_DTYPE)
    t["tile"][:] = -1
    t["nb_flows"] = 1
    t["tile"][:, 0] = 0
    t["body"] = L.BODY_CHECK_I32
    t["access"][:, 0] = L.ACCESS_READ
    t["iparam"][:, 0] = [4, 4, 4, 3, 4, 4, 4, 4]
    # a CTL root (NOP, no flows) releases the eight readers, so they form one group
    root = np.zeros(1, L.TASK_DTYPE)
    root["tile"][:] = -1
    t = np.concatenate([root, t])
    t["dep_goal"][1:] = 1
    t["succ_begin"][0], t["succ_count"][0] = 0, 8
    t["succ_begin"][1:] = 8
    dag = dags.Dag(t, np.arange(1, 9, dtype=np.uint32), np.array([0], np.int32), ntiles=1, tile_bytes=tb, name="wide")
    host = np.full(tb // 4, 4, np.int32)
    host[12345] = 0
    layout = Layout.packed(dag, host)
    ref = run_oracle(dag, layout)
    with Engine(0, part_bytes=64 * 1024) as e:
        run = run_engine(e, dag, layout)
    assert_like_oracle(run, ref, dag)
    assert run.stats["bytes_h2d"] == tb and run.stats["stage_ins"] == 1
    assert len(set(run.res["worker"][1:].tolist())) == 1
