"""Read groups of HBM windows: consecutive CHECK readers of one tile version run as one task that streams the tile once.
Every per-task output must be what the same window computes with groups off, and what the sequential oracle computes."""
import numpy as np
import pytest

from parsec_b200 import _lib as L
from oracle import orc
from oracle import orc_dags as dags
from parsec_b200.engine import Engine

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engines():
    on, off = Engine(0), Engine(0, read_groups=-1)
    yield on, off
    on.close()
    off.close()


def run_on(e, dag, host, valid):
    """One run of dag on engine e, tiles in a fresh slab (resident copies of host, or staged in from it)."""
    tb = dag.tile_bytes
    slot = (tb + 511) // 512 * 512
    slab = e.malloc(max(dag.ntiles * slot, 16))
    alias = e.host_register(host)
    tiles = np.zeros(dag.ntiles, L.TILE_DTYPE)
    tiles["dev_ptr"] = slab + np.arange(dag.ntiles, dtype=np.uint64) * np.uint64(slot)
    tiles["src_ptr"] = alias + np.arange(dag.ntiles, dtype=np.uint64) * np.uint64(tb)
    tiles["bytes"] = tb
    tiles["state"] = L.TILE_VALID if valid else L.TILE_INVALID
    if valid:
        for i in range(dag.ntiles):
            e.h2d(int(tiles["dev_ptr"][i]), host.view(np.uint8)[i * tb:(i + 1) * tb])
    w = e.window(0, dag.tasks, dag.succ, tiles, dag.ready)
    st = w.run()
    res = w.results()
    w.close()
    data = np.empty(dag.ntiles * tb, np.uint8)
    for i in range(dag.ntiles):
        e.d2h(data[i * tb:(i + 1) * tb], int(tiles["dev_ptr"][i]))
    e.host_unregister(host)
    e.free(slab)
    return st, res, data


def oracle(dag, host):
    """The sequential oracle's run of dag, every tile staged in from host."""
    spec = np.zeros(dag.ntiles, orc.TILE_DTYPE)
    spec["bytes"] = dag.tile_bytes
    spec["src_ptr"] = np.arange(dag.ntiles, dtype=np.uint64) * np.uint64(dag.tile_bytes)
    spec["state"] = orc.TILE_INVALID
    ref = orc.run_window(dag.tasks, dag.succ, spec, dag.ready, host.copy())
    assert ref["rc"] == 0
    return ref


def assert_same(a, b):
    (st_a, res_a, data_a), (st_b, res_b, data_b) = a, b
    assert np.array_equal(res_a["result"], res_b["result"])
    assert np.array_equal(res_a["seen_version"], res_b["seen_version"])
    assert np.array_equal(res_a["tiles"]["version"], res_b["tiles"]["version"])
    assert np.array_equal(res_a["tiles"]["state"], res_b["tiles"]["state"])
    assert np.array_equal(data_a, data_b)
    for k in ("tasks_retired", "bytes_h2d", "stage_ins", "body_errors"):
        assert st_a[k] == st_b[k], k


@pytest.mark.parametrize("valid", [False, True], ids=["staged", "resident"])
@pytest.mark.parametrize("K,NB,tile_bytes", [(8, 6, 4), (64, 14, 256 * 256 * 4), (33, 4, 1000), (1, 0, 16), (512, 14, 256 * 256 * 4)])
def test_ex05_groups_on_off_identical(engines, K, NB, tile_bytes, valid):
    on, off = engines
    dag = dags.ex05_broadcast(K, NB, tile_bytes)
    F = dag.meta["F"]
    host = np.full(K * tile_bytes // 4, -7, np.int32)
    a = run_on(on, dag, host, valid)
    b = run_on(off, dag, host, valid)
    assert_same(a, b)
    st, res, _ = a
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


def readers_dag(producer_body, producer_k, reader_ks, tile_bytes):
    """Task 0 writes tile 0 (FILL k / IOTA), tasks 1.. read it with CHECK constants reader_ks (ints: CHECK_I32, floats:
    CHECK_F32 with those bits)."""
    n = 1 + len(reader_ks)
    t = np.zeros(n, L.TASK_DTYPE)
    t["tile"][:] = -1
    t["nb_flows"] = 1
    t["tile"][:, 0] = 0
    t["body"][0], t["iparam"][0, 0], t["access"][0, 0] = producer_body, producer_k, L.ACCESS_WRITE
    for i, k in enumerate(reader_ks, start=1):
        t["access"][i, 0] = L.ACCESS_READ
        t["dep_goal"][i] = 1
        if isinstance(k, float):
            t["body"][i], t["fparam"][i] = L.BODY_CHECK_F32, np.float32(k)
        else:
            t["body"][i], t["iparam"][i, 0] = L.BODY_CHECK_I32, k
    t["succ_begin"][0], t["succ_count"][0] = 0, n - 1
    t["succ_begin"][1:] = n - 1
    succ = np.arange(1, n, dtype=np.uint32)
    return dags.Dag(t, succ, np.array([0], np.int32), ntiles=1, tile_bytes=tile_bytes, name="readers")


f5 = float(np.array([5], np.int32).view(np.float32)[0])     # a CHECK_F32 constant whose bits are the integer 5


@pytest.mark.parametrize("producer", ["fill5", "iota"])
@pytest.mark.parametrize("tile_bytes,part_bytes", [(4096 + 12, 0), (1 << 20, 64 * 1024)])
def test_mismatches_inside_a_group(producer, tile_bytes, part_bytes):
    """Members with different constants, some of which fail: per-member results and body_errors are the oracle's."""
    body, k = (L.BODY_FILL_I32, 5) if producer == "fill5" else (L.BODY_IOTA_I32, 0)
    dag = readers_dag(body, k, [5, 5, 6, f5, 0, 7, 1, 5], tile_bytes)
    host = np.zeros(tile_bytes // 4, np.int32)
    ref = oracle(dag, host)
    with Engine(0, part_bytes=part_bytes) as e:
        st, res, data = run_on(e, dag, host, False)
    assert np.array_equal(res["result"], ref["result"])
    assert np.array_equal(res["seen_version"], ref["seen_version"])
    assert st["body_errors"] == ref["stats"]["body_errors"] > 0
    assert np.array_equal(data, ref["device"][0][:tile_bytes])
    assert len(set(res["worker"][1:].tolist())) == 1                  # the eight readers ran as one group
    assert all(v == 0 for v in dags.check_execution(dag, res).values())


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
    host = np.arange(2 * 256, dtype=np.int32)
    ref = oracle(dag, host)
    for workers in (0, 1):
        with Engine(0, max_workers=workers) as e:
            st, res, data = run_on(e, dag, host, False)
        assert np.array_equal(res["result"], ref["result"])
        assert np.array_equal(res["seen_version"], ref["seen_version"])
        assert np.array_equal(data[1024:].view(np.int32), ref["device"][1].view(np.int32))
        assert st["body_errors"] == ref["stats"]["body_errors"] == 256
        assert all(v == 0 for v in dags.check_execution(dag, res).values())
        if workers == 1:
            assert np.array_equal(res["retire_order"], ref["retire_order"])
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
    ref = oracle(dag, host)
    with Engine(0, part_bytes=64 * 1024) as e:
        st, res, data = run_on(e, dag, host, False)
    assert st["bytes_h2d"] == tb == ref["stats"]["bytes_h2d"] and st["stage_ins"] == 1
    assert np.array_equal(res["result"], ref["result"])
    assert np.array_equal(res["seen_version"], ref["seen_version"])
    assert st["body_errors"] == ref["stats"]["body_errors"]
    assert len(set(res["worker"][1:].tolist())) == 1
    assert all(v == 0 for v in dags.check_execution(dag, res).values())
