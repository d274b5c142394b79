"""Fused units of HBM windows: a producer and the read group that checks the tile it writes run as one unit, chunk by
chunk.  Every per-task output must be what the same window computes with fusion off, and what the sequential oracle
computes; the dependency order must hold on every edge."""
import numpy as np
import pytest

from parsec_b200 import _lib as L
from oracle import orc_dags as dags
from parsec_b200.engine import Engine
from window_harness import (KS, Layout, assert_like_oracle, assert_same_run, check_pair, engines, fused,  # noqa: F401
                            not_fused, readers_dag, run_engine, run_oracle)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("valid", [False, True], ids=["staged", "resident"])
@pytest.mark.parametrize("K,NB,tile_bytes", [(8, 6, 4), (64, 14, 256 * 256 * 4), (33, 4, 1000), (1, 0, 16), (512, 14, 256 * 256 * 4)])
def test_ex05_fused_on_off_identical(engines, K, NB, tile_bytes, valid):
    dag = dags.ex05_broadcast(K, NB, tile_bytes)
    F = dag.meta["F"]
    on, off = check_pair(engines, dag, Layout.packed(dag, np.full(K * tile_bytes // 4, -7, np.int32), valid))
    assert np.array_equal(on["result"][K:], np.repeat(np.arange(K, dtype=np.uint64), F))   # 0 mismatches, first element k
    if F >= 2:
        units = [(k, list(range(K + k * F, K + (k + 1) * F))) for k in range(K)]
        assert all(fused(on, k, m) for k, m in units)
        assert not all(fused(off, k, m) for k, m in units)


@pytest.mark.parametrize("producer", ["fill5", "iota"])
@pytest.mark.parametrize("tile_bytes,part_bytes", [(4096 + 12, 0), (40000, 0), (1 << 20, 64 * 1024)],
                         ids=["ragged16", "ragged_chunk", "wide_parts"])
def test_mismatches_inside_a_fused_group(producer, tile_bytes, part_bytes):
    """Members with different constants, some of which fail, checking what FILL or IOTA writes: tiles that are not a
    multiple of 16 bytes, not a multiple of the chunk, or split into 16 parts."""
    body, k = (L.BODY_FILL_I32, 5) if producer == "fill5" else (L.BODY_IOTA_I32, 0)
    dag = readers_dag(body, k, KS, tile_bytes)
    layout = Layout.packed(dag, np.zeros(tile_bytes // 4, np.int32))
    with Engine(0, part_bytes=part_bytes) as on, Engine(0, part_bytes=part_bytes, fuse_readers=-1) as off:
        a, b = check_pair((on, off), dag, layout)
    assert a["result"][1:].any() and (a["result"][1:] >> np.uint64(32)).any()
    assert fused(a, 0, list(range(1, 9)))
    assert not_fused(b, 0, list(range(1, 9)))


@pytest.mark.parametrize("chunk", [16, 4096 + 48])
def test_chunk_sizes(engines, monkeypatch, chunk):
    """A 16-byte chunk, and a chunk that does not divide the slice, give the same results."""
    monkeypatch.setenv("PB2_FUSE_CHUNK_BYTES", str(chunk))
    with Engine(0) as e:
        for body, k, tb in ((L.BODY_IOTA_I32, 0, 4096 + 12), (L.BODY_FILL_I32, 5, 40000)):
            dag = readers_dag(body, k, KS, tb)
            layout = Layout.packed(dag, np.zeros(tb // 4, np.int32))
            a = run_engine(e, dag, layout)
            assert_same_run(a, run_engine(engines[1], dag, layout))
            assert_like_oracle(a, run_oracle(dag, layout), dag)
            assert fused(a.res, 0, list(range(1, 9)))
        dag = dags.ex05_broadcast(16, 14, 4096 + 16)
        layout = Layout.packed(dag, np.full(16 * (4096 + 16) // 4, -7, np.int32), True)
        a = run_engine(e, dag, layout)
        assert_same_run(a, run_engine(engines[1], dag, layout))
        assert_like_oracle(a, run_oracle(dag, layout), dag)


def around_dag(mask):
    """P fills tile 0; its out-edges are [X0, R1, R2, X, R3, R4] with X0, X NOPs: {R1, R2} is fused with P, {R3, R4}
    (a second group on the same tile) runs on its own.  R2 has a successor of its own, S (INCR on tile 1), and so does
    R4 (T, INCR on tile 2).  Counter or mask dependency words."""
    P, X0, R1, R2, X, R3, R4, S, T = range(9)
    t = np.zeros(9, L.TASK_DTYPE)
    t["tile"][:] = -1
    t["nb_flows"] = 1
    t["tile"][:, 0] = 0
    t["body"][P], t["iparam"][P, 0], t["access"][P, 0] = L.BODY_FILL_I32, 9, L.ACCESS_WRITE
    for r, k in ((R1, 9), (R2, 8), (R3, 9), (R4, 8)):
        t["body"][r], t["iparam"][r, 0], t["access"][r, 0] = L.BODY_CHECK_I32, k, L.ACCESS_READ
    for x in (X0, X):
        t["body"][x], t["nb_flows"][x], t["tile"][x, 0] = L.BODY_NOP, 0, -1
    t["body"][S], t["iparam"][S, 0], t["tile"][S, 0], t["access"][S, 0] = L.BODY_INCR_I32, 3, 1, L.ACCESS_RW
    t["body"][T], t["iparam"][T, 0], t["tile"][T, 0], t["access"][T, 0] = L.BODY_INCR_I32, 4, 2, L.ACCESS_RW
    src = [P, P, P, P, P, P, R2, R4]
    dst = [X0, R1, R2, X, R3, R4, S, T]
    begin, count, succ = dags._csr_from_edges(9, src, dst, np.zeros(8, np.int64))
    t["succ_begin"], t["succ_count"] = begin, count
    if mask:
        t["flags"] = L.TASK_DEPS_MASK
        t["dep_goal"] = 0x1
    else:
        t["dep_goal"] = 1
    t["dep_goal"][P] = 0
    return dags.Dag(t, succ, np.array([P], np.int32), ntiles=3, tile_bytes=1024, name="around")


@pytest.mark.parametrize("mask", [False, True], ids=["counter", "mask"])
def test_other_successors_and_a_second_group(engines, mask):
    dag = around_dag(mask)
    on, off = check_pair(engines, dag, Layout.packed(dag, np.arange(3 * 256, dtype=np.int32)))
    assert fused(on, 0, [2, 3])
    assert not_fused(on, 0, [5, 6]) and on["worker"][5] == on["worker"][6]
    assert not_fused(off, 0, [2, 3])


def copy_dag(tile_bytes):
    """P copies tile 0 (read) into tile 1 (written, flow 1); eight readers check tile 1."""
    dag = readers_dag(L.BODY_COPY, 0, KS, tile_bytes)
    t = dag.tasks
    t["nb_flows"][0] = 2
    t["access"][0, 0], t["access"][0, 1] = L.ACCESS_READ, L.ACCESS_WRITE
    t["tile"][0, 1] = 1
    t["tile"][1:, 0] = 1
    return dags.Dag(t, dag.succ, dag.ready, ntiles=2, tile_bytes=tile_bytes, name="copy")


def test_two_flow_producer(engines):
    tb = 40000
    dag = copy_dag(tb)
    host = np.concatenate([np.full(tb // 4, 5, np.int32), np.zeros(tb // 4, np.int32)])
    host[17] = 6
    on, off = check_pair(engines, dag, Layout.packed(dag, host))
    assert fused(on, 0, list(range(1, 9)))


def test_not_fused_when_the_read_tile_is_not_the_widest(engines):
    """P fills tile 1 while it also reads the wider tile 0: its parts follow tile 0, so its group runs on its own."""
    dag = copy_dag(4096)
    t = dag.tasks
    t["body"][0], t["iparam"][0, 0] = L.BODY_FILL_I32, 5
    t["tile"][0, 0], t["tile"][0, 1] = 1, 0
    t["access"][0, 0], t["access"][0, 1] = L.ACCESS_WRITE, L.ACCESS_READ
    on, _ = check_pair(engines, dag, Layout.packed(dag, np.zeros((8192 + 4096) // 4, np.int32), sizes=[8192, 4096]))
    assert not_fused(on, 0, list(range(1, 9)))


def test_not_fused_with_pushout(engines):
    dag = readers_dag(L.BODY_FILL_I32, 5, KS, 4096, access=L.ACCESS_WRITE | L.FLOW_PUSHOUT)
    on, _ = check_pair(engines, dag, Layout.packed(dag, np.zeros(1024, np.int32)))
    assert not_fused(on, 0, list(range(1, 9)))


def test_not_fused_without_read_groups():
    dag = readers_dag(L.BODY_FILL_I32, 5, KS, 4096)
    layout = Layout.packed(dag, np.zeros(1024, np.int32))
    with Engine(0, read_groups=-1) as e:
        run = run_engine(e, dag, layout)
    assert_like_oracle(run, run_oracle(dag, layout), dag)
    assert not_fused(run.res, 0, list(range(1, 9)))


def test_single_worker_keeps_fifo_order():
    """With one worker nothing is fused: two producers retire before their readers, as the oracle's FIFO has it."""
    dag = dags.ex05_broadcast(8, 6, 4096)
    layout = Layout.packed(dag, np.full(8 * 1024, -7, np.int32))
    ref = run_oracle(dag, layout)
    with Engine(0, max_workers=1) as e:
        run = run_engine(e, dag, layout)
    assert_like_oracle(run, ref, dag)
    assert np.array_equal(run.res["retire_order"], ref.res["retire_order"])
