"""Priority ready order on the H100 (queue_policy 1): with one worker the windows retire in the oracle's 16-lane priority
order; with every worker they compute exactly what the FIFO policy computes, in a dependency-respecting order."""
import ctypes as C

import numpy as np
import pytest

from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200 import multigpu as M
from parsec_b200 import runtime as R
from parsec_b200.bf16 import bf16_bits_to_f32, f32_to_bf16_bits
from parsec_b200.engine import Engine
from priority_order import LANES, priority_order, replay
from test_priority import random_dag
from window_harness import Layout, run_engine, run_oracle

pytestmark = pytest.mark.gpu


def morton(x, y):
    """The Z-order key build_gemm2_units (pb2_window_plan.cpp) sorts the initial ready GEMM units by."""
    r = 0
    for b in range(16):
        r |= (((x >> b) & 1) << (2 * b + 1)) | (((y >> b) & 1) << (2 * b))
    return r


def resident(dag):
    """The DAG with its tiles kept in HBM: no flow is pushed out to a home copy."""
    dag.tasks["access"] &= ~np.uint8(L.FLOW_PUSHOUT)
    return dag


def no_violations(dag, res):
    assert all(v == 0 for v in dags.check_execution(dag, res).values())


@pytest.mark.parametrize("seed,nprio,part_bytes", [(11, 5, 0), (12, 200, 4096), (13, 16, 4096)])
def test_hbm_one_worker_retires_in_oracle_lane_order(seed, nprio, part_bytes):
    """Random DAGs with few and many distinct priorities, tiles staged in from host memory; part_bytes 4096 cuts every
    task into four parts that share their lane."""
    dag = random_dag(500, seed, nprio, tile_bytes=16384)
    host = np.random.default_rng(seed).integers(-100, 100, dag.ntiles * dag.tile_bytes // 4).astype(np.int32)
    layout = Layout.contiguous(dag, host=host, valid=False)
    ref = replay(dag, priority_order(dag, LANES), layout.offsets(), layout.host.copy())
    with Engine(0, max_workers=1, queue_policy=1, part_bytes=part_bytes) as e:
        st, res, got, _, _, _ = run_engine(e, dag, layout)
    assert st["tasks_retired"] == dag.ntasks
    assert np.array_equal(res["retire_order"], ref["retire_order"])
    assert np.array_equal(res["result"], ref["result"])
    assert np.array_equal(res["seen_version"], ref["seen_version"])
    assert np.array_equal(res["tiles"]["version"], ref["tiles"]["version"])
    assert np.array_equal(got, np.concatenate(ref["device"]))


@pytest.mark.parametrize("NT", [3, 5])
def test_gemm_one_worker_retires_in_oracle_lane_order(NT):
    """dtd_gemm with the reference's priorities (NT^3 - i*NT + j: 9 distinct at NT = 3, 25 quantised into 16 lanes at
    NT = 5), every task its own unit; the ready list is given in the Z-order the window keeps within a lane."""
    T = 64
    dag = resident(dags.dtd_gemm(NT, T))
    loc = dag.tasks["locals"][dag.ready]
    dag.ready = dag.ready[np.argsort([morton(int(i), int(j)) for i, j in loc], kind="stable")]
    rng = np.random.default_rng(NT)
    layout = Layout.contiguous(dag, dev=f32_to_bf16_bits(rng.uniform(-0.5, 0.5, dag.ntiles * T * T).astype(np.float32)))
    ref = replay(dag, priority_order(dag, LANES), layout.offsets(), np.zeros(dag.ntiles * dag.tile_bytes, np.uint8))
    outs = {}
    for pol in (0, 1):
        with Engine(0, max_workers=1, gemm_mode=2, queue_policy=pol) as e:
            st, res, outs[pol], _, _, _ = run_engine(e, dag, layout)
        assert st["tasks_retired"] == dag.ntasks
        no_violations(dag, res)
    assert np.array_equal(res["retire_order"], ref["retire_order"])
    assert np.array_equal(outs[0], outs[1])


def test_equal_priorities_one_worker_retire_as_fifo():
    for dag in (random_dag(400, 14, 1), dags.ex05_broadcast(64, 14, 4096)):
        dag.tasks["priority"] = -3
        orders = []
        for pol in (0, 1):
            with Engine(0, max_workers=1, queue_policy=pol) as e:
                orders.append(run_engine(e, dag, Layout.contiguous(dag)).res["retire_order"])
        assert np.array_equal(orders[0], orders[1])


def test_ex05_all_workers_priority_policy():
    """K = 4096 tiles staged in from host memory: read groups and fused producer units run in their lanes."""
    K, NB, tb = 4096, 14, 16384
    dag = dags.ex05_broadcast(K, NB, tb)
    layout = Layout.contiguous(dag, host=np.full(K * tb // 4, -7, np.int32), valid=False)
    ref = run_oracle(dag, layout).res
    with Engine(0, queue_policy=1) as e:
        st, res, _, _, _, _ = run_engine(e, dag, layout)
    assert st["tasks_retired"] == dag.ntasks and st["body_errors"] == 0
    no_violations(dag, res)
    recv = res["result"][K:]
    assert np.all((recv >> np.uint64(32)) == 0)
    assert np.array_equal((recv & np.uint64(0xFFFFFFFF)).astype(np.int64), np.repeat(np.arange(K), dag.meta["F"]))
    assert np.array_equal(res["seen_version"], ref["seen_version"])


def _policies_agree(dag, init, **engine_kw):
    """Both policies leave the same tile bytes, and every task sees the tile versions it sees in the oracle's run."""
    layout = Layout.contiguous(dag, dev=init)
    ref = run_oracle(dag, layout).res
    outs = {}
    for pol in (0, 1):
        with Engine(0, queue_policy=pol, **engine_kw) as e:
            st, res, outs[pol], _, _, _ = run_engine(e, dag, layout)
        assert st["tasks_retired"] == dag.ntasks
        no_violations(dag, res)
        assert np.array_equal(res["seen_version"], ref["seen_version"])
    assert np.array_equal(outs[0], outs[1])


def test_dtd_gemm_fused_chains_all_workers_priority_policy():
    NT, T = 4, 128
    dag = resident(dags.dtd_gemm(NT, T))
    rng = np.random.default_rng(4)
    init = f32_to_bf16_bits(rng.uniform(-0.5, 0.5, dag.ntiles * T * T).astype(np.float32)).view(np.uint8)
    _policies_agree(dag, init)


def cholesky_dag(NT, nb):
    """The Cholesky shape with the classes and priorities of pb2_ptg_cholesky_shape_new (POTRF 4(NT-k) > TRSM
    3(NT-k) > SYRK 2(NT-k) > GEMM NT-k), as one window on one GPU."""
    tasks, succ, tiles, ready, _, _ = M.cholesky_global(NT, nb, 1, 1)
    return dags.Dag(tasks, succ, ready, ntiles=len(tiles), tile_bytes=nb * nb * 2, kind=1, name="cholesky_shape")


def test_cholesky_shape_all_workers_priority_policy():
    NT, nb = 8, 128
    dag = cholesky_dag(NT, nb)
    assert len(np.unique(dag.tasks["priority"])) > LANES             # quantised lanes
    rng = np.random.default_rng(8)
    init = f32_to_bf16_bits(rng.uniform(-0.05, 0.05, dag.ntiles * nb * nb).astype(np.float32)).view(np.uint8)
    _policies_agree(dag, init)


def test_shared_windows_refuse_the_priority_policy():
    dag = dags.ex02_chain(4)
    with Engine(0, queue_policy=1) as e:
        e.set_shared_windows(True)
        with pytest.raises(L.Pb2Error) as ei:
            e.window(0, dag.tasks, dag.succ, np.zeros(1, L.TILE_DTYPE), dag.ready)
        assert ei.value.rc == L.PB2_ERR_NOT_SUPPORTED
        assert "shared windows" in str(ei.value)


def test_runtime_pools_with_the_priority_policy():
    """device_engine_queue_policy = 1: the Ex05 pool gives its known answers, the Cholesky-shape pool runs every task
    on the GPU and leaves the same bits as with the FIFO policy."""
    K, NB, tb = 64, 14, 65536
    host = np.full(K * tb // 4, -3, np.int32)
    with R.Context(cuda_devices=(0,), mca={"device_engine_queue_policy": 1}) as ctx:
        dc = ctx.block_cyclic(4, tb // 4, 1, K * tb // 4, 1, mat=host)
        tp = C.c_void_p(ctx.l.pb2_ptg_ex05_broadcast_new(ctx.h, dc, K, NB))
        ctx.wait()
        info = ctx.task_info(tp)
        recv = info["class_id"] == 1
        assert np.all((info["result"][recv] >> np.uint64(32)) == 0)
        assert np.array_equal(info["result"][recv] & np.uint64(0xFFFFFFFF), info["locals"][recv, 0].astype(np.uint64))
        assert ctx.l.pb2_device_memory_release(ctx.devices[0]) == 0
    assert np.array_equal(host.reshape(K, -1)[:, 0], np.arange(K))

    NT, nb = 5, 128
    finals = {}
    for pol in (0, 1):
        bits = f32_to_bf16_bits(np.random.default_rng(5).uniform(-0.01, 0.01, NT * NT * nb * nb).astype(np.float32))
        with R.Context(cuda_devices=(0,), mca={"device_engine_queue_policy": pol}) as ctx:
            dc = ctx.block_cyclic(2, nb, nb, NT * nb, NT * nb, mat=bits)
            tp = C.c_void_p(ctx.l.pb2_ptg_cholesky_shape_new(ctx.h, dc, NT))
            n = ctx.l.pb2_taskpool_nb_tasks(tp)
            ctx.wait()
            t, dev = ctx.trace(tp)
            assert sorted(t.tolist()) == list(range(n)) and np.all(dev == 2)
            assert ctx.l.pb2_device_memory_release(ctx.devices[0]) == 0
        assert np.all(np.isfinite(bf16_bits_to_f32(bits)))
        finals[pol] = bits
    assert np.array_equal(finals[0], finals[1])
