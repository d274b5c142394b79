"""Compressible tile memory (pb2_engine_malloc_ex): which allocations get it, that it holds what is written to it, that
it comes back when freed, and that windows on it compute what they compute on cudaMalloc memory."""
import ctypes as C

import numpy as np
import pytest

from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200 import runtime as R
from parsec_b200.engine import Engine
from window_harness import Layout, assert_same_run, placed

pytestmark = pytest.mark.gpu

MIB = 1 << 20


@pytest.fixture(scope="module")
def engine():
    with Engine(0) as e:
        if not e.info()["compression_supported"]:
            pytest.skip("the device or the driver offers no compressible memory (CU_DEVICE_ATTRIBUTE_GENERIC_COMPRESSION_SUPPORTED)")
        yield e


def test_slab_sized_allocations_are_compressible(engine):
    p = engine.malloc(64 * MIB)
    try:
        assert engine.info()["slab_compressible"] == 1
    finally:
        engine.free(p)


def test_small_and_ipc_allocations_are_plain(engine):
    big = engine.malloc(64 * MIB)
    small = engine.malloc(512)
    try:
        assert engine.info()["slab_compressible"] == 1        # a request under one granule is no slab: the flag stays
        ipc = engine.malloc(64 * MIB, ipc=True)
        try:
            assert engine.info()["slab_compressible"] == 0
            assert len(engine.ipc_export(ipc)) == 64           # cudaMalloc memory: CUDA IPC exports it
            assert len(engine.ipc_export(small)) == 64
        finally:
            engine.free(ipc)
    finally:
        engine.free(small)
        engine.free(big)


def test_ipc_export_of_compressible_memory_is_refused(engine):
    p = engine.malloc(64 * MIB)
    try:
        for ptr in (p, p + 3 * MIB):                           # the base and an address inside
            with pytest.raises(L.Pb2Error) as err:
                engine.ipc_export(ptr)
            assert err.value.rc == L.PB2_ERR_NOT_SUPPORTED
            assert "compressible" in str(err.value) and "PB2_MALLOC_IPC" in str(err.value)
    finally:
        engine.free(p)


@pytest.mark.parametrize("nbytes", [2 * MIB, 5 * MIB + 12_345, 64 * MIB])
def test_copies_round_trip(engine, nbytes):
    rng = np.random.default_rng(nbytes)
    data = rng.integers(0, 256, nbytes, dtype=np.uint8)
    p = engine.malloc(nbytes)
    try:
        assert engine.info()["slab_compressible"] == 1
        engine.h2d(p, data)
        got = engine.d2h(np.empty(nbytes, np.uint8), p)
        assert np.array_equal(got, data)
        engine.h2d(p, np.zeros(nbytes, np.uint8))              # uniform data, the case the L2 compresses
        assert not engine.d2h(np.empty(nbytes, np.uint8), p).any()
    finally:
        engine.free(p)


def test_free_returns_the_memory(engine):
    nbytes = 256 * MIB + 1
    p = engine.malloc(nbytes)
    engine.free(p)
    before = engine.info()["free_mem"]
    for _ in range(20):
        p = engine.malloc(nbytes)
        assert engine.info()["slab_compressible"] == 1
        engine.free(p)
    assert abs(engine.info()["free_mem"] - before) <= 2 * MIB


def run_on(engine, dag, layout, ipc):
    """One window of dag over layout in a slab that is plain (ipc) or compressible: the harness's Run of it."""
    slab = engine.malloc(len(layout.dev), ipc=ipc)
    try:
        assert engine.info()["slab_compressible"] == (0 if ipc else 1)
        with placed(engine, layout, slab) as p:
            w = engine.window(dag.kind, dag.tasks, dag.succ, p.tiles, dag.ready)
            try:
                st = w.run()
                res = w.results()
            finally:
                w.close()
        return p.run(st, res, (), (p.dev, p.host))
    finally:
        engine.free(slab)


def test_ex05_window_on_compressible_memory(engine):
    K = 512
    dag = dags.ex05_broadcast(K, 14, 256 * 1024)
    layout = Layout.contiguous(dag)
    plain, comp = run_on(engine, dag, layout, True), run_on(engine, dag, layout, False)
    assert plain.stats["body_errors"] == 0 and plain.stats["tasks_retired"] == dag.ntasks
    assert_same_run(plain, comp)


def test_gemm_window_on_compressible_memory(engine):
    NT, T = 4, 512
    dag = dags.dtd_gemm(NT, T)
    dag.tasks["access"][:, 2] &= ~np.uint8(L.FLOW_PUSHOUT)     # C stays in the slab
    rng = np.random.default_rng(3)
    bits = (rng.integers(0, 1 << 16, dag.ntiles * T * T, dtype=np.uint32).astype(np.uint16) & 0xBFFF)   # finite bf16
    layout = Layout.contiguous(dag, dev=bits)
    plain, comp = run_on(engine, dag, layout, True), run_on(engine, dag, layout, False)
    assert plain.stats["tasks_retired"] == NT ** 3
    assert np.any(plain.dev != layout.dev)
    assert_same_run(plain, comp)


def test_standalone_runtime_heap_on_compressible_memory(engine):
    """The stand-alone runtime's device heap comes from pb2_engine_malloc: at 512 blocks of 256 KiB it is compressible."""
    K, NB, tb = 256, 14, 256 * 1024
    host = np.full(K * tb // 4, -3, np.int32)
    with R.Context(cuda_devices=(0,), mca={"device_cuda_memory_number_of_blocks": 512, "device_cuda_memory_block_size": tb}) as ctx:
        dc = ctx.block_cyclic(4, tb // 4, 1, K * tb // 4, 1, mat=host)
        tp = C.c_void_p(ctx.l.pb2_ptg_ex05_broadcast_new(ctx.h, dc, K, NB))
        ctx.wait()
        info = ctx.task_info(tp)
        recv = info["class_id"] == 1
        assert np.all((info["result"][recv] >> np.uint64(32)) == 0)
        assert np.array_equal(info["result"][recv] & np.uint64(0xFFFFFFFF), info["locals"][recv, 0].astype(np.uint64))
        st = ctx.stats(ctx.devices[0])
        assert st["executed_tasks"] == K * (1 + NB // 2 + 1)
        assert ctx.l.pb2_device_memory_release(ctx.devices[0]) == 0
    assert np.array_equal(host.reshape(K, -1)[:, 0], np.arange(K))
