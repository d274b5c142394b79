"""Linked bodies with a checked form (pb2_engine_link_bodies_checked) fused with their read groups, on the H100.

The bodies are those of tests/cuda/checked_bodies.cu, built by the Makefile into a relocatable sm_90a cubin and PTX:
LINKED_0 a FILL, LINKED_1 y = m x + b, both sliceable and declared checked.  A fused linked producer must compute what
the built-in fused FILL and the oracle compute (results, versions, images, retire order), its readers must get every
mismatch count and first element that numpy and the unfused run give them, and the linked kernels must keep the
engine's worker count."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200 import runtime as R
from parsec_b200.engine import Engine
from window_harness import Layout, assert_like_oracle, assert_same_run, fused, not_fused, run_engine, run_oracle
from test_part_trace_gpu import check_parts, run_traced
from test_linked_bodies import int32_collection, linked_class

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FILL, AXPB = L.BODY_LINKED_0, L.BODY_LINKED_0 + 1
MASK = 0b11


def image(fmt):
    with open(os.path.join(HERE, "cuda", "checked_bodies." + ("ptx" if fmt == L.IMAGE_PTX else "cubin")), "rb") as f:
        return f.read()


def checked_engine(fmt=L.IMAGE_CUBIN, checked=MASK, **kw):
    e = Engine(0, **kw)
    e.link_bodies(image(fmt), fmt, MASK, checked)
    info = e.linked_info()
    print("linked kernel (%s, checked %#x, %s): %s" % ("PTX" if fmt == L.IMAGE_PTX else "cubin", checked, kw, info))
    assert info["nworkers"] == e.info()["nworkers"], "the linked kernel must keep the engine's worker count"
    return e


def linked_ex05(dag):
    """dag (dags.ex05_broadcast) with TaskBcast's FILL_I32 as the linked FILL."""
    t = dag.tasks.copy()
    t["body"][t["body"] == L.BODY_FILL_I32] = FILL
    return dags.Dag(t, dag.succ, dag.ready, ntiles=dag.ntiles, tile_bytes=dag.tile_bytes, name="linked_ex05", meta=dag.meta)


def ex05_members(dag, k):
    K, F = dag.ntiles, dag.meta["F"]
    return [K + k * F + n for n in range(F)]


# ----------------------------------------------------------------------------------------------------------------------
# the Ex05 window with TaskBcast as the checked linked FILL
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt,checked", [(L.IMAGE_CUBIN, MASK), (L.IMAGE_PTX, MASK), (L.IMAGE_CUBIN, 0)],
                         ids=["cubin", "ptx", "undeclared"])
def test_ex05_checked_fill(fmt, checked):
    builtin = dags.ex05_broadcast(512, 14, 64 * 1024)          # F = 8 readers per tile
    assert builtin.meta["F"] == 8
    dag = linked_ex05(builtin)
    host = np.full(builtin.ntiles * builtin.tile_bytes // 4, -1, np.int32)
    layout = lambda: Layout.contiguous(builtin, dev=host)
    ref = run_oracle(builtin, layout())
    with Engine(0) as e:
        want = run_engine(e, builtin, layout())
    e = checked_engine(fmt, checked)
    try:
        plain = run_engine(e, dag, layout())
        traced, out, _ = run_traced(e, dag, layout())
    finally:
        e.close()
    assert_same_run(plain, traced)
    assert_like_oracle(plain, ref, builtin)
    assert_same_run(plain, want)                                  # the built-in fused window
    unit = out[0][1]["unit"]
    for k in range(builtin.ntiles):
        m = ex05_members(builtin, k)
        if checked:
            assert fused(plain.res, k, m) and np.all(unit[m] == k), k
        else:
            assert not_fused(plain.res, k, m) and np.all(unit[m] == m[0]), k


# ----------------------------------------------------------------------------------------------------------------------
# y = m x + b fused with readers of mixed constants: the mismatch path
# ----------------------------------------------------------------------------------------------------------------------
def axpb_case(n=48, tb=64 * 1024, m=3, b=-7, seed=5):
    """Producer i (task i) runs AXPB from tile i (A_i) into tile n + i (X_i); tasks n + 8 i .. + 7 CHECK X_i.  A_i holds
    one constant c_i, and every third tile but the first of each three has some other values too (at element 0 on
    some), so its unit takes the mismatch path.  Readers' constants: k0_i = m c_i + b (leader), k0_i, k0_i + 1, the
    first value of Y_i, k0_i again, 0, k0_i, -1.  Returns the DAG, the slab image it starts from and the expected X."""
    R_ = 8
    rng = np.random.default_rng(seed)
    t = dags._new_tasks(n + n * R_)
    A = np.empty((n, tb // 4), np.int32)
    src, dst = [], []
    with np.errstate(over="ignore"):
        for i in range(n):
            c = np.int32(rng.integers(-1000, 1000))
            A[i] = c
            if i % 3:
                at = rng.choice(tb // 4, size=int(rng.integers(1, 40)), replace=False)
                if i % 3 == 2:
                    at[0] = 0
                A[i, at] = rng.integers(-1000, 1000, len(at)).astype(np.int32) + c + 1
            t["body"][i], t["nb_flows"][i] = AXPB, 2
            t["tile"][i, :2], t["access"][i, :2] = (i, n + i), (L.ACCESS_READ, L.ACCESS_WRITE)
            t["iparam"][i, :2] = (m, b)
            y = A[i] * np.int32(m) + np.int32(b)
            k0 = int(np.int32(c) * np.int32(m) + np.int32(b))
            ks = [k0, k0, k0 + 1, int(y[0]), k0, 0, k0, -1]
            for j, k in enumerate(ks):
                r = n + i * R_ + j
                t["body"][r], t["nb_flows"][r], t["tile"][r, 0], t["access"][r, 0] = L.BODY_CHECK_I32, 1, n + i, L.ACCESS_READ
                t["iparam"][r, 0] = k
                src.append(i); dst.append(r)
        Y = A * np.int32(m) + np.int32(b)
    src, dst = np.array(src, np.int64), np.array(dst, np.int64)
    t["succ_begin"], t["succ_count"], succ = dags._csr_from_edges(len(t), src, dst, np.zeros(len(src), np.int64))
    t["dep_goal"] = np.bincount(dst, minlength=len(t))
    dag = dags.Dag(t, succ, np.arange(n, dtype=np.int32), ntiles=2 * n, tile_bytes=tb, name="axpb_readers")
    garbage = rng.integers(-2 ** 31, 2 ** 31, n * tb // 4, dtype=np.int64).astype(np.int32)
    return dag, np.concatenate([A.reshape(-1), garbage]), Y


def expected_checks(dag, Y):
    """(count of elements != k) << 32 | the tile's first element, per CHECK task; 0 for the producers."""
    t = dag.tasks
    want = np.zeros(dag.ntasks, np.uint64)
    n = Y.shape[0]
    for r in np.flatnonzero(t["body"] == L.BODY_CHECK_I32):
        y = Y[int(t["tile"][r, 0]) - n]
        k = np.int32(t["iparam"][r, 0])
        want[r] = (np.uint64(np.count_nonzero(y != k)) << np.uint64(32)) | np.uint64(np.uint32(y[0]))
    return want


# (queue_policy, trace, part_bytes): all four linked kernels, 64 KiB tiles whole or in four parts
VARIANTS = [(0, False, 16 * 1024), (1, False, 0), (0, True, 0), (1, True, 16 * 1024)]


@pytest.mark.parametrize("queue_policy,trace,part_bytes", VARIANTS,
                         ids=["fifo-%s-%d" % ("traced" if v[1] else "plain", v[2]) if v[0] == 0 else
                              "prio-%s-%d" % ("traced" if v[1] else "plain", v[2]) for v in VARIANTS])
def test_mismatch_path(queue_policy, trace, part_bytes):
    dag, start, Y = axpb_case()
    n = Y.shape[0]
    layout = lambda: Layout.contiguous(dag, dev=start)
    kw = dict(queue_policy=queue_policy, part_bytes=part_bytes)
    e = checked_engine(**kw)
    try:
        if trace:
            run, out, entries = run_traced(e, dag, layout())
            sm_count = e.info()["sm_count"]
        else:
            run = run_engine(e, dag, layout())
    finally:
        e.close()
    e = checked_engine(fuse_readers=-1, **kw)
    try:
        unfused = run_engine(e, dag, layout())
    finally:
        e.close()
    assert_same_run(run, unfused)
    bad = dags.check_execution(dag, run.res)
    assert all(v == 0 for v in bad.values()), bad
    assert np.array_equal(run.res["result"], expected_checks(dag, Y))
    assert np.array_equal(run.dev.view(np.int32)[n * dag.tile_bytes // 4:], Y.reshape(-1))
    assert run.stats["body_errors"] == int(np.sum(expected_checks(dag, Y) >> np.uint64(32)))
    for i in range(n):
        m = list(range(n + 8 * i, n + 8 * i + 8))
        assert fused(run.res, i, m) and not_fused(unfused.res, i, m), i
    if trace:
        st, tr, rec = out[0]
        check_parts(dag, entries, st, tr, rec, sm_count, True, "checked axpb %s" % (kw,))
        assert np.all(tr["unit"][n:] == np.repeat(np.arange(n), 8))
        assert rec["nparts"].max() == (4 if part_bytes else 1)


def test_one_worker_fuses_nothing_and_keeps_fifo_order():
    builtin = dags.ex05_broadcast(8, 6, 4096)
    dag = linked_ex05(builtin)
    layout = lambda: Layout.packed(builtin, np.full(8 * 1024, -7, np.int32))
    ref = run_oracle(builtin, layout())
    e = checked_engine(max_workers=1)
    try:
        run = run_engine(e, dag, layout())
    finally:
        e.close()
    assert_like_oracle(run, ref, builtin)
    assert np.array_equal(run.res["retire_order"], ref.res["retire_order"])
    for k in range(8):
        assert not_fused(run.res, k, ex05_members(builtin, k))


def test_engine_refusals():
    with Engine(0) as e:
        for sliceable, checked, why in ((0b01, 0b11, "sliceable"), (0xFF, 0x100, "bits above bit 7")):
            with pytest.raises(L.Pb2Error) as ex:
                e.link_bodies(image(L.IMAGE_CUBIN), L.IMAGE_CUBIN, sliceable, checked)
            assert ex.value.rc == L.PB2_ERR_BAD_PARAM and why in str(ex.value), str(ex.value)
        e.link_bodies(image(L.IMAGE_CUBIN), L.IMAGE_CUBIN, MASK, MASK)      # nothing was left behind


# ----------------------------------------------------------------------------------------------------------------------
# the stand-alone runtime
# ----------------------------------------------------------------------------------------------------------------------
def test_runtime_checked_fill_pool():
    """A DTD pool: FILL tile i with k_i (the checked linked FILL), then eight CHECK readers of tile i, the last with
    k_i + 1.  Host data written back, every reader's result as numpy has it."""
    n, F, tb = 64, 8, 256 * 1024
    ks = (np.arange(n, dtype=np.int32) * 7 - 100)
    host = np.full(n * tb // 4, -1, np.int32)
    with R.Context(cuda_devices=(0,)) as ctx:
        ctx.link_bodies(ctx.devices[0], image(L.IMAGE_CUBIN), L.IMAGE_CUBIN, MASK, MASK)
        tp = C.c_void_p(ctx.l.pb2_dtd_taskpool_new(ctx.h))
        rc, fill = linked_class(ctx, tp, FILL, 1)
        assert rc == 0
        check = linked_class(ctx, tp, L.BODY_CHECK_I32, 1)[1]
        dc = int32_collection(ctx, n, tb, host)
        keep, checks = [], []

        def put(tc, i, op, k):
            arr = (C.c_void_p * 1)(ctx.l.pb2_dtd_tile_of(tp, dc, ctx.l.pb2_dc_data_key(dc, i, 0)))
            o, p = np.array([op], np.int32), np.array([k, 0, 0], np.int32)
            keep.extend((arr, o, p))
            t = ctx.l.pb2_dtd_insert_task_with_task_class(tp, tc, 0, R.DEV_CUDA, arr, o.ctypes.data_as(C.c_void_p),
                                                          p.ctypes.data_as(C.c_void_p), 0.0)
            assert t >= 0
            return t

        for i in range(n):
            put(fill, i, R.OUTPUT, int(ks[i]))
            checks += [(put(check, i, R.INPUT, int(ks[i]) + (j == F - 1)), i, j == F - 1) for j in range(F)]
        ctx.wait()
        st = ctx.stats(ctx.devices[0])
        info = ctx.task_info(tp)
        assert ctx.l.pb2_device_memory_release(ctx.devices[0]) == 0
    assert st["executed_tasks"] == n * (1 + F)
    assert np.array_equal(host.reshape(n, -1), np.repeat(ks[:, None], tb // 4, axis=1))
    for t, i, off in checks:
        want = (np.uint64(tb // 4 if off else 0) << np.uint64(32)) | np.uint64(np.uint32(ks[i]))
        assert info["result"][t] == want, (t, i, off)
