"""Linked readers with the group form (PB2_LINK_READER_GROUPS) on the H100.

Every case runs on two engines and against numpy: one linked with tests/cuda/reader_group_bodies.cubin and its readers
declared with the group form, so that each read group calls pb2_linked_reader_group once per chunk; one linked with
tests/cuda/reader_bodies.cubin, the same readers called one by one.  Results, seen versions, tile versions, images and
stats are equal bit for bit, and every reader's result is numpy's over its tile (test_linked_readers_gpu.readers_case)."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200 import runtime as R
from parsec_b200.engine import Engine
from gemm_chain_dags import C_WORD, ex05_beside_gemm
from test_gemm_groups_gpu import ran_as_unit
from test_linked_bodies import int32_collection, linked_class
from test_linked_readers_gpu import (AXPB, COUNT_GT, COUNT_NE, FAIL, FILL, RAGGED, READERS, SLICEABLE, SUM_I64,
                                     assert_results, layout_of, reader_result, reader_spec, readers_case, tiles_hold)
from test_part_trace_gpu import check_parts, run_traced
from window_harness import Layout, assert_same_run, fused, run_engine

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GROUPS = READERS


def fixture(name):
    with open(os.path.join(HERE, "cuda", name + ".cubin"), "rb") as f:
        return f.read()


def engine(groups=GROUPS, gemm_windows=False, **kw):
    """An engine linked with the group fixture and `groups` declared (0: the per-member fixture, nothing declared)."""
    e = Engine(0, **kw)
    try:
        e.link_bodies(fixture("reader_group_bodies" if groups else "reader_bodies"), L.IMAGE_CUBIN, SLICEABLE, 0,
                      gemm_windows=gemm_windows, readers=READERS, reader_groups=groups)
        info = e.linked_info()
        assert info["nworkers"] == e.info()["nworkers"] and info["regs"] <= 80, info
    except BaseException:
        e.close()
        raise
    return e


def both(dag, layout, groups=GROUPS, **kw):
    """(group run, per-member run) of dag on the two engines, equal bit for bit."""
    runs = []
    for g in (groups, 0):
        e = engine(g, **kw)
        try:
            runs.append(run_engine(e, dag, layout))
        finally:
            e.close()
    assert_same_run(runs[0], runs[1])
    return runs


# ----------------------------------------------------------------------------------------------------------------------
# the Ex05 shape: TaskRecv as COUNT_NE, unfused, fused with the built-in FILL and with the linked FILL
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("producer,kw", [(L.BODY_FILL_I32, dict(fuse_readers=-1)), (L.BODY_FILL_I32, {}), (FILL, {})],
                         ids=["unfused", "fused_builtin_fill", "fused_linked_fill"])
def test_ex05(producer, kw):
    K, F, tb = 256, 8, 256 * 1024
    dag = dags.ex05_broadcast(K, 14, tb)
    t = dag.tasks
    t["body"][t["body"] == L.BODY_CHECK_I32] = COUNT_NE
    t["body"][t["body"] == L.BODY_FILL_I32] = producer
    runs = both(dag, Layout.packed(dag, valid=True), **kw)
    res = runs[0].res
    bad = dags.check_execution(dag, res)
    assert all(v == 0 for v in bad.values()), bad
    # every TaskRecv(k, n) compares tile k, filled with k, with n's constant: 0 or every element
    for r in range(K, dag.ntasks):
        k = int(t["tile"][r, 0])
        x = np.full(tb // 4, int(t["iparam"][k, 0]), np.int32)
        assert res["result"][r] == reader_result(COUNT_NE, int(t["iparam"][r, 0]), x), r
    for k in range(K):
        assert fused(res, k, list(range(K + k * F, K + k * F + F))) == ("fuse_readers" not in kw), k


# ----------------------------------------------------------------------------------------------------------------------
# groups of 1 to 8 mixed members, ragged tiles, small parts, staged tiles, one worker
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("F", [1, 2, 3, 5, 8])
def test_group_sizes(F):
    K = 48
    dag, init, X, want, sizes = readers_case(K, F, [256 * 1024 + 48] * K, L.BODY_ADD_IOTA_I32, seed=F)
    # rotate each tile's reader bodies so every position sees every body
    t = dag.tasks
    for k in range(K):
        for j in range(F):
            r = K + k * F + j
            body, dk = reader_spec(j + k)
            c = int(X[k][0])
            t["body"][r], t["iparam"][r, 0] = body, (np.int64(c + dk).astype(np.int32) if body != SUM_I64 else 0)
            want[r] = reader_result(body, int(t["iparam"][r, 0]), X[k])
    runs = both(dag, layout_of(dag, init, sizes), part_bytes=64 * 1024)
    for run in runs:
        assert_results(run, dag, want)
        tiles_hold(run, layout_of(dag, init, sizes), X)


@pytest.mark.parametrize("part_bytes", [0, 4096], ids=["whole", "many"])
@pytest.mark.parametrize("producer,staged", [(L.BODY_ADD_IOTA_I32, False), (AXPB, True)], ids=["add_iota", "axpb_staged"])
def test_ragged_tiles_and_parts(part_bytes, producer, staged):
    K, F = len(RAGGED), 8
    dag, init, X, want, sizes = readers_case(K, F, RAGGED, producer, seed=11)
    for run in both(dag, layout_of(dag, init, sizes, staged), part_bytes=part_bytes):
        assert_results(run, dag, want)
        tiles_hold(run, layout_of(dag, init, sizes), X)


def test_some_members_declared():
    """SUM_I64 not declared with the group form: it is called one by one beside the group call of the others."""
    K, F = 32, 8
    dag, init, X, want, sizes = readers_case(K, F, [256 * 1024] * K, FILL, seed=4)
    for run in both(dag, layout_of(dag, init, sizes), groups=GROUPS & ~(1 << (SUM_I64 - L.BODY_LINKED_0))):
        assert_results(run, dag, want)


def test_one_worker_retires_alike():
    K, F = 16, 8
    dag, init, X, want, sizes = readers_case(K, F, [64 * 1024] * K, L.BODY_IOTA_I32, seed=6)
    runs = both(dag, layout_of(dag, init, sizes), max_workers=1)
    assert np.array_equal(runs[0].res["retire_order"], runs[1].res["retire_order"])
    assert_results(runs[0], dag, want)


def test_read_groups_off():
    K, F = 32, 8
    dag, init, X, want, sizes = readers_case(K, F, [256 * 1024] * K, FILL, seed=7)
    for run in both(dag, layout_of(dag, init, sizes), read_groups=-1):
        assert_results(run, dag, want)


# ----------------------------------------------------------------------------------------------------------------------
# the four kernel variants
# ----------------------------------------------------------------------------------------------------------------------
VARIANTS = [(0, False, 64 * 1024), (1, False, 0), (0, True, 0), (1, True, 64 * 1024)]


@pytest.mark.parametrize("queue_policy,trace,part_bytes", VARIANTS,
                         ids=["%s-%s-%d" % ("prio" if v[0] else "fifo", "traced" if v[1] else "plain", v[2]) for v in VARIANTS])
def test_kernel_variants(queue_policy, trace, part_bytes):
    K, F = 64, 8
    dag, init, X, want, sizes = readers_case(K, F, [256 * 1024] * K, FILL, seed=5)
    e = engine(queue_policy=queue_policy, part_bytes=part_bytes)
    try:
        if trace:
            run, out, entries = run_traced(e, dag, layout_of(dag, init, sizes))
            st, tr, rec = out[0]
            check_parts(dag, entries, st, tr, rec, e.info()["sm_count"], True, "group readers %d %d" % (queue_policy, part_bytes))
        else:
            run = run_engine(e, dag, layout_of(dag, init, sizes))
    finally:
        e.close()
    assert_results(run, dag, want)
    tiles_hold(run, layout_of(dag, init, sizes), X)


# ----------------------------------------------------------------------------------------------------------------------
# a bad member, and the link mismatches
# ----------------------------------------------------------------------------------------------------------------------
def test_group_fail():
    """FAIL's group form sets its result to ~0 and returns ~0: the window is bad (PB2_ERR_BAD_PARAM from the wait, as
    for any bad body; the workers stop at their next idle pop, so a window whose last tasks were already queued may
    still retire them all), and no result of a member of that call is added: FAIL's and its group's stay 0."""
    K, F = 4, 8
    dag, init, X, want, sizes = readers_case(K, F, [64 * 1024] * K, L.BODY_IOTA_I32)
    bad = K + F + 3
    dag.tasks["body"][bad] = FAIL
    e = engine(part_bytes=16 * 1024)
    try:
        try:
            run = run_engine(e, dag, layout_of(dag, init, sizes))
        except L.Pb2Error as ex:
            assert ex.rc == L.PB2_ERR_BAD_PARAM, str(ex)
        else:
            got = run.res["result"]
            assert np.all(got[K + F:K + 2 * F] == 0), got[K + F:K + 2 * F]
            idx = [r for r in range(K, dag.ntasks) if not K + F <= r < K + 2 * F]
            assert np.array_equal(got[idx], np.array([want[r] for r in idx], np.uint64))
    finally:
        e.close()


def test_link_mismatches():
    with Engine(0) as e:
        # the mask without the group form: the group-call kernels have an undefined reference
        img = fixture("reader_bodies")
        assert e._lib.pb2_engine_link_bodies_ex(e._h, img, len(img), L.IMAGE_CUBIN, SLICEABLE, 0,
                                                 L.LINK_READERS(READERS) | L.LINK_READER_GROUPS(GROUPS)) == L.PB2_ERR_BAD_PARAM
        msg = (e._lib.pb2_engine_last_error(e._h) or b"").decode()
        assert "pb2_linked_reader_group" in msg, msg
        with pytest.raises(L.Pb2Error):
            e.linked_info()
        # a mask that is not a subset of the readers mask
        img = fixture("reader_group_bodies")
        assert e._lib.pb2_engine_link_bodies_ex(e._h, img, len(img), L.IMAGE_CUBIN, SLICEABLE, 0,
                                                 L.LINK_READERS(0b1) | L.LINK_READER_GROUPS(0b11)) == L.PB2_ERR_BAD_PARAM
        assert "reader groups" in (e._lib.pb2_engine_last_error(e._h) or b"").decode()
        # nothing was left behind: the right link succeeds
        e.link_bodies(img, L.IMAGE_CUBIN, SLICEABLE, 0, readers=READERS, reader_groups=GROUPS)
        assert e.linked_info()["regs"] <= 80


def test_group_image_without_the_mask():
    """An image with the group form linked without the mask runs the plain kernels, which call its members one by one."""
    K, F = 16, 8
    dag, init, X, want, sizes = readers_case(K, F, [256 * 1024] * K, FILL, seed=8)
    e = Engine(0)
    try:
        e.link_bodies(fixture("reader_group_bodies"), L.IMAGE_CUBIN, SLICEABLE, 0, readers=READERS)
        assert_results(run_engine(e, dag, layout_of(dag, init, sizes)), dag, want)
    finally:
        e.close()


# ----------------------------------------------------------------------------------------------------------------------
# a GEMM window linked with PB2_LINK_GEMM_WINDOWS
# ----------------------------------------------------------------------------------------------------------------------
def test_gemm_window():
    K = 128
    dag, ex, sizes, host = ex05_beside_gemm(K)
    t = dag.tasks
    F = ex.meta["F"]
    for k in range(K):
        for j in range(F):
            r = K + k * F + j
            body, dk = reader_spec(j + k)
            t["body"][r], t["iparam"][r, 0] = body, (k + dk if body != SUM_I64 else 0)
    creaders = list(range(ex.ntasks + 2, dag.ntasks))
    for j, r in enumerate(creaders):
        t["body"][r] = (COUNT_NE, SUM_I64, COUNT_GT, COUNT_NE)[j]
        t["iparam"][r, 0] = (C_WORD, 0, 0, C_WORD + 1)[j]
    runs = both(dag, Layout.packed(dag, host=host, valid=True, sizes=sizes), gemm_windows=True, part_bytes=64 * 1024)
    res = runs[0].res
    bad = dags.check_execution(dag, res)
    assert all(v == 0 for v in bad.values()), bad
    for k in range(K):
        x = np.full(ex.tile_bytes // 4, k, np.int32)
        for j in range(F):
            r = K + k * F + j
            assert res["result"][r] == reader_result(int(t["body"][r]), int(t["iparam"][r, 0]), x), (k, j)
        assert ran_as_unit(res, [k] + list(range(K + k * F, K + k * F + F))), k
    assert ran_as_unit(res, creaders)
    c = np.full(128 * 128 // 2, C_WORD, np.uint32).view(np.int32)
    for r in creaders:
        assert res["result"][r] == reader_result(int(t["body"][r]), int(t["iparam"][r, 0]), c), r


# ----------------------------------------------------------------------------------------------------------------------
# the stand-alone runtime
# ----------------------------------------------------------------------------------------------------------------------
def test_runtime_reader_pool():
    """A DTD pool: the linked FILL writes tile i with k_i, then eight linked readers of tile i, declared with the group
    form.  Every reader's result as numpy has it, the host data written back."""
    n, F, tb = 64, 8, 256 * 1024
    ks = np.arange(n, dtype=np.int32) * 7 - 100
    host = np.full(n * tb // 4, -1, np.int32)
    with R.Context(cuda_devices=(0,)) as ctx:
        ctx.link_bodies(ctx.devices[0], fixture("reader_group_bodies"), L.IMAGE_CUBIN, SLICEABLE, readers=READERS,
                        reader_groups=GROUPS)
        tp = C.c_void_p(ctx.l.pb2_dtd_taskpool_new(ctx.h))
        rc, fill = linked_class(ctx, tp, FILL, 1)
        assert rc == 0
        classes = {b: linked_class(ctx, tp, b, 1)[1] for b in (COUNT_NE, SUM_I64, COUNT_GT)}
        dc = int32_collection(ctx, n, tb, host)
        keep, readers = [], []

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
            for j in range(F):
                body, dk = reader_spec(j + i)
                k = int(ks[i]) + dk if body != SUM_I64 else 0
                readers.append((put(classes[body], i, R.INPUT, k), body, k, i))
        ctx.wait()
        info = ctx.task_info(tp)
        assert ctx.l.pb2_device_memory_release(ctx.devices[0]) == 0
    assert np.array_equal(host.reshape(n, -1), np.repeat(ks[:, None], tb // 4, axis=1))
    for t, body, k, i in readers:
        assert info["result"][t] == reader_result(body, k, np.full(tb // 4, ks[i], np.int32)), (t, body, k, i)
