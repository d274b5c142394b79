"""Linked readers (PB2_LINK_READERS) in read groups and fused units, on the H100.

The bodies are those of tests/cuda/reader_bodies.cu: the readers COUNT_NE, SUM_I64 and COUNT_GT, the producers AXPB and
FILL, the control SUM_CTL (SUM_I64, not declared a reader) and FAIL.  A reader's result is the sum of what its calls
return, so it must equal numpy's over the whole tile whether the engine groups the task, fuses it with its producer,
runs it alone or cuts it into parts; and every such run must compute the same results, versions and images."""
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
from test_part_trace_gpu import check_parts, run_traced
from window_harness import Layout, assert_same_run, fused, run_engine, run_oracle

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
COUNT_NE, SUM_I64, COUNT_GT, AXPB, FILL, SUM_CTL, FAIL = (L.BODY_LINKED_0 + i for i in range(7))
READERS = 0b1000111
SLICEABLE = 0x7F
U64 = np.uint64


def image(fmt=L.IMAGE_CUBIN):
    with open(os.path.join(HERE, "cuda", "reader_bodies." + ("ptx" if fmt == L.IMAGE_PTX else "cubin")), "rb") as f:
        return f.read()


def reader_engine(fmt=L.IMAGE_CUBIN, gemm_windows=False, **kw):
    e = Engine(0, **kw)
    e.link_bodies(image(fmt), fmt, SLICEABLE, 0, gemm_windows=gemm_windows, readers=READERS)
    info = e.linked_info()
    print("linked kernel (%s): %s" % (kw, info))
    assert info["nworkers"] == e.info()["nworkers"], "the linked kernel must keep the engine's worker count"
    return e


def reader_result(body, k, x):
    """What reader `body` with constant k returns over the int32 elements x."""
    x = np.asarray(x, np.int32)
    if body == COUNT_NE:
        return U64(np.count_nonzero(x != np.int32(k)))
    if body == COUNT_GT:
        return U64(np.count_nonzero(x > np.int32(k)))
    return U64(int(x.astype(np.int64).sum()) % (1 << 64))


# (body, constant) of reader j of a tile whose producer wrote constant c_k (a reader's constant is relative to it)
def reader_spec(j):
    return [(COUNT_NE, 0), (SUM_I64, 0), (COUNT_GT, 100), (COUNT_NE, 7), (SUM_I64, 0), (COUNT_GT, -5), (COUNT_NE, 0),
            (COUNT_GT, 1000)][j % 8]


def readers_case(K, F, sizes, producer, seed=3, m=3, b=-11):
    """Producer k writes tile k (sizes[k] bytes), then F readers of tile k (reader_spec) in one out-edge run.  Producers:
    IOTA, ADD_IOTA (RW over random data), AXPB (from tile K + k, y = m x + b), FILL (iparam k * 13 - 40), the last two
    the linked bodies.  Returns (dag, the tiles' initial int32 contents, their contents after their producers, per task
    its expected result or None, the tiles' bytes)."""
    rng = np.random.default_rng(seed)
    sizes = list(sizes)
    ntiles = 2 * K if producer == AXPB else K
    all_sizes = sizes + (sizes if producer == AXPB else [])
    init = [rng.integers(-2 ** 31, 2 ** 31, s // 4, dtype=np.int64).astype(np.int32) for s in all_sizes]
    n = K + K * F
    t = dags._new_tasks(n)
    src, dst = [], []
    X = []
    with np.errstate(over="ignore"):
        for k in range(K):
            ne = sizes[k] // 4
            t["nb_flows"][k] = 1
            t["tile"][k, 0], t["access"][k, 0] = k, L.ACCESS_WRITE
            if producer == L.BODY_IOTA_I32:
                t["body"][k] = producer
                X.append(np.arange(ne, dtype=np.int64).astype(np.int32))
            elif producer == L.BODY_ADD_IOTA_I32:
                t["body"][k], t["access"][k, 0] = producer, L.ACCESS_RW
                X.append(init[k] + np.arange(ne, dtype=np.int64).astype(np.int32))
            elif producer == AXPB:
                t["body"][k], t["nb_flows"][k] = AXPB, 2
                t["tile"][k, :2], t["access"][k, :2] = (K + k, k), (L.ACCESS_READ, L.ACCESS_WRITE)
                t["iparam"][k, :2] = (m, b)
                X.append(init[K + k] * np.int32(m) + np.int32(b))
            else:
                t["body"][k], t["iparam"][k, 0] = FILL, k * 13 - 40
                X.append(np.full(ne, k * 13 - 40, np.int32))
            for j in range(F):
                r = K + k * F + j
                body, dk = reader_spec(j)
                c = int(X[k][0]) if len(X[k]) else 0
                t["body"][r], t["nb_flows"][r], t["tile"][r, 0], t["access"][r, 0] = body, 1, k, L.ACCESS_READ
                t["iparam"][r, 0] = np.int32(np.int64(c + dk).astype(np.int32)) if body != SUM_I64 else 0
                t["dep_goal"][r] = 1
                src.append(k); dst.append(r)
    t["succ_begin"], t["succ_count"], succ = dags._csr_from_edges(n, np.array(src, np.int64), np.array(dst, np.int64),
                                                                  np.zeros(len(src), np.int64))
    dag = dags.Dag(t, succ, np.arange(K, dtype=np.int32), ntiles=ntiles, tile_bytes=max(all_sizes), name="readers")
    want = [None] * n
    for r in range(K, n):
        want[r] = reader_result(int(t["body"][r]), int(t["iparam"][r, 0]), X[(r - K) // F])
    return dag, init, X, want, all_sizes


def layout_of(dag, init, sizes, staged=False):
    """Layout.packed over tiles that start holding init: resident, or staged in from their host copies."""
    host = np.concatenate([np.pad(x.view(np.uint8), (0, s - 4 * len(x))) for x, s in zip(init, sizes)])
    return Layout.packed(dag, host=host, valid=not staged, sizes=sizes)


def assert_results(run, dag, want):
    bad = dags.check_execution(dag, run.res)
    assert all(v == 0 for v in bad.values()), bad
    got = run.res["result"]
    idx = [i for i, w in enumerate(want) if w is not None]
    assert np.array_equal(got[idx], np.array([want[i] for i in idx], np.uint64)), \
        [(i, int(got[i]), int(want[i])) for i in idx if got[i] != want[i]][:8]


def tiles_hold(run, layout, X):
    for k, x in enumerate(X):
        assert np.array_equal(layout.tile_bytes(run.dev, k)[:len(x) * 4].view(np.int32), x), k


# ----------------------------------------------------------------------------------------------------------------------
# the Ex05 shape: grouped, fused, alone and on one worker
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("producer", [L.BODY_IOTA_I32, L.BODY_ADD_IOTA_I32, AXPB, FILL],
                         ids=["iota", "add_iota", "linked_axpb", "linked_fill"])
def test_ex05_shape(producer):
    K, F, tb = 96, 8, 256 * 1024
    dag, init, X, want, sizes = readers_case(K, F, [tb] * K, producer)
    runs = {}
    for name, kw in (("fused", {}), ("no_groups", dict(read_groups=-1)), ("groups_only", dict(fuse_readers=-1)),
                     ("one_worker", dict(max_workers=1))):
        e = reader_engine(**kw)
        try:
            runs[name] = run_engine(e, dag, layout_of(dag, init, sizes))
        finally:
            e.close()
    for name, run in runs.items():
        assert_results(run, dag, want)
        tiles_hold(run, layout_of(dag, init, sizes), X)
        assert_same_run(run, runs["fused"])
    for k in range(K):
        m = list(range(K + k * F, K + k * F + F))
        assert fused(runs["fused"].res, k, m), k
        res = runs["groups_only"].res
        assert len(set(res["worker"][m].tolist())) == 1 and not fused(res, k, m), k
    if producer == L.BODY_IOTA_I32:
        # the oracle models the same DAG with its readers as CHECK: the same versions, images and order rules
        chk = dag.tasks.copy()
        chk["body"][K:] = L.BODY_CHECK_I32
        cdag = dags.Dag(chk, dag.succ, dag.ready, ntiles=dag.ntiles, tile_bytes=dag.tile_bytes)
        ref = run_oracle(cdag, layout_of(dag, init, sizes))
        for k in ("seen_version",):
            assert np.array_equal(runs["fused"].res[k], ref.res[k]), k
        assert np.array_equal(runs["fused"].res["tiles"]["version"], ref.res["tiles"]["version"])
        assert np.array_equal(runs["fused"].dev, ref.dev)


# ----------------------------------------------------------------------------------------------------------------------
# ragged tiles, 1, 4 and many parts, staged tiles
# ----------------------------------------------------------------------------------------------------------------------
RAGGED = [256 * 1024 + 20, 100 * 1024 + 4, 12 * 1024 + 12, 36, 4, 64 * 1024 + 1028, 48 * 1024 - 4, 16 * 1024 + 8]


@pytest.mark.parametrize("part_bytes", [0, 64 * 1024 + 16, 4096], ids=["whole", "about_four", "many"])
@pytest.mark.parametrize("producer,staged", [(L.BODY_ADD_IOTA_I32, False), (AXPB, True)], ids=["add_iota", "axpb_staged"])
def test_ragged_tiles_and_parts(part_bytes, producer, staged):
    K, F = len(RAGGED), 8
    dag, init, X, want, sizes = readers_case(K, F, RAGGED, producer, seed=11)
    runs = []
    for kw in ({}, dict(read_groups=-1)):
        e = reader_engine(part_bytes=part_bytes, **kw)
        try:
            runs.append(run_engine(e, dag, layout_of(dag, init, sizes, staged)))
        finally:
            e.close()
    for run in runs:
        assert_results(run, dag, want)
        tiles_hold(run, layout_of(dag, init, sizes), X)
    assert_same_run(runs[0], runs[1])


# ----------------------------------------------------------------------------------------------------------------------
# all four linked kernels, with part records
# ----------------------------------------------------------------------------------------------------------------------
VARIANTS = [(0, False, 64 * 1024), (1, False, 0), (0, True, 0), (1, True, 64 * 1024)]


@pytest.mark.parametrize("queue_policy,trace,part_bytes", VARIANTS,
                         ids=["%s-%s-%d" % ("prio" if v[0] else "fifo", "traced" if v[1] else "plain", v[2]) for v in VARIANTS])
def test_kernel_variants(queue_policy, trace, part_bytes):
    K, F = 64, 8
    dag, init, X, want, sizes = readers_case(K, F, [256 * 1024] * K, FILL, seed=5)
    e = reader_engine(queue_policy=queue_policy, part_bytes=part_bytes)
    try:
        if trace:
            run, out, entries = run_traced(e, dag, layout_of(dag, init, sizes))
            st, tr, rec = out[0]
            check_parts(dag, entries, st, tr, rec, e.info()["sm_count"], True, "linked readers %d %d" % (queue_policy, part_bytes))
            assert np.all(tr["unit"][K:] == np.repeat(np.arange(K), F))
        else:
            run = run_engine(e, dag, layout_of(dag, init, sizes))
    finally:
        e.close()
    assert_results(run, dag, want)
    tiles_hold(run, layout_of(dag, init, sizes), X)


# ----------------------------------------------------------------------------------------------------------------------
# members with successors, a bad reader, the control
# ----------------------------------------------------------------------------------------------------------------------
def test_war_writer_after_the_readers():
    """IOTA writes tile 0, four readers read it (a group fused with IOTA), FILL overwrites it after all four."""
    t = dags._new_tasks(6)
    t["body"][0], t["nb_flows"][0], t["tile"][0, 0], t["access"][0, 0] = L.BODY_IOTA_I32, 1, 0, L.ACCESS_WRITE
    for r, (body, k) in zip(range(1, 5), [(COUNT_NE, 0), (SUM_I64, 0), (COUNT_GT, 1000), (SUM_I64, 0)]):
        t["body"][r], t["nb_flows"][r], t["tile"][r, 0], t["access"][r, 0] = body, 1, 0, L.ACCESS_READ
        t["iparam"][r, 0], t["dep_goal"][r] = k, 1
    t["body"][5], t["nb_flows"][5], t["tile"][5, 0], t["access"][5, 0] = FILL, 1, 0, L.ACCESS_WRITE
    t["iparam"][5, 0], t["dep_goal"][5] = 99, 4
    src, dst = [0, 0, 0, 0, 1, 2, 3, 4], [1, 2, 3, 4, 5, 5, 5, 5]
    t["succ_begin"], t["succ_count"], succ = dags._csr_from_edges(6, np.array(src), np.array(dst), np.zeros(8, np.int64))
    tb = 256 * 1024
    dag = dags.Dag(t, succ, np.array([0], np.int32), ntiles=1, tile_bytes=tb, name="war")
    x = np.arange(tb // 4, dtype=np.int32)
    for part_bytes in (0, 64 * 1024):
        e = reader_engine(part_bytes=part_bytes)
        try:
            run = run_engine(e, dag, Layout.packed(dag))
        finally:
            e.close()
        res = run.res
        assert fused(res, 0, [1, 2, 3, 4])
        assert [int(v) for v in res["result"][1:5]] == [int(reader_result(b, k, x)) for b, k in
                                                        [(COUNT_NE, 0), (SUM_I64, 0), (COUNT_GT, 1000), (SUM_I64, 0)]]
        assert all(res["end_seq"][r] < res["start_seq"][5] for r in range(1, 5))
        assert np.all(res["seen_version"][1:5, 0] == res["seen_version"][5, 0])
        assert res["tiles"]["version"][0] == res["seen_version"][5, 0] + 1
        assert np.all(run.dev[:tb].view(np.int32) == 99)
        bad = dags.check_execution(dag, res)
        assert all(v == 0 for v in bad.values()), bad


@pytest.mark.parametrize("kw", [{}, dict(read_groups=-1)], ids=["grouped", "alone"])
def test_bad_reader_is_not_added(kw):
    """A reader returning ~0 marks the window bad (PB2_ERR_BAD_PARAM from the wait, as for any body; the workers stop
    at their next idle pop, so a window whose last tasks were already queued may still retire them all) and its ~0 is
    not added: its result stays 0, and every other reader's is numpy's."""
    dag, init, X, want, sizes = readers_case(4, 8, [64 * 1024] * 4, L.BODY_IOTA_I32)
    bad = 4 + 8 + 3
    dag.tasks["body"][bad] = FAIL
    want[bad] = U64(0)
    e = reader_engine(part_bytes=16 * 1024, **kw)
    try:
        try:
            run = run_engine(e, dag, layout_of(dag, init, sizes))
        except L.Pb2Error as ex:
            assert ex.rc == L.PB2_ERR_BAD_PARAM, str(ex)
        else:
            assert_results(run, dag, want)
    finally:
        e.close()


def test_non_reader_keeps_part_zero():
    """SUM_CTL is SUM_I64 without the reader declaration: cut into parts, a task keeps part 0's sum; SUM_I64 adds."""
    dag, init, X, want, sizes = readers_case(8, 8, [256 * 1024] * 8, L.BODY_ADD_IOTA_I32, seed=9)
    ctl = [r for r in range(8, dag.ntasks) if dag.tasks["body"][r] == SUM_I64][::2]
    dag.tasks["body"][ctl] = SUM_CTL
    for part_bytes, nparts in ((0, 1), (64 * 1024, 4)):
        e = reader_engine(part_bytes=part_bytes)
        try:
            run = run_engine(e, dag, layout_of(dag, init, sizes))
        finally:
            e.close()
        per = (256 * 1024 // nparts + 15) // 16 * 16
        for r in range(8, dag.ntasks):
            x = X[(r - 8) // 8]
            w = reader_result(SUM_I64, 0, x[:per // 4]) if r in ctl else want[r]
            assert run.res["result"][r] == w, (r, part_bytes)


def test_engine_refusals():
    with Engine(0) as e:
        img = image()
        for sliceable, flags, why in ((0b01, L.LINK_READERS(0b11), "sliceable"), (0xFF, 0x10000, "unknown bit")):
            assert e._lib.pb2_engine_link_bodies_ex(e._h, img, len(img), L.IMAGE_CUBIN, sliceable, 0, flags) == L.PB2_ERR_BAD_PARAM
            msg = (e._lib.pb2_engine_last_error(e._h) or b"").decode()
            assert why in msg, msg
        e.link_bodies(img, L.IMAGE_CUBIN, SLICEABLE, 0, readers=READERS)     # nothing was left behind


# ----------------------------------------------------------------------------------------------------------------------
# a GEMM window linked with PB2_LINK_GEMM_WINDOWS
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("part_bytes", [0, 64 * 1024], ids=["whole", "parts"])
def test_gemm_window(part_bytes):
    K = 128
    dag, ex, sizes, host = ex05_beside_gemm(K)
    t = dag.tasks
    F = ex.meta["F"]
    for k in range(K):
        for j in range(F):
            r = K + k * F + j
            body, dk = reader_spec(j)
            t["body"][r], t["iparam"][r, 0] = body, (k + dk if body != SUM_I64 else 0)
    creaders = list(range(ex.ntasks + 2, dag.ntasks))
    for j, r in enumerate(creaders):
        t["body"][r] = (COUNT_NE, SUM_I64, COUNT_GT, COUNT_NE)[j]
        t["iparam"][r, 0] = (C_WORD, 0, 0, C_WORD + 1)[j]
    runs = []
    for kw in ({}, dict(read_groups=-1)):
        e = reader_engine(gemm_windows=True, part_bytes=part_bytes, **kw)
        try:
            runs.append(run_engine(e, dag, Layout.packed(dag, host=host, valid=True, sizes=sizes)))
        finally:
            e.close()
    assert_same_run(runs[0], runs[1])
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
    """A DTD pool: the linked FILL writes tile i with k_i, then eight linked readers of tile i.  Every reader's result
    as numpy has it, the host data written back."""
    n, F, tb = 64, 8, 256 * 1024
    ks = np.arange(n, dtype=np.int32) * 7 - 100
    host = np.full(n * tb // 4, -1, np.int32)
    with R.Context(cuda_devices=(0,)) as ctx:
        ctx.link_bodies(ctx.devices[0], image(), L.IMAGE_CUBIN, SLICEABLE, readers=READERS)
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
                body, dk = reader_spec(j)
                k = int(ks[i]) + dk if body != SUM_I64 else 0
                readers.append((put(classes[body], i, R.INPUT, k), body, k, i))
        ctx.wait()
        info = ctx.task_info(tp)
        assert ctx.l.pb2_device_memory_release(ctx.devices[0]) == 0
    assert np.array_equal(host.reshape(n, -1), np.repeat(ks[:, None], tb // 4, axis=1))
    for t, body, k, i in readers:
        assert info["result"][t] == reader_result(body, k, np.full(tb // 4, ks[i], np.int32)), (t, body, k, i)
