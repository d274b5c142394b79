"""Window building of the stand-alone runtime (no GPU): a task pool that mixes tile GEMMs with HBM-body tasks is one
engine window, so its edges across the two kinds are released on the device."""
import ctypes as C

import numpy as np

from parsec_b200 import _lib as L
from parsec_b200 import runtime as R
import mixed_pool as P


def pool_edges(ctx, tp):
    """(src, dst) of every dependency edge of the pool, from the runtime's own successor lists via the window arrays
    of a pool whose tasks all fit one window."""
    win = ctx.export_window(tp, ctx.devices[0])
    ids = win["task_ids"].astype(np.int64)
    cnt = win["tasks"]["succ_count"].astype(np.int64)
    src = np.repeat(ids, cnt)
    dst = ids[(win["succ"] & np.uint32(0x07FFFFFF)).astype(np.int64)]
    return win, sorted(zip(src.tolist(), dst.tolist()))


def dtd_edges(ids, NT):
    """The edges the DTD rule gives the mixed pool: FILL -> first GEMM -> ... -> last GEMM -> CHECK on each C tile
    (A, B, X are only read, every Y has one writer)."""
    e = []
    for i in range(NT):
        for j in range(NT):
            chain = [ids[("fill", i, j)]] + [ids[("gemm", i, j, k)] for k in range(NT)] + [ids[("check", i, j)]]
            e += list(zip(chain[:-1], chain[1:]))
    return sorted(e)


def test_mixed_pool_is_one_window():
    NT, T = 3, 64
    data = P.Data(NT, T)
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        tp, ids = P.insert(ctx, data)
        n = ctx.l.pb2_taskpool_nb_tasks(tp)
        assert n == P.ntasks(NT)
        win, edges = pool_edges(ctx, tp)
        # one window holds every task, the GEMMs and the HBM bodies together
        assert sorted(win["task_ids"].tolist()) == list(range(n))
        bodies = win["tasks"]["body"]
        assert np.count_nonzero(bodies == L.BODY_GEMM_BF16) == NT ** 3
        assert np.count_nonzero(bodies == L.BODY_FILL_I32) == NT * NT
        assert np.count_nonzero(bodies == L.BODY_CHECK_I32) == NT * NT
        assert np.count_nonzero(bodies == L.BODY_AXPY_F32) == NT * NT
        # its successor lists are the pool's edges, its ready tasks the pool's tasks without predecessor
        assert edges == dtd_edges(ids, NT)
        roots = sorted([ids[("fill", i, j)] for i in range(NT) for j in range(NT)] +
                       [ids[("axpy", i, j)] for i in range(NT) for j in range(NT)])
        assert sorted(win["task_ids"][win["ready"]].tolist()) == roots
        assert len(win["ready"]) == P.nready(NT)
        # in-window dependency goals: what each task still waits for inside the window
        indeg = np.bincount([d for _, d in edges], minlength=n)
        assert np.array_equal(win["tasks"]["dep_goal"], indeg[win["task_ids"]])


def test_mixed_pool_runs_in_one_dry_run_window():
    """Run to completion in dry-run mode: one window, every edge of the pool released on the device."""
    NT, T = 2, 64
    data = P.Data(NT, T)
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        tp, ids = P.insert(ctx, data)
        ctx.wait()
        st = ctx.stats(ctx.devices[0])
        t, dev = ctx.trace(tp)
    assert sorted(t.tolist()) == list(range(P.ntasks(NT))) and np.all(dev == 2)
    assert st["windows_launched"] == 1 and st["executed_tasks"] == P.ntasks(NT)
    assert st["tasks_released_on_device"] == P.ntasks(NT) - P.nready(NT)


def test_cholesky_shape_pool_is_one_window():
    """pb2_ptg_cholesky_shape_new: its POTRF stand-ins are NOP (an HBM body) and everything else is GEMM.  The first
    ready task is POTRF(0), and the whole pool is one GEMM-kind window: every edge, NOP -> GEMM included, is released on
    the device."""
    NT, nb = 6, 64
    bits = np.zeros(NT * NT * nb * nb, np.uint16)
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        dc = ctx.block_cyclic(2, nb, nb, NT * nb, NT * nb, mat=bits)
        tp = C.c_void_p(ctx.l.pb2_ptg_cholesky_shape_new(ctx.h, dc, NT))
        n = ctx.l.pb2_taskpool_nb_tasks(tp)
        win = ctx.export_window(tp, ctx.devices[0])
        assert sorted(win["task_ids"].tolist()) == list(range(n))
        assert np.count_nonzero(win["tasks"]["body"] == L.BODY_NOP) == NT
        assert len(win["ready"]) == 1 and win["tasks"]["body"][win["ready"][0]] == L.BODY_NOP
        ctx.wait()
        st = ctx.stats(ctx.devices[0])
    assert st["windows_launched"] == 1 and st["executed_tasks"] == n
    assert st["tasks_released_on_device"] == n - 1


def test_user_submit_task_still_splits_a_mixed_pool():
    """A user submit task between engine tasks still runs in the host-driven lane of its own: FILL -> GEMM (engine)
    -> user -> CHECK (engine) is three windows."""
    T = 64
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        cb = R.GPU_SUBMIT(lambda d, g, s: 0)
        tp = C.c_void_p(ctx.l.pb2_dtd_taskpool_new(ctx.h))
        nc = lambda nf: C.c_void_p(ctx.l.pb2_dtd_create_task_class(tp, b"k", nf, np.array([R.INOUT] * nf, np.int32).ctypes.data_as(C.c_void_p)))
        fill, gemm, user, chk = nc(1), nc(3), nc(1), nc(1)
        assert ctx.l.pb2_dtd_task_class_add_chore(tp, fill, R.DEV_CUDA, L.BODY_FILL_I32, None) == 0
        assert ctx.l.pb2_dtd_task_class_add_chore(tp, gemm, R.DEV_CUDA, L.BODY_GEMM_BF16, None) == 0
        assert ctx.l.pb2_dtd_task_class_add_submit(tp, user, cb) == 0
        assert ctx.l.pb2_dtd_task_class_add_chore(tp, chk, R.DEV_CUDA, L.BODY_CHECK_I32, None) == 0
        a, b, c = (C.c_void_p(ctx.l.pb2_dtd_tile_new(tp, T * T * 2)) for _ in range(3))
        p = lambda *v: np.array(v, np.int32).ctypes.data_as(C.c_void_p)
        ctx.l.pb2_dtd_insert_task_with_task_class(tp, fill, 0, R.DEV_CUDA, (C.c_void_p * 1)(c), p(R.OUTPUT), p(P.ONES, 0, 0), 0.0)
        ctx.l.pb2_dtd_insert_task_with_task_class(tp, gemm, 0, R.DEV_CUDA, (C.c_void_p * 3)(a, b, c),
                                                  p(R.INPUT, R.INPUT, R.INOUT), p(T, T, T), 0.0)
        ctx.l.pb2_dtd_insert_task_with_task_class(tp, user, 0, R.DEV_CUDA, (C.c_void_p * 1)(c), p(R.INOUT), p(1, 0, 0), 0.0)
        ctx.l.pb2_dtd_insert_task_with_task_class(tp, chk, 0, R.DEV_CUDA, (C.c_void_p * 1)(c), p(R.INPUT), p(0, 0, 0), 0.0)
        ctx.wait()
        st = ctx.stats(ctx.devices[0])
        t, _ = ctx.trace(tp)
    assert st["executed_tasks"] == 4 and st["windows_launched"] == 3
    assert t.tolist() == [0, 1, 2, 3]
