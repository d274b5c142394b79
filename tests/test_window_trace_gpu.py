"""Device time stamps of engine windows (pb2_engine_set_window_trace, pb2_window_trace) on the H100.

A traced window must compute bit for bit what the same window computes untraced, and its trace must be consistent with
the DAG: every task has 0 < t_start <= t_end on an existing SM, the tasks of one scheduling entity (read group, fused
producer unit, GEMM unit) share one interval, and across every edge u -> v between different entities v starts no
earlier than u ended.  %globaltimer is read on different SMs and may advance in steps of about a microsecond, so that
last check allows TOL_NS."""
import ctypes as C

import numpy as np
import pytest

from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200 import runtime as R
from parsec_b200.engine import Engine
from window_harness import Layout, assert_same_run, placed, run_engine
from test_priority import random_dag
from test_rearm_gpu import gemm_chains_dag

pytestmark = pytest.mark.gpu

TOL_NS = 2000


def groups_dag(seed, n_rmw=300, ngroups=24, tile_bytes=64 * 1024):
    """A random DAG with read groups and fusable producers: the read-modify-write tasks of test_priority.random_dag on
    six tiles, each also waiting for the previous writer of its tile (so that every run computes the same thing), and
    ngroups broadcasts, each a FILL producer of a tile of its own (released by a random RMW task, or ready) followed by
    2..8 CHECK readers of that tile (one of which may fail), whose last reader releases a later RMW task.  Counter
    dependency words."""
    rng = np.random.default_rng(seed)
    base = random_dag(n_rmw, seed, 1, tile_bytes=tile_bytes)
    bt = base.tasks
    src, dst, _ = base.edges()
    edges = set(zip(src.tolist(), dst.tolist()))
    last = {}
    for j in range(n_rmw):
        x = int(bt["tile"][j, 0])
        if x in last:
            edges.add((last[x], j))
        last[x] = j
    edges = sorted(edges)
    src, dst = [e[0] for e in edges], [e[1] for e in edges]
    rows = []                       # (body, tile, access, k)
    for g in range(ngroups):
        tile = 6 + g
        k = int(rng.integers(0, 1000))
        p = n_rmw + len(rows)
        rows.append((L.BODY_FILL_I32, tile, L.ACCESS_WRITE, k))
        a = int(rng.integers(0, n_rmw - 1)) if rng.random() < 0.5 else -1
        if a >= 0:
            src.append(a); dst.append(p)
        nr = int(rng.integers(2, 9))
        for i in range(nr):
            kk = k + 1 if (i == nr - 1 and rng.random() < 0.3) else k
            src.append(p); dst.append(n_rmw + len(rows))
            rows.append((L.BODY_CHECK_I32, tile, L.ACCESS_READ, kk))
        b = int(rng.integers(max(a, 0) + 1, n_rmw))
        src.append(n_rmw + len(rows) - 1); dst.append(b)
    n = n_rmw + len(rows)
    t = dags._new_tasks(n)
    t[:n_rmw] = bt
    for i, (body, tile, acc, k) in enumerate(rows):
        j = n_rmw + i
        t["body"][j], t["nb_flows"][j], t["tile"][j, 0], t["access"][j, 0], t["iparam"][j, 0] = body, 1, tile, acc, k
    t["priority"] = 0
    src, dst = np.array(src, np.int64), np.array(dst, np.int64)
    begin, count, succ = dags._csr_from_edges(n, src, dst, np.zeros(len(src), np.int64))
    t["succ_begin"], t["succ_count"] = begin, count
    t["dep_goal"] = np.bincount(dst, minlength=n)
    t["flags"] = 0
    ready = np.flatnonzero(t["dep_goal"] == 0).astype(np.int32)
    return dags.Dag(t, succ, ready, ntiles=6 + ngroups, tile_bytes=tile_bytes, name="groups")


def check_trace(dag, tr, sm_count, what):
    t0, t1, sm, unit = (tr[k].astype(np.int64) for k in ("t_start_ns", "t_end_ns", "smid", "unit"))
    assert np.all(t0 > 0) and np.all(t0 <= t1), what
    assert np.all(sm < sm_count), what
    # one interval and one SM per entity: the entity's leader holds them
    assert np.all(unit >= 0) and np.all(unit < dag.ntasks) and np.all(unit[unit] == unit), what
    for a in (t0, t1, sm):
        assert np.array_equal(a, a[unit]), what
    src, dst, _ = dag.edges()
    cross = unit[src] != unit[dst]
    gap = t0[dst[cross]] - t1[src[cross]]
    worst = int(gap.min()) if len(gap) else 0
    print("%s: %d tasks, %d entities, %d cross-entity edges, largest negative gap %d ns (tol %d)"
          % (what, dag.ntasks, len(np.unique(unit)), int(cross.sum()), min(worst, 0), TOL_NS))
    assert worst >= -TOL_NS, what
    return unit


def run_twice(e, dag, host):
    """The window over tiles resident in HBM (holding host), untraced and traced: both compute the same thing, in an
    order that respects every edge.  Returns the traced run."""
    plain = run_engine(e, dag, Layout.contiguous(dag, dev=host))
    traced = run_engine(e, dag, Layout.contiguous(dag, dev=host), trace=True)
    assert_same_run(plain, traced)
    assert traced.stats["tasks_retired"] == dag.ntasks
    assert all(v == 0 for v in dags.check_execution(dag, traced.res).values())     # end_seq[u] < start_seq[v] on every edge
    return traced


@pytest.mark.parametrize("seed,part_bytes,queue_policy", [(1, 0, 0), (2, 16 * 1024, 0), (3, 0, 1), (4, 16 * 1024, 1)])
def test_random_hbm_dags_with_groups(seed, part_bytes, queue_policy):
    dag = groups_dag(seed)
    host = np.random.default_rng(seed).integers(-100, 100, dag.ntiles * dag.tile_bytes // 4).astype(np.int32)
    with Engine(0, part_bytes=part_bytes, queue_policy=queue_policy) as e:
        traced = run_twice(e, dag, host)
        sm_count = e.info()["sm_count"]
    unit = check_trace(dag, traced.traces[0], sm_count, "groups seed %d part_bytes %d policy %d" % (seed, part_bytes, queue_policy))
    # every producer runs fused with its readers and leads them
    fills = np.flatnonzero(dag.tasks["body"] == L.BODY_FILL_I32)
    readers = np.flatnonzero(dag.tasks["body"] == L.BODY_CHECK_I32)
    assert np.all(unit[fills] == fills)
    assert np.all(np.isin(unit[readers], fills))


@pytest.mark.parametrize("fuse_readers", [0, -1], ids=["fused", "groups_only"])
def test_ex05_window(fuse_readers):
    dag = dags.ex05_broadcast(256, 14, 256 * 1024)
    host = np.full(dag.ntiles * dag.tile_bytes // 4, -1, np.int32)
    with Engine(0, fuse_readers=fuse_readers) as e:
        traced = run_twice(e, dag, host)
        sm_count = e.info()["sm_count"]
    K, F = 256, dag.meta["F"]
    unit = check_trace(dag, traced.traces[0], sm_count, "ex05 fuse_readers %d" % fuse_readers)
    lead = np.repeat(np.arange(K), F) if fuse_readers == 0 else K + np.repeat(np.arange(K) * F, F)
    assert np.array_equal(unit[K:], lead)


@pytest.mark.parametrize("gemm_mode,queue_policy", [(0, 0), (2, 0), (0, 1)])
@pytest.mark.parametrize("make", [gemm_chains_dag, lambda: dags.dtd_gemm(3, 256)], ids=["chains", "dtd_gemm"])
def test_gemm_window(make, gemm_mode, queue_policy):
    dag = make()
    dag.tasks["access"] &= ~np.uint8(L.FLOW_PUSHOUT)             # tiles stay resident
    if "host" not in dag.meta:
        rng = np.random.default_rng(5)
        bits = (rng.integers(-64, 64, dag.ntiles * dag.tile_bytes // 2) * 0x10 + 0x3C00).astype(np.uint16)   # small bf16
        dag.meta["host"] = bits.view(np.int32)
    with Engine(0, gemm_mode=gemm_mode, queue_policy=queue_policy, part_bytes=32 * 1024) as e:
        traced = run_twice(e, dag, dag.meta["host"])
        sm_count = e.info()["sm_count"]
    unit = check_trace(dag, traced.traces[0], sm_count, "gemm mode %d policy %d" % (gemm_mode, queue_policy))
    gemm = dag.tasks["body"] == L.BODY_GEMM_BF16
    fused = int(np.sum(unit[gemm] != np.flatnonzero(gemm)))
    if gemm_mode == 2:
        assert np.array_equal(unit, np.arange(dag.ntasks))       # every task its own unit
    else:
        assert fused > 0                                         # k-chains share their first task's interval


def test_rearmed_window_reads_the_copy_each_launch_used():
    dag = groups_dag(9)
    host = np.random.default_rng(9).integers(-100, 100, dag.ntiles * dag.tile_bytes // 4).astype(np.int32)
    with Engine(0) as e:
        traces = run_engine(e, dag, Layout.contiguous(dag, dev=host), launches=3, trace=True).traces
        sm_count = e.info()["sm_count"]
    prev_end = 0
    for i, tr in enumerate(traces):
        check_trace(dag, tr, sm_count, "launch %d" % i)
        assert int(tr["t_start_ns"].min()) > prev_end, i
        prev_end = int(tr["t_end_ns"].max())


def test_untraced_window_refuses_trace():
    dag = dags.ex05_broadcast(4, 2, 4096)
    with Engine(0) as e, placed(e, Layout.contiguous(dag)) as p:
        w = e.window(0, dag.tasks, dag.succ, p.tiles, dag.ready)
        w.run()
        with pytest.raises(L.Pb2Error) as exc:
            w.trace()
        assert exc.value.rc == L.PB2_ERR_NOT_SUPPORTED and "without trace" in str(exc.value)
        w.close()


@pytest.mark.parametrize("max_workers", [0, 1], ids=["fused", "one_worker"])
def test_runtime_ex05_pool_device_trace(max_workers):
    """Every TaskRecv(k, .) starts no earlier than TaskBcast(k) ended, unless it ran in one fused unit with it: then it
    has TaskBcast(k)'s interval and SM.  With one worker the engine does not fuse (the read groups stay), so every
    receiver is checked against the end of its broadcast."""
    K, NB, tb = 64, 6, 64 * 1024
    host = np.full(K * tb // 4, -1, np.int32)
    with R.Context(cuda_devices=(0,), mca={"device_engine_trace": 1, "device_engine_max_workers": max_workers}) as ctx:
        dc = ctx.block_cyclic(4, tb // 4, 1, K * tb // 4, 1, mat=host)
        tp = C.c_void_p(ctx.l.pb2_ptg_ex05_broadcast_new(ctx.h, dc, K, NB))
        ctx.wait()
        info = ctx.task_info(tp)
        tr = ctx.device_trace(tp)
        gpu = ctx.l.pb2_device_index(ctx.devices[0])
    n = len(info["class_id"])
    assert n == K * (1 + NB // 2 + 1)
    assert np.all(tr["device"] == gpu)
    t0, t1, sm = (tr[k].astype(np.int64) for k in ("t_start_ns", "t_end_ns", "smid"))
    assert np.all(t0 > 0) and np.all(t0 <= t1)
    bcast = np.flatnonzero(info["class_id"] == 0)
    recv = np.flatnonzero(info["class_id"] == 1)
    of = np.zeros(K, np.int64)
    of[info["locals"][bcast, 0]] = bcast
    b = of[info["locals"][recv, 0]]                           # TaskBcast(k) of each TaskRecv(k, .)
    fused = (t0[recv] == t0[b]) & (t1[recv] == t1[b]) & (sm[recv] == sm[b])
    gap = t0[recv] - t1[b]
    worst = int(gap[~fused].min()) if np.any(~fused) else 0
    print("runtime Ex05 max_workers %d: %d tasks, %d receivers fused with their broadcast, largest negative "
          "TaskBcast -> TaskRecv gap of the others %d ns (tol %d)" % (max_workers, n, int(fused.sum()), min(worst, 0), TOL_NS))
    assert worst >= -TOL_NS
    if max_workers == 1:
        assert not np.any(fused & (t1[b] > t0[b]))
    assert np.all(info["result"][recv] == info["locals"][recv, 0].astype(np.uint64))
