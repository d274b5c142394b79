"""GEMM-worker bodies (PB2_LINK_GEMM_BODIES) on the H100: the application's bodies that get the GEMM worker's operand
ring as shared memory, in GEMM windows beside the built-in bf16 GEMM units.

  - the fp64 DTD GEMM (tests/fp64_gemm.py) through the fixture's DMMA tile body, on the engine and through the
    stand-alone runtime: every C tile within the float64 bound of NumPy's, the k-order in the seen versions, the same
    bits from a second run;
  - the ring hazard: ring probes between the units of bf16 GEMM chains on one worker and on all, with fp64 tasks
    beside them: the bf16 C tiles bit for bit those of the window without them, every probe clean;
  - queue_policy 1 and traced windows, whose part records show one part per GEMM-worker task;
  - the refusals: HBM windows, shared windows and engines without an image.
The host side is tests/test_gemm_worker_bodies.py."""
import numpy as np
import pytest

from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200 import runtime as R
from parsec_b200.bf16 import f32_to_bf16_bits
from parsec_b200.engine import Engine
import fp64_gemm as F
from window_harness import Layout, placed, run_engine

pytestmark = pytest.mark.gpu


def linked_engine(fmt=L.IMAGE_CUBIN, **kw):
    e = Engine(0, timeout_ms=20000, **kw)
    e.link_bodies(F.image(fmt), fmt, 0, gemm_windows=True, gemm_bodies=F.GEMM_BODIES)
    info = e.linked_gemm_info()
    print("linked GEMM kernel with the GEMM-worker bodies (%s): %s" % (kw, info))
    assert info["regs"] <= 168 and 0 < info["nworkers"] <= e.info()["nworkers_gemm"]
    return e


def fp64_layout(dag, sizes, t):
    host = np.concatenate([x.reshape(-1) for x in t]).view(np.uint8)
    return Layout.packed(dag, host=host, valid=True, sizes=sizes)


def c_tile(run, layout, tid, M, N):
    return layout.tile_bytes(run.dev, tid).view(np.float64).reshape(M, N)


def check_fp64(run, layout, t, NT, M, N, base=0, ctile0=None):
    """Every C tile of the fp64 DAG (task ids from base, C tile ids from ctile0) against NumPy, and the k-order."""
    ctile0 = 2 * NT * NT if ctile0 is None else ctile0
    for i in range(NT):
        for j in range(NT):
            want, bound = F.reference(t, NT, i, j)
            got = c_tile(run, layout, ctile0 + i * NT + j, M, N)
            err = np.abs(got - want)
            assert np.all(err <= bound), (i, j, float(err.max()), float(bound.min()))
    ids = base + np.arange(NT ** 3)
    k = np.arange(NT ** 3) % NT
    assert np.array_equal(run.res["seen_version"][ids, 2], k), "C versions seen out of k-order"
    assert not np.any(run.res["seen_version"][ids, :2]) and not np.any(run.res["result"][ids])


SHAPES = [(4, 256, 256, 256), (3, 200, 150, 99), (2, 130, 50, 40)]


@pytest.mark.parametrize("NT,M,N,K", SHAPES, ids=["nt4_256", "ragged_odd_k", "ragged_even_k"])
def test_fp64_dtd_gemm_on_the_engine(NT, M, N, K):
    dag, sizes = F.dag(NT, M, N, K)
    t = F.tiles(NT, M, N, K)
    layout = fp64_layout(dag, sizes, t)
    e = linked_engine()
    try:
        a = run_engine(e, dag, layout)
        b = run_engine(e, dag, layout)
    finally:
        e.close()
    check_fp64(a, layout, t, NT, M, N)
    assert np.array_equal(a.dev, b.dev) and np.array_equal(a.host, b.host), "a second run gave other bits"
    # the last k of every chain pushed C(i,j) out to its host home
    for c in range(2 * NT * NT, 3 * NT * NT):
        o = int(layout.hoff[c])
        assert np.array_equal(a.host[o:o + int(sizes[c])], layout.tile_bytes(a.dev, c))


def test_fp64_dtd_gemm_through_the_runtime():
    """The same pool as DTD tasks whose chore names the linked id: every window it runs in is a GEMM window (an HBM
    window refuses a GEMM-worker body, which would fail the pool)."""
    NT, M, N, K = 3, 256, 192, 128
    t = F.tiles(NT, M, N, K)
    with R.Context(cuda_devices=(0,)) as ctx:
        ctx.link_bodies(ctx.devices[0], F.image(), L.IMAGE_CUBIN, 0, gemm_windows=True, gemm_bodies=F.GEMM_BODIES)
        tp, bufs = F.insert(ctx, NT, M, N, K, t)
        ctx.wait()
        st = ctx.stats(ctx.devices[0])
        info = ctx.task_info(tp)
        assert ctx.l.pb2_device_memory_release(ctx.devices[0]) == 0
    assert st["executed_tasks"] == NT ** 3
    assert not np.any(info["result"])
    for i in range(NT):
        for j in range(NT):
            want, bound = F.reference(t, NT, i, j)
            got = F.runtime_tile(bufs, "C", i, j, NT, M, N)
            assert np.all(np.abs(got - want) <= bound), (i, j)


# ----------------------------------------------------------------------------------------------------------------------
# the ring hazard
# ----------------------------------------------------------------------------------------------------------------------
def hazard_dag(NT=3, T=256, fNT=2, fM=96, fN=80, fK=72):
    """bf16 dtd_gemm(NT, T) chains serialised through ring probes: chain c's last task releases probe c, which releases
    the head of chain c + 1, so a probe overwrites the ring between two chains' units on whatever worker runs them.
    Beside them, the fp64 dtd_gemm(fNT) on tiles of its own, ready at start.  Returns (dag, sizes, ids of the probes,
    first fp64 task, first fp64 tile)."""
    g = dags.dtd_gemm(NT, tile=T)
    f, fsizes = F.dag(fNT, fM, fN, fK)
    nchain, n0, t0 = NT * NT, g.ntasks, g.ntiles
    probes = n0 + np.arange(nchain)
    fbase = n0 + nchain
    tasks = np.concatenate([g.tasks, dags._new_tasks(nchain), f.tasks])
    p = tasks[n0:fbase]
    p["body"], p["dep_goal"], p["iparam"][:, 0], p["iparam"][:, 1] = F.PROBE, 1, np.arange(nchain), 7
    ft = tasks[fbase:]
    ft["tile"][:, :3] += t0
    edges = [(int(s), int(d), int(fl)) for s, d, fl in zip(*g.edges())]
    edges += [(int(s) + fbase, int(d) + fbase, int(fl)) for s, d, fl in zip(*f.edges())]
    heads = [c * NT for c in range(nchain)]                     # task (i, j, 0) of chain c = i * NT + j
    for c in range(nchain):
        edges.append((heads[c] + NT - 1, int(probes[c]), 0))
        if c + 1 < nchain:
            edges.append((int(probes[c]), heads[c + 1], 0))
            tasks["dep_goal"][heads[c + 1]] = 1
    src, dst, fl = (np.array(x, np.int64) for x in zip(*edges))
    begin, count, succ = dags._csr_from_edges(len(tasks), src, dst, fl)
    tasks["succ_begin"], tasks["succ_count"] = begin, count
    ready = np.array([heads[0]] + list(fbase + f.ready), np.int32)
    sizes = np.concatenate([np.full(t0, T * T * 2, np.int64), fsizes])
    dag = dags.Dag(tasks, succ, ready, ntiles=t0 + f.ntiles, tile_bytes=0, kind=1, name="ring_hazard")
    return dag, sizes, probes, fbase, t0


def bf16_host(NT, T, seed=11):
    rng = np.random.default_rng(seed)
    return f32_to_bf16_bits(rng.uniform(-1, 1, 3 * NT * NT * T * T).astype(np.float32)).view(np.uint8)


@pytest.mark.parametrize("max_workers", [1, 0], ids=["one_worker", "all_workers"])
def test_probes_between_gemm_units_leave_the_bf16_results_unchanged(max_workers):
    NT, T, fNT, fM, fN, fK = 3, 256, 2, 96, 80, 72
    dag, sizes, probes, fbase, t0 = hazard_dag(NT, T, fNT, fM, fN, fK)
    ft = F.tiles(fNT, fM, fN, fK)
    host = np.concatenate([bf16_host(NT, T)] + [x.reshape(-1).view(np.uint8) for x in ft])
    layout = Layout.packed(dag, host=host, valid=True, sizes=sizes)
    plain = dags.dtd_gemm(NT, tile=T)
    plain_layout = Layout.packed(plain, host=bf16_host(NT, T), valid=True)
    with Engine(0) as e:
        want = run_engine(e, plain, plain_layout)
    e = linked_engine(max_workers=max_workers)
    try:
        got = run_engine(e, dag, layout)
    finally:
        e.close()
    for c in range(2 * NT * NT, 3 * NT * NT):
        assert np.array_equal(layout.tile_bytes(got.dev, c), plain_layout.tile_bytes(want.dev, c)), c
    assert np.array_equal(got.res["result"][probes], np.zeros(len(probes), np.uint64)), got.res["result"][probes]
    assert np.array_equal(got.res["seen_version"][:NT ** 3], want.res["seen_version"])
    check_fp64(got, layout, ft, fNT, fM, fN, base=fbase, ctile0=t0 + 2 * fNT * fNT)
    if max_workers == 1:                            # chain, probe, chain, ... on the one worker
        order = got.res["retire_order"]
        pos = {int(x): i for i, x in enumerate(order)}
        for c in range(NT * NT - 1):
            assert pos[c * NT + NT - 1] < pos[int(probes[c])] < pos[(c + 1) * NT]


# ----------------------------------------------------------------------------------------------------------------------
# variants and refusals
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("queue_policy", [0, 1])
def test_traced_and_priority_windows(queue_policy):
    NT, M, N, K = 3, 128, 128, 64
    dag, sizes = F.dag(NT, M, N, K)
    t = F.tiles(NT, M, N, K)
    layout = fp64_layout(dag, sizes, t)
    e = linked_engine(queue_policy=queue_policy, part_bytes=4096)
    try:
        with placed(e, layout) as p:
            e.set_window_trace(True)
            try:
                w = e.window(dag.kind, dag.tasks, dag.succ, p.tiles, dag.ready)
            finally:
                e.set_window_trace(False)
            try:
                st = w.run()
                res = w.results()
                parts = w.part_trace()
            finally:
                w.close()
        run = p.run(st, res, images=(p.dev, p.host))
    finally:
        e.close()
    check_fp64(run, layout, t, NT, M, N)
    # one record per task, part 0 of 1, although part_bytes would cut 128 KiB tiles into 32 parts
    assert sorted(parts["task"].tolist()) == list(range(NT ** 3))
    assert np.all(parts["part"] == 0) and np.all(parts["nparts"] == 1)
    assert np.all(parts["t_exec_ns"] >= parts["t_in_ns"]) and np.all(parts["t_in_ns"] >= parts["t_pop_ns"])


def test_refusals():
    dag, sizes = F.dag(2, 64, 64, 64)
    layout = fp64_layout(dag, sizes, F.tiles(2, 64, 64, 64))
    e = linked_engine()
    try:
        with placed(e, layout) as p:
            with pytest.raises(L.Pb2Error) as ex:
                e.window(0, dag.tasks, dag.succ, p.tiles, dag.ready)
            assert ex.value.rc == L.PB2_ERR_NOT_SUPPORTED and "HBM window" in str(ex.value)
            e.set_shared_windows(True)
            with pytest.raises(L.Pb2Error) as ex:
                e.window(1, dag.tasks, dag.succ, p.tiles, dag.ready)
            assert ex.value.rc == L.PB2_ERR_NOT_SUPPORTED and "shared window" in str(ex.value)
            e.set_shared_windows(False)
    finally:
        e.close()
    with Engine(0) as e, placed(e, layout) as p:
        with pytest.raises(L.Pb2Error) as ex:
            e.window(1, dag.tasks, dag.succ, p.tiles, dag.ready)
        assert ex.value.rc == L.PB2_ERR_NOT_SUPPORTED and "linked body in a GEMM window" in str(ex.value)
        with pytest.raises(L.Pb2Error) as ex:
            e.window(0, dag.tasks, dag.succ, p.tiles, dag.ready)
        assert ex.value.rc == L.PB2_ERR_NOT_SUPPORTED and "has not linked an image" in str(ex.value)
