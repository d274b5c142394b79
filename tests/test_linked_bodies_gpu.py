"""Application device bodies linked into HBM windows (pb2_engine_link_bodies) on the H100.

The bodies are those of tests/cuda/linked_bodies.cu, built by the Makefile into a relocatable sm_90a cubin and PTX:
LINKED_0 y = m x + b (sliceable), LINKED_1 a 3-point halo stencil over whole tiles, LINKED_2 a CTA sum through the
scratch words (sliceable).  Every output is integer, so numpy replays it bit for bit.  Flow versions and results do not
depend on what a body computes: they must equal the oracle's for the same DAG with each linked task replaced by an
INCR of 0."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200 import runtime as R
from parsec_b200.bf16 import bf16_bits_to_f32
from parsec_b200.engine import Engine
from window_harness import Layout, assert_same_run, placed, run_engine, run_oracle
from test_part_trace_gpu import check_parts, run_traced
from test_window_trace_gpu import groups_dag
from test_linked_bodies import insert_linked, int32_collection
import mixed_pool as P

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
AXPB, STENCIL, SUM = L.BODY_LINKED_0, L.BODY_LINKED_0 + 1, L.BODY_LINKED_0 + 2
SLICEABLE = (1 << 0) | (1 << 2)                 # AXPB and SUM; the stencil runs over whole tiles


def image(fmt):
    with open(os.path.join(HERE, "cuda", "linked_bodies." + ("ptx" if fmt == L.IMAGE_PTX else "cubin")), "rb") as f:
        return f.read()


def linked_engine(fmt=L.IMAGE_CUBIN, **kw):
    e = Engine(0, **kw)
    e.link_bodies(image(fmt), fmt, SLICEABLE)
    info = e.linked_info()
    print("linked kernel (%s, queue_policy %d): %s" % ("PTX" if fmt == L.IMAGE_PTX else "cubin", kw.get("queue_policy", 0), info))
    assert info["regs"] > 0 and 0 < info["nworkers"] <= e.info()["nworkers"]
    return e


# ----------------------------------------------------------------------------------------------------------------------
# random HBM DAGs: built-in bodies and LINKED_0 together
# ----------------------------------------------------------------------------------------------------------------------
def with_linked(dag, seed, naxpb=24):
    """dag (test_window_trace_gpu.groups_dag: RMW tasks on tiles 0-5, FILL + CHECK groups on their own tiles) with naxpb
    AXPB tasks.  AXPB q reads RMW tile X after RMW task j has written it, writes a fresh tile Y_q, and holds back the
    next writer of X (write after read); an INCR of Y_q follows it.  Returns the DAG and the linked task ids."""
    rng = np.random.default_rng(seed + 1000)
    t0 = dag.tasks
    src, dst, _ = dag.edges()
    src, dst = src.tolist(), dst.tolist()
    n0, nrmw = dag.ntasks, int(np.count_nonzero(np.isin(t0["body"], [L.BODY_INCR_I32, L.BODY_SCALE_I32, L.BODY_ADD_IOTA_I32])))
    t = dags._new_tasks(n0 + 2 * naxpb)
    t[:n0] = t0
    linked = []
    for q in range(naxpb):
        j = int(rng.integers(0, nrmw))
        x = int(t0["tile"][j, 0])
        later = [i for i in range(j + 1, nrmw) if int(t0["tile"][i, 0]) == x]
        a, inc, y = n0 + 2 * q, n0 + 2 * q + 1, dag.ntiles + q
        t["body"][a], t["nb_flows"][a] = AXPB, 2
        t["tile"][a, :2], t["access"][a, :2] = (x, y), (L.ACCESS_READ, L.ACCESS_WRITE)
        t["iparam"][a, :2] = (int(rng.integers(-9, 10)), int(rng.integers(-1000, 1000)))
        t["body"][inc], t["nb_flows"][inc], t["tile"][inc, 0], t["access"][inc, 0] = L.BODY_INCR_I32, 1, y, L.ACCESS_RW
        t["iparam"][inc, 0] = int(rng.integers(-5, 6))
        src += [j, a]; dst += [a, inc]
        if later:
            src.append(a); dst.append(later[0])
        linked.append(a)
    src, dst = np.array(src, np.int64), np.array(dst, np.int64)
    t["succ_begin"], t["succ_count"], succ = dags._csr_from_edges(len(t), src, dst, np.zeros(len(src), np.int64))
    t["dep_goal"] = np.bincount(dst, minlength=len(t))
    ready = np.flatnonzero(t["dep_goal"] == 0).astype(np.int32)
    out = dags.Dag(t, succ, ready, ntiles=dag.ntiles + naxpb, tile_bytes=dag.tile_bytes, name="linked_" + dag.name)
    return out, np.array(linked, np.int64)


def with_pushout(dag):
    """Every written flow of every task but the FILL producers (which stay fusable) pushed out to its host home."""
    t = dag.tasks.copy()
    for i in np.flatnonzero(t["body"] != L.BODY_FILL_I32):
        for f in range(int(t["nb_flows"][i])):
            if t["tile"][i, f] >= 0 and t["access"][i, f] & L.ACCESS_WRITE:
                t["access"][i, f] |= L.FLOW_PUSHOUT
    return dags.Dag(t, dag.succ, dag.ready, ntiles=dag.ntiles, tile_bytes=dag.tile_bytes, name=dag.name + "_pushout")


def replay(dag, start):
    """The tiles after dag, every task applied in a topological order to int32 tiles that start as `start`."""
    tiles = start.view(np.int32).reshape(dag.ntiles, -1).copy()
    idx = np.arange(tiles.shape[1], dtype=np.int64)
    src, dst, _ = dag.edges()
    indeg = np.bincount(dst, minlength=dag.ntasks)
    ready = list(np.flatnonzero(indeg == 0))
    t = dag.tasks
    with np.errstate(over="ignore"):
        while ready:
            i = int(ready.pop())
            b, tl, k = int(t["body"][i]), t["tile"][i], t["iparam"][i]
            x = tiles[tl[0]]
            if b == L.BODY_FILL_I32:
                x[:] = k[0]
            elif b == L.BODY_INCR_I32:
                x += np.int32(k[0])
            elif b == L.BODY_SCALE_I32:
                x *= np.int32(k[0])
            elif b == L.BODY_ADD_IOTA_I32:
                x += idx.astype(np.int32)
            elif b == AXPB:
                tiles[tl[1]] = x * np.int32(k[0]) + np.int32(k[1])
            else:
                assert b == L.BODY_CHECK_I32
            for s in dag.succ[t["succ_begin"][i]:t["succ_begin"][i] + t["succ_count"][i]]:
                s = int(s) & 0x7FFFFFF
                indeg[s] -= 1
                if indeg[s] == 0:
                    ready.append(s)
    return tiles.view(np.uint8).reshape(-1)


def as_incr(dag):
    """The same DAG with every linked task an INCR of 0 (the oracle runs built-in bodies only)."""
    t = dag.tasks.copy()
    lk = (t["body"] >= L.BODY_LINKED_0) & (t["body"] <= L.BODY_LINKED_7)
    t["body"][lk], t["iparam"][lk] = L.BODY_INCR_I32, 0
    return dags.Dag(t, dag.succ, dag.ready, ntiles=dag.ntiles, tile_bytes=dag.tile_bytes, name=dag.name + "_incr")


def layout_of(dag, host, staged, pushout):
    if staged:
        return Layout.contiguous(dag, host=host, valid=False)
    return Layout.contiguous(dag, host=host, valid=True) if pushout else Layout.contiguous(dag, dev=host)


def random_case(seed, pushout):
    dag, linked = with_linked(groups_dag(seed), seed)
    if pushout:
        dag = with_pushout(dag)
    host = np.random.default_rng(seed).integers(-100, 100, dag.ntiles * dag.tile_bytes // 4).astype(np.int32)
    return dag, linked, host


def check_against_replay(dag, run, host, staged, pushout):
    want = replay(dag, host.view(np.uint8))
    assert np.array_equal(run.dev, want), "slab image differs from the numpy replay"
    if pushout:
        t = dag.tasks
        pushed = np.unique(t["tile"][(t["access"] & L.FLOW_PUSHOUT) != 0])
        tb = dag.tile_bytes
        want_host = host.view(np.uint8).copy()
        for x in pushed:
            want_host[x * tb:(x + 1) * tb] = want[x * tb:(x + 1) * tb]
        assert np.array_equal(run.host, want_host), "host image differs from the numpy replay"


# (seed, queue_policy, part_bytes, staged, pushout)
RANDOM_CASES = [
    (1, 0, 16 * 1024, False, False),
    (2, 1, 16 * 1024, True, True),
    (3, 0, 0, True, False),
    (4, 1, 0, False, True),
]


@pytest.mark.parametrize("seed,queue_policy,part_bytes,staged,pushout", RANDOM_CASES,
                         ids=["-".join(map(str, c)) for c in RANDOM_CASES])
def test_random_dags_with_linked_bodies(seed, queue_policy, part_bytes, staged, pushout):
    dag, linked, host = random_case(seed, pushout)
    e = linked_engine(queue_policy=queue_policy, part_bytes=part_bytes)
    try:
        plain = run_engine(e, dag, layout_of(dag, host, staged, pushout))
        traced, out, entries = run_traced(e, dag, layout_of(dag, host, staged, pushout))
        sm_count = e.info()["sm_count"]
    finally:
        e.close()
    assert_same_run(plain, traced)
    st, tr, rec = out[0]
    check_parts(dag, entries, st, tr, rec, sm_count, not staged, "linked dag %s" % (RANDOM_CASES[seed - 1],))
    bad = dags.check_execution(dag, plain.res)
    assert all(v == 0 for v in bad.values()), bad
    ref = run_oracle(as_incr(dag), layout_of(dag, host, staged, pushout))
    for k in ("result", "seen_version"):
        assert np.array_equal(plain.res[k], ref.res[k]), k
    for k in ("version", "state"):
        assert np.array_equal(plain.res["tiles"][k], ref.res["tiles"][k]), "tile " + k
    assert plain.stats["body_errors"] == ref.stats["body_errors"]
    check_against_replay(dag, plain, host, staged, pushout)
    parts = (entries[linked].astype(np.uint32) >> np.uint32(22)) + 1
    assert np.all(parts == (4 if part_bytes else 1)), parts       # 64 KiB tiles in 16 KiB parts


def test_ptx_and_cubin_images_compute_the_same():
    dag, _, host = random_case(5, True)
    runs = []
    for fmt in (L.IMAGE_PTX, L.IMAGE_CUBIN):
        e = linked_engine(fmt, part_bytes=16 * 1024)
        try:
            runs.append(run_engine(e, dag, layout_of(dag, host, True, True)))
        finally:
            e.close()
    assert_same_run(*runs)
    check_against_replay(dag, runs[0], host, True, True)


def test_builtin_windows_on_a_linked_engine():
    """A window without linked tasks runs the built-in kernels on a linked engine: outputs identical to an unlinked
    engine's."""
    dag = groups_dag(7)
    host = np.random.default_rng(7).integers(-100, 100, dag.ntiles * dag.tile_bytes // 4).astype(np.int32)
    runs = []
    for linked in (True, False):
        e = linked_engine(part_bytes=16 * 1024) if linked else Engine(0, part_bytes=16 * 1024)
        try:
            runs.append(run_engine(e, dag, layout_of(dag, host, True, False)))
        finally:
            e.close()
    assert_same_run(*runs)
    ex05 = dags.ex05_broadcast(64, 9, 64 * 1024)
    h = np.full(ex05.ntiles * ex05.tile_bytes // 4, -1, np.int32)
    runs = []
    for linked in (True, False):
        e = linked_engine() if linked else Engine(0)
        try:
            runs.append(run_engine(e, ex05, Layout.contiguous(ex05, host=h, valid=False)))
        finally:
            e.close()
    assert_same_run(*runs)
    assert runs[0].stats["body_errors"] == 0


# ----------------------------------------------------------------------------------------------------------------------
# the stencil over whole tiles, the CTA sum
# ----------------------------------------------------------------------------------------------------------------------
def stencil_dag(nt, sweeps, tile_bytes, w=(1, -2, 3)):
    """Sweep s reads buffer s % 2 (tiles 0..nt-1, then nt..2nt-1) and writes the other: task (s, i) runs STENCIL over
    the left, centre and right tiles of i (no tile past either end) into tile i of the other buffer.  It waits for
    tasks (s-1, i-1 .. i+1): they wrote what it reads, and read what it overwrites."""
    n = nt * sweeps
    t = dags._new_tasks(n)
    src, dst = [], []
    for s in range(sweeps):
        a, b = (s % 2) * nt, ((s + 1) % 2) * nt
        for i in range(nt):
            j = s * nt + i
            t["body"][j], t["nb_flows"][j] = STENCIL, 4
            t["tile"][j] = (a + i - 1 if i > 0 else -1, a + i, a + i + 1 if i < nt - 1 else -1, b + i)
            t["access"][j] = (L.ACCESS_READ, L.ACCESS_READ, L.ACCESS_READ, L.ACCESS_WRITE)
            t["iparam"][j] = w
            if s:
                for p in range(max(i - 1, 0), min(i + 2, nt)):
                    src.append((s - 1) * nt + p); dst.append(j)
    src, dst = np.array(src, np.int64), np.array(dst, np.int64)
    t["succ_begin"], t["succ_count"], succ = dags._csr_from_edges(n, src, dst, np.zeros(len(src), np.int64))
    t["dep_goal"] = np.bincount(dst, minlength=n)
    return dags.Dag(t, succ, np.arange(nt, dtype=np.int32), ntiles=2 * nt, tile_bytes=tile_bytes, name="stencil")


def test_stencil_sweeps():
    nt, sweeps, tb, w = 16, 6, 64 * 1024, (1, -2, 3)
    dag = stencil_dag(nt, sweeps, tb, w)
    host = np.random.default_rng(11).integers(-1000, 1000, dag.ntiles * tb // 4).astype(np.int32)
    e = linked_engine(part_bytes=16 * 1024)            # would cut 64 KiB tiles into 4 parts: the stencil is not cut
    try:
        run = run_engine(e, dag, Layout.contiguous(dag, host=host, valid=False))
    finally:
        e.close()
    bad = dags.check_execution(dag, run.res)
    assert all(v == 0 for v in bad.values()), bad
    buf = [host[:nt * tb // 4].copy(), host[nt * tb // 4:].copy()]
    with np.errstate(over="ignore"):
        for s in range(sweeps):
            c = buf[s % 2]
            left, right = np.concatenate([[0], c[:-1]]), np.concatenate([c[1:], [0]])
            buf[(s + 1) % 2] = np.int32(w[0]) * left + np.int32(w[1]) * c + np.int32(w[2]) * right
    assert np.array_equal(run.dev.view(np.int32), np.concatenate(buf))
    assert np.all(run.res["result"] == 0)


@pytest.mark.parametrize("part_bytes", [0, 16 * 1024], ids=["one_part", "four_parts"])
def test_cta_sum(part_bytes):
    nt, tb = 40, 64 * 1024
    t = dags._new_tasks(nt)
    t["body"], t["nb_flows"], t["tile"][:, 0], t["access"][:, 0] = SUM, 1, np.arange(nt), L.ACCESS_READ
    t["succ_begin"] = 0
    dag = dags.Dag(t, np.zeros(0, np.uint32), np.arange(nt, dtype=np.int32), ntiles=nt, tile_bytes=tb, name="sum")
    host = np.random.default_rng(12).integers(-2 ** 31, 2 ** 31, nt * tb // 4, dtype=np.int64).astype(np.int32)
    e = linked_engine(part_bytes=part_bytes)
    try:
        run = run_engine(e, dag, Layout.contiguous(dag, dev=host))
    finally:
        e.close()
    per = tb // 4 if not part_bytes else part_bytes // 4      # a multi-part task keeps part 0's result
    want = host.reshape(nt, -1)[:, :per].astype(np.int64).sum(axis=1) & 0xFFFFFFFF
    assert np.array_equal(run.res["result"].astype(np.int64), want)


# ----------------------------------------------------------------------------------------------------------------------
# refusals
# ----------------------------------------------------------------------------------------------------------------------
def one_task_window(engine, body, kind=0):
    t = dags._new_tasks(1)
    t["body"], t["nb_flows"], t["tile"][0, :2], t["access"][0, :2] = body, 2, (0, 1), (L.ACCESS_READ, L.ACCESS_WRITE)
    dag = dags.Dag(t, np.zeros(0, np.uint32), np.array([0], np.int32), ntiles=2, tile_bytes=4096, name="one")
    with placed(engine, Layout.contiguous(dag)) as p:
        w = engine.window(kind, dag.tasks, dag.succ, p.tiles, dag.ready)
        w.run()
        w.close()


def test_refusals():
    with Engine(0) as e:
        with pytest.raises(L.Pb2Error) as ex:
            one_task_window(e, AXPB)
        assert ex.value.rc == L.PB2_ERR_NOT_SUPPORTED and "not linked" in str(ex.value)
        with pytest.raises(L.Pb2Error) as ex:
            e.linked_info()
        assert ex.value.rc == L.PB2_ERR_NOT_FOUND
        lib = e._lib
        for img, n, fmt, mask in ((None, 8, L.IMAGE_CUBIN, 0), (b"x", 0, L.IMAGE_PTX, 0), (b"x", 1, 7, 0), (b"x", 1, L.IMAGE_PTX, 1 << 8)):
            assert lib.pb2_engine_link_bodies(e._h, img, n, fmt, mask) == L.PB2_ERR_BAD_PARAM
        # a link error: PTX that does not define pb2_linked_body; the linker's log is in last_error
        ptx = b".version 8.0\n.target sm_90a\n.address_size 64\n.visible .func nothing()\n{\n\tret;\n}\n"
        with pytest.raises(L.Pb2Error) as ex:
            e.link_bodies(ptx, L.IMAGE_PTX)
        assert ex.value.rc == L.PB2_ERR_BAD_PARAM and "pb2_linked_body" in str(ex.value), str(ex.value)
        # the failed link left nothing behind: the engine links an image, then refuses a second one
        e.link_bodies(image(L.IMAGE_CUBIN), L.IMAGE_CUBIN, SLICEABLE)
        with pytest.raises(L.Pb2Error) as ex:
            e.link_bodies(image(L.IMAGE_CUBIN), L.IMAGE_CUBIN, SLICEABLE)
        assert ex.value.rc == L.PB2_ERR_EXISTS
        with pytest.raises(L.Pb2Error) as ex:
            one_task_window(e, AXPB, kind=1)
        assert ex.value.rc == L.PB2_ERR_NOT_SUPPORTED and "GEMM window" in str(ex.value)
        one_task_window(e, AXPB)                         # and runs it in an HBM window


# ----------------------------------------------------------------------------------------------------------------------
# the stand-alone runtime
# ----------------------------------------------------------------------------------------------------------------------
def test_runtime_linked_pool_host_fed():
    n, tb, m, b, k = 32, 256 * 1024, 3, -7, 5
    host = np.full(2 * n * tb // 4, -1, np.int32)
    with R.Context(cuda_devices=(0,)) as ctx:
        ctx.link_bodies(ctx.devices[0], image(L.IMAGE_CUBIN), L.IMAGE_CUBIN, SLICEABLE)
        tp = C.c_void_p(ctx.l.pb2_dtd_taskpool_new(ctx.h))
        ids = insert_linked(ctx, tp, int32_collection(ctx, 2 * n, tb, host), n, m, b, k)
        ctx.wait()
        st = ctx.stats(ctx.devices[0])
        info = ctx.task_info(tp)
        assert ctx.l.pb2_device_memory_release(ctx.devices[0]) == 0
    assert st["windows_launched"] == 1 and st["executed_tasks"] == 3 * n
    assert st["tasks_released_on_device"] == 2 * n
    assert np.all(info["result"][ids["check"]] >> np.uint64(32) == 0)         # no CHECK mismatch
    assert np.all(host[n * tb // 4:] == m * k + b) and np.all(host[:n * tb // 4] == k)


def test_runtime_gemm_and_linked_pool():
    NT, T, n, tb, m, b, k = 2, 128, 8, 64 * 1024, -4, 11, 9
    data = P.Data(NT, T, seed=2)
    init = data.host.copy()
    host = np.zeros(2 * n * tb // 4, np.int32)
    with R.Context(cuda_devices=(0,)) as ctx:
        ctx.link_bodies(ctx.devices[0], image(L.IMAGE_PTX), L.IMAGE_PTX, SLICEABLE)
        tp, gids = P.insert(ctx, data)
        ids = insert_linked(ctx, tp, int32_collection(ctx, 2 * n, tb, host), n, m, b, k)
        ctx.wait()
        st = ctx.stats(ctx.devices[0])
        info = ctx.task_info(tp)
        assert ctx.l.pb2_device_memory_release(ctx.devices[0]) == 0
    assert st["executed_tasks"] == P.ntasks(NT) + 3 * n and st["windows_launched"] >= 2
    assert np.all(info["result"][ids["check"]] >> np.uint64(32) == 0)
    assert np.all(host[n * tb // 4:] == m * k + b)
    x0 = init[P.NAMES.index("X") * data.mat_bytes:][:data.mat_bytes].view(np.float32)
    y0 = init[P.NAMES.index("Y") * data.mat_bytes:][:data.mat_bytes].view(np.float32)
    assert np.array_equal(data.view("Y").view(np.float32), y0 + np.float32(P.ALPHA) * x0)
    for i in range(NT):
        for j in range(NT):
            acc = np.ones((T, T), np.float64)
            big = np.abs(acc)
            for kk in range(NT):
                a = bf16_bits_to_f32(data.tile("A", i, kk).view(np.uint16)).reshape(T, T).astype(np.float64)
                bb = bf16_bits_to_f32(data.tile("B", kk, j).view(np.uint16)).reshape(T, T).astype(np.float64)
                acc = acc + a @ bb.T
                big = np.maximum(big, np.abs(acc))
            gc = bf16_bits_to_f32(data.tile("C", i, j).view(np.uint16)).reshape(T, T).astype(np.float64)
            assert np.all(np.abs(gc - acc) <= 2.0 ** -7 * big), (i, j)
