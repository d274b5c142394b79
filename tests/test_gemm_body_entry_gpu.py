"""The GEMM-worker entry point (PB2_LINK_GEMM_BODY_ENTRY) on the H100: GEMM-worker bodies called through the
application's pb2_linked_gemm_body, at the GEMM window kernels' 168 registers, beside the built-in bf16 GEMM units and
the application's other bodies.

  - the fp64 DTD GEMM (tests/fp64_gemm.py) through the fixture's 32 x 32-per-warp DMMA body
    (tests/cuda/gemm_entry_bodies.cu), on the engine and through the stand-alone runtime, at small NT, ragged M, N and K
    and odd K: within the float64 bound of NumPy's C, and bit for bit the C of the 80-register body of
    tests/cuda/gemm_worker_bodies.cu on the same data (each C element gets the same DMMA sequence in the same k order);
  - ring probes through the entry point between the units of bf16 GEMM chains, on one worker and on all: the bf16 C
    bit for bit that of the window without them, every probe clean;
  - all four kernel variants, queue_policy 0 / 1 x untraced / traced;
  - a window of GEMM-worker tasks, a linked element-wise producer and linked readers of its tile, on the entry link and
    on the reader groups x entry link; the same producer and readers in an HBM window;
  - without the flag, the same image runs its probes through pb2_linked_body;
  - the link refusals: an image without pb2_linked_gemm_body, and the fixture's PTX, which the driver's JIT compiles
    without the register cap; the engine stays unlinked and then links the right image.
The host side is tests/test_gemm_body_entry.py."""
import os

import numpy as np
import pytest

from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200 import runtime as R
from parsec_b200.engine import Engine
import fp64_gemm as F
from test_gemm_worker_bodies_gpu import bf16_host, check_fp64, fp64_layout, hazard_dag
from window_harness import Layout, run_engine

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ADD, SUM = L.BODY_LINKED_0 + 2, L.BODY_LINKED_0 + 3
SLICEABLE, READERS = 0x0C, 0x08                 # ADD and SUM may be cut into parts; SUM is a reader
ENTRY_BIT = 1 << 35                             # a probe's result bit: reached through pb2_linked_body


def image(name, fmt=L.IMAGE_CUBIN):
    path = os.path.join(ROOT, "tests", "cuda", name + (".ptx" if fmt == L.IMAGE_PTX else ".cubin"))
    assert os.path.exists(path), "build() makes " + path
    return open(path, "rb").read()


def entry_engine(name="gemm_entry_bodies", groups=False, **kw):
    e = Engine(0, timeout_ms=20000, **kw)
    e.link_bodies(image(name), L.IMAGE_CUBIN, SLICEABLE, gemm_windows=True, readers=READERS,
                  reader_groups=READERS if groups else 0, gemm_bodies=F.GEMM_BODIES, gemm_body_entry=True)
    info = e.linked_gemm_info()
    print("linked GEMM kernel with the entry point (%s, %s): %s; HBM: %s" % (name, kw, info, e.linked_info()))
    assert info["regs"] <= 168 and e.linked_info()["regs"] <= 80
    return e


def worker_engine(**kw):
    """The 80-register fixture through pb2_linked_body, as tests/test_gemm_worker_bodies_gpu.py links it."""
    e = Engine(0, timeout_ms=20000, **kw)
    e.link_bodies(F.image(), L.IMAGE_CUBIN, 0, gemm_windows=True, gemm_bodies=F.GEMM_BODIES)
    return e


def on(engine, dag, layout, **kw):
    try:
        return run_engine(engine, dag, layout, **kw)
    finally:
        engine.close()


SHAPES = [(2, 128, 96, 64), (3, 200, 150, 99), (2, 130, 50, 40), (2, 64, 48, 7)]


@pytest.mark.parametrize("NT,M,N,K", SHAPES, ids=["small_nt", "ragged_odd_k", "ragged_even_k", "k_below_one_block"])
def test_fp64_dtd_gemm_on_the_engine(NT, M, N, K):
    dag, sizes = F.dag(NT, M, N, K)
    t = F.tiles(NT, M, N, K)
    layout = fp64_layout(dag, sizes, t)
    got = on(entry_engine(), dag, layout)
    check_fp64(got, layout, t, NT, M, N)
    assert np.array_equal(got.res["result"], np.zeros(dag.ntasks, np.uint64))
    want = on(worker_engine(), dag, layout)
    assert np.array_equal(got.dev, want.dev) and np.array_equal(got.host, want.host), \
        "C differs from the 80-register body's"


def test_fp64_dtd_gemm_through_the_runtime():
    NT, M, N, K = 3, 200, 136, 77
    t = F.tiles(NT, M, N, K)
    out = {}
    for entry in (True, False):
        with R.Context(cuda_devices=(0,)) as ctx:
            if entry:
                ctx.link_bodies(ctx.devices[0], image("gemm_entry_bodies"), L.IMAGE_CUBIN, 0, gemm_windows=True,
                                gemm_bodies=F.GEMM_BODIES, gemm_body_entry=True)
            else:
                ctx.link_bodies(ctx.devices[0], F.image(), L.IMAGE_CUBIN, 0, gemm_windows=True, gemm_bodies=F.GEMM_BODIES)
            tp, bufs = F.insert(ctx, NT, M, N, K, t)
            ctx.wait()
            st = ctx.stats(ctx.devices[0])
            info = ctx.task_info(tp)
            assert ctx.l.pb2_device_memory_release(ctx.devices[0]) == 0
        assert st["executed_tasks"] == NT ** 3 and not np.any(info["result"])
        out[entry] = bufs["C"].copy()
    for i in range(NT):
        for j in range(NT):
            want, bound = F.reference(t, NT, i, j)
            assert np.all(np.abs(F.runtime_tile({"C": out[True]}, "C", i, j, NT, M, N) - want) <= bound), (i, j)
    assert np.array_equal(out[True], out[False]), "C differs from the 80-register body's"


# ----------------------------------------------------------------------------------------------------------------------
# the ring hazard, through the entry point
# ----------------------------------------------------------------------------------------------------------------------
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
    got = on(entry_engine(max_workers=max_workers), dag, layout)
    for c in range(2 * NT * NT, 3 * NT * NT):
        assert np.array_equal(layout.tile_bytes(got.dev, c), plain_layout.tile_bytes(want.dev, c)), c
    assert np.array_equal(got.res["result"][probes], np.zeros(len(probes), np.uint64)), got.res["result"][probes]
    assert np.array_equal(got.res["seen_version"][:NT ** 3], want.res["seen_version"])
    check_fp64(got, layout, ft, fNT, fM, fN, base=fbase, ctile0=t0 + 2 * fNT * fNT)
    if max_workers == 1:                            # chain, probe, chain, ... on the one worker
        pos = {int(x): i for i, x in enumerate(got.res["retire_order"])}
        for c in range(NT * NT - 1):
            assert pos[c * NT + NT - 1] < pos[int(probes[c])] < pos[(c + 1) * NT]


@pytest.mark.parametrize("queue_policy,trace", [(0, False), (1, False), (0, True), (1, True)],
                         ids=["fifo", "prio", "fifo_traced", "prio_traced"])
def test_kernel_variants(queue_policy, trace):
    NT, M, N, K = 3, 136, 104, 57
    dag, sizes = F.dag(NT, M, N, K)
    t = F.tiles(NT, M, N, K)
    layout = fp64_layout(dag, sizes, t)
    got = on(entry_engine(queue_policy=queue_policy), dag, layout, trace=trace)
    check_fp64(got, layout, t, NT, M, N)
    if trace:
        assert len(got.traces) == 1
    want = on(worker_engine(queue_policy=queue_policy), dag, layout)
    assert np.array_equal(got.dev, want.dev)


# ----------------------------------------------------------------------------------------------------------------------
# GEMM-worker tasks beside the application's other bodies
# ----------------------------------------------------------------------------------------------------------------------
def mixed_dag(NT, M, N, K, add_k, nsum, x_bytes, kind=1):
    """The fp64 dtd_gemm (kind 1 only) and, on a tile X of its own (the last tile), ADD add_k then nsum SUM readers of
    X, which the ADD releases together (a read group).  Returns (dag, sizes, id of the ADD)."""
    parts, sizes, edges, ready = [], [], [], []
    n0 = nt0 = 0
    if kind == 1:
        f, fs = F.dag(NT, M, N, K)
        parts.append(f.tasks)
        sizes.append(fs)
        edges += list(zip(*f.edges()))
        ready += list(f.ready)
        n0, nt0 = f.ntasks, f.ntiles
    x = dags._new_tasks(1 + nsum)
    x["nb_flows"] = 1
    x["tile"][:, 0] = nt0
    x["body"][0], x["iparam"][0, 0], x["access"][0, 0] = ADD, add_k, L.ACCESS_RW
    x["body"][1:], x["access"][1:, 0], x["dep_goal"][1:] = SUM, L.ACCESS_READ, 1
    parts.append(x)
    sizes.append([x_bytes])
    edges += [(n0, n0 + 1 + i, 0) for i in range(nsum)]
    ready.append(n0)
    tasks = np.concatenate(parts)
    src, dst, fl = (np.array(v, np.int64) for v in zip(*edges))
    begin, count, succ = dags._csr_from_edges(len(tasks), src, dst, fl)
    tasks["succ_begin"], tasks["succ_count"] = begin, count
    dag = dags.Dag(tasks, succ, np.array(ready, np.int32), ntiles=nt0 + 1, tile_bytes=0, kind=kind, name="mixed")
    return dag, np.concatenate([np.asarray(s, np.int64) for s in sizes]), n0


@pytest.mark.parametrize("groups", [False, True], ids=["entry", "reader_groups_and_entry"])
def test_window_with_gemm_worker_tasks_a_linked_producer_and_a_read_group(groups):
    NT, M, N, K, k, nsum, xb = 2, 160, 72, 48, -12345, 4, 3 << 20
    rng = np.random.default_rng(5)
    x0 = rng.integers(-1 << 31, 1 << 31, xb // 4, dtype=np.int64).astype(np.int32)
    x1 = (x0.astype(np.int64) + k).astype(np.int32)         # int32 wrap-around, as the body adds
    total = np.uint64(int(x1.astype(np.int64).sum()) % (1 << 64))
    t = F.tiles(NT, M, N, K)
    name = "gemm_entry_group_bodies" if groups else "gemm_entry_bodies"
    for kind in (1, 0):
        dag, sizes, add = mixed_dag(NT, M, N, K, k, nsum, xb, kind)
        host = np.concatenate(([x.reshape(-1).view(np.uint8) for x in t] if kind == 1 else []) + [x0.view(np.uint8)])
        layout = Layout.packed(dag, host=host, valid=True, sizes=sizes)
        got = on(entry_engine(name, groups=groups, part_bytes=256 * 1024), dag, layout)
        if kind == 1:
            check_fp64(got, layout, t, NT, M, N)
        assert np.array_equal(layout.tile_bytes(got.dev, dag.ntiles - 1).view(np.int32), x1), kind
        assert got.res["result"][add] == 0
        assert np.array_equal(got.res["result"][add + 1:], np.full(nsum, total, np.uint64)), (kind, got.res["result"][add + 1:])


def probe_dag(n=6):
    """n ring probes, ready at start, and nothing else: a GEMM window of GEMM-worker tasks alone."""
    t = dags._new_tasks(n)
    t["body"], t["iparam"][:, 0], t["iparam"][:, 1] = F.PROBE, np.arange(n), 3
    return dags.Dag(t, np.zeros(0, np.uint32), np.arange(n, dtype=np.int32), ntiles=1, tile_bytes=512, kind=1, name="probes")


def test_without_the_flag_the_same_image_runs_through_pb2_linked_body():
    dag = probe_dag()
    layout = Layout.packed(dag)
    e = Engine(0, timeout_ms=20000)
    e.link_bodies(image("gemm_entry_bodies"), L.IMAGE_CUBIN, 0, gemm_windows=True, gemm_bodies=F.GEMM_BODIES)
    plain = on(e, dag, layout)
    assert np.array_equal(plain.res["result"], np.full(dag.ntasks, ENTRY_BIT, np.uint64)), plain.res["result"]
    entry = on(entry_engine(), dag, layout)
    assert np.array_equal(entry.res["result"], np.zeros(dag.ntasks, np.uint64)), entry.res["result"]


# ----------------------------------------------------------------------------------------------------------------------
# link refusals
# ----------------------------------------------------------------------------------------------------------------------
def test_image_without_the_entry_point_is_refused_then_the_right_one_links():
    NT, M, N, K = 2, 64, 64, 64
    dag, sizes = F.dag(NT, M, N, K)
    t = F.tiles(NT, M, N, K)
    layout = fp64_layout(dag, sizes, t)
    e = Engine(0, timeout_ms=20000)
    try:
        with pytest.raises(L.Pb2Error) as ex:
            e.link_bodies(F.image(), L.IMAGE_CUBIN, 0, gemm_windows=True, gemm_bodies=F.GEMM_BODIES, gemm_body_entry=True)
        assert ex.value.rc == L.PB2_ERR_BAD_PARAM and "pb2_linked_gemm_body" in str(ex.value), str(ex.value)
        with pytest.raises(L.Pb2Error) as ex:
            e.linked_gemm_info()
        assert ex.value.rc == L.PB2_ERR_NOT_FOUND                  # the engine stayed unlinked
        e.link_bodies(image("gemm_entry_bodies"), L.IMAGE_CUBIN, 0, gemm_windows=True, gemm_bodies=F.GEMM_BODIES,
                      gemm_body_entry=True)
        got = run_engine(e, dag, layout)
    finally:
        e.close()
    check_fp64(got, layout, t, NT, M, N)


def test_ptx_form_is_compiled_without_the_cap():
    """The driver's JIT compiles PTX without a register cap: pb2_linked_gemm_body then needs more than the GEMM
    kernels' 168 registers and the entry link fails.  Without the flag the kernels never reach that function, and the
    same PTX links and runs its probes through pb2_linked_body."""
    ptx = image("gemm_entry_bodies", L.IMAGE_PTX)
    e = Engine(0, timeout_ms=20000)
    try:
        with pytest.raises(L.Pb2Error) as ex:
            e.link_bodies(ptx, L.IMAGE_PTX, 0, gemm_windows=True, gemm_bodies=F.GEMM_BODIES, gemm_body_entry=True)
        print("entry link of the PTX form:", ex.value)
        assert ex.value.rc == L.PB2_ERR_BAD_PARAM and "pb2_linked_gemm_body" in str(ex.value), str(ex.value)
        e.link_bodies(ptx, L.IMAGE_PTX, 0, gemm_windows=True, gemm_bodies=F.GEMM_BODIES)
        dag = probe_dag()
        got = run_engine(e, dag, Layout.packed(dag))
    finally:
        e.close()
    assert np.array_equal(got.res["result"], np.full(dag.ntasks, ENTRY_BIT, np.uint64)), got.res["result"]
