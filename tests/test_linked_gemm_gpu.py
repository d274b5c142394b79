"""Application device bodies linked into GEMM windows (pb2_engine_link_bodies_ex with PB2_LINK_GEMM_WINDOWS) on the
H100.

The random mixed DAGs of tests/test_mixed_windows_gpu.py run with every FILL_I32 task replaced by the fixture's linked
FILL (tests/cuda/linked_bodies.cu, LINKED_3, the same function).  The linked GEMM kernel must compute exactly what the
built-in GEMM kernel computes on the original DAG -- GEMM outputs bit for bit, every result, version and seen version
-- and what the oracle computes.  The CTA sum through the scratch words runs on the 384 threads of a GEMM worker beside
a GEMM chain, and the stand-alone runtime runs a GEMM pool and a linked pool in one window."""
import numpy as np
import pytest

from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200 import runtime as R
from parsec_b200.bf16 import bf16_bits_to_f32, f32_to_bf16_bits
from parsec_b200.engine import Engine
from window_harness import Layout, assert_like_oracle, assert_same_run, run_engine, run_oracle
from test_mixed_windows_gpu import MixedDag
from test_linked_bodies import insert_linked, int32_collection
from test_linked_bodies_gpu import image
import mixed_pool as P

pytestmark = pytest.mark.gpu

SUM, FILL = L.BODY_LINKED_0 + 2, L.BODY_LINKED_0 + 3
SLICEABLE = 0xFF & ~(1 << 1)                   # every fixture body but the stencil


def linked_gemm_engine(fmt=L.IMAGE_CUBIN, **kw):
    e = Engine(0, **kw)
    e.link_bodies(image(fmt), fmt, SLICEABLE, gemm_windows=True)
    info = e.linked_gemm_info()
    print("linked GEMM kernel (%s, %s): %s" % ("PTX" if fmt == L.IMAGE_PTX else "cubin", kw, info))
    assert info["regs"] > 0 and 0 < info["nworkers"] <= e.info()["nworkers_gemm"]
    return e


def with_linked_fill(dag):
    t = dag.tasks.copy()
    assert np.any(t["body"] == L.BODY_FILL_I32)
    t["body"][t["body"] == L.BODY_FILL_I32] = FILL
    return dags.Dag(t, dag.succ, dag.ready, ntiles=dag.ntiles, tile_bytes=dag.tile_bytes, kind=1)


CASES = [  # seed, engine parameters, image format, traced
    (21, dict(), L.IMAGE_CUBIN, False),
    (22, dict(part_bytes=65536), L.IMAGE_CUBIN, True),
    (23, dict(part_bytes=16384, queue_policy=1), L.IMAGE_CUBIN, False),
    (24, dict(part_bytes=16384, gemm_mode=2), L.IMAGE_PTX, False),
    (25, dict(queue_policy=1), L.IMAGE_PTX, True),
    (26, dict(max_workers=1, gemm_mode=2), L.IMAGE_CUBIN, False),
]


@pytest.mark.parametrize("seed,kw,fmt,trace", CASES, ids=["default", "parts64k_traced", "prio_parts16k",
                                                          "per_task_units_ptx", "prio_ptx_traced", "one_worker"])
def test_random_mixed_dag_with_linked_fills(seed, kw, fmt, trace):
    md = MixedDag(seed)
    linked = with_linked_fill(md.dag)
    with Engine(0, timeout_ms=8000, **kw) as e:
        want = run_engine(e, md.dag, md.layout, trace=trace)
    e = linked_gemm_engine(fmt, timeout_ms=8000, **kw)
    try:
        got = run_engine(e, linked, md.layout, trace=trace)
    finally:
        e.close()
    # the same tile bytes (GEMM outputs bit for bit), results, versions and seen versions as the built-in kernel's run
    assert_same_run(got, want)
    assert_like_oracle(got, run_oracle(md.dag, md.layout), md.dag)
    if kw.get("max_workers") == 1:
        assert np.array_equal(got.res["retire_order"], want.res["retire_order"])


@pytest.mark.parametrize("part_bytes", [0, 16 * 1024], ids=["one_part", "eight_parts"])
def test_cta_sum_beside_a_gemm_chain(part_bytes):
    """SUM through the 32 scratch words on the 12 warps of a GEMM worker, in a window with a GEMM k-chain."""
    NT, T = 2, 256
    g = dags.dtd_gemm(NT, tile=T)
    tb, nsum = T * T * 2, 24
    t = np.concatenate([g.tasks, dags._new_tasks(nsum)])
    s = t[g.ntasks:]
    s["body"], s["nb_flows"], s["access"][:, 0], s["succ_begin"] = SUM, 1, L.ACCESS_READ, len(g.succ)
    s["tile"][:, 0] = g.ntiles + np.arange(nsum)
    t["access"][:, 2] &= ~np.uint8(L.FLOW_PUSHOUT)
    ready = np.concatenate([g.ready, g.ntasks + np.arange(nsum)]).astype(np.int32)
    dag = dags.Dag(t, g.succ, ready, ntiles=g.ntiles + nsum, tile_bytes=tb, kind=1)
    rng = np.random.default_rng(5)
    ops = f32_to_bf16_bits(rng.integers(-1, 2, 3 * NT * NT * T * T).astype(np.float32))
    ints = rng.integers(-2 ** 31, 2 ** 31, nsum * tb // 4, dtype=np.int64).astype(np.int32)
    dev = np.concatenate([ops.view(np.uint8), ints.view(np.uint8)])
    e = linked_gemm_engine(part_bytes=part_bytes)
    try:
        run = run_engine(e, dag, Layout.contiguous(dag, dev=dev))
    finally:
        e.close()
    per = tb // 4 if not part_bytes else part_bytes // 4       # a multi-part task keeps part 0's result
    want = ints.reshape(nsum, -1)[:, :per].astype(np.int64).sum(axis=1) & 0xFFFFFFFF
    assert np.array_equal(run.res["result"][g.ntasks:].astype(np.int64), want)
    tile = lambda image, i: bf16_bits_to_f32(image[i * tb:(i + 1) * tb].view(np.uint16)).reshape(T, T)
    for i in range(NT):
        for j in range(NT):
            acc = tile(dev, 2 * NT * NT + i * NT + j).astype(np.float64)
            for k in range(NT):
                acc = acc + tile(dev, i * NT + k).astype(np.float64) @ tile(dev, NT * NT + k * NT + j).astype(np.float64).T
            want = bf16_bits_to_f32(f32_to_bf16_bits(acc.astype(np.float32))).reshape(T, T)
            assert np.array_equal(tile(run.dev, 2 * NT * NT + i * NT + j), want), (i, j)


def test_runtime_gemm_and_linked_pool_in_one_window():
    NT, T, n, tb, m, b, k = 2, 128, 8, 64 * 1024, -4, 11, 9
    data = P.Data(NT, T, seed=2)
    init = data.host.copy()
    host = np.zeros(2 * n * tb // 4, np.int32)
    with R.Context(cuda_devices=(0,)) as ctx:
        ctx.link_bodies(ctx.devices[0], image(L.IMAGE_PTX), L.IMAGE_PTX, 0x01, gemm_windows=True)
        tp, gids = P.insert(ctx, data)
        ids = insert_linked(ctx, tp, int32_collection(ctx, 2 * n, tb, host), n, m, b, k)
        ctx.wait()
        st = ctx.stats(ctx.devices[0])
        info = ctx.task_info(tp)
        assert ctx.l.pb2_device_memory_release(ctx.devices[0]) == 0
    assert st["executed_tasks"] == P.ntasks(NT) + 3 * n and st["windows_launched"] == 1
    assert np.all(info["result"][ids["check"]] >> np.uint64(32) == 0)
    assert np.all(host[n * tb // 4:] == m * k + b) and np.all(host[:n * tb // 4] == k)
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


def test_gemm_windows_without_the_flag_are_refused_on_a_linked_engine():
    e = Engine(0)
    try:
        e.link_bodies(image(L.IMAGE_CUBIN), L.IMAGE_CUBIN, SLICEABLE)
        with pytest.raises(L.Pb2Error) as ex:
            e.linked_gemm_info()
        assert ex.value.rc == L.PB2_ERR_NOT_FOUND
        md = MixedDag(21)
        with pytest.raises(L.Pb2Error) as ex:
            run_engine(e, with_linked_fill(md.dag), md.layout)
        assert ex.value.rc == L.PB2_ERR_NOT_SUPPORTED and "GEMM window" in str(ex.value)
    finally:
        e.close()
