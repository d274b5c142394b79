"""Every window kernel of the engine's kernel table on the H100: kind (HBM, GEMM) x bodies (built-in, linked) x
queue_policy (0, 1) x window trace (off, on).

One engine per queue policy, linked with PB2_LINK_GEMM_WINDOWS to tests/cuda/linked_bodies.cubin, runs a small HBM DAG
and a small GEMM DAG.  A window whose tasks name no linked body runs the built-in kernel; the linked variant of a DAG
has every FILL_I32 replaced by the fixture's linked FILL (LINKED_3, the same function), so its window runs the linked
kernel.  Each run must compute what the oracle computes on the original DAG, on no more workers than the kernel's grid,
and a traced run must leave one part record per popped ring entry.  The worker counts are the ones each kernel has
always launched with: 8 HBM workers per SM, one GEMM worker per SM, and on the H100 the linked kernels fit as many."""
import numpy as np
import pytest

from parsec_b200 import _lib as L
from parsec_b200.engine import Engine
from window_harness import Layout, assert_like_oracle, run_engine, run_oracle
from test_linked_bodies_gpu import image
from test_linked_gemm_gpu import SLICEABLE
from test_mixed_windows_gpu import MixedDag
from test_part_trace_gpu import check_parts, run_traced
from test_window_trace_gpu import groups_dag
from oracle import orc_dags as dags

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engines():
    """An engine per queue policy, linked for HBM and GEMM windows."""
    out = {}
    try:
        for policy in (0, 1):
            e = out[policy] = Engine(0, queue_policy=policy, timeout_ms=8000)
            e.link_bodies(image(L.IMAGE_CUBIN), L.IMAGE_CUBIN, SLICEABLE, gemm_windows=True)
        yield out
    finally:
        for e in out.values():
            e.close()


def hbm_case():
    dag = groups_dag(7, n_rmw=80, ngroups=8)
    host = np.random.default_rng(7).integers(-100, 100, dag.ntiles * dag.tile_bytes // 4).astype(np.int32)
    return dag, Layout.contiguous(dag, dev=host)


def gemm_case():
    md = MixedDag(21)
    return md.dag, md.layout


def with_linked_fill(dag):
    t = dag.tasks.copy()
    assert np.any(t["body"] == L.BODY_FILL_I32)
    t["body"][t["body"] == L.BODY_FILL_I32] = L.BODY_LINKED_0 + 3
    return dags.Dag(t, dag.succ, dag.ready, ntiles=dag.ntiles, tile_bytes=dag.tile_bytes, kind=dag.kind, name=dag.name)


@pytest.mark.parametrize("policy", [0, 1], ids=["fifo", "prio"])
def test_worker_counts(engines, policy):
    e = engines[policy]
    info = e.info()
    assert info["nworkers"] == 8 * info["sm_count"] and info["nworkers_gemm"] == info["sm_count"], info
    assert e.linked_info()["nworkers"] == info["nworkers"]
    assert e.linked_gemm_info()["nworkers"] == info["nworkers_gemm"]


@pytest.mark.parametrize("trace", [False, True], ids=["untraced", "traced"])
@pytest.mark.parametrize("policy", [0, 1], ids=["fifo", "prio"])
@pytest.mark.parametrize("linked", [False, True], ids=["builtin", "linked"])
@pytest.mark.parametrize("kind", [0, 1], ids=["hbm", "gemm"])
def test_window_kernel(engines, kind, linked, policy, trace):
    e = engines[policy]
    dag, layout = hbm_case() if kind == 0 else gemm_case()
    run_dag = with_linked_fill(dag) if linked else dag
    if trace:
        run, out, entries = run_traced(e, run_dag, layout)
        st, tr, rec = out[0]
        check_parts(run_dag, entries, st, tr, rec, e.info()["sm_count"], bool(np.all(layout.valid)),
                    "kind %d linked %d policy %d" % (kind, linked, policy))
    else:
        run = run_engine(e, run_dag, layout)
    assert_like_oracle(run, run_oracle(dag, layout), dag)
    if linked:
        grid = (e.linked_gemm_info() if kind else e.linked_info())["nworkers"]
    else:
        grid = e.info()["nworkers_gemm" if kind else "nworkers"]
    assert 0 <= run.res["worker"].min() and run.res["worker"].max() < grid
