"""Part records of traced engine windows (pb2_window_part_trace) on the H100.

Every ring entry a run pops is one part of a scheduling entity, and the worker that ran it records four %globaltimer
stamps (pop, stage-in done, body done, pushout done), the bytes it moved in and pushed out, its SM and two flags.  A
traced window must compute bit for bit what the untraced window computes, and its part records must agree with the
window trace and the window's statistics exactly:
  1. every (leading task, part) that owns ring entries appears once, ordered by task, then part;
  2. each record's stamps are ordered;
  3. exactly one part retired each entity, and the window trace gives every task of the entity its earliest pop, its
     latest pushout end and the SM of that part;
  4. the bytes moved in add up to bytes_h2d + bytes_d2d and those pushed out to bytes_d2h.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200 import runtime as R
from parsec_b200.engine import Engine
from window_harness import Layout, assert_same_run, placed, run_engine
from test_rearm_gpu import gemm_chains_dag
from test_window_trace_gpu import groups_dag
import mixed_pool as P

pytestmark = pytest.mark.gpu

TOL_NS = 2000


def run_traced(e, dag, layout, launches=1):
    """`launches` runs of one traced window of dag over layout.  Returns the Run of the last one and, per launch,
    (stats, trace, part records), and the window's ring entry per task (parts - 1 in its part field)."""
    with placed(e, layout) as p:
        e.set_window_trace(True)
        try:
            w = e.window(dag.kind, dag.tasks, dag.succ, p.tiles, dag.ready)
        finally:
            e.set_window_trace(False)
        try:
            entries = w.task_entries()
            out = []
            for _ in range(launches):
                st = w.run()
                out.append((st, w.trace(), w.part_trace()))
            res = w.results()
        finally:
            w.close()
    return p.run(st, res, [o[1] for o in out], (p.dev, p.host)), out, entries


def entry_parts(dag, entries):
    """Parts of the entity each task belongs to, from its ring entry."""
    e = entries.astype(np.uint32)
    return (e >> np.uint32(27 if dag.kind == 1 else 22)).astype(np.int64) + 1


def check_parts(dag, entries, st, tr, rec, sm_count, resident, what):
    unit = tr["unit"].astype(np.int64)
    lead = np.unique(unit)
    nparts = entry_parts(dag, entries)[lead]
    # 1. one record per (leading task, part), by task then part
    assert len(rec) == int(nparts.sum()), what
    assert np.array_equal(rec["task"], np.repeat(lead, nparts)), what
    assert np.array_equal(rec["part"], np.concatenate([np.arange(n) for n in nparts])), what
    assert np.array_equal(rec["nparts"], np.repeat(nparts, nparts)), what
    assert np.all(unit[rec["task"]] == rec["task"]), what
    # 2. ordered stamps on an existing SM
    t = [rec[k].astype(np.int64) for k in ("t_pop_ns", "t_in_ns", "t_exec_ns", "t_out_ns")]
    assert np.all(t[0] > 0) and np.all(t[0] <= t[1]) and np.all(t[1] <= t[2]) and np.all(t[2] <= t[3]), what
    assert np.all(rec["smid"] < sm_count), what
    # 3. the window trace is derived from the records, entity by entity (every part was popped: t_pop > 0 above)
    first = np.concatenate([[0], np.cumsum(nparts)[:-1]])
    retired = (rec["flags"] & L.PART_RETIRED) != 0
    assert np.array_equal(np.add.reduceat(retired.astype(np.int64), first), np.ones(len(lead), np.int64)), what
    want = {k: np.zeros(dag.ntasks, np.int64) for k in ("t_start_ns", "t_end_ns", "smid")}
    want["t_start_ns"][lead] = np.minimum.reduceat(t[0], first)
    want["t_end_ns"][lead] = np.maximum.reduceat(t[3], first)
    want["smid"][rec["task"][retired]] = rec["smid"][retired]
    for k, v in want.items():
        assert np.array_equal(tr[k].astype(np.int64), v[unit]), (what, k)
    # 4. bytes
    assert int(rec["in_bytes"].sum()) == st["bytes_h2d"] + st["bytes_d2d"], what
    assert int(rec["out_bytes"].sum()) == st["bytes_d2h"], what
    if resident:
        assert np.all(rec["in_bytes"] == 0), what
    assert np.all((rec["flags"][rec["in_bytes"] > 0] & L.PART_WAITED_INPUT) != 0), what
    print("%s: %d entities, %d parts, %d waited for input, %d bytes in, %d bytes out"
          % (what, len(lead), len(rec), int(np.sum(rec["flags"] & L.PART_WAITED_INPUT != 0)),
             int(rec["in_bytes"].sum()), int(rec["out_bytes"].sum())))


def layout_of(dag, host, staged, pushout):
    """Tiles resident in the slab, or staged in from a pinned host image; a host home whenever something is pushed out."""
    if staged:
        return Layout.contiguous(dag, host=host, valid=False)
    return Layout.contiguous(dag, host=host, valid=True) if pushout else Layout.contiguous(dag, dev=host)


def run_and_check(engine_kw, dag, host, staged, pushout, what):
    with Engine(0, **engine_kw) as e:
        plain = run_engine(e, dag, layout_of(dag, host, staged, pushout))
        traced, out, entries = run_traced(e, dag, layout_of(dag, host, staged, pushout))
        sm_count = e.info()["sm_count"]
    assert_same_run(plain, traced)
    st, tr, rec = out[0]
    check_parts(dag, entries, st, tr, rec, sm_count, not staged, what)
    return rec


def with_pushout(dag, tasks):
    """The same DAG with every written flow of `tasks` pushed out to its host home."""
    t = dag.tasks.copy()
    for i in tasks:
        for f in range(int(t["nb_flows"][i])):
            if t["tile"][i, f] >= 0 and t["access"][i, f] & L.ACCESS_WRITE:
                t["access"][i, f] |= L.FLOW_PUSHOUT
    return dags.Dag(t, dag.succ, dag.ready, ntiles=dag.ntiles, tile_bytes=dag.tile_bytes, kind=dag.kind,
                    name=dag.name + "_pushout", meta=dag.meta)


GROUPS = {"fused": {}, "groups_only": {"fuse_readers": -1}, "no_groups": {"read_groups": -1}}
# (seed, queue_policy, read groups / fusion, part_bytes, staged, pushout)
HBM_CASES = [
    (1, 0, "fused", 0, False, False),
    (2, 1, "fused", 16 * 1024, True, True),
    (3, 0, "groups_only", 16 * 1024, True, False),
    (4, 1, "groups_only", 0, False, True),
    (5, 0, "no_groups", 16 * 1024, False, True),
    (6, 1, "no_groups", 0, True, False),
]


@pytest.mark.parametrize("seed,queue_policy,groups,part_bytes,staged,pushout", HBM_CASES,
                         ids=["-".join(map(str, c)) for c in HBM_CASES])
def test_random_hbm_dags(seed, queue_policy, groups, part_bytes, staged, pushout):
    dag = groups_dag(seed)
    if pushout:                                         # the read-modify-write tasks; producers stay fusable
        dag = with_pushout(dag, np.flatnonzero(~np.isin(dag.tasks["body"], [L.BODY_FILL_I32, L.BODY_CHECK_I32])))
    host = np.random.default_rng(seed).integers(-100, 100, dag.ntiles * dag.tile_bytes // 4).astype(np.int32)
    rec = run_and_check(dict(GROUPS[groups], queue_policy=queue_policy, part_bytes=part_bytes), dag, host, staged,
                        pushout, "groups dag %s" % ((seed, queue_policy, groups, part_bytes, staged, pushout),))
    if part_bytes:
        assert rec["nparts"].max() > 1                  # 64 KiB tiles in 16 KiB parts
    if pushout:
        assert rec["out_bytes"].sum() > 0


@pytest.mark.parametrize("staged,part_bytes", [(False, 0), (True, 0), (True, 64 * 1024)],
                         ids=["resident", "host_fed", "host_fed_parts"])
def test_ex05_window(staged, part_bytes):
    dag = dags.ex05_broadcast(256, 14, 256 * 1024)
    host = np.full(dag.ntiles * dag.tile_bytes // 4, -1, np.int32)
    rec = run_and_check({"part_bytes": part_bytes}, dag, host, staged, False, "ex05 staged %d part_bytes %d" % (staged, part_bytes))
    if staged:
        assert rec["in_bytes"].sum() == dag.ntiles * dag.tile_bytes


@pytest.mark.parametrize("queue_policy", [0, 1])
@pytest.mark.parametrize("staged", [False, True], ids=["resident", "host_fed"])
@pytest.mark.parametrize("make", [lambda: with_pushout(gemm_chains_dag(), [2, 4, 9]), lambda: dags.dtd_gemm(3, 256)],
                         ids=["chains_pushout", "dtd_gemm"])
def test_gemm_window(make, staged, queue_policy):
    dag = make()
    if "host" not in dag.meta:
        rng = np.random.default_rng(5)
        bits = (rng.integers(-64, 64, dag.ntiles * dag.tile_bytes // 2) * 0x10 + 0x3C00).astype(np.uint16)   # small bf16
        dag.meta["host"] = bits.view(np.int32)
    rec = run_and_check({"queue_policy": queue_policy, "part_bytes": 32 * 1024}, dag, dag.meta["host"], staged, True,
                        "%s staged %d policy %d" % (dag.name, staged, queue_policy))
    gemm = dag.tasks["body"][rec["task"]] == L.BODY_GEMM_BF16
    assert np.all(rec["nparts"][gemm] == 2)             # 256 x 256 C tiles: two 128-row sub-tiles
    assert rec["out_bytes"][gemm].sum() > 0


def test_rearmed_window_records_each_launch():
    dag = groups_dag(9)
    host = np.random.default_rng(9).integers(-100, 100, dag.ntiles * dag.tile_bytes // 4).astype(np.int32)
    with Engine(0, part_bytes=16 * 1024) as e:
        _, out, entries = run_traced(e, dag, Layout.contiguous(dag, host=host, valid=False), launches=3)
        sm_count = e.info()["sm_count"]
    prev_out = 0
    for i, (st, tr, rec) in enumerate(out):
        check_parts(dag, entries, st, tr, rec, sm_count, False, "launch %d" % i)
        assert int(rec["t_pop_ns"].min()) >= prev_out - TOL_NS, i
        prev_out = int(rec["t_out_ns"].max())


def test_untraced_window_refuses_part_trace():
    dag = dags.ex05_broadcast(4, 2, 4096)
    with Engine(0) as e, placed(e, Layout.contiguous(dag)) as p:
        w = e.window(0, dag.tasks, dag.succ, p.tiles, dag.ready)
        w.run()
        with pytest.raises(L.Pb2Error) as exc:
            w.part_trace()
        assert exc.value.rc == L.PB2_ERR_NOT_SUPPORTED and "without trace" in str(exc.value)
        w.close()


def check_pool_records(rec, dev, ntasks, gpu, what):
    assert len(rec) > 0 and np.all(dev == gpu), what
    assert np.all((rec["task"] >= 0) & (rec["task"] < ntasks)), what
    t = [rec[k].astype(np.int64) for k in ("t_pop_ns", "t_in_ns", "t_exec_ns", "t_out_ns")]
    assert np.all(t[0] > 0) and np.all(t[0] <= t[1]) and np.all(t[1] <= t[2]) and np.all(t[2] <= t[3]), what
    for task in np.unique(rec["task"]):
        r = rec[rec["task"] == task]
        assert sorted(r["part"].tolist()) == list(range(int(r["nparts"][0]))), (what, task)
        assert np.all(r["nparts"] == r["nparts"][0]), (what, task)
        assert int(np.sum((r["flags"] & L.PART_RETIRED) != 0)) == 1, (what, task)


# tiles come in through the kernels' stage-in, not the copy engine
RUNTIME_MCA = {"device_engine_trace": 1, "device_engine_dma_prefetch_min_bytes": 0}


def test_runtime_ex05_pool_part_trace():
    K, NB, tb = 32, 6, 64 * 1024
    host = np.full(K * tb // 4, -1, np.int32)
    with R.Context(cuda_devices=(0,), mca=RUNTIME_MCA) as ctx:
        dc = ctx.block_cyclic(4, tb // 4, 1, K * tb // 4, 1, mat=host)
        before = ctx.stats(ctx.devices[0])["data_in_from_device"][0]
        tp = C.c_void_p(ctx.l.pb2_ptg_ex05_broadcast_new(ctx.h, dc, K, NB))
        ctx.wait()
        grown = ctx.stats(ctx.devices[0])["data_in_from_device"][0] - before
        info = ctx.task_info(tp)
        tr = ctx.device_trace(tp)
        rec, dev = ctx.device_part_trace(tp)
    n = len(info["class_id"])
    check_pool_records(rec, dev, n, 2, "runtime ex05")
    assert grown == K * tb
    assert int(rec["in_bytes"].sum()) == grown
    # every entity is led by a task that ran there, and its earliest pop is that task's t_start
    for task in np.unique(rec["task"]):
        assert int(rec["t_pop_ns"][rec["task"] == task].min()) == int(tr["t_start_ns"][task])
    assert np.isin(np.flatnonzero(info["class_id"] == 0), rec["task"]).all()     # every TaskBcast leads an entity


def test_runtime_mixed_pool_part_trace():
    NT, T = 2, 1024
    data = P.Data(NT, T, seed=1)
    with R.Context(cuda_devices=(0,), mca=RUNTIME_MCA) as ctx:
        before = ctx.stats(ctx.devices[0])["data_in_from_device"][0]
        tp, ids = P.insert(ctx, data)
        ctx.wait()
        grown = ctx.stats(ctx.devices[0])["data_in_from_device"][0] - before
        rec, dev = ctx.device_part_trace(tp)
        assert ctx.l.pb2_device_memory_release(ctx.devices[0]) == 0
    check_pool_records(rec, dev, P.ntasks(NT), 2, "runtime mixed pool")
    # the runtime counts the C tiles as data in when FILL takes them (the reference's accounting, device_gpu.c:2133),
    # but FILL only writes them: the kernel moves the A, B, X and Y tiles
    c_bytes = NT * NT * data.tile_bytes
    assert grown > c_bytes and int(rec["in_bytes"].sum()) == grown - c_bytes
    gemm = {v for k, v in ids.items() if k[0] == "gemm"}
    axpy = {v for k, v in ids.items() if k[0] == "axpy"}
    assert any(int(t) in gemm for t in rec["task"]) and any(int(t) in axpy for t in rec["task"])
    assert rec["nparts"][np.isin(rec["task"], list(axpy))].min() > 1     # 2 MiB tiles in 256 KiB parts
