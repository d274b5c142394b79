"""Read groups and fused producer units in GEMM windows, on the H100.

A GEMM window plans and runs its HBM-body tasks as an HBM window does (form_read_groups, DESIGN §5): the Ex05
broadcast beside a small GEMM chain, in one kind-1 window, must compute what the oracle computes and what the HBM
window computes for the Ex05 tasks alone -- results, seen versions, tile bytes, stats -- with fusion, with groups
only and with neither, under both queue policies, traced or not, resident or staged in, in whole tiles or in parts.
The CHECK readers of the chain's C tile run as one group beside it.  The stand-alone runtime runs a DTD pool of GEMM
chains and check fan-outs as one GEMM window with its groups, and computes what that window computes without them."""
import ctypes as C

import numpy as np
import pytest

from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200 import runtime as R
from parsec_b200.engine import Engine
from window_harness import Layout, assert_like_oracle, assert_same_run, run_engine, run_oracle
from test_part_trace_gpu import check_parts, run_traced
from test_checked_linked_gpu import MASK, image, linked_ex05
from gemm_chain_dags import C_WORD, ex05_beside_gemm
import mixed_pool as P

pytestmark = pytest.mark.gpu

KCHAIN = 2                                  # GEMMs in ex05_beside_gemm's chain
GROUPS = {"fused": {}, "groups_only": {"fuse_readers": -1}, "no_groups": {"read_groups": -1}}


def layout_of(dag, sizes, host, staged):
    return Layout.packed(dag, host=host, valid=not staged, sizes=sizes)


def ran_as_unit(res, seq):
    """The tasks seq ran as one unit of a GEMM window: on one worker, retired back to back in this order (each member's
    start and end are consecutive events, retire_unit_warp)."""
    ss, es = res["start_seq"].astype(np.int64), res["end_seq"].astype(np.int64)
    return (len(set(res["worker"][seq].tolist())) == 1 and np.array_equal(es[seq], ss[seq] + 1)
            and np.array_equal(ss[seq], ss[seq[0]] + 2 * np.arange(len(seq))))


def ex05_members(ex, k):
    F = ex.meta["F"]
    return [ex.ntiles + k * F + n for n in range(F)]


def assert_ex05_as_hbm(run, hbm, ex, layout):
    """The Ex05 tasks of a kind-1 run computed what the HBM window computed for them alone."""
    n0 = ex.ntasks
    for k in ("result", "seen_version"):
        assert np.array_equal(run.res[k][:n0], hbm.res[k]), k
    for i in range(ex.ntiles):
        assert np.array_equal(layout.tile_bytes(run.dev, i), hbm.dev[i * ex.tile_bytes:(i + 1) * ex.tile_bytes]), i


CASES = [  # groups, queue_policy, trace, staged, part_bytes
    ("fused", 0, False, False, 0),
    ("fused", 1, True, False, 16 * 1024),
    ("fused", 0, True, True, 0),
    ("fused", 1, False, True, 16 * 1024),
    ("groups_only", 0, False, False, 16 * 1024),
    ("groups_only", 1, True, True, 0),
    ("no_groups", 0, True, False, 0),
    ("no_groups", 1, False, True, 16 * 1024),
]


@pytest.mark.parametrize("groups,queue_policy,trace,staged,part_bytes", CASES,
                         ids=["-".join(str(x) for x in c) for c in CASES])
def test_ex05_beside_a_gemm_chain(groups, queue_policy, trace, staged, part_bytes):
    dag, ex, sizes, host = ex05_beside_gemm(256)
    kw = dict(GROUPS[groups], queue_policy=queue_policy, part_bytes=part_bytes)
    ref = run_oracle(dag, layout_of(dag, sizes, host, staged))
    with Engine(0, **kw) as e:
        hbm = run_engine(e, ex, Layout.contiguous(ex, dev=host[:ex.ntiles * ex.tile_bytes]))
        if trace:
            got, out, entries = run_traced(e, dag, layout_of(dag, sizes, host, staged))
            st, tr, rec = out[0]
            check_parts(dag, entries, st, tr, rec, e.info()["sm_count"], not staged, "ex05 beside GEMM %s" % (kw,))
        else:
            got = run_engine(e, dag, layout_of(dag, sizes, host, staged))
    assert_like_oracle(got, ref, dag)
    assert_ex05_as_hbm(got, hbm, ex, layout_of(dag, sizes, host, staged))
    readers = list(range(ex.ntasks + KCHAIN, dag.ntasks))
    res = got.res
    for k in range(ex.ntiles):
        m = ex05_members(ex, k)
        if groups == "fused":
            assert ran_as_unit(res, [k] + m), k
        elif groups == "groups_only":
            assert ran_as_unit(res, m) and not ran_as_unit(res, [k] + m), k
    if groups != "no_groups":
        assert ran_as_unit(res, readers)
    if trace:
        unit = tr["unit"]
        for k in range(ex.ntiles):
            m = ex05_members(ex, k)
            lead = {"fused": k, "groups_only": m[0], "no_groups": None}[groups]
            assert np.all(unit[m] == (lead if lead is not None else m)), k
        assert np.all(unit[readers] == (readers[0] if groups != "no_groups" else readers))


def test_one_worker_retires_in_oracle_order():
    """With one worker fusion is off and groups keep the ungrouped FIFO order (every task its own unit otherwise, as
    gemm_mode 2 makes it: a fused k-chain runs its members back to back)."""
    dag, ex, sizes, host = ex05_beside_gemm(64)
    ref = run_oracle(dag, layout_of(dag, sizes, host, False))
    with Engine(0, max_workers=1, gemm_mode=2) as e:
        got = run_engine(e, dag, layout_of(dag, sizes, host, False))
    assert_like_oracle(got, ref, dag)
    assert np.array_equal(got.res["retire_order"], ref.res["retire_order"])
    F = ex.meta["F"]
    assert ran_as_unit(got.res, [ex.ntiles + n for n in range(F)])


def test_planted_mismatches_are_counted_exactly():
    """Leaders whose constant is not what the producer wrote take the fused unit's exact recount, and members with
    other constants count every element or recount, exactly as the oracle's CHECKs count."""
    dag, ex, sizes, host = ex05_beside_gemm(96, readers=[C_WORD + 2, C_WORD, C_WORD + 2, 7])
    t = dag.tasks
    for k in range(ex.ntiles):
        m = ex05_members(ex, k)
        if k % 3 == 0:
            t["iparam"][m[0], 0] = k + 1               # the leader mismatches everything: the exact recount
        if k % 3 == 1:
            t["iparam"][m[2], 0] = -5                 # one member mismatches, the leader does not
    for staged in (False, True):
        ref = run_oracle(dag, layout_of(dag, sizes, host, staged))
        assert ref.stats["body_errors"] > 0
        for kw in (dict(), dict(part_bytes=16 * 1024)):
            with Engine(0, **kw) as e:
                got = run_engine(e, dag, layout_of(dag, sizes, host, staged))
            assert_like_oracle(got, ref, dag)


@pytest.mark.parametrize("fmt", [L.IMAGE_CUBIN, L.IMAGE_PTX], ids=["cubin", "ptx"])
def test_checked_linked_fill_in_a_linked_gemm_window(fmt):
    """The checked linked FILL fused with its readers in a PB2_LINK_GEMM_WINDOWS window: the same run as unfused, as
    the HBM window's fused run, and as the oracle's."""
    dag, ex, sizes, host = ex05_beside_gemm(128, 64 * 1024)
    lt = linked_ex05(dag).tasks
    ldag = dags.Dag(lt, dag.succ, dag.ready, ntiles=dag.ntiles, tile_bytes=dag.tile_bytes, kind=1, meta=dag.meta)
    lex = linked_ex05(ex)
    ref = run_oracle(dag, layout_of(dag, sizes, host, False))
    runs = {}
    for name, kw in (("fused", {}), ("unfused", {"fuse_readers": -1})):
        e = Engine(0, **kw)
        try:
            e.link_bodies(image(fmt), fmt, MASK, MASK, gemm_windows=True)
            runs[name] = run_engine(e, ldag, layout_of(dag, sizes, host, False))
            if name == "fused":
                hbm = run_engine(e, lex, Layout.contiguous(ex, dev=host[:ex.ntiles * ex.tile_bytes]))
        finally:
            e.close()
    assert_same_run(runs["fused"], runs["unfused"])
    assert_like_oracle(runs["fused"], ref, dag)
    assert_ex05_as_hbm(runs["fused"], hbm, ex, layout_of(dag, sizes, host, False))
    for k in range(ex.ntiles):
        assert ran_as_unit(runs["fused"].res, [k] + ex05_members(ex, k)), k
        assert not ran_as_unit(runs["unfused"].res, [k] + ex05_members(ex, k)), k


# ----------------------------------------------------------------------------------------------------------------------
# the stand-alone runtime: a DTD pool with GEMM chains and broadcast / check fan-outs runs as one GEMM window
# ----------------------------------------------------------------------------------------------------------------------
FAN = 4


def insert_fanout_pool(ctx, data):
    """For every C tile (i, j) of mixed_pool.Data: FILL C, the GEMM k-chain (the last one pushed out), then FAN CHECK
    readers of C (one with another constant); and FILL X(i, j) = i * NT + j, then FAN CHECK readers of X (one with
    another constant).  Returns (taskpool, ids) with ids[(kind, i, j[, k])] = pool task id."""
    NT, T = data.NT, data.T
    dcs = P.collections(ctx, data)
    tp = C.c_void_p(ctx.l.pb2_dtd_taskpool_new(ctx.h))

    def klass(name, nf, body):
        ops = np.array([R.INOUT] * nf, np.int32)
        tc = C.c_void_p(ctx.l.pb2_dtd_create_task_class(tp, name, nf, ops.ctypes.data_as(C.c_void_p)))
        assert ctx.l.pb2_dtd_task_class_add_chore(tp, tc, R.DEV_CUDA, body, None) == 0
        return tc

    fill, gemm, check = klass(b"FILL", 1, L.BODY_FILL_I32), klass(b"GEMM", 3, L.BODY_GEMM_BF16), klass(b"CHECK", 1, L.BODY_CHECK_I32)
    tile = lambda name, m, n: ctx.l.pb2_dtd_tile_of(tp, dcs[name], ctx.l.pb2_dc_data_key(dcs[name], m, n))
    keep, ids = [], {}

    def put(key, tc, tiles, ops, iparam=(0, 0, 0)):
        arr = (C.c_void_p * len(tiles))(*tiles)
        o, p = np.array(ops, np.int32), np.array(iparam, np.int32)
        keep.extend((arr, o, p))
        ids[key] = ctx.l.pb2_dtd_insert_task_with_task_class(tp, tc, 0, R.DEV_CUDA, arr, o.ctypes.data_as(C.c_void_p),
                                                             p.ctypes.data_as(C.c_void_p), 0.0)
        assert ids[key] >= 0

    for i in range(NT):
        for j in range(NT):
            c, x, kx = tile("C", i, j), tile("X", i, j), i * NT + j
            put(("fill", i, j), fill, [c], [R.OUTPUT], (P.ONES, 0, 0))
            for k in range(NT):
                put(("gemm", i, j, k), gemm, [tile("A", i, k), tile("B", k, j), c],
                    [R.INPUT, R.INPUT, (R.INOUT | R.PUSHOUT) if k == NT - 1 else R.INOUT], (T, T, T))
            for n in range(FAN):
                put(("check_c", i, j, n), check, [c], [R.INPUT], (P.ONES + (n == 2), 0, 0))
            put(("fill_x", i, j), fill, [x], [R.OUTPUT], (kx, 0, 0))
            for n in range(FAN):
                put(("check_x", i, j, n), check, [x], [R.INPUT], (kx + (n == 1), 0, 0))
    return tp, ids


def exported_layout(win, data):
    """The exported window's tiles as a Layout over a copy of data.host: host-fed, each at its offset in the image."""
    t = win["tiles"]
    nbytes = t["bytes"].astype(np.int64)
    slots = (nbytes + 511) // 512 * 512
    doff = np.concatenate([[0], np.cumsum(slots)[:-1]]).astype(np.int64)
    hoff = (t["src_ptr"] - np.uint64(data.host.ctypes.data)).astype(np.int64)
    return Layout(doff, hoff, nbytes, np.zeros(len(t), bool), np.zeros(int(slots.sum()), np.uint8), data.host.copy())


def test_runtime_pool_groups_beside_gemm_chains():
    """The stand-alone runtime runs the pool as one GEMM window (take_closure), with its fan-outs as read groups and
    the X fan-outs fused with their FILL; its data, results and seen versions are what the same window computes on an
    engine with read_groups = -1, and, off the GEMM chains' C tiles, what the oracle computes."""
    NT, T = 2, 512
    # the window the runtime builds for the pool, on an engine without read groups and in the oracle
    odata = P.Data(NT, T, seed=3)
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        tp, oids = insert_fanout_pool(ctx, odata)
        win = ctx.export_window(tp, ctx.devices[0])
    dag = dags.Dag(win["tasks"], win["succ"], win["ready"], ntiles=len(win["tiles"]), tile_bytes=0, kind=1)
    assert np.any(dag.tasks["body"] == L.BODY_GEMM_BF16)
    layout = exported_layout(win, odata)
    with Engine(0, read_groups=-1) as e:
        plain = run_engine(e, dag, layout)
    # the fused k-chains round C once, the oracle once per GEMM: only the tasks off the chains' tiles compare with it
    ref = run_oracle(dag, layout)
    off_c = np.flatnonzero(dag.tasks["body"] != L.BODY_GEMM_BF16)
    off_c = off_c[~np.isin(dag.tasks["tile"][off_c, 0], dag.tasks["tile"][dag.tasks["body"] == L.BODY_GEMM_BF16, 2])]
    assert len(off_c) == NT * NT * (1 + FAN)
    assert np.array_equal(plain.res["result"][off_c], ref.res["result"][off_c])
    data = P.Data(NT, T, seed=3)
    with R.Context(cuda_devices=(0,), mca={"device_engine_trace": 1, "device_engine_dma_prefetch_min_bytes": 0}) as ctx:
        tp, ids = insert_fanout_pool(ctx, data)
        ctx.wait()
        st = ctx.stats(ctx.devices[0])
        info = ctx.task_info(tp)
        rec, _ = ctx.device_part_trace(tp)
        assert ctx.l.pb2_device_memory_release(ctx.devices[0]) == 0
    assert ids == oids
    n = len(win["tasks"])
    assert st["windows_launched"] == 1 and st["executed_tasks"] == n
    # what the engine without groups computed, task by task and byte by byte
    pool = win["task_ids"]
    assert np.array_equal(info["result"][pool], plain.res["result"])
    assert np.array_equal(info["seen_version"][pool], plain.res["seen_version"])
    for name in ("A", "B", "C"):
        i = P.NAMES.index(name)
        assert np.array_equal(data.view(name), plain.host[i * data.mat_bytes:(i + 1) * data.mat_bytes]), name
    # the fan-outs ran as groups: only their first reader leads an entity, and a fused X group is led by its FILL
    leads = set(rec["task"].tolist())
    for i in range(NT):
        for j in range(NT):
            cc = [ids[("check_c", i, j, m)] for m in range(FAN)]
            cx = [ids[("check_x", i, j, m)] for m in range(FAN)]
            assert cc[0] in leads and not leads & set(cc[1:]), (i, j)
            assert ids[("fill_x", i, j)] in leads and not leads & set(cx), (i, j)
            assert int(info["result"][cx[1]]) >> 32 == T * T * 2 // 4 and int(info["result"][cx[0]]) >> 32 == 0
