"""GEMM-worker bodies in parts (pb2_engine_set_gemm_body_parts) on the H100: every task of a declared body runs as
nparts parts, each on a worker of its own where workers are free, each over the task's whole tiles.

  - the engine setter's refusals and their messages;
  - the fp64 DTD GEMM (tests/fp64_gemm.py) through the fixture's parted DGEMM (tests/cuda/gemm_part_bodies.cu) at
    NT 1, 2, 4 and 8, ragged M and N, odd K, with nparts 1, 2, 3, 4, 8 and 32 set on one engine between windows: C bit
    for bit that of nparts = 1 and of the DGEMM of tests/cuda/gemm_entry_bodies.cu, within the float64 bound of NumPy's
    C; the last k's PUSHOUT leaves the host C equal to the slab's, counted once in bytes_d2h;
  - the same on one worker and with queue_policy 1;
  - PART probes through both entry points: every task's tile holds 1..nparts, the result is part 0's, a traced window
    has nparts records per task and one PB2_PART_RETIRED among them, and a PUSHOUT flow goes home whole and once;
  - parted tasks between the units of bf16 GEMM chains, leaving the bf16 C bit for bit unchanged;
  - a parted DGEMM beside a linked producer and its read group on the reader groups x entry link;
  - the stand-alone runtime's narrow DTD fp64 GEMM with parts and pushout.
The host side is tests/test_gemm_body_parts.py."""
import os

import numpy as np
import pytest

from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200 import runtime as R
from parsec_b200.engine import Engine
import fp64_gemm as F
from test_gemm_body_entry_gpu import mixed_dag
from test_gemm_worker_bodies_gpu import bf16_host, check_fp64, fp64_layout, hazard_dag
from window_harness import Layout, placed, run_engine

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DGEMM, PART = L.BODY_LINKED_0, L.BODY_LINKED_0 + 1
SLICEABLE, READERS = 0x0C, 0x08                 # ADD and SUM may be cut into parts; SUM is a reader
ENTRY_BIT = 1 << 35                             # a probe's result bit: reached through pb2_linked_body


def image(name):
    path = os.path.join(ROOT, "tests", "cuda", name + ".cubin")
    assert os.path.exists(path), "build() makes " + path
    return open(path, "rb").read()


def part_engine(groups=False, entry=True, **kw):
    e = Engine(0, timeout_ms=20000, **kw)
    e.link_bodies(image("gemm_part_group_bodies" if groups else "gemm_part_bodies"), L.IMAGE_CUBIN, SLICEABLE,
                  gemm_windows=True, readers=READERS, reader_groups=READERS if groups else 0, gemm_bodies=F.GEMM_BODIES,
                  gemm_body_entry=entry)
    return e


def entry_engine():
    e = Engine(0, timeout_ms=20000)
    e.link_bodies(image("gemm_entry_bodies"), L.IMAGE_CUBIN, 0, gemm_windows=True, gemm_bodies=F.GEMM_BODIES,
                  gemm_body_entry=True)
    return e


def run_parts(engine, dag, layout):
    """One traced run of dag: (Run, part records)."""
    with placed(engine, layout) as p:
        engine.set_window_trace(True)
        try:
            w = engine.window(dag.kind, dag.tasks, dag.succ, p.tiles, dag.ready)
        finally:
            engine.set_window_trace(False)
        try:
            st = w.run()
            rec = w.part_trace()
            res = w.results()
        finally:
            w.close()
    return p.run(st, res, (), (p.dev, p.host)), rec


# ----------------------------------------------------------------------------------------------------------------------
# the setter
# ----------------------------------------------------------------------------------------------------------------------
def test_engine_setter_refusals():
    with Engine(0, timeout_ms=20000) as e:
        with pytest.raises(L.Pb2Error) as ex:
            e.set_gemm_body_parts(DGEMM, 2)
        assert ex.value.rc == L.PB2_ERR_NOT_FOUND and "no image is linked" in str(ex.value)
        e.link_bodies(image("gemm_part_bodies"), L.IMAGE_CUBIN, SLICEABLE, gemm_windows=True, readers=READERS,
                      gemm_bodies=F.GEMM_BODIES, gemm_body_entry=True)
        for body, n, rc, msg in [(L.BODY_LINKED_0 - 1, 2, L.PB2_ERR_BAD_PARAM, "PB2_BODY_LINKED_0 .. _7"),
                                 (L.BODY_LINKED_7 + 1, 2, L.PB2_ERR_BAD_PARAM, "PB2_BODY_LINKED_0 .. _7"),
                                 (L.BODY_LINKED_0 + 2, 2, L.PB2_ERR_BAD_PARAM, "PB2_LINK_GEMM_BODIES"),
                                 (DGEMM, 0, L.PB2_ERR_VALUE_OUT_OF_BOUNDS, "PB2_GEMM_BODY_MAX_PARTS"),
                                 (DGEMM, 33, L.PB2_ERR_VALUE_OUT_OF_BOUNDS, "PB2_GEMM_BODY_MAX_PARTS")]:
            with pytest.raises(L.Pb2Error) as ex:
                e.set_gemm_body_parts(body, n)
            assert ex.value.rc == rc and msg in str(ex.value), (body, n, str(ex.value))
        e.set_gemm_body_parts(DGEMM, L.GEMM_BODY_MAX_PARTS)
        e.set_gemm_body_parts(DGEMM, 1)


# ----------------------------------------------------------------------------------------------------------------------
# the fp64 DTD GEMM
# ----------------------------------------------------------------------------------------------------------------------
NPARTS = (1, 2, 3, 4, 8, 32)


def host_tile(run, layout, i):
    """Tile i's bytes in the host image after the run (its home)."""
    return run.host[int(layout.hoff[i]):int(layout.hoff[i]) + int(layout.nbytes[i])]


def check_pushout(run, layout, dag, NT, M, N):
    """The last k pushed every C tile out whole, once: the host C equals the slab's, and bytes_d2h counts it once."""
    for c in range(2 * NT * NT, 3 * NT * NT):
        assert np.array_equal(host_tile(run, layout, c), layout.tile_bytes(run.dev, c)), c
    assert run.stats["bytes_d2h"] == NT * NT * M * N * 8, run.stats["bytes_d2h"]


@pytest.mark.parametrize("NT,M,N,K", [(1, 300, 200, 77), (2, 200, 150, 99), (4, 136, 104, 57), (8, 130, 98, 33)],
                         ids=["nt1", "nt2", "nt4", "nt8"])
def test_fp64_dtd_gemm_in_parts(NT, M, N, K):
    dag, sizes = F.dag(NT, M, N, K)
    t = F.tiles(NT, M, N, K)
    layout = fp64_layout(dag, sizes, t)
    e = entry_engine()
    try:
        want = run_engine(e, dag, layout)
    finally:
        e.close()
    got = {}
    e = part_engine()
    try:
        for n in NPARTS:
            e.set_gemm_body_parts(DGEMM, n)
            got[n] = run_engine(e, dag, layout)
    finally:
        e.close()
    check_fp64(got[1], layout, t, NT, M, N)
    for n in NPARTS:
        assert np.array_equal(got[n].dev, want.dev), "C of %d parts differs from the entry fixture's" % n
        assert np.array_equal(got[n].dev, got[1].dev), n
        check_pushout(got[n], layout, dag, NT, M, N)
        assert np.array_equal(got[n].res["seen_version"], got[1].res["seen_version"]), n
        assert not np.any(got[n].res["result"]), n


@pytest.mark.parametrize("kw", [dict(max_workers=1), dict(queue_policy=1)], ids=["one_worker", "queue_policy_1"])
def test_fp64_dtd_gemm_in_parts_one_worker_and_priority(kw):
    NT, M, N, K = 2, 260, 200, 65
    dag, sizes = F.dag(NT, M, N, K)
    dag.tasks["priority"] = np.arange(dag.ntasks, dtype=np.int32) % 3
    t = F.tiles(NT, M, N, K)
    layout = fp64_layout(dag, sizes, t)
    e = part_engine(**kw)
    try:
        got = {}
        for n in (1, 3, 8):
            e.set_gemm_body_parts(DGEMM, n)
            got[n] = run_engine(e, dag, layout)
    finally:
        e.close()
    check_fp64(got[1], layout, t, NT, M, N)
    for n in (3, 8):
        assert np.array_equal(got[n].dev, got[1].dev), n
        check_pushout(got[n], layout, dag, NT, M, N)


# ----------------------------------------------------------------------------------------------------------------------
# PART probes
# ----------------------------------------------------------------------------------------------------------------------
def probe_dag(n, tile_bytes=4096, pushout=False):
    """n PART probes, ready at start, each on a tile of its own."""
    t = dags._new_tasks(n)
    t["body"], t["nb_flows"], t["iparam"][:, 0] = PART, 1, tile_bytes
    t["tile"][:, 0] = np.arange(n)
    t["access"][:, 0] = L.ACCESS_WRITE | (L.FLOW_PUSHOUT if pushout else 0)
    return dags.Dag(t, np.zeros(0, np.uint32), np.arange(n, dtype=np.int32), ntiles=n, tile_bytes=tile_bytes, kind=1,
                    name="part_probes")


@pytest.mark.parametrize("entry", [True, False], ids=["entry", "pb2_linked_body"])
@pytest.mark.parametrize("nparts", [1, 3, 32])
def test_part_probes(entry, nparts):
    n, tb = 40, 4096
    for pushout in (False, True):
        dag = probe_dag(n, tb, pushout)
        layout = Layout.packed(dag, host=np.full(n * tb, 0xEE, np.uint8), valid=True)
        layout.dev[:] = 0
        e = part_engine(entry=entry)
        try:
            e.set_gemm_body_parts(PART, nparts)
            run, rec = run_parts(e, dag, layout)
        finally:
            e.close()
        want_res = (nparts << 40) | (0 if entry else ENTRY_BIT)
        assert np.array_equal(run.res["result"], np.full(n, want_res, np.uint64)), [hex(x) for x in run.res["result"][:4]]
        for i in range(n):
            words = layout.tile_bytes(run.dev, i).view(np.uint32)
            assert np.array_equal(words[:nparts], (nparts << 16) | (np.arange(nparts, dtype=np.uint32) + 1)), i
            assert not np.any(words[nparts:]), i
            if pushout:
                assert np.array_equal(host_tile(run, layout, i), layout.tile_bytes(run.dev, i)), i
        assert run.stats["bytes_d2h"] == (n * tb if pushout else 0)
        assert len(rec) == n * nparts
        for i in range(n):
            r = rec[rec["task"] == i]
            assert sorted(r["part"].tolist()) == list(range(nparts)) and np.all(r["nparts"] == nparts)
            retired = (r["flags"] & L.PART_RETIRED) != 0
            assert retired.sum() == 1, r
            # the retiring part pushed the tile out, once; no other part pushed anything
            assert r["out_bytes"][retired][0] == (tb if pushout else 0) and not np.any(r["out_bytes"][~retired])
        if nparts > 1:                              # the parts of a task ran on more than one SM
            assert max(len(set(rec["smid"][rec["task"] == i].tolist())) for i in range(n)) > 1


# ----------------------------------------------------------------------------------------------------------------------
# beside the application's other work
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("max_workers", [1, 0], ids=["one_worker", "all_workers"])
def test_parted_tasks_between_gemm_units_leave_the_bf16_results_unchanged(max_workers):
    NT, T, fNT, fM, fN, fK = 3, 256, 2, 260, 200, 72
    dag, sizes, probes, fbase, t0 = hazard_dag(NT, T, fNT, fM, fN, fK)
    dag.tasks["iparam"][probes, 0] = 0              # the probes have no tile: bytes[0] == iparam[0] == 0
    ft = F.tiles(fNT, fM, fN, fK)
    host = np.concatenate([bf16_host(NT, T)] + [x.reshape(-1).view(np.uint8) for x in ft])
    layout = Layout.packed(dag, host=host, valid=True, sizes=sizes)
    plain = dags.dtd_gemm(NT, tile=T)
    plain_layout = Layout.packed(plain, host=bf16_host(NT, T), valid=True)
    with Engine(0) as e:
        want = run_engine(e, plain, plain_layout)
    e = part_engine(max_workers=max_workers)
    try:
        e.set_gemm_body_parts(DGEMM, 4)
        e.set_gemm_body_parts(PART, 5)
        got = run_engine(e, dag, layout)
    finally:
        e.close()
    for c in range(2 * NT * NT, 3 * NT * NT):
        assert np.array_equal(layout.tile_bytes(got.dev, c), plain_layout.tile_bytes(want.dev, c)), c
    assert np.array_equal(got.res["result"][probes], np.full(len(probes), 5 << 40, np.uint64)), got.res["result"][probes]
    assert np.array_equal(got.res["seen_version"][:NT ** 3], want.res["seen_version"])
    check_fp64(got, layout, ft, fNT, fM, fN, base=fbase, ctile0=t0 + 2 * fNT * fNT)


def test_parted_dgemm_beside_a_read_group_on_the_reader_groups_and_entry_link():
    NT, M, N, K, k, nsum, xb = 2, 300, 136, 48, -12345, 4, 3 << 20
    rng = np.random.default_rng(5)
    x0 = rng.integers(-1 << 31, 1 << 31, xb // 4, dtype=np.int64).astype(np.int32)
    x1 = (x0.astype(np.int64) + k).astype(np.int32)
    total = np.uint64(int(x1.astype(np.int64).sum()) % (1 << 64))
    t = F.tiles(NT, M, N, K)
    dag, sizes, add = mixed_dag(NT, M, N, K, k, nsum, xb, 1)
    host = np.concatenate([x.reshape(-1).view(np.uint8) for x in t] + [x0.view(np.uint8)])
    layout = Layout.packed(dag, host=host, valid=True, sizes=sizes)
    got = {}
    e = part_engine(groups=True, part_bytes=256 * 1024)
    try:
        for n in (1, 6):
            e.set_gemm_body_parts(DGEMM, n)
            got[n] = run_engine(e, dag, layout)
    finally:
        e.close()
    check_fp64(got[6], layout, t, NT, M, N)
    assert np.array_equal(got[6].dev, got[1].dev)
    assert np.array_equal(layout.tile_bytes(got[6].dev, dag.ntiles - 1).view(np.int32), x1)
    assert got[6].res["result"][add] == 0
    assert np.array_equal(got[6].res["result"][add + 1:], np.full(nsum, total, np.uint64)), got[6].res["result"][add + 1:]


# ----------------------------------------------------------------------------------------------------------------------
# the stand-alone runtime
# ----------------------------------------------------------------------------------------------------------------------
def test_fp64_dtd_gemm_through_the_runtime_in_parts():
    NT, M, N, K = 2, 300, 200, 77
    t = F.tiles(NT, M, N, K)
    out = {}
    for n in (1, 8):
        with R.Context(cuda_devices=(0,)) as ctx:
            dev = ctx.devices[0]
            ctx.link_bodies(dev, image("gemm_part_bodies"), L.IMAGE_CUBIN, 0, gemm_windows=True, gemm_bodies=F.GEMM_BODIES,
                            gemm_body_entry=True)
            ctx.set_gemm_body_parts(dev, DGEMM, n)
            assert ctx.gemm_body_parts(dev, DGEMM) == n
            tp, bufs = F.insert(ctx, NT, M, N, K, t)
            ctx.wait()
            st = ctx.stats(dev)
            info = ctx.task_info(tp)
            assert ctx.l.pb2_device_memory_release(dev) == 0
        assert st["executed_tasks"] == NT ** 3 and not np.any(info["result"])
        out[n] = bufs["C"].copy()
    for i in range(NT):
        for j in range(NT):
            want, bound = F.reference(t, NT, i, j)
            assert np.all(np.abs(F.runtime_tile({"C": out[8]}, "C", i, j, NT, M, N) - want) <= bound), (i, j)
    assert np.array_equal(out[8], out[1]), "C of 8 parts differs from one part's"
