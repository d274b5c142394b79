"""CPU tests of the window planner (parsec_b200/csrc/pb2_window_plan.cpp): what pb2_window_create uploads for a DAG --
read groups and fused producers, parts, priority lanes and the ring image, GEMM units, part records -- and the windows
it refuses.  The planner is built with g++ and no CUDA include path, through the shim tests/cpp/window_plan_shim.cpp.
Each expectation restates a rule of DESIGN.md §5 or tests/priority_order.py, not the C++."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from priority_order import lane_of
from test_priority import random_dag
from window_harness import KS, readers_dag

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GROUP_FUSED, GROUP_MAX, MAX_PARTS, GEMM_MAX_PARTS, EMPTY = 0x80000000, 8, 512, 32, -1
NWORKERS, NWORKERS_GEMM = 1056, 132
UNIT_DTYPE = np.dtype([(n, "<i4") for n in ("seg_begin", "seg_count", "succ_begin", "succ_count", "dep_goal", "nparts",
                                            "tileC", "M", "N", "K", "flags", "pad")])
SEG_DTYPE = np.dtype([(n, "<i4") for n in ("task", "tileA", "tileB", "pad")])
ENTITY_DTYPE = np.dtype([(n, "<i4") for n in ("lead", "base", "nparts")])
ARRAYS = {"tasks": L.TASK_DTYPE, "succ": np.uint32, "group": np.uint32, "group_mem": np.int32, "nparts": np.uint16,
          "units": UNIT_DTYPE, "segs": SEG_DTYPE, "usucc": np.int32, "lane": np.uint8, "part_base": np.int32,
          "ring_image": np.int32, "operand_rows": np.int32, "operand_inner": np.int32, "task_entry": np.int32,
          "task_unit": np.int32, "part_entities": ENTITY_DTYPE, "lane_begin": np.uint32, "lane_ninit": np.uint32}
SCALARS = ("slice_bytes", "nlanes", "linked", "ring", "nunits", "parts", "claims", "lanes", "trace", "part_records")
PARAMS = ("kind", "shared", "trace", "linked_image", "queue_policy", "gemm_mode", "read_groups", "fuse_readers",
          "nworkers", "nworkers_gemm", "part_bytes", "stage_slice_bytes", "linked_sliceable")
DEFAULTS = dict(kind=0, shared=0, trace=0, linked_image=0, queue_policy=0, gemm_mode=0, read_groups=0, fuse_readers=0,
                nworkers=NWORKERS, nworkers_gemm=NWORKERS_GEMM, part_bytes=256 * 1024, stage_slice_bytes=64 * 1024,
                linked_sliceable=0)


@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("plan") / "window_plan.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-Iinclude", "-Iparsec_b200/csrc",
                    "tests/cpp/window_plan_shim.cpp", "parsec_b200/csrc/pb2_window_plan.cpp", "-o", so],
                   cwd=ROOT, check=True)
    lib = C.CDLL(so)
    lib.wp_plan.restype = C.c_void_p
    lib.wp_plan.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                            C.c_void_p, C.c_int32, C.POINTER(C.c_int), C.POINTER(C.c_char_p)]
    lib.wp_free.argtypes = [C.c_void_p]
    lib.wp_array.restype = C.c_int64
    lib.wp_array.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p)]
    lib.wp_scalar.restype = C.c_int64
    lib.wp_scalar.argtypes = [C.c_void_p, C.c_char_p]
    return lib


def tiles_for(ntiles, nbytes, state=L.TILE_VALID):
    tiles = np.zeros(ntiles, L.TILE_DTYPE)
    tiles["bytes"] = nbytes
    tiles["state"] = state
    tiles["dev_ptr"] = 0x10000 + np.arange(ntiles, dtype=np.uint64) * np.uint64(1 << 24)
    return tiles


def plan_of(lib, tasks, succ, tiles, ready, next_rs_begin=None, **kw):
    """(rc, why, plan): plan maps every array and scalar name of the plan to its value (None when refused)."""
    prm = np.array([kw.get(k, DEFAULTS[k]) for k in PARAMS], np.int64)
    tasks = np.ascontiguousarray(tasks, L.TASK_DTYPE)
    succ = np.ascontiguousarray(succ, np.uint32)
    tiles = np.ascontiguousarray(tiles, L.TILE_DTYPE)
    ready = np.ascontiguousarray(ready, np.int32)
    rs = None if next_rs_begin is None else np.ascontiguousarray(next_rs_begin, np.int32)
    rc, why = C.c_int(0), C.c_char_p()
    h = lib.wp_plan(prm.ctypes.data, rs.ctypes.data if rs is not None else None, tasks.ctypes.data, len(tasks),
                    succ.ctypes.data, len(succ), tiles.ctypes.data, len(tiles), ready.ctypes.data, len(ready),
                    C.byref(rc), C.byref(why))
    if not h:
        return rc.value, why.value.decode() if why.value else None, None
    try:
        out = {}
        for name, dt in ARRAYS.items():
            p = C.c_void_p()
            n = lib.wp_array(h, name.encode(), C.byref(p))
            assert n >= 0, name
            out[name] = np.frombuffer(C.string_at(p.value, n) if n else b"", dtype=dt).copy()
        for name in SCALARS:
            out[name] = lib.wp_scalar(h, name.encode())
        return rc.value, None, out
    finally:
        lib.wp_free(h)


def plan_dag(lib, dag, tiles=None, **kw):
    if tiles is None:
        tiles = tiles_for(dag.ntiles, dag.tile_bytes)
    rc, why, p = plan_of(lib, dag.tasks, dag.succ, tiles, dag.ready, **kw)
    assert rc == 0, why
    return p


def members(p, word):
    b = (int(word) & ~GROUP_FUSED & 0xFFFFFFFF) >> 4
    return [int(m) for m in p["group_mem"][b:b + (int(word) & 15)]]


def device_edges(p, u):
    t = p["tasks"][u]
    return [int(s) for s in p["succ"][t["succ_begin"]:t["succ_begin"] + t["succ_count"]]]


def expanded_edges(p, u):
    """Task u's out-edges as the device releases them: an edge to a group leader reaches every member, and a fused
    producer's group is released with it."""
    out = []
    for s in device_edges(p, u):
        t, flow = s & 0x07FFFFFF, s >> 27
        w = int(p["group"][t]) if len(p["group"]) else 0
        out += [(flow << 27) | m for m in members(p, w)] if w & 15 and not w & GROUP_FUSED else [s]
    if len(p["group"]) and p["group"][u] & GROUP_FUSED:
        out += members(p, p["group"][u])
    return sorted(out)


def original_edges(dag, u):
    t = dag.tasks[u]
    return sorted(int(s) for s in dag.succ[t["succ_begin"]:t["succ_begin"] + t["succ_count"]])


# ---------------------------------------------------------------------------------------------------------------
# read groups and fused producers (DESIGN.md §5)
# ---------------------------------------------------------------------------------------------------------------
def test_ex05_readers_run_as_one_group_fused_with_their_producer(planner):
    dag = dags.ex05_broadcast(6)
    K, F = 6, dag.meta["F"]
    assert F == 8
    p = plan_dag(planner, dag)
    for k in range(K):
        recv = [K + k * F + n for n in range(F)]
        assert p["group"][k] & GROUP_FUSED and members(p, p["group"][k]) == recv
        assert int(p["group"][recv[0]]) == int(p["group"][k]) & ~GROUP_FUSED
        assert recv[0] not in [s & 0x07FFFFFF for s in device_edges(p, k)]
        assert all(p["group"][r] == 0 for r in recv[1:])


@pytest.mark.parametrize("kw", [dict(nworkers=1), dict(fuse_readers=-1)])
def test_ex05_groups_stay_plain_without_fusion(planner, kw):
    dag = dags.ex05_broadcast(4)
    K, F = 4, dag.meta["F"]
    p = plan_dag(planner, dag, **kw)
    for k in range(K):
        recv = [K + k * F + n for n in range(F)]
        assert p["group"][k] == 0
        assert members(p, p["group"][recv[0]]) == recv
        assert device_edges(p, k) == [recv[0]]


@pytest.mark.parametrize("kw", [dict(read_groups=-1), dict(shared=1)])
def test_no_groups_keep_the_input_csr(planner, kw):
    dag = dags.ex05_broadcast(4)
    p = plan_dag(planner, dag, **kw)
    assert len(p["group"]) == 0 and len(p["group_mem"]) == 0
    assert np.array_equal(p["succ"], dag.succ)
    assert np.array_equal(p["tasks"]["succ_begin"], dag.tasks["succ_begin"])
    assert np.array_equal(p["tasks"]["succ_count"], dag.tasks["succ_count"])


@pytest.mark.parametrize("NB", [30, 34])
def test_long_runs_of_readers_split_at_group_max(planner, NB):
    dag = dags.ex05_broadcast(3, NB=NB)
    K, F = 3, dag.meta["F"]
    assert F > GROUP_MAX
    p = plan_dag(planner, dag)
    for k in range(K):
        recv = [K + k * F + n for n in range(F)]
        runs = [recv[i:i + GROUP_MAX] for i in range(0, F, GROUP_MAX)]
        runs = [r for r in runs if len(r) >= 2]
        assert members(p, p["group"][k]) == runs[0]             # the first group runs with the producer
        for r in runs:
            assert members(p, p["group"][r[0]]) == r
        assert expanded_edges(p, k) == original_edges(dag, k)


def mixed_readers_dag(n, seed):
    """random_dag with CHECK readers of one tile: task j reads when its body is CHECK_I32."""
    dag = random_dag(n, seed, 3, tile_bytes=4096, ntiles=2, body_mix=(L.BODY_INCR_I32, L.BODY_CHECK_I32, L.BODY_CHECK_I32))
    chk = dag.tasks["body"] == L.BODY_CHECK_I32
    dag.tasks["access"][chk, 0] = L.ACCESS_READ
    return dag


@pytest.mark.parametrize("make", [lambda: mixed_readers_dag(300, 1), lambda: mixed_readers_dag(500, 2),
                                  lambda: random_dag(200, 3, 5), lambda: readers_dag(L.BODY_FILL_I32, 5, KS, 4096),
                                  lambda: readers_dag(L.BODY_IOTA_I32, 0, KS + KS[:3], 4096)])
@pytest.mark.parametrize("kw", [dict(), dict(nworkers=1)])
def test_groups_keep_every_edge(planner, make, kw):
    dag = make()
    p = plan_dag(planner, dag, **kw)
    for u in range(dag.ntasks):
        assert expanded_edges(p, u) == original_edges(dag, u)


def test_random_readers_form_groups(planner):
    p = plan_dag(planner, mixed_readers_dag(500, 2))
    assert len(p["group_mem"]) > 0 and (p["group"] & GROUP_FUSED).any()


# ---------------------------------------------------------------------------------------------------------------
# parts and the ring
# ---------------------------------------------------------------------------------------------------------------
def expected_parts(tasks, tile_bytes, part_bytes, sliceable=0):
    out = []
    for t in tasks:
        linked = L.BODY_LINKED_0 <= t["body"] <= L.BODY_LINKED_7
        if t["body"] == L.BODY_NOP or (linked and not (sliceable >> (t["body"] - L.BODY_LINKED_0)) & 1):
            out.append(1)
            continue
        widest = max([int(tile_bytes[f]) for f in t["tile"][:t["nb_flows"]] if f >= 0], default=0)
        out.append(max(1, min(math.ceil(widest / part_bytes), MAX_PARTS)))
    return np.array(out)


def ent(task, part):
    return np.int32(np.uint32((part << 22) | task).view(np.int32))


def ring_for(slots, nworkers=NWORKERS):
    cap = 1024
    while cap < slots + nworkers + 2:
        cap <<= 1
    return cap


def test_parts_entries_and_ring(planner):
    dag = random_dag(120, 7, 4, ntiles=8)
    rng = np.random.default_rng(7)
    sizes = np.array([16, 5000, 65536, 100000, 4 << 20, 1 << 20, 64, 3000], np.uint32)
    dag.tasks["body"][5] = L.BODY_NOP
    dag.tasks["body"][[6, 7]] = [L.BODY_LINKED_0, L.BODY_LINKED_0 + 1]
    dag.tasks["nb_flows"][9], dag.tasks["tile"][9, 1] = 2, int(rng.integers(0, 8))
    part_bytes = 4096
    p = plan_dag(planner, dag, tiles_for(8, sizes), part_bytes=part_bytes, linked_image=1, linked_sliceable=0b10)
    parts = expected_parts(dag.tasks, sizes, part_bytes, 0b10)
    assert parts.max() == MAX_PARTS and parts[6] == 1
    assert np.array_equal(p["task_entry"], [ent(t, n - 1) for t, n in enumerate(parts)])
    assert np.array_equal(p["nparts"], parts)
    assert p["parts"] == 1 and p["claims"] == 1 and p["linked"] == 1
    assert np.array_equal(p["ring_image"], [ent(int(t), q) for t in dag.ready for q in range(parts[t])])
    assert p["ring"] == ring_for(dag.ntasks + int((parts - 1).sum()))
    assert p["slice_bytes"] == part_bytes          # the smaller of stage_slice_bytes and part_bytes


def test_one_part_windows_claim_only_for_wide_tiles_to_stage(planner):
    dag = random_dag(50, 8, 2, tile_bytes=100000)
    p = plan_dag(planner, dag, tiles_for(dag.ntiles, 100000))
    assert p["parts"] == 0 and p["claims"] == 0 and len(p["nparts"]) == 0
    assert np.array_equal(p["task_entry"], np.arange(dag.ntasks))
    tiles = tiles_for(dag.ntiles, 100000)
    tiles["state"][2] = L.TILE_INVALID
    p = plan_dag(planner, dag, tiles)
    assert p["parts"] == 0 and p["claims"] == 1            # 100000 bytes > a 64 KiB stage-in slice


# ---------------------------------------------------------------------------------------------------------------
# priority lanes (queue_policy 1, tests/priority_order.py)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nprio", [1, 16, 40])
def test_priority_lanes_and_ring_image(planner, nprio):
    dag = random_dag(300, nprio, nprio, tile_bytes=1000)
    part_bytes = 400                                       # three parts per task
    p = plan_dag(planner, dag, queue_policy=1, part_bytes=part_bytes)
    lane = lane_of(dag.tasks["priority"], 16)
    parts = expected_parts(dag.tasks, np.full(dag.ntiles, 1000), part_bytes)
    assert p["lanes"] == 1 and p["nlanes"] == min(len(np.unique(dag.tasks["priority"])), 16)
    assert np.array_equal(p["lane"], lane)
    pushes = np.bincount(lane, weights=parts, minlength=16).astype(np.int64)
    begin = np.concatenate([[0], np.cumsum(pushes)[:-1]])
    assert np.array_equal(p["lane_begin"], begin)
    ring = np.full(int(pushes.sum()), EMPTY, np.int64)
    for ln in range(16):
        first = [ent(int(t), q) for t in dag.ready if lane[t] == ln for q in range(parts[t])]
        assert p["lane_ninit"][ln] == len(first)
        ring[begin[ln]:begin[ln] + len(first)] = first
    assert np.array_equal(p["ring_image"], ring)


# ---------------------------------------------------------------------------------------------------------------
# GEMM windows: units (pb2_gemm.cuh)
# ---------------------------------------------------------------------------------------------------------------
def morton(x, y):
    return sum((((x >> b) & 1) << (2 * b + 1)) | (((y >> b) & 1) << (2 * b)) for b in range(16))


@pytest.mark.parametrize("NT,tile", [(3, 512), (4, 256), (2, 384)])
def test_gemm_k_chains_become_units(planner, NT, tile):
    dag = dags.dtd_gemm(NT, tile=tile)
    p = plan_dag(planner, dag, kind=1)
    units, segs = p["units"], p["segs"]
    assert p["nunits"] == len(units) == NT * NT
    nparts = min(math.ceil(tile / 128) * math.ceil(tile / 256), GEMM_MAX_PARTS)
    for u in units:
        chain = segs["task"][u["seg_begin"]:u["seg_begin"] + u["seg_count"]]
        assert u["seg_count"] == NT and np.array_equal(chain, chain[0] + np.arange(NT)) and chain[0] % NT == 0
        assert u["nparts"] == nparts and u["flags"] == 3 and u["dep_goal"] == 0
    # dtd_gemm has no edges besides the chain links
    assert len(p["usucc"]) == 0 and (units["succ_count"] == 0).all()
    unit_of = {int(segs["task"][u["seg_begin"]]) // NT: i for i, u in enumerate(units)}
    ij = sorted(((i, j) for i in range(NT) for j in range(NT)), key=lambda c: morton(*c))
    expect = [(q << 27) | unit_of[i * NT + j] for i, j in ij for q in range(nparts)]
    assert np.array_equal(p["ring_image"].view(np.uint32), expect)
    assert np.array_equal(p["task_entry"].view(np.uint32),
                          [((nparts - 1) << 27) | unit_of[t // NT] for t in range(dag.ntasks)])
    assert np.array_equal(p["operand_rows"][:2 * NT * NT], np.full(2 * NT * NT, tile))
    assert (p["operand_rows"][2 * NT * NT:] == 0).all()
    assert p["claims"] == 1 and p["slice_bytes"] == 64 * 1024


def test_gemm_mode_2_runs_every_task_as_a_unit(planner):
    dag = dags.dtd_gemm(3)
    p = plan_dag(planner, dag, kind=1, gemm_mode=2)
    assert len(p["units"]) == dag.ntasks and (p["units"]["seg_count"] == 1).all()
    assert np.array_equal(p["segs"]["task"], np.arange(dag.ntasks))
    # every chain link is now an edge between units
    assert sorted(p["usucc"]) == sorted(int(s) & 0x07FFFFFF for s in dag.succ)


def mixed_pool(K, c_bytes):
    """FILL C -> K GEMMs accumulating into C -> CHECK C: the GEMM chain between two HBM bodies."""
    n = K + 2
    t = dags._new_tasks(n)
    t["body"][0], t["body"][1:K + 1], t["body"][K + 1] = L.BODY_FILL_I32, L.BODY_GEMM_BF16, L.BODY_CHECK_I32
    t["nb_flows"][0], t["tile"][0, 0], t["access"][0, 0] = 1, 0, L.ACCESS_WRITE
    t["nb_flows"][K + 1], t["tile"][K + 1, 0], t["access"][K + 1, 0] = 1, 0, L.ACCESS_READ
    g = t[1:K + 1]
    g["nb_flows"] = 3
    g["tile"][:, 0], g["tile"][:, 1], g["tile"][:, 2] = np.arange(K) + 1, np.arange(K) + 1 + K, 0
    g["access"][:, 0], g["access"][:, 1], g["access"][:, 2] = L.ACCESS_READ, L.ACCESS_READ, L.ACCESS_RW
    g["iparam"][:] = 256
    t["dep_goal"][1:] = 1
    flows = [2] * (K + 1)
    flows[-1] = 0
    begin, count, succ = dags._csr_from_edges(n, np.arange(K + 1), np.arange(1, K + 2), np.array(flows))
    t["succ_begin"], t["succ_count"] = begin, count
    tiles = tiles_for(1 + 2 * K, 256 * 256 * 2)
    tiles["bytes"][0] = c_bytes
    return dags.Dag(t, succ, np.array([0], np.int32), ntiles=1 + 2 * K, tile_bytes=0, kind=1), tiles


@pytest.mark.parametrize("shared", [0, 1])
def test_mixed_pool_cuts_hbm_units_by_the_part_rule(planner, shared):
    K, c_bytes, part_bytes = 4, 1 << 20, 64 * 1024
    dag, tiles = mixed_pool(K, c_bytes)
    p = plan_dag(planner, dag, tiles, kind=1, shared=shared, part_bytes=part_bytes)
    units, segs = p["units"], p["segs"]
    assert len(units) == 3
    hbm = 1 if shared else min(c_bytes // part_bytes, GEMM_MAX_PARTS)
    assert list(units["nparts"]) == [hbm, 2, hbm]           # C is 256 x 256: two 128 x 256 sub-tiles
    assert list(units["seg_count"]) == [1, K, 1] and list(units["flags"]) == [0, 1, 0]
    assert list(segs["task"]) == list(range(K + 2))
    assert list(p["usucc"]) == [1, 2]


# ---------------------------------------------------------------------------------------------------------------
# part records of traced windows (DESIGN.md §5)
# ---------------------------------------------------------------------------------------------------------------
def check_records(p, owner_parts, owner_lead):
    owner_parts = np.asarray(owner_parts)
    assert np.array_equal(p["part_base"], np.concatenate([[0], np.cumsum(owner_parts)[:-1]]))
    assert p["part_records"] == owner_parts.sum()
    ents = p["part_entities"]
    own = np.flatnonzero(owner_parts > 0)
    assert sorted(zip(ents["lead"], ents["base"], ents["nparts"])) == \
        sorted(zip(np.asarray(owner_lead)[own], p["part_base"][own], owner_parts[own]))
    assert (np.diff(ents["lead"]) >= 0).all()


@pytest.mark.parametrize("kw", [dict(), dict(nworkers=1), dict(read_groups=-1)])
def test_part_records_of_hbm_windows(planner, kw):
    dag = dags.ex05_broadcast(5, tile_bytes=1 << 20)
    K, F = 5, dag.meta["F"]
    p = plan_dag(planner, dag, trace=1, part_bytes=256 * 1024, **kw)
    parts = np.full(dag.ntasks, 4)
    lead = np.arange(dag.ntasks)
    if kw.get("read_groups", 0) >= 0:
        for k in range(K):
            recv = K + k * F + np.arange(F)
            lead[recv] = k if not kw else recv[0]
    assert np.array_equal(p["task_unit"], lead)
    check_records(p, np.where(lead == np.arange(dag.ntasks), parts, 0), np.arange(dag.ntasks))


def test_part_records_of_gemm_windows(planner):
    NT = 3
    dag = dags.dtd_gemm(NT)
    p = plan_dag(planner, dag, kind=1, trace=1)
    heads = p["segs"]["task"][p["units"]["seg_begin"]]
    assert np.array_equal(p["task_unit"], np.arange(dag.ntasks) // NT * NT)
    check_records(p, p["units"]["nparts"], heads)


def test_untraced_windows_have_no_records(planner):
    p = plan_dag(planner, dags.ex05_broadcast(3))
    assert len(p["task_unit"]) == 0 and len(p["part_base"]) == 0 and p["part_records"] == 0


# ---------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------
def refused(lib, dag, tiles=None, **kw):
    if tiles is None:
        tiles = tiles_for(dag.ntiles, dag.tile_bytes)
    rc, why, p = plan_of(lib, dag.tasks, dag.succ, tiles, dag.ready, **kw)
    assert p is None
    return rc, why


def test_refusals_of_the_argument_checks(planner):
    dag = dags.ex05_broadcast(2)
    assert refused(planner, dag, kind=2) == (L.PB2_ERR_BAD_PARAM, "window kind must be 0 (HBM bodies) or 1 (GEMM bodies)")
    bad = dags.ex05_broadcast(2)
    bad.tasks["tile"][3, 0] = 7
    assert refused(planner, bad) == (L.PB2_ERR_VALUE_OUT_OF_BOUNDS, "tile id out of bounds")
    bad = dags.ex05_broadcast(2)
    bad.succ = bad.succ.copy()
    bad.succ[0] = 99
    assert refused(planner, bad) == (L.PB2_ERR_VALUE_OUT_OF_BOUNDS, "successor id out of bounds")
    bad = dags.ex05_broadcast(2)
    bad.ready = np.array([0, 40], np.int32)
    assert refused(planner, bad) == (L.PB2_ERR_VALUE_OUT_OF_BOUNDS, "ready id out of bounds")
    bad = dags.ex05_broadcast(2)
    bad.tasks["body"][0] = L.BODY_GEMM_BF16
    assert refused(planner, bad) == (L.PB2_ERR_BAD_PARAM, "GEMM body in an HBM-kind window (use kind 1)")
    bad = dags.ex05_broadcast(2)
    bad.tasks["body"][0] = L.BODY_LINKED_0
    assert refused(planner, bad) == (L.PB2_ERR_NOT_SUPPORTED,
                                     "linked body id, but the engine has not linked an image (pb2_engine_link_bodies)")
    assert refused(planner, bad, linked_image=1, shared=1) == (L.PB2_ERR_NOT_SUPPORTED,
                                                               "linked body in a shared window (not supported)")
    assert refused(planner, dag, queue_policy=1, shared=1) == (
        L.PB2_ERR_NOT_SUPPORTED,
        "queue_policy 1 (priority lanes) is not supported with shared windows: peers push into one FIFO ring")


def test_refusals_of_gemm_windows(planner):
    dag = dags.dtd_gemm(2)
    bad = dags.dtd_gemm(2)
    bad.tasks["iparam"][3, 1] = 100
    assert refused(planner, bad, kind=1) == (L.PB2_ERR_NOT_SUPPORTED, "GEMM tile: need M,N,K > 0, K % 8 == 0, N % 8 == 0")
    bad = dags.dtd_gemm(2)
    bad.tasks["iparam"][3, 1] = 256
    assert refused(planner, bad, kind=1) == (L.PB2_ERR_NOT_SUPPORTED, "tile used with two different operand shapes")
    tiles = tiles_for(dag.ntiles, dag.tile_bytes)
    tiles["bytes"][1] = 1024
    assert refused(planner, dag, tiles, kind=1) == (L.PB2_ERR_VALUE_OUT_OF_BOUNDS, "GEMM operand larger than its tile")
    tiles = tiles_for(dag.ntiles, dag.tile_bytes)
    tiles["bytes"][-1] = 1024
    assert refused(planner, dag, tiles, kind=1) == (L.PB2_ERR_VALUE_OUT_OF_BOUNDS, "GEMM C larger than its tile")
    tiles = tiles_for(dag.ntiles, dag.tile_bytes)
    tiles["dev_ptr"][2] += 8
    assert refused(planner, dag, tiles, kind=1) == (L.PB2_ERR_BAD_PARAM, "GEMM tile not 16-byte aligned")
    bad = dags.dtd_gemm(2)
    bad.ready = np.array([0, 1], np.int32)
    assert refused(planner, bad, kind=1, gemm_mode=2) == (L.PB2_ERR_BAD_PARAM, "ready task has in-window predecessors")
    bad = dags.dtd_gemm(2)
    bad.tasks["dep_goal"][:] = 0
    bad.ready = np.array([0], np.int32)
    assert refused(planner, bad, kind=1, shared=1) == (L.PB2_ERR_BAD_PARAM,
                                                       "dependency goal smaller than the in-window in-degree")
