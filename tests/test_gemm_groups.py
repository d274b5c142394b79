"""CPU tests of read groups and fused producers in GEMM windows (pb2_window_plan.cpp): a kind-1 window plans its HBM-body
tasks as an HBM window plans them -- the same groups, fused producers, device CSR and part records, with the GEMM
window's part rule -- and runs each group as one unit, in its leader's (or its producer's) priority lane.  A GEMM
window with priority lanes and one worker forms no group."""
import os
import re

import numpy as np
import pytest

from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from test_window_plan import (GEMM_MAX_PARTS, GROUP_FUSED, NWORKERS_GEMM, device_edges, members, mixed_readers_dag,
                              plan_dag, planner, tiles_for)  # noqa: F401  (planner is a fixture)
from priority_order import lane_of
from gemm_chain_dags import MNK, with_gemm_chain

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PART = 256 * 1024


def sizes_of(dag, elementwise_bytes):
    return np.array([elementwise_bytes] * (dag.ntiles - 3) + [MNK * MNK * 2] * 3, np.uint32)


def unit_of(p):
    """Per task, the unit that holds it (from the units' segments)."""
    out = np.full(len(p["tasks"]), -1, np.int64)
    for u, unit in enumerate(p["units"]):
        out[p["segs"]["task"][unit["seg_begin"]:unit["seg_begin"] + unit["seg_count"]]] = u
    return out


def assert_plans_as_hbm(lib, base, gemm, sizes, **kw):
    """The kind-1 plan of `gemm` (base's tasks first, then a GEMM chain and its C readers) treats base's tasks as the HBM
    plan of base does: groups, fused producers, device out-edges, units of the groups, part records (GEMM part rule)."""
    n0 = base.ntasks
    p0 = plan_dag(lib, base, tiles_for(base.ntiles, sizes[:base.ntiles]), kind=0, trace=1, **kw)
    p1 = plan_dag(lib, gemm, tiles_for(gemm.ntiles, sizes), kind=1, trace=1, **kw)
    g0 = p0["group"] if len(p0["group"]) else np.zeros(n0, np.uint32)
    g1 = p1["group"] if len(p1["group"]) else np.zeros(gemm.ntasks, np.uint32)
    for u in range(n0):
        assert int(g1[u]) & (GROUP_FUSED | 15) == int(g0[u]) & (GROUP_FUSED | 15), u
        if g0[u] & 15:
            assert members(p1, g1[u]) == members(p0, g0[u]), u
        assert device_edges(p1, u) == device_edges(p0, u), u
    assert np.array_equal(p1["task_unit"][:n0], p0["task_unit"])
    # a group is one unit: its first task (producer or leader), then its members in order; flag bit 2 for a producer
    units = unit_of(p1)
    for u in range(n0):
        if not g1[u] & 15:
            continue
        m = members(p1, g1[u])
        seq = ([u] if g1[u] & GROUP_FUSED else []) + m
        unit = p1["units"][units[u]]
        if g1[u] & GROUP_FUSED or not (p0["group"][u] and any(g1[v] & GROUP_FUSED and members(p1, g1[v]) == m for v in range(n0))):
            assert p1["segs"]["task"][unit["seg_begin"]:unit["seg_begin"] + unit["seg_count"]].tolist() == seq, u
            assert bool(unit["flags"] & 4) == bool(g1[u] & GROUP_FUSED), u
            assert np.all(units[seq] == units[u]), u
    # part records: the HBM plan's entities, each with the GEMM window's part count
    e0 = {int(e["lead"]): int(e["nparts"]) for e in p0["part_entities"]}
    e1 = {int(e["lead"]): int(e["nparts"]) for e in p1["part_entities"] if e["lead"] < n0}
    assert e1.keys() == e0.keys()
    pb = kw.get("part_bytes", PART)
    for lead, n in e1.items():
        t = base.tasks[lead]
        widest = max(int(sizes[f]) for f in t["tile"][:t["nb_flows"]] if f >= 0)
        assert n == (max(1, min(-(-widest // pb), GEMM_MAX_PARTS)) if pb > 0 else 1), lead
    return p0, p1


@pytest.mark.parametrize("kw", [dict(), dict(fuse_readers=-1), dict(part_bytes=16384), dict(queue_policy=1)])
def test_ex05_beside_a_chain_plans_as_the_hbm_window(planner, kw):
    ex = dags.ex05_broadcast(8, tile_bytes=256 * 1024)
    gemm = with_gemm_chain(ex)
    p0, p1 = assert_plans_as_hbm(planner, ex, gemm, sizes_of(gemm, 256 * 1024), **kw)
    F = ex.meta["F"]
    for k in range(8):
        recv = [8 + k * F + n for n in range(F)]
        fusedw = not kw.get("fuse_readers")
        assert bool(p1["group"][k] & GROUP_FUSED) == fusedw and members(p1, p1["group"][k] if fusedw else p1["group"][recv[0]]) == recv


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("kw", [dict(), dict(nworkers=1, nworkers_gemm=1), dict(queue_policy=1), dict(gemm_mode=2)])
def test_random_dags_beside_a_chain_plan_as_the_hbm_window(planner, seed, kw):
    base = mixed_readers_dag(300 + 100 * seed, seed)
    gemm = with_gemm_chain(base)
    assert_plans_as_hbm(planner, base, gemm, sizes_of(gemm, 4096), **kw)


@pytest.mark.parametrize("gemm_mode", [0, 2])
def test_readers_of_a_chains_c_form_a_group(planner, gemm_mode):
    gemm = with_gemm_chain(dags.ex05_broadcast(2, tile_bytes=4096), nchain=3, readers=(5, 5, 6, 5))
    p = plan_dag(planner, gemm, tiles_for(gemm.ntiles, sizes_of(gemm, 4096)), kind=1, gemm_mode=gemm_mode)
    last, readers = gemm.ntasks - 5, list(range(gemm.ntasks - 4, gemm.ntasks))
    assert members(p, p["group"][readers[0]]) == readers
    assert p["group"][last] == 0                         # a GEMM task never runs with a group
    assert [s & 0x07FFFFFF for s in device_edges(p, last)] == [readers[0]]
    u = unit_of(p)
    assert len(set(u[readers].tolist())) == 1 and u[last] != u[readers[0]]
    assert p["units"][u[readers[0]]]["flags"] & 5 == 0
    # the chain itself: one unit with gemm_mode 0, one per task with 2
    assert len(set(u[last - 2:last + 1].tolist())) == (1 if gemm_mode == 0 else 3)


def test_gemm_tasks_are_never_fused_or_grouped(planner):
    """A GEMM task is neither a fused producer nor a group member, even when it is the only writer of the readers' tile."""
    gemm = with_gemm_chain(dags.ex05_broadcast(2, tile_bytes=4096), nchain=1, readers=(1, 1, 1))
    p = plan_dag(planner, gemm, tiles_for(gemm.ntiles, sizes_of(gemm, 4096)), kind=1)
    isg = gemm.tasks["body"] == L.BODY_GEMM_BF16
    assert not np.any(p["group"][isg]) and not np.isin(p["group_mem"], np.flatnonzero(isg)).any()
    assert len(p["group_mem"]) > 0


@pytest.mark.parametrize("kw", [dict(shared=1), dict(read_groups=-1)])
def test_no_groups_in_shared_windows_or_with_groups_off(planner, kw):
    gemm = with_gemm_chain(dags.ex05_broadcast(4, tile_bytes=4096))
    p = plan_dag(planner, gemm, tiles_for(gemm.ntiles, sizes_of(gemm, 4096)), kind=1, **kw)
    assert len(p["group"]) == 0 and len(p["group_mem"]) == 0
    assert np.array_equal(p["succ"], gemm.succ)
    assert len(p["units"]) == gemm.ntasks - 1             # the k-chain of two is one unit, every other task its own


@pytest.mark.parametrize("kw", [dict(fuse_readers=-1), dict(nworkers_gemm=1)])
def test_no_fusion_with_fusion_off_or_one_worker(planner, kw):
    gemm = with_gemm_chain(dags.ex05_broadcast(4, tile_bytes=4096))
    p = plan_dag(planner, gemm, tiles_for(gemm.ntiles, sizes_of(gemm, 4096)), kind=1, **kw)
    assert len(p["group_mem"]) > 0 and not np.any(p["group"] & GROUP_FUSED)
    assert not np.any(p["units"]["flags"] & 4)


def test_lanes_of_groups_and_fused_units(planner):
    """queue_policy 1: a group runs in its leader's lane and a fused unit in its producer's, whatever lanes its other
    members are in, as in an HBM window."""
    ex = dags.ex05_broadcast(6, tile_bytes=4096)
    F = ex.meta["F"]
    ex.tasks["priority"][:6] = [5, 4, 3, 2, 1, 0]                    # producers
    for k in range(6):
        ex.tasks["priority"][6 + k * F:6 + (k + 1) * F] = k % 3     # their readers, one lane per tile
    ex.tasks["priority"][6 + 5 * F + 3] = 9                         # tile 5: one reader in a lane of its own
    gemm = with_gemm_chain(ex, priority=7)
    lanes = lane_of(gemm.tasks["priority"], 16)
    for kw in (dict(), dict(fuse_readers=-1)):
        assert_plans_as_hbm(planner, ex, gemm, sizes_of(gemm, 4096), queue_policy=1, **kw)
        p = plan_dag(planner, gemm, tiles_for(gemm.ntiles, sizes_of(gemm, 4096)), kind=1, queue_policy=1, **kw)
        first = p["segs"]["task"][p["units"]["seg_begin"]]
        assert np.array_equal(p["lane"], lanes[first])
        u = unit_of(p)
        for k in range(6):
            recv = [6 + k * F + n for n in range(F)]
            lead = k if not kw else recv[0]
            assert np.all(u[recv] == u[lead]) and p["lane"][u[lead]] == lanes[lead], k
        assert lanes[6 + 5 * F + 3] != lanes[6 + 5 * F]


@pytest.mark.parametrize("gemm_mode", [0, 2])
def test_one_worker_priority_lanes_form_no_groups(planner, gemm_mode):
    """queue_policy 1 with one GEMM worker retires in the oracle's priority order (DESIGN §6), which a group need not
    keep: such a window forms none.  With the FIFO ring, or with more workers, it does."""
    ex = dags.ex05_broadcast(4, tile_bytes=4096)
    ex.tasks["priority"][4:] = np.arange(ex.ntasks - 4) % 3
    gemm = with_gemm_chain(ex)
    tiles = tiles_for(gemm.ntiles, sizes_of(gemm, 4096))
    p = plan_dag(planner, gemm, tiles, kind=1, queue_policy=1, nworkers=1, nworkers_gemm=1, gemm_mode=gemm_mode)
    assert len(p["group_mem"]) == 0 and np.array_equal(p["succ"], gemm.succ)
    for kw in (dict(queue_policy=0, nworkers=1, nworkers_gemm=1), dict(queue_policy=1)):
        assert len(plan_dag(planner, gemm, tiles, kind=1, gemm_mode=gemm_mode, **kw)["group_mem"]) > 0, kw


def test_gemm_kernels_keep_registers_and_stay_spill_free():
    """-Xptxas -v of the library build: the built-in GEMM window kernels keep one 384-thread CTA per SM (168
    registers) without a stack frame or a spill, and the linked ones have no spill in the kernel itself and no
    serialized wgmma."""
    logs = [os.path.join(ROOT, "build_ptxas.log"), os.path.join(ROOT, "build", "linked_gemm_ptxas.log")]
    if not all(os.path.exists(f) for f in logs):
        pytest.skip("no ptxas logs: the library was not built through the Makefile")
    text = open(logs[0]).read()
    props = re.findall(r"Function properties for (_ZN3pb223pb2_engine_gemm2_kernel\w+)\n\s*(.*)\n.*Used (\d+) registers", text)
    assert len(props) >= 4
    for name, frame, regs in props:
        assert frame.startswith("0 bytes stack frame, 0 bytes spill stores") and int(regs) <= 168, (name, frame, regs)
    linked = open(logs[1]).read()
    assert "C7509" not in linked
    for name, frame in re.findall(r"Function properties for (_ZN3pb223pb2_engine_gemm2_kernel\w+)\n\s*(.*)", linked):
        assert "0 bytes spill stores" in frame, (name, frame)
