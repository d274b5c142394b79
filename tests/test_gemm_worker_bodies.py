"""GEMM-worker bodies (PB2_LINK_GEMM_BODIES), host side.

  - the link calls: the mask needs PB2_LINK_GEMM_WINDOWS and must not overlap `sliceable`, `checked` or the readers
    masks; otherwise bits 24..31 are accepted and recorded;
  - the planner: HBM windows refuse such a task; GEMM windows mark it PB2_TASK_GEMM_BODY and run it as one part of a
    unit of its own, never in a read group or fused with one, even when CHECK readers of its output follow it; a GEMM
    window of such tasks alone plans;
  - the device ABI header states the operand ring the engine's static_assert pins;
  - the stand-alone runtime, in dry run, takes a pool of such tasks;
  - the fixture's image links with the engine's linked kernels within their register budgets.
The GPU side is tests/test_gemm_worker_bodies_gpu.py."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from parsec_b200 import _lib as L
from parsec_b200 import runtime as R
from test_window_plan import ARRAYS, DEFAULTS, PARAMS, SCALARS, tiles_for
import fp64_gemm as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
TASK_GEMM_BODY = 0x20                   # pb2_window_layout.h
HBM_MSG = "GEMM-worker body in an HBM window (it runs in GEMM windows only, on the worker's operand ring)"


# ----------------------------------------------------------------------------------------------------------------------
# the link calls
# ----------------------------------------------------------------------------------------------------------------------
def link(**kw):
    """rc of a dry-run Context.link_bodies with these arguments, and whether a second link is then refused as one."""
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        dev = ctx.devices[0]
        try:
            ctx.link_bodies(dev, b"ptx", L.IMAGE_PTX, **kw)
            rc = 0
        except L.Pb2Error as e:
            rc = e.rc
        second = ctx.l.pb2_device_link_bodies_ex(dev, b"x", 1, L.IMAGE_PTX, 0, 0, 0)
    return rc, second


@pytest.mark.parametrize("kw", [
    dict(gemm_bodies=0x01),                                          # without gemm_windows
    dict(gemm_bodies=0x80, sliceable=0x80, gemm_windows=True),       # overlaps sliceable
    dict(gemm_bodies=0x06, sliceable=0x04, checked=0x04, gemm_windows=True),
    dict(gemm_bodies=0x10, sliceable=0x30, readers=0x10, gemm_windows=True),
    dict(gemm_bodies=0x20, sliceable=0x20, readers=0x20, reader_groups=0x20, gemm_windows=True),
], ids=["no_gemm_windows", "sliceable", "checked", "readers", "reader_groups"])
def test_link_refuses(kw):
    rc, second = link(**kw)
    assert rc == L.PB2_ERR_BAD_PARAM
    assert second == 0                  # nothing was recorded


@pytest.mark.parametrize("kw", [
    dict(gemm_bodies=0xFF, gemm_windows=True),
    dict(gemm_bodies=0x03, sliceable=0xFC, checked=0x04, readers=0x30, reader_groups=0x10, gemm_windows=True),
    dict(gemm_bodies=0x80, sliceable=0x7F, gemm_windows=True),
], ids=["all_eight", "beside_the_other_masks", "bit_31"])
def test_link_accepts(kw):
    rc, second = link(**kw)
    assert rc == 0 and second == L.PB2_ERR_EXISTS


def test_flag_helper():
    assert L.LINK_GEMM_BODIES(0xFF) == 0xFF000000 and L.LINK_GEMM_BODIES(0x01) == 1 << 24


def test_engine_link_refuses_a_null_engine():
    lib = L.load()
    flags = L.LINK_GEMM_WINDOWS | L.LINK_GEMM_BODIES(0x01)
    assert lib.pb2_engine_link_bodies_ex(None, b"x", 1, L.IMAGE_PTX, 0, 0, flags) == L.PB2_ERR_BAD_PARAM


# ----------------------------------------------------------------------------------------------------------------------
# the planner
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("gemm_body_plan") / "gemm_body_plan.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-Iinclude", "-Iparsec_b200/csrc",
                    "tests/cpp/gemm_body_plan_shim.cpp", "tests/cpp/window_plan_shim.cpp",
                    "parsec_b200/csrc/pb2_window_plan.cpp", "-o", so], cwd=ROOT, check=True)
    lib = C.CDLL(so)
    lib.wp_plan_gemm_bodies.restype = C.c_void_p
    lib.wp_plan_gemm_bodies.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_int32, C.c_void_p,
                                        C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.POINTER(C.c_int),
                                        C.POINTER(C.c_char_p)]
    lib.wp_free.argtypes = [C.c_void_p]
    lib.wp_array.restype = C.c_int64
    lib.wp_array.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p)]
    lib.wp_scalar.restype = C.c_int64
    lib.wp_scalar.argtypes = [C.c_void_p, C.c_char_p]
    return lib


def plan(lib, tasks, succ, ready, tiles, checked=0, readers=0, gemm_bodies=F.GEMM_BODIES, **kw):
    """(rc, why, plan) of a window of an engine linked with PB2_LINK_GEMM_WINDOWS (linked_image set)."""
    kw.setdefault("kind", 1)
    kw.setdefault("linked_image", 1)
    prm = np.array([kw.get(k, DEFAULTS[k]) for k in PARAMS], np.int64)
    tasks = np.ascontiguousarray(tasks, L.TASK_DTYPE)
    succ = np.ascontiguousarray(succ, np.uint32)
    tiles = np.ascontiguousarray(tiles, L.TILE_DTYPE)
    ready = np.ascontiguousarray(ready, np.int32)
    rc, why = C.c_int(0), C.c_char_p()
    h = lib.wp_plan_gemm_bodies(prm.ctypes.data, checked, readers, gemm_bodies, tasks.ctypes.data, len(tasks),
                                succ.ctypes.data, len(succ), tiles.ctypes.data, len(tiles), ready.ctypes.data, len(ready),
                                C.byref(rc), C.byref(why))
    if not h:
        return rc.value, why.value.decode() if why.value else None, None
    try:
        out = {}
        for name, dt in ARRAYS.items():
            p = C.c_void_p()
            n = lib.wp_array(h, name.encode(), C.byref(p))
            out[name] = np.frombuffer(C.string_at(p.value, n) if n else b"", dtype=dt).copy()
        for name in SCALARS:
            out[name] = lib.wp_scalar(h, name.encode())
        return rc.value, None, out
    finally:
        lib.wp_free(h)


def fp64_window(NT=3, M=128, N=128, K=64):
    dag, sizes = F.dag(NT, M, N, K)
    tiles = tiles_for(dag.ntiles, 0)
    tiles["bytes"] = sizes
    return dag, tiles


def test_hbm_window_refuses(planner):
    dag, tiles = fp64_window()
    rc, why, _ = plan(planner, dag.tasks, dag.succ, dag.ready, tiles, kind=0)
    assert rc == L.PB2_ERR_NOT_SUPPORTED and why == HBM_MSG
    # the same ids without the mask are ordinary linked bodies, which HBM windows run
    rc, why, _ = plan(planner, dag.tasks, dag.succ, dag.ready, tiles, kind=0, gemm_bodies=0)
    assert rc == 0, why


SHARED_MSG = "linked body in a shared window (not supported)"
UNLINKED_MSG = "linked body id, but the engine has not linked an image (pb2_engine_link_bodies)"
GEMM_MSG = "linked body in a GEMM window (linked bodies run in HBM windows only)"


@pytest.mark.parametrize("shared,linked_image,msgs", [(1, 1, (SHARED_MSG, SHARED_MSG)), (0, 0, (UNLINKED_MSG, GEMM_MSG))],
                         ids=["shared", "unlinked"])
def test_shared_and_unlinked_refuse_as_for_any_linked_body(planner, shared, linked_image, msgs):
    """The messages of any linked body: an engine without an image has no linked GEMM kernel either."""
    dag, tiles = fp64_window()
    for kind in (0, 1):
        rc, why, _ = plan(planner, dag.tasks, dag.succ, dag.ready, tiles, kind=kind, shared=shared, linked_image=linked_image)
        assert rc == L.PB2_ERR_NOT_SUPPORTED and why == msgs[kind], (kind, why)


@pytest.mark.parametrize("queue_policy,trace", [(0, 0), (1, 1)])
def test_window_of_gemm_worker_bodies_alone(planner, queue_policy, trace):
    """No bf16 GEMM in the window: one unit of one part per task, no operand tensor map, every task flagged."""
    NT = 3
    dag, tiles = fp64_window(NT)
    rc, why, p = plan(planner, dag.tasks, dag.succ, dag.ready, tiles, part_bytes=4096, queue_policy=queue_policy,
                      trace=trace)
    assert rc == 0, why
    assert p["linked"] == 1
    assert np.all(p["tasks"]["flags"] & TASK_GEMM_BODY)
    units = p["units"]
    assert len(units) == NT ** 3 and np.all(units["nparts"] == 1) and np.all(units["seg_count"] == 1)
    assert np.all(units["flags"] == 0) and np.all(units["tileC"] == -1)
    assert not np.any(p["operand_rows"]) and not len(p["group_mem"])
    assert sorted(p["segs"]["task"].tolist()) == list(range(NT ** 3))
    if trace:
        assert np.all(p["part_entities"]["nparts"] == 1) and p["part_records"] == NT ** 3


def body_and_checks(nchecks=4, tile_bytes=1 << 20):
    """Task 0 runs body LINKED_2 and writes tile 0; tasks 1.. CHECK it (a read group a fusable producer would run
    with); task nchecks + 1 runs LINKED_3, a sliceable linked FILL of tile 1."""
    n = nchecks + 2
    t = np.zeros(n, L.TASK_DTYPE)
    t["tile"][:] = -1
    t["nb_flows"] = 1
    t["tile"][:, 0] = 0
    t["body"][0], t["access"][0, 0] = L.BODY_LINKED_0 + 2, L.ACCESS_WRITE
    t["body"][1:n - 1], t["access"][1:n - 1, 0], t["dep_goal"][1:n - 1] = L.BODY_CHECK_I32, L.ACCESS_READ, 1
    t["body"][n - 1], t["access"][n - 1, 0], t["tile"][n - 1, 0] = L.BODY_LINKED_0 + 3, L.ACCESS_WRITE, 1
    t["succ_begin"][0], t["succ_count"][0] = 0, nchecks
    t["succ_begin"][1:] = nchecks
    succ = np.arange(1, nchecks + 1, dtype=np.uint32)
    return t, succ, np.array([0, n - 1], np.int32), tiles_for(2, tile_bytes)


@pytest.mark.parametrize("kind", [0, 1])
def test_never_grouped_fused_or_cut(planner, kind):
    """The same DAG with LINKED_2 declared sliceable and checked (a fused producer, cut into parts) and declared a
    GEMM-worker body (one part, alone; its CHECK readers still form their own group)."""
    t, succ, ready, tiles = body_and_checks()
    kw = dict(kind=kind, part_bytes=64 * 1024, nworkers=8, nworkers_gemm=8)
    rc, why, a = plan(planner, t, succ, ready, tiles, checked=0x04, gemm_bodies=0, linked_sliceable=0x0C, **kw)
    assert rc == 0, why
    assert a["group"][0] & 0x80000000                   # fused with its group
    if kind == 1:
        rc, why, b = plan(planner, t, succ, ready, tiles, gemm_bodies=0x04, linked_sliceable=0x08, **kw)
        assert rc == 0, why
        assert b["tasks"]["flags"][0] & TASK_GEMM_BODY and not np.any(b["tasks"]["flags"][1:] & TASK_GEMM_BODY)
        assert b["group"][0] == 0                       # neither fused nor a member
        assert b["group"][1] & 15 == 4                  # the CHECKs are a group of their own
        units, segs = b["units"], b["segs"]
        u0 = [u for u in units if segs["task"][u["seg_begin"]] == 0]
        assert len(u0) == 1 and u0[0]["seg_count"] == 1 and u0[0]["nparts"] == 1 and u0[0]["flags"] == 0
        fill = [u for u in units if segs["task"][u["seg_begin"]] == len(t) - 1]
        assert fill[0]["nparts"] == 16                  # the sliceable linked FILL is still cut: 1 MiB / 64 KiB
    else:
        rc, why, _ = plan(planner, t, succ, ready, tiles, gemm_bodies=0x04, linked_sliceable=0x08, **kw)
        assert rc == L.PB2_ERR_NOT_SUPPORTED and why == HBM_MSG


# ----------------------------------------------------------------------------------------------------------------------
# the device ABI header
# ----------------------------------------------------------------------------------------------------------------------
def test_header_states_the_operand_ring(tmp_path):
    src = tmp_path / "ring.c"
    src.write_text('#include <stdio.h>\n#include "pb2_device_body.h"\n'
                   'int main(void) { printf("%d %d\\n", PB2_GEMM_BODY_SMEM_BYTES, PB2_GEMM_BODY_SMEM_ALIGN); return 0; }\n')
    exe = tmp_path / "ring"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                   check=True)
    nbytes, align = map(int, subprocess.check_output([str(exe)], text=True).split())
    # what the GEMM kernel's static_asserts pin: kStages * (BM + BN) * BK * 2 bytes, aligned up from kSmemBytes' slack
    gemm = open(os.path.join(ROOT, "parsec_b200", "csrc", "pb2_gemm.cuh")).read()
    layout = open(os.path.join(ROOT, "parsec_b200", "csrc", "pb2_window_layout.h")).read()
    stages = int(re.search(r"kStages = (\d+);", gemm).group(1))
    bk = int(re.search(r"BK = (\d+)", gemm).group(1))
    bm, bn = map(int, re.search(r"BM = (\d+), BN = (\d+);", layout).groups())
    assert nbytes == stages * (bm + bn) * bk * 2 == 196608
    assert align == 1024 and "kStages * kStageBytes + 1024" in gemm
    assert "static_assert(PB2_GEMM_BODY_SMEM_BYTES == kStages * kStageBytes" in gemm


# ----------------------------------------------------------------------------------------------------------------------
# the stand-alone runtime in dry run, and the fixture
# ----------------------------------------------------------------------------------------------------------------------
def test_dry_run_pool_of_gemm_worker_tasks():
    NT, M, N, K = 2, 64, 48, 40
    t = F.tiles(NT, M, N, K)
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        ctx.link_bodies(ctx.devices[0], b"ptx", L.IMAGE_PTX, 0, gemm_windows=True, gemm_bodies=F.GEMM_BODIES)
        tp, _ = F.insert(ctx, NT, M, N, K, t)
        win = ctx.export_window(tp, ctx.devices[0])
        ctx.wait()
        st = ctx.stats(ctx.devices[0])
    assert np.all(win["tasks"]["body"] == F.DGEMM) and len(win["tasks"]) == NT ** 3
    assert st["executed_tasks"] == NT ** 3 and st["windows_launched"] == 1


def test_fixture_links_within_the_register_budgets(tmp_path):
    engine = [os.path.join(ROOT, "build", f) for f in ("pb2_engine_linked.cubin", "pb2_engine_linked_gemm.cubin")]
    bodies = os.path.join(ROOT, "tests", "cuda", "gemm_worker_bodies.cubin")
    assert all(os.path.exists(f) for f in engine + [bodies]), "build() makes the engine cubins and the fixture"
    out = tmp_path / "linked.cubin"
    subprocess.check_call([os.path.join(CUDA, "bin", "nvlink"), "-arch=sm_90a", "-o", str(out), *engine, bodies])
    res = subprocess.check_output([os.path.join(CUDA, "bin", "cuobjdump"), "-res-usage", str(out)], text=True)
    gemm = re.findall(r"Function (_ZN3pb223pb2_engine_gemm2_kernelI\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+)", res)
    hbm = re.findall(r"Function (_ZN3pb221pb2_engine_hbm_kernelI\w+):\s*\n\s*REG:(\d+)", res)
    assert len(gemm) == 4 and len(hbm) == 4, res
    assert all(int(r) <= 168 and int(s) + 196608 + 1024 <= 227 * 1024 for _, r, _, s in gemm), gemm
    assert all(int(r) <= 80 for _, r in hbm), hbm
    # the DGEMM body runs on the FP64 tensor cores
    sass = subprocess.check_output([os.path.join(CUDA, "bin", "cuobjdump"), "-sass", bodies], text=True)
    assert "DMMA.16x8x8" in sass
