"""Linked bodies with a checked form (pb2_engine_link_bodies_checked, include/pb2_device_body.h), host side.

  - the planner fuses a linked producer with the first read group among its out-edges only when its id is declared
    checked, and then exactly as it fuses a built-in FILL on the same DAG (members, group words, device CSR, parts);
  - it does not fuse one that writes a second tile, pushes its tile out, has a wider tile, or runs on one worker;
  - the link calls refuse a checked mask that is not a subset of the sliceable mask, or has bits above bit 7;
  - pb2_body_check_t is the 80-byte block the engine hands a linked body, as gcc and nvcc lay it out;
  - tests/cuda/checked_bodies.cu compiles to a relocatable cubin and to PTX, and nvlink links it with the engine's
    linked HBM window kernel within the kernel's 80-register budget.
The GPU side is tests/test_checked_linked_gpu.py."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200 import runtime as R
from test_window_plan import ARRAYS, DEFAULTS, GROUP_FUSED, PARAMS, SCALARS, members, tiles_for

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
NVCC = os.environ.get("NVCC", os.path.join(CUDA, "bin", "nvcc"))
LINKED_FILL = L.BODY_LINKED_0            # tests/cuda/checked_bodies.cu
LINKED_AXPB = L.BODY_LINKED_0 + 1


@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("checked_plan") / "checked_plan.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-Iinclude", "-Iparsec_b200/csrc",
                    "tests/cpp/checked_plan_shim.cpp", "tests/cpp/window_plan_shim.cpp",
                    "parsec_b200/csrc/pb2_window_plan.cpp", "-o", so], cwd=ROOT, check=True)
    lib = C.CDLL(so)
    lib.wp_plan_checked.restype = C.c_void_p
    lib.wp_plan_checked.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                    C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.POINTER(C.c_int),
                                    C.POINTER(C.c_char_p)]
    lib.wp_free.argtypes = [C.c_void_p]
    lib.wp_array.restype = C.c_int64
    lib.wp_array.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p)]
    lib.wp_scalar.restype = C.c_int64
    lib.wp_scalar.argtypes = [C.c_void_p, C.c_char_p]
    return lib


def plan(lib, dag, tiles=None, checked=0, **kw):
    """(rc, why, plan) of dag as test_window_plan.plan_of gives them, with PlanParams::linked_checked = checked."""
    if tiles is None:
        tiles = tiles_for(dag.ntiles, dag.tile_bytes)
    prm = np.array([kw.get(k, DEFAULTS[k]) for k in PARAMS], np.int64)
    tasks = np.ascontiguousarray(dag.tasks, L.TASK_DTYPE)
    succ = np.ascontiguousarray(dag.succ, np.uint32)
    tiles = np.ascontiguousarray(tiles, L.TILE_DTYPE)
    ready = np.ascontiguousarray(dag.ready, np.int32)
    rc, why = C.c_int(0), C.c_char_p()
    h = lib.wp_plan_checked(prm.ctypes.data, checked, None, tasks.ctypes.data, len(tasks), succ.ctypes.data, len(succ),
                            tiles.ctypes.data, len(tiles), ready.ctypes.data, len(ready), C.byref(rc), C.byref(why))
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


def linked_ex05(K=6, tile_bytes=256 * 1024, body=LINKED_FILL):
    """dags.ex05_broadcast with TaskBcast's FILL_I32 as the linked body `body` (same tile, access and constant)."""
    dag = dags.ex05_broadcast(K, 14, tile_bytes)
    t = dag.tasks.copy()
    t["body"][t["body"] == L.BODY_FILL_I32] = body
    return dags.Dag(t, dag.succ, dag.ready, ntiles=dag.ntiles, tile_bytes=dag.tile_bytes, name="linked_ex05", meta=dag.meta)


LINKED = dict(linked_image=1, linked_sliceable=0xFF)


def producers_fused(p, K):
    return [bool(p["group"][k] & GROUP_FUSED) for k in range(K)]


@pytest.mark.parametrize("part_bytes,trace", [(256 * 1024, 0), (64 * 1024, 1), (0, 1)],
                         ids=["one_part", "four_parts_traced", "whole_tiles_traced"])
def test_checked_fill_plans_as_the_builtin_fill(planner, part_bytes, trace):
    K = 6
    builtin = dags.ex05_broadcast(K, 14, 256 * 1024)
    rc, why, want = plan(planner, builtin, part_bytes=part_bytes, trace=trace)
    assert rc == 0, why
    rc, why, got = plan(planner, linked_ex05(K), checked=0b1, part_bytes=part_bytes, trace=trace, **LINKED)
    assert rc == 0, why
    assert all(producers_fused(got, K))
    F = builtin.meta["F"]
    for k in range(K):
        assert members(got, got["group"][k]) == [K + k * F + n for n in range(F)]
    for name in ARRAYS:
        a, b = want[name], got[name]
        if name == "tasks":
            a, b = a.copy(), b.copy()
            assert np.all(b["body"][:K] == LINKED_FILL)
            a["body"][:K] = b["body"][:K] = 0
        assert a.tobytes() == b.tobytes(), name
    for name in SCALARS:
        assert got[name] == want[name] or name == "linked", name
    assert got["linked"] == 1


@pytest.mark.parametrize("checked", [0, 0b10, 0xFE], ids=["none", "other_id", "all_but_it"])
def test_undeclared_linked_producer_is_not_fused(planner, checked):
    K = 6
    rc, why, want = plan(planner, dags.ex05_broadcast(K, 14, 256 * 1024), fuse_readers=-1)
    rc, why, got = plan(planner, linked_ex05(K), checked=checked, **LINKED)
    assert rc == 0, why
    assert not any(producers_fused(got, K))
    # the readers still form their groups, as with fusion off
    assert got["group"].tobytes() == want["group"].tobytes() and got["succ"].tobytes() == want["succ"].tobytes()


def one_producer(flows, sizes, readers=3):
    """Task 0 runs LINKED_AXPB over `flows` [(tile, access)], tasks 1.. CHECK tile 0; tile i has sizes[i] bytes."""
    n = 1 + readers
    t = dags._new_tasks(n)
    t["body"][0], t["nb_flows"][0] = LINKED_AXPB, len(flows)
    for f, (tile, acc) in enumerate(flows):
        t["tile"][0, f], t["access"][0, f] = tile, acc
    t["body"][1:], t["nb_flows"][1:], t["tile"][1:, 0], t["access"][1:, 0] = L.BODY_CHECK_I32, 1, 0, L.ACCESS_READ
    t["dep_goal"][1:] = 1
    t["succ_begin"][0], t["succ_count"][0], t["succ_begin"][1:] = 0, readers, readers
    dag = dags.Dag(t, np.arange(1, n, dtype=np.uint32), np.array([0], np.int32), ntiles=len(sizes),
                   tile_bytes=max(sizes), name="one_producer")
    tiles = tiles_for(len(sizes), 0)
    tiles["bytes"] = sizes
    return dag, tiles


W, R_, RW = L.ACCESS_WRITE, L.ACCESS_READ, L.ACCESS_RW
TB = 64 * 1024
# (name, producer flows, tile sizes, fused with checked = its bit)
SHAPES = [
    ("reads_a_tile_writes_x", [(1, R_), (0, W)], [TB, TB], True),          # the output is flow 1, not flow 0
    ("reads_a_narrower_tile", [(1, R_), (0, W)], [TB, TB // 2], True),
    ("rw_x", [(0, RW)], [TB], True),
    ("writes_a_second_tile", [(1, W), (0, W)], [TB, TB], False),
    ("writes_a_second_tile_first_flow_x", [(0, W), (1, RW)], [TB, TB], False),
    ("pushes_x_out", [(1, R_), (0, W | L.FLOW_PUSHOUT)], [TB, TB], False),
    ("reads_a_wider_tile", [(1, R_), (0, W)], [TB, 2 * TB], False),
    ("does_not_write_x", [(0, R_), (1, W)], [TB, TB], False),
]


@pytest.mark.parametrize("name,flows,sizes,fuses", SHAPES, ids=[s[0] for s in SHAPES])
def test_which_linked_producers_fuse(planner, name, flows, sizes, fuses):
    dag, tiles = one_producer(flows, sizes)
    for checked in (0, 1 << (LINKED_AXPB - L.BODY_LINKED_0)):
        rc, why, p = plan(planner, dag, tiles, checked=checked, part_bytes=16 * 1024, **LINKED)
        assert rc == 0, why
        assert members(p, p["group"][1]) == [1, 2, 3]                        # the group forms either way
        assert bool(p["group"][0] & GROUP_FUSED) == (fuses and checked != 0), (name, checked)


def test_one_worker_runs_the_oracle_order(planner):
    """With one worker the ready ring's FIFO order is the oracle's: no fused unit, checked or not."""
    rc, why, p = plan(planner, linked_ex05(), checked=0b1, nworkers=1, **LINKED)
    assert rc == 0, why
    assert not any(producers_fused(p, 6))


def test_shared_windows_refuse_linked_producers(planner):
    """A shared window runs its tasks alone and never fuses; it refuses a linked body whether or not it is checked."""
    rc, why, _ = plan(planner, linked_ex05(), checked=0b1, shared=1, **LINKED)
    assert rc == L.PB2_ERR_NOT_SUPPORTED and "shared window" in why


# ----------------------------------------------------------------------------------------------------------------------
# the link calls
# ----------------------------------------------------------------------------------------------------------------------
def test_engine_checked_link_refuses_a_null_engine():
    lib = L.load()
    assert lib.pb2_engine_link_bodies_checked(None, b"x", 1, L.IMAGE_PTX, 1, 1) == L.PB2_ERR_BAD_PARAM


@pytest.mark.parametrize("sliceable,checked", [(0, 1), (0b0110, 0b0111), (0xFF, 0x100), (0x1FF, 0x100),
                                               (0xFF, 0xFFFFFFFF)],
                         ids=["not_sliceable", "one_bit_not_sliceable", "bit8", "both_bit8", "all"])
def test_device_checked_link_argument_checks(sliceable, checked):
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        assert ctx.l.pb2_device_link_bodies_checked(ctx.devices[0], b"x", 1, L.IMAGE_PTX, sliceable, checked) == L.PB2_ERR_BAD_PARAM
        # nothing was recorded: a valid call still links, a second one is refused
        ctx.link_bodies(ctx.devices[0], b"x", L.IMAGE_PTX, 0b0110, 0b0100)
        assert ctx.l.pb2_device_link_bodies_checked(ctx.devices[0], b"x", 1, L.IMAGE_PTX, 0, 0) == L.PB2_ERR_EXISTS


# ----------------------------------------------------------------------------------------------------------------------
# the device ABI and the fixture
# ----------------------------------------------------------------------------------------------------------------------
def check_block_layout(tmp_path, compiler):
    src = tmp_path / ("check_layout" + (".cu" if compiler == NVCC else ".c"))
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pb2_device_body.h"\n'
                   'int main(void) { printf("%zu %zu %zu %zu %zu", sizeof(pb2_body_check_t), '
                   'offsetof(pb2_body_check_t, args), offsetof(pb2_body_check_t, check), '
                   'offsetof(pb2_body_check_t, k0), sizeof(pb2_body_args_t)); return 0; }\n')
    exe = tmp_path / "check_layout"
    arch = ["-gencode", "arch=compute_90a,code=sm_90a"] if compiler == NVCC else []
    subprocess.check_call([compiler, *arch, "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    return [int(v) for v in subprocess.check_output([str(exe)]).split()]


def test_check_block_layout(tmp_path):
    want = [80, 0, L.BODY_ARGS_DTYPE.itemsize, L.BODY_ARGS_DTYPE.itemsize + 4, L.BODY_ARGS_DTYPE.itemsize]
    assert want == [80, 0, 72, 76, 72]
    assert check_block_layout(tmp_path, "gcc") == want
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not found")
    assert check_block_layout(tmp_path, NVCC) == want


def test_fixture_links_with_the_engine_kernel(tmp_path):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not found")
    engine = os.path.join(ROOT, "build", "pb2_engine_linked.cubin")
    assert os.path.exists(engine), "build() makes build/pb2_engine_linked.cubin"
    src = os.path.join(ROOT, "tests", "cuda", "checked_bodies.cu")
    cubin, ptx, out = tmp_path / "checked.cubin", tmp_path / "checked.ptx", tmp_path / "linked.cubin"
    inc = ["-I", os.path.join(ROOT, "include")]
    subprocess.check_call([NVCC, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-rdc=true", "-cubin",
                           *inc, "-o", str(cubin), src])
    subprocess.check_call([NVCC, "-O3", "-std=c++17", "-arch=compute_90a", "-rdc=true", "-ptx", *inc, "-o", str(ptx), src])
    assert b"pb2_linked_body" in ptx.read_bytes()
    subprocess.check_call([os.path.join(CUDA, "bin", "nvlink"), "-arch=sm_90a", "-o", str(out), engine, str(cubin)])
    res = subprocess.check_output([os.path.join(CUDA, "bin", "cuobjdump"), "-res-usage", str(out)], text=True)
    kernels = re.findall(r"Function (_ZN3pb221pb2_engine_hbm_kernelI\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+)", res)
    assert len(kernels) == 4, res
    for name, reg, stack, smem in kernels:
        # 80 registers (the kernel's launch bounds), and 8 workers of 64 threads per SM fit in shared memory
        assert int(reg) <= 80 and 8 * int(smem) <= 227 * 1024, (name, reg, stack, smem)
