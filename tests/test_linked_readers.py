"""Linked readers (PB2_LINK_READERS, include/pb2_device_body.h), host side.

  - the link calls take a readers mask in bits 8..15 of their flags, refuse one that is not a subset of the sliceable
    mask and refuse any other unknown flag bit;
  - the planner makes consecutive linked readers of one tile a read group, apart from CHECK readers, at most 8 to a
    group, and leaves alone a reader that is not declared, or has a second flow, writes, or pushes out;
  - it fuses a built-in producer, or a sliceable linked one that writes only that tile, with such a group, under the
    rules of CHECK groups (no pushout, the widest tile, more than one worker);
  - a window with linked readers plans as the same window with CHECK readers, in both window kinds, except for the
    readers' body and PB2_TASK_READER mark;
  - tests/cuda/reader_bodies.cu links offline with both engine cubins within their register budgets.
The GPU side is tests/test_linked_readers_gpu.py."""
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
# tests/cuda/reader_bodies.cu
COUNT_NE, SUM_I64, COUNT_GT, AXPB, FILL, SUM_CTL = (L.BODY_LINKED_0 + i for i in range(6))
READERS = 0b1000111                         # COUNT_NE, SUM_I64, COUNT_GT, FAIL
SLICEABLE = 0xFF
TASK_READER = 0x80
W, R_, RW = L.ACCESS_WRITE, L.ACCESS_READ, L.ACCESS_RW
LINKED = dict(linked_image=1, linked_sliceable=SLICEABLE)


@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("reader_plan") / "reader_plan.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-Iinclude", "-Iparsec_b200/csrc",
                    "tests/cpp/reader_plan_shim.cpp", "tests/cpp/window_plan_shim.cpp",
                    "parsec_b200/csrc/pb2_window_plan.cpp", "-o", so], cwd=ROOT, check=True)
    lib = C.CDLL(so)
    lib.wp_plan_readers.restype = C.c_void_p
    lib.wp_plan_readers.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                    C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.POINTER(C.c_int),
                                    C.POINTER(C.c_char_p)]
    lib.wp_free.argtypes = [C.c_void_p]
    lib.wp_array.restype = C.c_int64
    lib.wp_array.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p)]
    lib.wp_scalar.restype = C.c_int64
    lib.wp_scalar.argtypes = [C.c_void_p, C.c_char_p]
    return lib


def plan(lib, dag, tiles=None, checked=0, readers=0, **kw):
    """(rc, why, plan) of dag as test_window_plan.plan_of gives them, with linked_checked and linked_readers."""
    if tiles is None:
        tiles = tiles_for(dag.ntiles, dag.tile_bytes)
    prm = np.array([kw.get(k, DEFAULTS[k]) for k in PARAMS], np.int64)
    tasks = np.ascontiguousarray(dag.tasks, L.TASK_DTYPE)
    succ = np.ascontiguousarray(dag.succ, np.uint32)
    tiles = np.ascontiguousarray(tiles, L.TILE_DTYPE)
    ready = np.ascontiguousarray(dag.ready, np.int32)
    rc, why = C.c_int(0), C.c_char_p()
    h = lib.wp_plan_readers(prm.ctypes.data, checked, readers, tasks.ctypes.data, len(tasks), succ.ctypes.data,
                            len(succ), tiles.ctypes.data, len(tiles), ready.ctypes.data, len(ready), C.byref(rc),
                            C.byref(why))
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


def with_bodies(dag, producer=None, reader=COUNT_NE):
    """dag (dags.ex05_broadcast) with its CHECK readers as `reader` and, if given, its FILL producers as `producer`."""
    t = dag.tasks.copy()
    t["body"][t["body"] == L.BODY_CHECK_I32] = reader
    if producer is not None:
        t["body"][t["body"] == L.BODY_FILL_I32] = producer
    return dags.Dag(t, dag.succ, dag.ready, ntiles=dag.ntiles, tile_bytes=dag.tile_bytes, name="linked_readers",
                    meta=dag.meta)


def fan_out(readers, producer=L.BODY_FILL_I32, flows=((0, W),), sizes=(64 * 1024,)):
    """Task 0 runs `producer` over `flows` [(tile, access)], tasks 1.. are `readers` [(body, flows)] released by task
    0 in that order; tile i has sizes[i] bytes."""
    n = 1 + len(readers)
    t = dags._new_tasks(n)
    t["body"][0], t["nb_flows"][0] = producer, len(flows)
    for f, (tile, acc) in enumerate(flows):
        t["tile"][0, f], t["access"][0, f] = tile, acc
    for i, (body, rflows) in enumerate(readers, start=1):
        t["body"][i], t["nb_flows"][i] = body, len(rflows)
        for f, (tile, acc) in enumerate(rflows):
            t["tile"][i, f], t["access"][i, f] = tile, acc
        t["dep_goal"][i] = 1
    t["succ_begin"][0], t["succ_count"][0], t["succ_begin"][1:] = 0, n - 1, n - 1
    dag = dags.Dag(t, np.arange(1, n, dtype=np.uint32), np.array([0], np.int32), ntiles=len(sizes),
                   tile_bytes=max(sizes), name="fan_out")
    tiles = tiles_for(len(sizes), 0)
    tiles["bytes"] = sizes
    return dag, tiles


def groups(p, tasks):
    """The member lists of the groups led by `tasks`' ids, in task order ([] for a task that leads none)."""
    return [members(p, p["group"][t]) if p["group"][t] & 15 and not p["group"][t] & GROUP_FUSED else [] for t in tasks]


def rd(body=COUNT_NE):
    return (body, [(0, R_)])


# ----------------------------------------------------------------------------------------------------------------------
# the link calls
# ----------------------------------------------------------------------------------------------------------------------
def test_link_readers_flag(tmp_path):
    assert L.LINK_READERS(0b101) == 0x500 and L.LINK_READERS(0xFF) == 0xFF00
    src = tmp_path / "flag.c"
    src.write_text('#include <stdio.h>\n#include <stdint.h>\n#include <stddef.h>\n#include "pb2_engine.h"\n'
                   'int main(void) { printf("%u %u", (unsigned)PB2_LINK_READERS(0x5u), (unsigned)PB2_LINK_READERS(0xFFu));'
                   ' return 0; }\n')
    exe = tmp_path / "flag"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    assert subprocess.check_output([str(exe)]).split() == [b"1280", b"65280"]


@pytest.mark.parametrize("sliceable,flags", [(0b0001, L.LINK_READERS(0b0011)), (0, L.LINK_READERS(1)),
                                             (0xFF, 0x2), (0xFF, 0x10000), (0xFF, 0x80), (0xFF, 0xFFFFFFFF)],
                         ids=["not_sliceable", "nothing_sliceable", "bit1", "bit16", "bit7", "all"])
def test_device_link_refusals(sliceable, flags):
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        d = ctx.devices[0]
        assert ctx.l.pb2_device_link_bodies_ex(d, b"x", 1, L.IMAGE_PTX, sliceable, 0, flags) == L.PB2_ERR_BAD_PARAM
        # nothing was recorded: a valid call still links, a second one is refused
        ctx.link_bodies(d, b"x", L.IMAGE_PTX, 0b0111, 0b0100, readers=0b0011)
        assert ctx.l.pb2_device_link_bodies_ex(d, b"x", 1, L.IMAGE_PTX, 0, 0, 0) == L.PB2_ERR_EXISTS


@pytest.mark.parametrize("readers,gemm", [(0b1, False), (0xFF, True), (0, True)], ids=["one", "all_gemm", "none_gemm"])
def test_device_link_accepts_readers(readers, gemm):
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        ctx.link_bodies(ctx.devices[0], b"x", L.IMAGE_PTX, 0xFF, 0, gemm_windows=gemm, readers=readers)


def test_engine_link_refuses_a_null_engine():
    lib = L.load()
    assert lib.pb2_engine_link_bodies_ex(None, b"x", 1, L.IMAGE_PTX, 1, 0, L.LINK_READERS(1)) == L.PB2_ERR_BAD_PARAM


# ----------------------------------------------------------------------------------------------------------------------
# read groups
# ----------------------------------------------------------------------------------------------------------------------
def test_readers_are_marked(planner):
    dag = with_bodies(dags.ex05_broadcast(4, 14, 64 * 1024))
    rc, why, p = plan(planner, dag, readers=READERS, **LINKED)
    assert rc == 0, why
    assert np.all(p["tasks"]["flags"][4:] == (L.TASK_DEPS_MASK | TASK_READER))
    assert np.all(p["tasks"]["flags"][:4] == L.TASK_DEPS_MASK)
    rc, why, p = plan(planner, dag, readers=0, **LINKED)
    assert np.all(p["tasks"]["flags"] == L.TASK_DEPS_MASK)


def test_linked_only_groups_with_mixed_bodies(planner):
    dag, tiles = fan_out([rd(COUNT_NE), rd(SUM_I64), rd(COUNT_GT), rd(COUNT_NE)])
    rc, why, p = plan(planner, dag, tiles, readers=READERS, fuse_readers=-1, **LINKED)
    assert rc == 0, why
    assert groups(p, [1]) == [[1, 2, 3, 4]]


def test_split_where_check_and_linked_readers_meet(planner):
    chk = (L.BODY_CHECK_I32, [(0, R_)])
    dag, tiles = fan_out([chk, chk, rd(), rd(), rd(SUM_I64), chk, rd()])
    rc, why, p = plan(planner, dag, tiles, readers=READERS, fuse_readers=-1, **LINKED)
    assert rc == 0, why
    assert groups(p, [1, 3, 6, 7]) == [[1, 2], [3, 4, 5], [], []]


def test_split_at_eight(planner):
    dag, tiles = fan_out([rd()] * 11)
    rc, why, p = plan(planner, dag, tiles, readers=READERS, fuse_readers=-1, **LINKED)
    assert rc == 0, why
    assert groups(p, [1, 9]) == [list(range(1, 9)), [9, 10, 11]]


@pytest.mark.parametrize("reader,readers", [
    (rd(SUM_CTL), READERS),                                      # not declared a reader
    (rd(COUNT_NE), READERS & ~1),                                # its bit is clear
    ((COUNT_NE, [(0, R_), (1, R_)]), READERS),                   # a second flow with a tile
    ((COUNT_NE, [(0, RW)]), READERS),                            # writes its tile
    ((COUNT_NE, [(0, R_ | L.FLOW_PUSHOUT)]), READERS),           # pushes it out
], ids=["undeclared_body", "bit_clear", "two_flows", "rw", "pushout"])
def test_readers_left_alone(planner, reader, readers):
    dag, tiles = fan_out([reader] * 4, sizes=(64 * 1024, 64 * 1024))
    rc, why, p = plan(planner, dag, tiles, readers=readers, **LINKED)
    assert rc == 0, why
    assert not p["group_mem"].size
    assert p["succ"].tolist() == dag.succ.tolist()


# ----------------------------------------------------------------------------------------------------------------------
# fused producers
# ----------------------------------------------------------------------------------------------------------------------
TB = 64 * 1024
# (name, producer body, producer flows, tile sizes, fused)
SHAPES = [
    ("builtin_fill", L.BODY_FILL_I32, [(0, W)], [TB], True),
    ("builtin_iota", L.BODY_IOTA_I32, [(0, W)], [TB], True),
    ("builtin_add_iota_rw", L.BODY_ADD_IOTA_I32, [(0, RW)], [TB], True),
    ("builtin_fill_pushout", L.BODY_FILL_I32, [(0, W | L.FLOW_PUSHOUT)], [TB], False),
    ("builtin_check", L.BODY_CHECK_I32, [(0, R_)], [TB], False),
    ("linked_fill", FILL, [(0, W)], [TB], True),
    ("linked_axpb", AXPB, [(1, R_), (0, W)], [TB, TB], True),
    ("linked_axpb_narrower_input", AXPB, [(1, R_), (0, W)], [TB, TB // 2], True),
    ("linked_axpb_wider_input", AXPB, [(1, R_), (0, W)], [TB, 2 * TB], False),
    ("linked_pushes_x_out", FILL, [(0, W | L.FLOW_PUSHOUT)], [TB], False),
    ("linked_writes_two_tiles", AXPB, [(1, W), (0, W)], [TB, TB], False),
    ("linked_does_not_write_x", AXPB, [(0, R_), (1, W)], [TB, TB], False),
]


@pytest.mark.parametrize("name,body,flows,sizes,fuses", SHAPES, ids=[s[0] for s in SHAPES])
def test_which_producers_fuse(planner, name, body, flows, sizes, fuses):
    dag, tiles = fan_out([rd()] * 3, body, flows, sizes)
    rc, why, p = plan(planner, dag, tiles, readers=READERS, part_bytes=16 * 1024, **LINKED)
    assert rc == 0, why
    assert members(p, p["group"][1] if not p["group"][0] & GROUP_FUSED else p["group"][0]) == [1, 2, 3]
    assert bool(p["group"][0] & GROUP_FUSED) == fuses, name


def test_linked_producer_needs_sliceable(planner):
    dag, tiles = fan_out([rd()] * 3, FILL)
    rc, why, p = plan(planner, dag, tiles, readers=READERS, linked_image=1, linked_sliceable=READERS)
    assert rc == 0, why
    assert not p["group"][0] & GROUP_FUSED


@pytest.mark.parametrize("kw", [dict(nworkers=1), dict(fuse_readers=-1), dict(kind=1, nworkers_gemm=1)],
                         ids=["one_worker", "fusion_off", "one_gemm_worker"])
def test_no_fusion(planner, kw):
    rc, why, p = plan(planner, with_bodies(dags.ex05_broadcast(6, 14, TB), FILL), readers=READERS,
                      **dict(LINKED, **kw))
    assert rc == 0, why
    assert not any(p["group"][k] & GROUP_FUSED for k in range(6))
    assert all(groups(p, [6 + 8 * k]) == [list(range(6 + 8 * k, 14 + 8 * k))] for k in range(6))


def test_no_groups_with_read_groups_off_or_prio_one_gemm_worker(planner):
    dag = with_bodies(dags.ex05_broadcast(6, 14, TB), FILL)
    for kw in (dict(read_groups=-1), dict(kind=1, queue_policy=1, nworkers_gemm=1)):
        rc, why, p = plan(planner, dag, readers=READERS, **dict(LINKED, **kw))
        assert rc == 0, why
        assert not p["group_mem"].size, kw


def test_shared_windows_refuse_linked_readers(planner):
    rc, why, _ = plan(planner, with_bodies(dags.ex05_broadcast(6, 14, TB)), readers=READERS, shared=1, **LINKED)
    assert rc == L.PB2_ERR_NOT_SUPPORTED and "shared window" in why


# ----------------------------------------------------------------------------------------------------------------------
# a window with linked readers plans as the same window with CHECK readers
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", [0, 1], ids=["hbm", "gemm"])
@pytest.mark.parametrize("producer,part_bytes,trace,queue_policy", [
    (None, 256 * 1024, 0, 0), (None, 64 * 1024, 1, 0), (FILL, 0, 1, 1), (FILL, 64 * 1024, 0, 1)],
    ids=["builtin_one_part", "builtin_four_parts_traced", "linked_whole_traced_prio", "linked_four_parts_prio"])
def test_plans_as_check_readers(planner, kind, producer, part_bytes, trace, queue_policy):
    K = 6
    base = dags.ex05_broadcast(K, 14, 256 * 1024)
    kw = dict(LINKED, kind=kind, part_bytes=part_bytes, trace=trace, queue_policy=queue_policy)
    # the CHECK window: its producers may be checked linked FILLs (fused either way)
    rc, why, want = plan(planner, with_bodies(base, producer, L.BODY_CHECK_I32), checked=0xFF, **kw)
    assert rc == 0, why
    rc, why, got = plan(planner, with_bodies(base, producer), readers=READERS, **kw)
    assert rc == 0, why
    assert all(got["group"][k] & GROUP_FUSED for k in range(K))
    for name in ARRAYS:
        a, b = want[name], got[name]
        if name == "tasks":
            a, b = a.copy(), b.copy()
            assert np.all(b["body"][K:] == COUNT_NE) and np.all(b["flags"][K:] & TASK_READER)
            a["body"][K:] = b["body"][K:] = 0
            b["flags"][K:] &= np.uint8(0x7F)
        assert a.tobytes() == b.tobytes(), name
    for name in SCALARS:
        assert got[name] == want[name] or name == "linked", name
    assert got["linked"] == 1


# ----------------------------------------------------------------------------------------------------------------------
# the fixture
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("engine,pattern,max_regs", [
    ("pb2_engine_linked.cubin", r"_ZN3pb221pb2_engine_hbm_kernelI\w+", 80),
    ("pb2_engine_linked_gemm.cubin", r"_ZN3pb223pb2_engine_gemm2_kernelI\w+", 168)], ids=["hbm", "gemm"])
def test_fixture_links_with_the_engine_kernels(tmp_path, engine, pattern, max_regs):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not found")
    engine = os.path.join(ROOT, "build", engine)
    assert os.path.exists(engine), "build() makes " + engine
    src = os.path.join(ROOT, "tests", "cuda", "reader_bodies.cu")
    cubin, ptx, out = tmp_path / "readers.cubin", tmp_path / "readers.ptx", tmp_path / "linked.cubin"
    inc = ["-I", os.path.join(ROOT, "include")]
    subprocess.check_call([NVCC, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-rdc=true", "-cubin",
                           *inc, "-o", str(cubin), src])
    subprocess.check_call([NVCC, "-O3", "-std=c++17", "-arch=compute_90a", "-rdc=true", "-ptx", *inc, "-o", str(ptx), src])
    assert b"pb2_linked_body" in ptx.read_bytes()
    subprocess.check_call([os.path.join(CUDA, "bin", "nvlink"), "-arch=sm_90a", "-o", str(out), engine, str(cubin)])
    res = subprocess.check_output([os.path.join(CUDA, "bin", "cuobjdump"), "-res-usage", str(out)], text=True)
    kernels = re.findall(r"Function (%s):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)" % pattern, res)
    assert len(kernels) == 4, res
    for name, reg, stack, smem, local in kernels:
        assert int(reg) <= max_regs and int(local) == 0, (name, reg, stack, smem, local)
        if max_regs == 80:      # 8 workers of 64 threads per SM fit in shared memory
            assert 8 * int(smem) <= 227 * 1024, (name, smem)
