"""Linked readers with the group form (PB2_LINK_READER_GROUPS, pb2_linked_reader_group), host side.

  - the link calls take a group mask in bits 16..23 of their flags and refuse one that is not a subset of the readers
    mask, or any bit above 23;
  - the planner makes the same groups, units, parts and ring image with and without the mask, and only marks the
    declared readers' descriptors with one more flag bit;
  - the kernels built with the group call link offline with tests/cuda/reader_group_bodies.cu within the budgets of the
    plain ones, and the two mismatches behave as pb2_engine_link_bodies_ex documents: the group-call kernels need the
    image's group form (undefined reference without it), and the plain kernels never name it;
  - the plain kernels do not name pb2_linked_reader_group.
The GPU side is tests/test_reader_groups_linked_gpu.py."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200 import runtime as R
from test_linked_readers import COUNT_GT, COUNT_NE, FILL, READERS, SUM_CTL, SUM_I64, fan_out, rd, with_bodies
from test_window_plan import ARRAYS, DEFAULTS, GROUP_FUSED, PARAMS, SCALARS, tiles_for

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
GROUPS = READERS                            # COUNT_NE, SUM_I64, COUNT_GT and FAIL have the group form
TASK_READER, TASK_READER_GROUP = 0x80, 0x40
LINKED = dict(linked_image=1, linked_sliceable=0xFF)


def test_flag_values(tmp_path):
    assert L.LINK_READER_GROUPS(0b101) == 0x50000 and L.LINK_READER_GROUPS(0xFF) == 0xFF0000
    src = tmp_path / "flag.c"
    src.write_text('#include <stdio.h>\n#include <stdint.h>\n#include <stddef.h>\n#include "pb2_engine.h"\n'
                   '#include "pb2_device_body.h"\n'
                   'int main(void) { printf("%u %zu %d", (unsigned)PB2_LINK_READER_GROUPS(0x5u), sizeof(pb2_reader_group_t),'
                   ' PB2_GROUP_MAX); return 0; }\n')
    exe = tmp_path / "flag"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    assert subprocess.check_output([str(exe)]).split() == [b"327680", b"184", b"8"]


# ----------------------------------------------------------------------------------------------------------------------
# the link calls
# ----------------------------------------------------------------------------------------------------------------------
REFUSED = [(0b0011, 0b0100), (0, 0b1), (0b0001, 0b0011), (0xFF, 0x100)]


@pytest.mark.parametrize("readers,groups", REFUSED, ids=["not_a_reader", "no_readers", "one_more", "bit24"])
def test_device_link_refusals(readers, groups):
    flags = L.LINK_READERS(readers) | (groups << 16)
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        d = ctx.devices[0]
        assert ctx.l.pb2_device_link_bodies_ex(d, b"x", 1, L.IMAGE_PTX, 0xFF, 0, flags) == L.PB2_ERR_BAD_PARAM
        # nothing was recorded: a valid call still links
        ctx.link_bodies(d, b"x", L.IMAGE_PTX, 0xFF, readers=0b0111, reader_groups=0b0101)


@pytest.mark.parametrize("readers,groups", REFUSED, ids=["not_a_reader", "no_readers", "one_more", "bit24"])
def test_engine_refusals_on_a_null_engine(readers, groups):
    lib = L.load()
    flags = L.LINK_READERS(readers) | (groups << 16)
    assert lib.pb2_engine_link_bodies_ex(None, b"x", 1, L.IMAGE_PTX, 0xFF, 0, flags) == L.PB2_ERR_BAD_PARAM


@pytest.mark.parametrize("readers,groups,gemm", [(0b1, 0b1, False), (0xFF, 0xFF, True), (READERS, 0b101, False),
                                                 (READERS, 0, True)],
                         ids=["one", "all_gemm", "some", "none_gemm"])
def test_device_link_accepts(readers, groups, gemm):
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        ctx.link_bodies(ctx.devices[0], b"x", L.IMAGE_PTX, 0xFF, gemm_windows=gemm, readers=readers, reader_groups=groups)


# ----------------------------------------------------------------------------------------------------------------------
# plans
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("reader_group_plan") / "reader_group_plan.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-Iinclude", "-Iparsec_b200/csrc",
                    "tests/cpp/reader_group_plan_shim.cpp", "tests/cpp/window_plan_shim.cpp",
                    "parsec_b200/csrc/pb2_window_plan.cpp", "-o", so], cwd=ROOT, check=True)
    lib = C.CDLL(so)
    lib.wp_plan_reader_groups.restype = C.c_void_p
    lib.wp_plan_reader_groups.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_int32,
                                          C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                          C.POINTER(C.c_int), C.POINTER(C.c_char_p)]
    lib.wp_free.argtypes = [C.c_void_p]
    lib.wp_array.restype = C.c_int64
    lib.wp_array.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p)]
    lib.wp_scalar.restype = C.c_int64
    lib.wp_scalar.argtypes = [C.c_void_p, C.c_char_p]
    return lib


def plan(lib, dag, tiles=None, readers=READERS, groups=0, **kw):
    """The plan of dag (every array and scalar of test_window_plan's), with linked_readers and linked_reader_groups."""
    if tiles is None:
        tiles = tiles_for(dag.ntiles, dag.tile_bytes)
    prm = np.array([kw.get(k, DEFAULTS[k]) for k in PARAMS], np.int64)
    tasks = np.ascontiguousarray(dag.tasks, L.TASK_DTYPE)
    succ = np.ascontiguousarray(dag.succ, np.uint32)
    tiles = np.ascontiguousarray(tiles, L.TILE_DTYPE)
    ready = np.ascontiguousarray(dag.ready, np.int32)
    rc, why = C.c_int(0), C.c_char_p()
    h = lib.wp_plan_reader_groups(prm.ctypes.data, 0, readers, groups, tasks.ctypes.data, len(tasks), succ.ctypes.data,
                                  len(succ), tiles.ctypes.data, len(tiles), ready.ctypes.data, len(ready), C.byref(rc),
                                  C.byref(why))
    assert h, (rc.value, why.value)
    try:
        out = {}
        for name, dt in ARRAYS.items():
            p = C.c_void_p()
            n = lib.wp_array(h, name.encode(), C.byref(p))
            out[name] = np.frombuffer(C.string_at(p.value, n) if n else b"", dtype=dt).copy()
        for name in SCALARS:
            out[name] = lib.wp_scalar(h, name.encode())
        return out
    finally:
        lib.wp_free(h)


def assert_same_but_the_mark(without, with_, groups):
    """Every array and scalar equal, except the group mark of the declared readers' descriptors."""
    for name in SCALARS:
        assert with_[name] == without[name], name
    for name in ARRAYS:
        if name != "tasks":
            assert with_[name].tobytes() == without[name].tobytes(), name
    a, b = without["tasks"], with_["tasks"]
    bodies = b["body"].astype(np.int64) - L.BODY_LINKED_0
    declared = (bodies >= 0) & (bodies < 8) & ((groups >> np.clip(bodies, 0, 7)) & 1).astype(bool)
    assert np.all(b["flags"][declared] == a["flags"][declared] | TASK_READER_GROUP)
    assert np.all(b["flags"][declared] & TASK_READER), "only readers carry the group mark"
    assert np.all(b["flags"][~declared] == a["flags"][~declared])
    assert not np.any(a["flags"] & TASK_READER_GROUP)
    a, b = a.copy(), b.copy()
    a["flags"] = b["flags"] = 0
    assert a.tobytes() == b.tobytes()
    return int(np.count_nonzero(declared))


@pytest.mark.parametrize("kind", [0, 1], ids=["hbm", "gemm"])
@pytest.mark.parametrize("producer,part_bytes,trace,queue_policy,groups", [
    (None, 256 * 1024, 0, 0, GROUPS), (None, 64 * 1024, 1, 0, 0b101), (FILL, 0, 1, 1, GROUPS),
    (FILL, 64 * 1024, 0, 1, 0b1)],
    ids=["builtin_one_part", "builtin_four_parts_traced_some", "linked_whole_traced_prio", "linked_four_parts_prio_one"])
def test_ex05_plans_alike(planner, kind, producer, part_bytes, trace, queue_policy, groups):
    base = with_bodies(dags.ex05_broadcast(6, 14, 256 * 1024), producer)
    # the readers of each tile mix COUNT_NE, SUM_I64 and COUNT_GT
    t = base.tasks
    t["body"][6:] = np.array([COUNT_NE, SUM_I64, COUNT_GT] * 100, np.uint8)[:len(t) - 6]
    kw = dict(LINKED, kind=kind, part_bytes=part_bytes, trace=trace, queue_policy=queue_policy)
    without = plan(planner, base, **kw)
    with_ = plan(planner, base, groups=groups, **kw)
    assert all(with_["group"][k] & GROUP_FUSED for k in range(6))
    assert assert_same_but_the_mark(without, with_, groups) > 0


@pytest.mark.parametrize("kw", [dict(read_groups=-1), dict(fuse_readers=-1), dict(nworkers=1), dict(shared=0)],
                         ids=["ungrouped", "unfused", "one_worker", "default"])
def test_fan_out_plans_alike(planner, kw):
    dag, tiles = fan_out([rd(COUNT_NE), rd(SUM_I64), rd(SUM_CTL), rd(COUNT_GT), rd(COUNT_NE)] * 2, FILL)
    without = plan(planner, dag, tiles, **dict(LINKED, **kw))
    with_ = plan(planner, dag, tiles, groups=GROUPS, **dict(LINKED, **kw))
    # SUM_CTL is no reader: it splits the groups and never carries the mark
    assert assert_same_but_the_mark(without, with_, GROUPS) == 8


# ----------------------------------------------------------------------------------------------------------------------
# the kernels and the fixture, linked offline
# ----------------------------------------------------------------------------------------------------------------------
def tool(name):
    path = os.path.join(CUDA, "bin", name)
    if not os.path.exists(path):
        pytest.skip(name + " not found")
    return path


def built(*parts):
    path = os.path.join(ROOT, *parts)
    assert os.path.exists(path), "build() makes " + path
    return path


@pytest.mark.parametrize("engine,pattern,max_regs", [
    ("pb2_engine_linked_groups.cubin", r"_ZN3pb221pb2_engine_hbm_kernelI\w+", 80),
    ("pb2_engine_linked_gemm_groups.cubin", r"_ZN3pb223pb2_engine_gemm2_kernelI\w+", 168)], ids=["hbm", "gemm"])
def test_group_kernels_link_with_the_fixture(tmp_path, engine, pattern, max_regs):
    out = tmp_path / "linked.cubin"
    subprocess.check_call([tool("nvlink"), "-arch=sm_90a", "-o", str(out), built("build", engine),
                           built("tests", "cuda", "reader_group_bodies.cubin")])
    res = subprocess.check_output([tool("cuobjdump"), "-res-usage", str(out)], text=True)
    kernels = re.findall(r"Function (%s):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)" % pattern, res)
    assert len(kernels) == 4, res
    for name, reg, stack, smem, local in kernels:
        assert int(reg) <= max_regs and int(local) == 0, (name, reg, stack, smem, local)
        if max_regs == 80:      # 8 workers of 64 threads per SM fit in shared memory
            assert 8 * int(smem) <= 227 * 1024, (name, smem)


def test_gemm_group_kernels_keep_their_wgmma():
    with open(built("build", "linked_gemm_groups_ptxas.log")) as f:
        text = f.read()
    assert "C7509" not in text and "serialized" not in text


def test_group_kernels_need_the_group_form(tmp_path):
    p = subprocess.run([tool("nvlink"), "-arch=sm_90a", "-o", str(tmp_path / "x.cubin"),
                        built("build", "pb2_engine_linked_groups.cubin"), built("tests", "cuda", "reader_bodies.cubin")],
                       capture_output=True, text=True)
    assert p.returncode != 0 and "pb2_linked_reader_group" in p.stdout + p.stderr, p


@pytest.mark.parametrize("engine", ["pb2_engine_linked.cubin", "pb2_engine_linked_gemm.cubin"])
def test_plain_kernels_never_name_the_group_form(tmp_path, engine):
    cubin = built("build", engine)
    with open(cubin, "rb") as f:
        assert b"pb2_linked_reader_group" not in f.read()
    # an image with the group form links with them too: the form is simply never called
    subprocess.check_call([tool("nvlink"), "-arch=sm_90a", "-o", str(tmp_path / "x.cubin"), cubin,
                           built("tests", "cuda", "reader_group_bodies.cubin")])


def test_fixture_ptx_defines_both_forms():
    with open(built("tests", "cuda", "reader_group_bodies.ptx"), "rb") as f:
        ptx = f.read()
    for name in (b"pb2_linked_reader_group", b"pb2_linked_body"):
        assert re.search(rb"\.visible \.func\s+\(\.param \.b64 func_retval0\)\s+" + name + rb"\(", ptx), name
