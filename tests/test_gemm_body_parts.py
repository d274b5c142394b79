"""GEMM-worker bodies in parts (pb2_engine_set_gemm_body_parts, pb2_device_set_gemm_body_parts), host side.

  - the module setter's refusals, and the counts a dry-run module records; the engine setter refuses a null engine;
  - the header constant PB2_GEMM_BODY_MAX_PARTS, the static_assert that ties it to the ring entry's part field, and the
    layout of pb2_gemm_body_args_t;
  - the planner (tests/cpp/gemm_body_parts_plan_shim.cpp): unit part counts, ring image, task entries, priority lanes
    and part records for declared counts 1, 2, 7 and 32; all-ones counts give the plan of a planner without them;
  - the fixture (tests/cuda/gemm_part_bodies.cu) links offline with the entry builds of the GEMM kernels within both
    register budgets, with no local memory between the DMMAs of its DGEMM.
The GPU side is tests/test_gemm_body_parts_gpu.py."""
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
BUILD = os.path.join(ROOT, "build")
DGEMM, PART, ADD = L.BODY_LINKED_0, L.BODY_LINKED_0 + 1, L.BODY_LINKED_0 + 2
GEMM_BODIES = 0x03
TASK_GEMM_BODY = 0x20


def tool(name):
    return os.path.join(CUDA, "bin", name)


# ----------------------------------------------------------------------------------------------------------------------
# the setters
# ----------------------------------------------------------------------------------------------------------------------
def test_module_setter_refusals_and_record():
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        dev = ctx.devices[0]
        set_parts = lambda body, n: ctx.l.pb2_device_set_gemm_body_parts(dev, body, n)
        assert set_parts(DGEMM, 4) == L.PB2_ERR_NOT_FOUND                     # before the link
        ctx.link_bodies(dev, b"ptx", L.IMAGE_PTX, 0x04, gemm_windows=True, gemm_bodies=GEMM_BODIES)
        assert [ctx.gemm_body_parts(dev, L.BODY_LINKED_0 + i) for i in range(8)] == [1] * 8
        for body in (L.BODY_LINKED_0 - 1, L.BODY_LINKED_7 + 1, L.BODY_GEMM_BF16, ADD, L.BODY_LINKED_7):
            assert set_parts(body, 2) == L.PB2_ERR_BAD_PARAM, body             # not an id, or not a GEMM-worker body
        for n in (0, -1, L.GEMM_BODY_MAX_PARTS + 1):
            assert set_parts(DGEMM, n) == L.PB2_ERR_VALUE_OUT_OF_BOUNDS, n
        assert [ctx.gemm_body_parts(dev, L.BODY_LINKED_0 + i) for i in range(8)] == [1] * 8   # refusals change nothing
        ctx.set_gemm_body_parts(dev, DGEMM, 7)
        ctx.set_gemm_body_parts(dev, PART, L.GEMM_BODY_MAX_PARTS)
        assert ctx.gemm_body_parts(dev, DGEMM) == 7 and ctx.gemm_body_parts(dev, PART) == 32
        ctx.set_gemm_body_parts(dev, DGEMM, 1)
        assert ctx.gemm_body_parts(dev, DGEMM) == 1
        with pytest.raises(L.Pb2Error) as ex:
            ctx.set_gemm_body_parts(dev, DGEMM, 33)
        assert ex.value.rc == L.PB2_ERR_VALUE_OUT_OF_BOUNDS
        assert ctx.gemm_body_parts(dev, DGEMM) == 1


def test_module_setter_without_gemm_worker_bodies():
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        dev = ctx.devices[0]
        ctx.link_bodies(dev, b"ptx", L.IMAGE_PTX, 0, gemm_windows=True)
        assert ctx.l.pb2_device_set_gemm_body_parts(dev, DGEMM, 2) == L.PB2_ERR_BAD_PARAM


def test_engine_setter_refuses_a_null_engine():
    lib = L.load()
    assert lib.pb2_engine_set_gemm_body_parts(None, DGEMM, 2) == L.PB2_ERR_BAD_PARAM


def test_refusal_messages(tmp_path):
    """gemm_body_parts_error, the check both setters make: its code and message for each refusal."""
    src = tmp_path / "why.cpp"
    src.write_text('#include <cstdio>\n#include <cstdlib>\n#include "pb2_engine_priv.hpp"\n'
                   'int main(int, char** v) { int rc; const char* w = gemm_body_parts_error(atoi(v[1]), '
                   '(uint32_t)strtoul(v[2], 0, 0), atoi(v[3]), atoi(v[4]), &rc); printf("%d %s", rc, w ? w : ""); }\n')
    exe = tmp_path / "why"
    subprocess.run(["g++", "-std=c++17", "-I" + os.path.join(CUDA, "include"), "-I" + os.path.join(ROOT, "parsec_b200", "csrc"),
                    str(src), "-o", str(exe)], check=True)
    why = lambda *a: subprocess.check_output([str(exe), *map(str, a)], text=True).split(" ", 1)
    assert why(0, 3, DGEMM, 2) == [str(L.PB2_ERR_NOT_FOUND), "no image is linked yet: part counts are declared for the "
                                   "GEMM-worker bodies of a link"]
    rc, msg = why(1, 3, 19, 2)
    assert int(rc) == L.PB2_ERR_BAD_PARAM and "PB2_BODY_LINKED_0 .. _7" in msg
    rc, msg = why(1, 3, ADD, 2)
    assert int(rc) == L.PB2_ERR_BAD_PARAM and "PB2_LINK_GEMM_BODIES" in msg
    rc, msg = why(1, 3, DGEMM, 33)
    assert int(rc) == L.PB2_ERR_VALUE_OUT_OF_BOUNDS and "PB2_GEMM_BODY_MAX_PARTS" in msg
    assert why(1, 3, DGEMM, 32) == ["0", ""] and why(1, 3, PART, 1) == ["0", ""]


# ----------------------------------------------------------------------------------------------------------------------
# the headers
# ----------------------------------------------------------------------------------------------------------------------
def test_header_constant_and_args_block(tmp_path):
    src = tmp_path / "parts.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include <stdint.h>\n#include "pb2_engine.h"\n'
                   '#include "pb2_device_body.h"\n'
                   'int main(void) { printf("%d %zu %zu %zu %zu", PB2_GEMM_BODY_MAX_PARTS, sizeof(pb2_gemm_body_args_t), '
                   'offsetof(pb2_gemm_body_args_t, check), offsetof(pb2_gemm_body_args_t, nparts), sizeof(pb2_body_check_t));'
                   ' return 0; }\n')
    exe = tmp_path / "parts"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                   check=True)
    maxp, size, check, nparts, check_size = map(int, subprocess.check_output([str(exe)], text=True).split())
    assert maxp == 32 == L.GEMM_BODY_MAX_PARTS
    # the words of pb2_body_check_t, then nparts right after its 80 bytes
    assert (size, check, nparts, check_size) == (88, 72, 80, 80)
    layout = open(os.path.join(ROOT, "parsec_b200", "csrc", "pb2_window_layout.h")).read()
    assert "constexpr int kMaxParts = 32;" in layout
    assert "static_assert(PB2_GEMM_BODY_MAX_PARTS == kMaxParts" in layout


def test_static_assert_holds_the_two_together(tmp_path):
    """The layout header does not compile against a header whose constant differs from the ring's part field."""
    inc = tmp_path / "include"
    inc.mkdir()
    hdr = open(os.path.join(ROOT, "include", "pb2_engine.h")).read()
    (inc / "pb2_engine.h").write_text(hdr.replace("#define PB2_GEMM_BODY_MAX_PARTS 32", "#define PB2_GEMM_BODY_MAX_PARTS 64"))
    csrc = tmp_path / "parsec_b200" / "csrc"
    csrc.mkdir(parents=True)
    (csrc / "pb2_window_layout.h").write_text(open(os.path.join(ROOT, "parsec_b200", "csrc", "pb2_window_layout.h")).read())
    src = csrc / "t.cpp"
    src.write_text('#include "pb2_window_layout.h"\nint main() { return 0; }\n')
    real = tmp_path / "real.cpp"
    real.write_text('#include "pb2_window_layout.h"\nint main() { return 0; }\n')
    ok = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I" + os.path.join(ROOT, "parsec_b200", "csrc"), str(real)],
                        capture_output=True, text=True)
    assert ok.returncode == 0, ok.stderr
    bad = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", str(src)], capture_output=True, text=True)
    assert bad.returncode != 0 and "ring entry's part field" in bad.stderr, bad.stderr


# ----------------------------------------------------------------------------------------------------------------------
# the planner
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("gemm_body_parts_plan") / "gemm_body_parts_plan.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-Iinclude", "-Iparsec_b200/csrc",
                    "tests/cpp/gemm_body_parts_plan_shim.cpp", "tests/cpp/gemm_body_plan_shim.cpp",
                    "tests/cpp/window_plan_shim.cpp", "parsec_b200/csrc/pb2_window_plan.cpp", "-o", so], cwd=ROOT, check=True)
    lib = C.CDLL(so)
    common = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
              C.POINTER(C.c_int), C.POINTER(C.c_char_p)]
    lib.wp_plan_gemm_body_parts.restype = C.c_void_p
    lib.wp_plan_gemm_body_parts.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p] + common
    lib.wp_plan_gemm_bodies.restype = C.c_void_p
    lib.wp_plan_gemm_bodies.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32] + common
    lib.wp_free.argtypes = [C.c_void_p]
    lib.wp_array.restype = C.c_int64
    lib.wp_array.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p)]
    lib.wp_scalar.restype = C.c_int64
    lib.wp_scalar.argtypes = [C.c_void_p, C.c_char_p]
    return lib


def plan(lib, tasks, succ, ready, tiles, parts=None, readers=0, gemm_bodies=GEMM_BODIES, **kw):
    """(rc, why, plan) of a GEMM window of an engine linked with PB2_LINK_GEMM_WINDOWS; parts: the 8 declared counts,
    or None for the planner without them (wp_plan_gemm_bodies)."""
    kw.setdefault("kind", 1)
    kw.setdefault("linked_image", 1)
    prm = np.array([kw.get(k, DEFAULTS[k]) for k in PARAMS], np.int64)
    tasks = np.ascontiguousarray(tasks, L.TASK_DTYPE)
    succ = np.ascontiguousarray(succ, np.uint32)
    tiles = np.ascontiguousarray(tiles, L.TILE_DTYPE)
    ready = np.ascontiguousarray(ready, np.int32)
    rc, why = C.c_int(0), C.c_char_p()
    rest = (tasks.ctypes.data, len(tasks), succ.ctypes.data, len(succ), tiles.ctypes.data, len(tiles), ready.ctypes.data,
            len(ready), C.byref(rc), C.byref(why))
    if parts is None:
        h = lib.wp_plan_gemm_bodies(prm.ctypes.data, 0, readers, gemm_bodies, *rest)
    else:
        p = np.ascontiguousarray(parts, np.int32)
        h = lib.wp_plan_gemm_body_parts(prm.ctypes.data, 0, readers, gemm_bodies, p.ctypes.data, *rest)
    if not h:
        return rc.value, why.value.decode() if why.value else None, None
    try:
        out = {}
        for name, dt in ARRAYS.items():
            q = C.c_void_p()
            n = lib.wp_array(h, name.encode(), C.byref(q))
            out[name] = np.frombuffer(C.string_at(q.value, n) if n else b"", dtype=dt).copy()
        for name in SCALARS:
            out[name] = lib.wp_scalar(h, name.encode())
        return rc.value, None, out
    finally:
        lib.wp_free(h)


def mixed_window(NT=3, M=128, N=128, K=64, prio=False):
    """The fp64 DTD GEMM (DGEMM tasks), plus one PART probe task on a tile of its own, ready at start.  With prio,
    the tasks get distinct priorities (the probe the highest)."""
    dag, sizes = F.dag(NT, M, N, K)
    t = np.concatenate([dag.tasks, np.zeros(1, L.TASK_DTYPE)])
    n = len(t) - 1
    t["tile"][n] = -1
    t["tile"][n, 0] = dag.ntiles
    t["nb_flows"][n], t["body"][n], t["access"][n, 0] = 1, PART, L.ACCESS_WRITE
    t["succ_begin"][n] = len(dag.succ)
    if prio:
        t["priority"] = np.arange(len(t), dtype=np.int32) % 5
        t["priority"][n] = 100
    tiles = tiles_for(dag.ntiles + 1, 0)
    tiles["bytes"][:dag.ntiles] = sizes
    tiles["bytes"][dag.ntiles] = 4096
    return t, dag.succ, np.concatenate([dag.ready, [n]]).astype(np.int32), tiles


def unit_of_task(p):
    u = np.full(len(p["tasks"]), -1, np.int64)
    for i, unit in enumerate(p["units"]):
        u[p["segs"]["task"][unit["seg_begin"]:unit["seg_begin"] + unit["seg_count"]]] = i
    return u


@pytest.mark.parametrize("queue_policy,trace", [(0, 0), (1, 1), (0, 1), (1, 0)], ids=["fifo", "lanes_traced", "traced", "lanes"])
@pytest.mark.parametrize("dgemm_parts,part_parts", [(1, 1), (2, 7), (7, 32), (32, 2)])
def test_units_ring_and_entries_follow_the_count(planner, queue_policy, trace, dgemm_parts, part_parts):
    t, succ, ready, tiles = mixed_window(prio=queue_policy == 1)
    parts = [dgemm_parts, part_parts, 1, 1, 1, 1, 1, 1]
    rc, why, p = plan(planner, t, succ, ready, tiles, parts=parts, queue_policy=queue_policy, trace=trace, part_bytes=4096)
    assert rc == 0, why
    assert np.all(p["tasks"]["flags"] & TASK_GEMM_BODY)
    units, segs = p["units"], p["segs"]
    assert len(units) == len(t) and np.all(units["seg_count"] == 1)            # never grouped or fused
    uot = unit_of_task(p)
    want = np.where(t["body"] == DGEMM, dgemm_parts, part_parts)
    assert np.array_equal(units["nparts"][uot], want)
    # every task's entry names its unit with (parts - 1) in the part field
    entry = p["task_entry"].astype(np.uint32)
    assert np.array_equal(entry & ((1 << 27) - 1), uot) and np.array_equal(entry >> 27, want - 1)
    # the ring image: every part of every ready unit, once
    img = p["ring_image"][p["ring_image"] != -1].astype(np.uint32)
    got = sorted(zip((img & ((1 << 27) - 1)).tolist(), (img >> 27).tolist()))
    assert got == sorted((int(uot[r]), q) for r in ready for q in range(want[r]))
    total = int(want.sum())
    if queue_policy == 1:
        # each lane's segment holds every entry its units can ever push
        assert p["lanes"] == 1 and len(p["ring_image"]) == total
        lanes = p["lane"]
        for l in range(8):
            size = int(units["nparts"][lanes == l].sum())
            nxt = p["lane_begin"][l + 1] if l + 1 < 8 else len(p["ring_image"])
            assert nxt - p["lane_begin"][l] == size
    assert p["ring"] >= len(t) + total
    if trace:
        assert p["part_records"] == total
        ent = p["part_entities"]
        assert len(ent) == len(t)
        assert np.array_equal(ent["nparts"], want[ent["lead"]])
        o = np.argsort(ent["base"])                     # owner order: each owner's records follow the previous one's
        assert np.array_equal(ent["base"][o], np.concatenate([[0], np.cumsum(ent["nparts"][o])[:-1]]))


@pytest.mark.parametrize("queue_policy,trace", [(0, 0), (1, 1)])
@pytest.mark.parametrize("window", ["fp64", "mixed"])
def test_all_ones_counts_give_the_plan_without_them(planner, queue_policy, trace, window):
    if window == "fp64":
        dag, sizes = F.dag(3, 130, 50, 40)
        t, succ, ready, tiles = dag.tasks, dag.succ, dag.ready, tiles_for(dag.ntiles, 0)
        tiles["bytes"] = sizes
    else:
        t, succ, ready, tiles = mixed_window(prio=queue_policy == 1)
    kw = dict(queue_policy=queue_policy, trace=trace, part_bytes=4096)
    rc0, _, a = plan(planner, t, succ, ready, tiles, parts=None, **kw)
    rc1, _, b = plan(planner, t, succ, ready, tiles, parts=[1] * 8, **kw)
    assert rc0 == rc1 == 0
    for name in ARRAYS:
        assert a[name].tobytes() == b[name].tobytes(), name
    for name in SCALARS:
        assert a[name] == b[name], name


def test_counts_apply_to_gemm_worker_bodies_only(planner):
    """A count set for a body outside the GEMM-worker mask plans nothing different: its tasks are ordinary linked
    bodies, cut into byte slices by part_bytes as before."""
    t, succ, ready, tiles = mixed_window()
    kw = dict(part_bytes=1024, linked_sliceable=0x02)
    rc0, _, a = plan(planner, t, succ, ready, tiles, parts=None, gemm_bodies=0x01, **kw)
    rc1, _, b = plan(planner, t, succ, ready, tiles, parts=[1, 9, 1, 1, 1, 1, 1, 1], gemm_bodies=0x01, **kw)
    assert rc0 == rc1 == 0
    assert a["units"].tobytes() == b["units"].tobytes() and a["ring_image"].tobytes() == b["ring_image"].tobytes()
    probe = unit_of_task(b)[len(t) - 1]
    assert b["units"]["nparts"][probe] == 4                                     # 4096 bytes in 1 KiB slices


# ----------------------------------------------------------------------------------------------------------------------
# the fixture, linked offline
# ----------------------------------------------------------------------------------------------------------------------
def built(*names):
    paths = [os.path.join(BUILD, n) if n.startswith("pb2_") else os.path.join(ROOT, "tests", "cuda", n) for n in names]
    assert all(os.path.exists(p) for p in paths), "build() makes the engine cubins and the fixtures"
    return paths


def resources(cubin):
    res = subprocess.check_output([tool("cuobjdump"), "-res-usage", str(cubin)], text=True)
    gemm = re.findall(r"Function _ZN3pb223pb2_engine_gemm2_kernelI\w+:\s*\n\s*REG:(\d+) STACK:\d+ SHARED:(\d+)", res)
    hbm = re.findall(r"Function _ZN3pb221pb2_engine_hbm_kernelI\w+:\s*\n\s*REG:(\d+)", res)
    return [(int(r), int(s)) for r, s in gemm], [int(r) for r in hbm]


@pytest.mark.parametrize("gemm_cubin,bodies", [("pb2_engine_linked_gemm_entry.cubin", "gemm_part_bodies.cubin"),
                                               ("pb2_engine_linked_gemm_entry_groups.cubin", "gemm_part_group_bodies.cubin"),
                                               ("pb2_engine_linked_gemm.cubin", "gemm_part_bodies.cubin")],
                         ids=["entry", "entry_groups", "plain"])
def test_fixture_links_within_both_budgets(tmp_path, gemm_cubin, bodies):
    hbm_cubin = "pb2_engine_linked_groups.cubin" if "groups" in gemm_cubin else "pb2_engine_linked.cubin"
    out = tmp_path / "linked.cubin"
    p = subprocess.run([tool("nvlink"), "-arch=sm_90a", "-o", str(out), *built(hbm_cubin, gemm_cubin, bodies)],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    assert "C7509" not in p.stdout + p.stderr
    gemm, hbm = resources(out)
    print("linked GEMM kernels (registers, static shared memory):", gemm)
    assert len(gemm) == 4 and len(hbm) == 4
    assert all(r <= 168 and s + 196608 + 1024 <= 227 * 1024 for r, s in gemm), gemm
    assert all(r == 80 for r in hbm), hbm


def test_dgemm_keeps_local_memory_out_of_its_dmma_loop():
    sass = subprocess.check_output([tool("cuobjdump"), "-sass", "-fun", "pb2_linked_gemm_body",
                                    *built("gemm_part_bodies.cubin")], text=True).splitlines()
    dmma = [i for i, l in enumerate(sass) if "DMMA.8x8x4" in l or "DMMA.16x8x8" in l]
    assert len(dmma) >= 16, "the DGEMM body runs on the FP64 tensor cores"
    local = [l.strip() for l in sass[dmma[0]:dmma[-1]] if re.search(r"\b(LDL|STL)\b", l)]
    assert not local, local[:8]
    log = open(os.path.join(ROOT, "tests", "cuda", "gemm_part_bodies.log")).read()
    body = re.search(r"Function properties for pb2_linked_body\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores", log)
    assert body and body.group(2) == "0", log
