"""Linked bodies in GEMM windows (pb2_engine_link_bodies_ex with PB2_LINK_GEMM_WINDOWS), host side.

  - the planner refuses a linked body in a GEMM window unless the engine linked with the flag, and a shared window
    either way, with the messages it gives without the flag;
  - with the flag, a linked unit is cut into parts as a built-in HBM unit is when its sliceable bit is set, and runs as
    one part over whole tiles when it is clear; the Morton ready order and the ring image are those of the same DAG
    with built-in bodies in place of the linked ones;
  - the link calls refuse unknown flag bits;
  - in dry run, the stand-alone runtime puts GEMM chains and linked tasks into one window only with the flag;
  - the linked GEMM kernels compile without serialized wgmma (no C7509), their wgmma loop makes no call and no local
    memory access, and the cubin links offline with both test fixtures.
The GPU side is tests/test_linked_gemm_gpu.py."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200 import runtime as R
from test_window_plan import ARRAYS, DEFAULTS, GEMM_MAX_PARTS, PARAMS, SCALARS, morton, tiles_for
from test_linked_bodies import insert_linked, int32_collection
import mixed_pool as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
LINKED_FILL = L.BODY_LINKED_0 + 3        # tests/cuda/linked_bodies.cu: FILL_I32 through the link
GEMM_MSG = "linked body in a GEMM window (linked bodies run in HBM windows only)"


@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("linked_gemm_plan") / "linked_gemm_plan.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-Iinclude", "-Iparsec_b200/csrc",
                    "tests/cpp/linked_gemm_plan_shim.cpp", "tests/cpp/window_plan_shim.cpp",
                    "parsec_b200/csrc/pb2_window_plan.cpp", "-o", so], cwd=ROOT, check=True)
    lib = C.CDLL(so)
    lib.wp_plan_linked_gemm.restype = C.c_void_p
    lib.wp_plan_linked_gemm.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p,
                                        C.c_int32, C.c_void_p, C.c_int32, C.POINTER(C.c_int), C.POINTER(C.c_char_p)]
    lib.wp_free.argtypes = [C.c_void_p]
    lib.wp_array.restype = C.c_int64
    lib.wp_array.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p)]
    lib.wp_scalar.restype = C.c_int64
    lib.wp_scalar.argtypes = [C.c_void_p, C.c_char_p]
    return lib


def plan(lib, dag, tiles, linked_gemm=0, **kw):
    """(rc, why, plan) of a GEMM window over dag, with PlanParams::linked_gemm = linked_gemm."""
    kw.setdefault("kind", 1)
    prm = np.array([kw.get(k, DEFAULTS[k]) for k in PARAMS], np.int64)
    tasks = np.ascontiguousarray(dag.tasks, L.TASK_DTYPE)
    succ = np.ascontiguousarray(dag.succ, np.uint32)
    tiles = np.ascontiguousarray(tiles, L.TILE_DTYPE)
    ready = np.ascontiguousarray(dag.ready, np.int32)
    rc, why = C.c_int(0), C.c_char_p()
    h = lib.wp_plan_linked_gemm(prm.ctypes.data, linked_gemm, tasks.ctypes.data, len(tasks), succ.ctypes.data,
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


def chains_and_fills(NT=3, tile=256, nfill=5, fill_bytes=1 << 20, body=L.BODY_FILL_I32):
    """dags.dtd_gemm(NT, tile) beside nfill independent `body` tasks, each writing a tile of its own of fill_bytes.
    The ready list interleaves the fills with the chain heads, so that the ring image mixes both kinds of unit."""
    g = dags.dtd_gemm(NT, tile=tile)
    n0, t0 = g.ntasks, g.ntiles
    t = np.concatenate([g.tasks, dags._new_tasks(nfill)])
    f = t[n0:]
    f["body"], f["nb_flows"], f["access"][:, 0], f["iparam"][:, 0] = body, 1, L.ACCESS_WRITE, 7
    f["tile"][:, 0] = t0 + np.arange(nfill)
    f["succ_begin"] = len(g.succ)
    heads = [int(r) for r in g.ready]
    ready = []
    for i in range(max(len(heads), nfill)):
        ready += heads[i:i + 1] + ([n0 + i] if i < nfill else [])
    dag = dags.Dag(t, g.succ, np.array(ready, np.int32), ntiles=t0 + nfill, tile_bytes=0, kind=1)
    tiles = tiles_for(t0 + nfill, tile * tile * 2)
    tiles["bytes"][t0:] = fill_bytes
    return dag, tiles


def linked_version(dag, body=LINKED_FILL):
    t = dag.tasks.copy()
    t["body"][t["body"] == L.BODY_FILL_I32] = body
    return dags.Dag(t, dag.succ, dag.ready, ntiles=dag.ntiles, tile_bytes=dag.tile_bytes, kind=1)


LINKED = dict(linked_image=1, linked_sliceable=0xFF)


def test_gemm_window_refuses_linked_bodies_without_the_flag(planner):
    dag, tiles = chains_and_fills()
    rc, why, _ = plan(planner, linked_version(dag), tiles, **LINKED)
    assert rc == L.PB2_ERR_NOT_SUPPORTED and why == GEMM_MSG
    rc, why, p = plan(planner, linked_version(dag), tiles, linked_gemm=1, **LINKED)
    assert rc == 0, why
    assert p["linked"] == 1
    # the flag changes nothing for a window without linked tasks
    rc, why, p = plan(planner, dag, tiles, linked_gemm=1, **LINKED)
    assert rc == 0 and p["linked"] == 0


@pytest.mark.parametrize("linked_gemm", [0, 1])
def test_shared_gemm_window_still_refuses_linked_bodies(planner, linked_gemm):
    dag, tiles = chains_and_fills()
    rc, why, _ = plan(planner, linked_version(dag), tiles, linked_gemm=linked_gemm, shared=1, **LINKED)
    assert rc == L.PB2_ERR_NOT_SUPPORTED
    assert why == (GEMM_MSG if not linked_gemm else "linked body in a shared window (not supported)")


def test_engine_without_an_image_refuses_linked_bodies_in_gemm_windows(planner):
    dag, tiles = chains_and_fills()
    rc, why, _ = plan(planner, linked_version(dag), tiles, linked_gemm=1, linked_image=0)
    assert rc == L.PB2_ERR_NOT_SUPPORTED and "has not linked an image" in why


@pytest.mark.parametrize("part_bytes,fill_bytes", [(64 * 1024, 1 << 20), (256 * 1024, 1 << 20), (16 * 1024, 1 << 20),
                                                   (256 * 1024, 64 * 1024)],
                         ids=["16_parts", "4_parts", "capped_at_32", "one_part"])
def test_linked_units_are_cut_by_their_sliceable_bit(planner, part_bytes, fill_bytes):
    dag, tiles = chains_and_fills(fill_bytes=fill_bytes)
    nfill = 5
    want = min(-(-fill_bytes // part_bytes), GEMM_MAX_PARTS)
    sliced = 1 << (LINKED_FILL - L.BODY_LINKED_0)
    for mask, parts in ((sliced, want), (0xFF & ~sliced, 1)):
        rc, why, p = plan(planner, linked_version(dag), tiles, linked_gemm=1, part_bytes=part_bytes, linked_image=1,
                          linked_sliceable=mask)
        assert rc == 0, why
        units = p["units"]
        fills = units[units["flags"] == 0]
        assert len(fills) == nfill and (fills["nparts"] == parts).all(), (mask, fills["nparts"])
        assert (units[units["flags"] == 1]["nparts"] == 2).all()       # 256 x 256 C: two 128 x 256 sub-tiles


@pytest.mark.parametrize("queue_policy,trace", [(0, 0), (1, 0), (0, 1), (1, 1)])
def test_linked_window_plans_as_the_builtin_one(planner, queue_policy, trace):
    """Sliceable linked FILLs in place of built-in ones: the same units, ready order, ring image, lanes and records."""
    NT = 3
    dag, tiles = chains_and_fills(NT=NT)
    kw = dict(part_bytes=128 * 1024, queue_policy=queue_policy, trace=trace)
    rc, why, want = plan(planner, dag, tiles, **kw)
    assert rc == 0, why
    rc, why, got = plan(planner, linked_version(dag), tiles, linked_gemm=1, **LINKED, **kw)
    assert rc == 0, why
    for name in ARRAYS:
        a, b = want[name], got[name]
        if name == "tasks":
            a, b = a.copy(), b.copy()
            assert np.count_nonzero(b["body"] == LINKED_FILL) == 5
            a["body"][a["body"] == L.BODY_FILL_I32] = 0
            b["body"][b["body"] == LINKED_FILL] = 0
        assert a.tobytes() == b.tobytes(), name
    for name in SCALARS:
        assert got[name] == want[name] or name == "linked", name
    assert got["linked"] == 1 and want["linked"] == 0
    if queue_policy == 0:
        # the ready units in the Morton order of their C(i,j), a fill's key being 0, ties in ready-list order
        units, segs = got["units"], got["segs"]
        owners = [int(e) & 0x07FFFFFF for e in got["ring_image"].view(np.uint32)]
        firsts = [o for i, o in enumerate(owners) if i == 0 or owners[i - 1] != o]
        lead = [int(segs["task"][units[u]["seg_begin"]]) for u in firsts]
        key = lambda t: morton(t // (NT * NT), (t // NT) % NT) if t < NT ** 3 else 0
        assert lead == sorted(dag.ready.tolist(), key=key)


# ----------------------------------------------------------------------------------------------------------------------
# the link calls
# ----------------------------------------------------------------------------------------------------------------------
def test_engine_link_ex_refuses_a_null_engine():
    lib = L.load()
    assert lib.pb2_engine_link_bodies_ex(None, b"x", 1, L.IMAGE_PTX, 1, 0, L.LINK_GEMM_WINDOWS) == L.PB2_ERR_BAD_PARAM
    assert lib.pb2_engine_linked_gemm_info(None, None, None, None, None) == L.PB2_ERR_BAD_PARAM


@pytest.mark.parametrize("flags", [0x2, 0x3, 0x80000000, 0xFFFFFFFF])
def test_device_link_ex_refuses_unknown_flags(flags):
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        dev = ctx.devices[0]
        assert ctx.l.pb2_device_link_bodies_ex(dev, b"x", 1, L.IMAGE_PTX, 1, 0, flags) == L.PB2_ERR_BAD_PARAM
        # nothing was recorded: a valid call still links, a second one is refused
        assert ctx.l.pb2_device_link_bodies_ex(dev, b"x", 1, L.IMAGE_PTX, 1, 0, L.LINK_GEMM_WINDOWS) == 0
        assert ctx.l.pb2_device_link_bodies_ex(dev, b"x", 1, L.IMAGE_PTX, 1, 0, 0) == L.PB2_ERR_EXISTS


# ----------------------------------------------------------------------------------------------------------------------
# the stand-alone runtime, in dry run
# ----------------------------------------------------------------------------------------------------------------------
def gemm_and_linked_pool(gemm_windows):
    """The pool of test_runtime_gemm_and_linked_pool in dry run: the first exported window, and the run's stats."""
    NT, T, n, tb = 2, 128, 8, 64 * 1024
    data = P.Data(NT, T, seed=2)
    host = np.zeros(2 * n * tb // 4, np.int32)
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        ctx.link_bodies(ctx.devices[0], b"ptx", L.IMAGE_PTX, 0x01, gemm_windows=gemm_windows)
        tp, _ = P.insert(ctx, data)
        ids = insert_linked(ctx, tp, int32_collection(ctx, 2 * n, tb, host), n, -4, 11, 9)
        win = ctx.export_window(tp, ctx.devices[0])
        ctx.wait()
        st = ctx.stats(ctx.devices[0])
        t, dev = ctx.trace(tp)
    total = P.ntasks(NT) + 3 * n
    assert sorted(t.tolist()) == list(range(total)) and np.all(dev == 2)
    assert st["executed_tasks"] == total
    return win, st, ids, NT, n


def test_dry_run_gemm_and_linked_pool_is_one_window_with_the_flag():
    win, st, ids, NT, n = gemm_and_linked_pool(True)
    bodies = win["tasks"]["body"]
    assert np.count_nonzero(bodies == L.BODY_GEMM_BF16) == NT ** 3
    assert np.count_nonzero(bodies == L.BODY_LINKED_0) == n
    assert sorted(win["task_ids"].tolist()) == list(range(P.ntasks(NT) + 3 * n))
    assert st["windows_launched"] == 1


def test_dry_run_gemm_and_linked_pool_without_the_flag_is_unchanged():
    win, st, ids, NT, n = gemm_and_linked_pool(False)
    bodies = win["tasks"]["body"]
    assert np.count_nonzero(bodies == L.BODY_GEMM_BF16) == NT ** 3
    assert not np.any((bodies >= L.BODY_LINKED_0) & (bodies <= L.BODY_LINKED_7))
    assert st["windows_launched"] >= 2


# ----------------------------------------------------------------------------------------------------------------------
# the linked GEMM kernels
# ----------------------------------------------------------------------------------------------------------------------
def test_linked_gemm_kernels_keep_the_wgmma_pipeline():
    log = os.path.join(ROOT, "build", "linked_gemm_ptxas.log")
    cubin = os.path.join(ROOT, "build", "pb2_engine_linked_gemm.cubin")
    assert os.path.exists(log) and os.path.exists(cubin), "build() makes build/pb2_engine_linked_gemm.cubin"
    text = open(log).read()
    assert "C7509" not in text and "serialized" not in text
    assert len(re.findall(r"Compiling entry function '_ZN3pb223pb2_engine_gemm2_kernelI\w+Lb1EEEvNS_7Win2DevE'", text)) == 4
    # every kernel's own frame is spill-free: the new stack use is the out-of-line calls
    for name, frame in re.findall(r"Function properties for (_ZN3pb223pb2_engine_gemm2_kernel\w+)\n\s*(.*)", text):
        assert "0 bytes spill stores" in frame, (name, frame)
    sass = subprocess.check_output([os.path.join(CUDA, "bin", "cuobjdump"), "-sass", cubin], text=True)
    funcs = dict(re.findall(r"Function : (\S+)\n(.*?)(?=\n\s*\.{10,}|\n\t\tFunction :|\Z)", sass, re.S))
    holders = [f for f, body in funcs.items() if "HGMMA" in body]
    assert len(holders) == 1 and "consume_part_outlined" in holders[0], holders
    body = funcs[holders[0]]
    # pipelined: one wgmma group of four per k-block, waited on once (a serialized loop waits after every HGMMA)
    hg = [l for l in body.splitlines() if "HGMMA" in l]
    assert sum("gsb0" in l for l in hg) == len(hg) // 4, hg
    assert "CALL" not in body
    # local memory only in the prologue and epilogue that save and restore callee-saved registers, never between
    # the first and the last HGMMA
    lines = body.splitlines()
    first = next(i for i, l in enumerate(lines) if "HGMMA" in l)
    last = max(i for i, l in enumerate(lines) if "HGMMA" in l)
    assert not any(("STL" in l or "LDL" in l) for l in lines[first:last + 1])


@pytest.mark.parametrize("fixture", ["linked_bodies", "checked_bodies"])
def test_fixtures_link_with_the_linked_gemm_kernels(tmp_path, fixture):
    engine = [os.path.join(ROOT, "build", f) for f in ("pb2_engine_linked.cubin", "pb2_engine_linked_gemm.cubin")]
    bodies = os.path.join(ROOT, "tests", "cuda", fixture + ".cubin")
    assert all(os.path.exists(f) for f in engine + [bodies]), "build() makes the engine cubins and the fixtures"
    out = tmp_path / "linked.cubin"
    subprocess.check_call([os.path.join(CUDA, "bin", "nvlink"), "-arch=sm_90a", "-o", str(out), *engine, bodies])
    res = subprocess.check_output([os.path.join(CUDA, "bin", "cuobjdump"), "-res-usage", str(out)], text=True)
    kernels = re.findall(r"Function (_ZN3pb223pb2_engine_gemm2_kernelI\w+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+)", res)
    assert len(kernels) == 4, res
    for name, reg, stack, smem in kernels:
        # 168 registers (one 384-thread CTA per SM), and the static shared memory fits beside the 193 KiB operand ring
        assert int(reg) <= 168 and int(smem) + 4 * (16 + 32) * 1024 + 1024 <= 227 * 1024, (name, reg, stack, smem)
    hbm = re.findall(r"Function (_ZN3pb221pb2_engine_hbm_kernelI\w+):\s*\n\s*REG:(\d+)", res)
    assert len(hbm) == 4 and all(int(r) <= 80 for _, r in hbm)
