"""Application device bodies linked into HBM windows (include/pb2_device_body.h, pb2_engine_link_bodies), host side.

  - pb2_body_args_t as gcc lays it out is the engine's BodyArgs (nvcc) and BODY_ARGS_DTYPE;
  - the link calls refuse a NULL or empty image, an unknown format and mask bits above bit 7, and a module links once;
  - a DTD chore naming a linked body is refused until every GPU module has linked an image;
  - the stand-alone runtime never puts GEMM tasks and linked-body tasks into one window.
The GPU side is tests/test_linked_bodies_gpu.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from parsec_b200 import _lib as L
from parsec_b200 import runtime as R
import mixed_pool as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FIELDS = ("flow", "bytes", "elem0", "part", "iparam", "fparam")


def layout(tmp_path, compiler, source, name):
    """sizeof, then offsetof each of FIELDS, of the struct `name` as a host program built by `compiler` prints them."""
    src = tmp_path / ("layout" + (".cu" if compiler == NVCC else ".c"))
    body = "".join('printf(" %%zu", (size_t)offsetof(%s, %s));' % (name, f) for f in FIELDS)
    src.write_text(source + '\n#include <stdio.h>\n#include <stddef.h>\nint main(void) { printf("%%zu", sizeof(%s)); %s return 0; }\n'
                   % (name, body))
    exe = tmp_path / "layout"
    arch = ["-gencode", "arch=compute_90a,code=sm_90a"] if compiler == NVCC else []
    subprocess.check_call([compiler, *arch, "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    return [int(v) for v in subprocess.check_output([str(exe)]).split()]


def test_body_args_layout(tmp_path):
    want = [L.BODY_ARGS_DTYPE.itemsize] + [L.BODY_ARGS_DTYPE.fields[f][1] for f in FIELDS]
    assert want == [72, 0, 32, 48, 52, 56, 68]
    assert layout(tmp_path, "gcc", '#include "pb2_device_body.h"', "pb2_body_args_t") == want
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not found: BodyArgs is checked against pb2_body_args_t by a static_assert in the build")
    assert layout(tmp_path, NVCC, '#include "%s/parsec_b200/csrc/pb2_sched.cuh"\nusing pb2::BodyArgs;' % ROOT, "BodyArgs") == want


def test_engine_link_refuses_a_null_engine():
    lib = L.load()
    assert lib.pb2_engine_link_bodies(None, b"x", 1, L.IMAGE_PTX, 0) == L.PB2_ERR_BAD_PARAM
    assert lib.pb2_engine_linked_info(None, None, None, None, None) == L.PB2_ERR_BAD_PARAM


@pytest.mark.parametrize("image,nbytes,fmt,mask", [
    (None, 16, L.IMAGE_PTX, 0),               # NULL image
    (b"x", 0, L.IMAGE_CUBIN, 0),              # empty image
    (b"x", 1, 0, 0),                          # unknown formats
    (b"x", 1, 3, 0),
    (b"x", 1, L.IMAGE_PTX, 0x100),            # a ninth body id
    (b"x", 1, L.IMAGE_CUBIN, 0xFFFFFFFF),
], ids=["null", "empty", "format0", "format3", "mask_bit8", "mask_all"])
def test_device_link_argument_checks(image, nbytes, fmt, mask):
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        assert ctx.l.pb2_device_link_bodies(ctx.devices[0], image, nbytes, fmt, mask) == L.PB2_ERR_BAD_PARAM
        # nothing was recorded: a valid call still links, a second one is refused
        assert ctx.l.pb2_device_link_bodies(ctx.devices[0], b"x", 1, L.IMAGE_PTX, 0xFF) == 0
        assert ctx.l.pb2_device_link_bodies(ctx.devices[0], b"x", 1, L.IMAGE_PTX, 0) == L.PB2_ERR_EXISTS


def linked_class(ctx, tp, body, nflows):
    """A DTD task class of nflows INOUT flows whose CUDA chore is `body`; returns (rc of add_chore, class)."""
    ops = np.array([R.INOUT] * nflows, np.int32)
    tc = C.c_void_p(ctx.l.pb2_dtd_create_task_class(tp, b"LINKED", nflows, ops.ctypes.data_as(C.c_void_p)))
    return ctx.l.pb2_dtd_task_class_add_chore(tp, tc, R.DEV_CUDA, body, None), tc


def test_linked_chore_needs_an_image_on_every_gpu_module():
    with R.Context(cuda_devices=(0, 1), dry_run=True) as ctx:
        tp = C.c_void_p(ctx.l.pb2_dtd_taskpool_new(ctx.h))
        for body in (L.BODY_LINKED_0, L.BODY_LINKED_7):
            assert linked_class(ctx, tp, body, 2)[0] == L.PB2_ERR_NOT_SUPPORTED
        ctx.link_bodies(ctx.devices[0], b"ptx", L.IMAGE_PTX)
        assert linked_class(ctx, tp, L.BODY_LINKED_0, 2)[0] == L.PB2_ERR_NOT_SUPPORTED     # module 1 has none yet
        ctx.link_bodies(ctx.devices[1], b"cubin", L.IMAGE_CUBIN, 0x01)
        for body in (L.BODY_LINKED_0, L.BODY_LINKED_7):
            assert linked_class(ctx, tp, body, 2)[0] == 0
        assert linked_class(ctx, tp, L.BODY_FILL_I32, 1)[0] == 0                        # built-in bodies as before
        ctx.l.pb2_taskpool_free(tp)


def insert_linked(ctx, tp, dc, n, m, b, k, pushout=True):
    """Into pool tp over the int32 collection dc of 2n tiles: for i < n, FILL X_i = k; LINKED_0 (y = m x + b) from X_i
    into Y_i (pushed out); CHECK Y_i against m k + b.  X_i is tile i, Y_i tile n + i.  Returns the pool ids by kind."""
    fill = linked_class(ctx, tp, L.BODY_FILL_I32, 1)[1]
    check = linked_class(ctx, tp, L.BODY_CHECK_I32, 1)[1]
    rc, axpb = linked_class(ctx, tp, L.BODY_LINKED_0, 2)
    assert rc == 0
    tile = lambda i: ctx.l.pb2_dtd_tile_of(tp, dc, ctx.l.pb2_dc_data_key(dc, i, 0))
    ids, keep = {"fill": [], "axpb": [], "check": []}, []

    def put(kind, tc, tiles, ops, iparam):
        arr, o, p = (C.c_void_p * len(tiles))(*tiles), np.array(ops, np.int32), np.array(iparam, np.int32)
        keep.extend((arr, o, p))
        t = ctx.l.pb2_dtd_insert_task_with_task_class(tp, tc, 0, R.DEV_CUDA, arr, o.ctypes.data_as(C.c_void_p),
                                                      p.ctypes.data_as(C.c_void_p), 0.0)
        assert t >= 0
        ids[kind].append(t)

    y_op = (R.OUTPUT | R.PUSHOUT) if pushout else R.OUTPUT
    for i in range(n):
        put("fill", fill, [tile(i)], [R.OUTPUT], (k, 0, 0))
        put("axpb", axpb, [tile(i), tile(n + i)], [R.INPUT, y_op], (m, b, 0))
        put("check", check, [tile(n + i)], [R.INPUT], (np.int32(m * k + b), 0, 0))
    return ids


def int32_collection(ctx, ntiles, tile_bytes, host):
    """A 1-D collection of ntiles int32 tiles over host (tile i at byte i * tile_bytes)."""
    return ctx.block_cyclic(4, tile_bytes // 4, 1, ntiles * tile_bytes // 4, 1, mat=host)


def test_dry_run_windows_never_mix_gemm_and_linked_tasks():
    NT, T, n, tb = 2, 64, 4, 4096
    data = P.Data(NT, T)
    host = np.zeros(2 * n * tb // 4, np.int32)
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        ctx.link_bodies(ctx.devices[0], b"ptx", L.IMAGE_PTX, 0x01)
        tp, _ = P.insert(ctx, data)
        ids = insert_linked(ctx, tp, int32_collection(ctx, 2 * n, tb, host), n, 3, -7, 5)
        win = ctx.export_window(tp, ctx.devices[0])
        bodies = win["tasks"]["body"]
        # the closure of the ready tasks reaches GEMMs first: the linked tasks wait for a window of their own
        assert np.count_nonzero(bodies == L.BODY_GEMM_BF16) == NT ** 3
        assert not np.any((bodies >= L.BODY_LINKED_0) & (bodies <= L.BODY_LINKED_7))
        assert set(ids["fill"]) <= set(win["task_ids"].tolist())
        ctx.wait()
        st = ctx.stats(ctx.devices[0])
        t, dev = ctx.trace(tp)
    total = P.ntasks(NT) + 3 * n
    assert sorted(t.tolist()) == list(range(total)) and np.all(dev == 2)
    assert st["executed_tasks"] == total and st["windows_launched"] >= 2


def test_dry_run_linked_pool_is_one_window():
    n, tb = 6, 4096
    host = np.zeros(2 * n * tb // 4, np.int32)
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        ctx.link_bodies(ctx.devices[0], b"ptx", L.IMAGE_PTX, 0x01)
        tp = C.c_void_p(ctx.l.pb2_dtd_taskpool_new(ctx.h))
        ids = insert_linked(ctx, tp, int32_collection(ctx, 2 * n, tb, host), n, 3, -7, 5)
        win = ctx.export_window(tp, ctx.devices[0])
        assert sorted(win["task_ids"].tolist()) == sorted(sum(ids.values(), []))
        assert np.count_nonzero(win["tasks"]["body"] == L.BODY_LINKED_0) == n
        ctx.wait()
        st = ctx.stats(ctx.devices[0])
    assert st["windows_launched"] == 1 and st["executed_tasks"] == 3 * n
    assert st["tasks_released_on_device"] == 2 * n


def test_link_after_the_first_window_is_refused():
    n, tb = 2, 4096
    host = np.zeros(2 * n * tb // 4, np.int32)
    with R.Context(cuda_devices=(0,), dry_run=True) as ctx:
        tp = C.c_void_p(ctx.l.pb2_dtd_taskpool_new(ctx.h))
        fill = linked_class(ctx, tp, L.BODY_FILL_I32, 1)[1]
        dc = int32_collection(ctx, 2 * n, tb, host)
        arr, o, p = (C.c_void_p * 1)(ctx.l.pb2_dtd_tile_of(tp, dc, ctx.l.pb2_dc_data_key(dc, 0, 0))), np.array([R.OUTPUT], np.int32), np.zeros(3, np.int32)
        assert ctx.l.pb2_dtd_insert_task_with_task_class(tp, fill, 0, R.DEV_CUDA, arr, o.ctypes.data_as(C.c_void_p),
                                                         p.ctypes.data_as(C.c_void_p), 0.0) >= 0
        ctx.wait()
        assert ctx.stats(ctx.devices[0])["windows_launched"] == 1
        assert ctx.l.pb2_device_link_bodies(ctx.devices[0], b"x", 1, L.IMAGE_PTX, 0) == L.PB2_ERR_NOT_SUPPORTED
