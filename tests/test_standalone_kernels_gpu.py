"""The two device entry points that run outside any engine window, against the NumPy reference (body_ref.py):
pb2_body_launch (the in-kernel bodies as one stand-alone launch, what a CUDA body runs under another device module) and
pb2_engine_copy_batch (the component's batched stage-in and write-back copies).  Every flow and copy sits in one
allocation between guard bytes that must come out unchanged.  The refusals are checked on the host and launch nothing."""
import ctypes as C
import itertools

import numpy as np
import pytest

import body_ref as R
from parsec_b200 import _lib as L

gpu = pytest.mark.gpu
GUARD = 64
SENTINEL = 0xA5


def lib():
    return L.load()


def c_array(ctype, values):
    return (ctype * max(len(values), 1))(*values)


def body_launch(stream, body, ptrs, nbytes, iparam=(0, 0, 0), fparam=0.0):
    p = c_array(C.c_void_p, ptrs)
    b = c_array(C.c_uint64, nbytes)
    ip = c_array(C.c_int32, iparam)
    return lib().pb2_body_launch(stream, body, len(ptrs), C.cast(p, C.c_void_p), C.cast(b, C.c_void_p),
                                 C.cast(ip, C.c_void_p), C.c_float(fparam))


def launch_errors(reset):
    v = C.c_uint64(0)
    assert lib().pb2_body_launch_errors(C.byref(v), reset) == L.PB2_SUCCESS
    return v.value


# ----------------------------------------------------------------------------------------------------------------------
# refusals (host side; the stand-alone launch is refused without a GPU, test_slot_alignment.py)
# ----------------------------------------------------------------------------------------------------------------------
@gpu
def test_copy_batch_refuses_copies_of_4_gib(engine):
    """Copies of 4 GiB or more (the copy loops index bytes with 32 bits) are refused before anything is allocated or
    launched: the pointers here are never dereferenced."""
    for sizes in ([1 << 32], [16, (1 << 32) + 5], [1 << 40, 0]):
        n = len(sizes)
        dst = np.arange(n, dtype=np.uint64) * np.uint64(4096) + np.uint64(0x10000)
        src = dst + np.uint64(1 << 20)
        b = np.array(sizes, np.uint64)
        rc = lib().pb2_engine_copy_batch(engine._h, dst.ctypes.data, src.ctypes.data, b.ctypes.data, n)
        assert rc == L.PB2_ERR_VALUE_OUT_OF_BOUNDS, sizes
    engine.synchronize()


# ----------------------------------------------------------------------------------------------------------------------
# pb2_body_launch
# ----------------------------------------------------------------------------------------------------------------------
def packed(flows):
    """One image holding the flows at 16-byte aligned offsets, each between GUARD sentinel bytes or more."""
    offs, o = [], GUARD
    for f in flows:
        offs.append(o)
        o = (o + len(f) + GUARD + 15) // 16 * 16
    img = np.full(o, SENTINEL, np.uint8)
    for off, f in zip(offs, flows):
        img[off:off + len(f)] = f
    return img, offs


def run_launch(engine, body, flows, iparam=(0, 0, 0), fparam=0.0):
    """The body over the flows in one allocation on the engine's stream; asserts the whole allocation equals what the
    reference makes of it.  Returns the reference's result."""
    img, offs = packed(flows)
    dev = engine.malloc(len(img))
    try:
        engine.h2d(dev, img)
        stream = lib().pb2_engine_get_stream(engine._h)
        rc = body_launch(stream, body, [dev + o for o in offs], [len(f) for f in flows], iparam, fparam)
        assert rc == L.PB2_SUCCESS
        engine.synchronize()
        got = engine.d2h(np.empty_like(img), dev)
        engine.synchronize()
    finally:
        engine.free(dev)
    want = img.copy()
    r = R.run_body(body, [want[o:o + len(f)] for o, f in zip(offs, flows)], iparam, fparam)
    diff = np.flatnonzero(got != want)
    assert not len(diff), f"body {body}: {len(diff)} bytes differ, first at {diff[0]} (flows at {offs})"
    return r


# one CTA, several, and the 1 056-CTA cap (32 KiB per CTA)
LAUNCH_SIZES = [17, 4096 + 12, 32768 - 4, 300000 + 12, (40 << 20) + 12]


def flows_for(rng, body, n):
    """Flow contents for body at n bytes (flow 1 of COPY and AXPY is 37 bytes longer, or 5 shorter at odd sizes)."""
    def ints(m):
        return rng.integers(0, 4, m, dtype=np.uint8)

    def floats(m):
        return np.concatenate([R.float_values(rng, m // 4).view(np.uint8), ints(m % 4)])

    if body == L.BODY_COPY:
        return [ints(n), ints(n + 37 if n % 2 else n - 5)]
    if body == L.BODY_AXPY_F32:
        m = n + 37 if n % 2 else n - 5
        x, y, _ = R.fma_pair_values(rng, max(n, m) // 4)
        return [np.concatenate([x.view(np.uint8), ints(n % 4)])[:n], np.concatenate([y.view(np.uint8), ints(m % 4)])[:m]]
    if body in (L.BODY_INCR_F32, L.BODY_CHECK_F32):
        return [floats(n)]
    return [ints(n)]


PARAMS = {L.BODY_FILL_I32: ((0x01020304, 0, 0), 0.0), L.BODY_CHECK_I32: ((0x01000000, 0, 0), 0.0),
          L.BODY_INCR_I32: ((-7, 0, 0), 0.0), L.BODY_ADD_IOTA_I32: ((0, 0, 0), 0.0),
          L.BODY_SCALE_I32: ((-3, 0, 0), 0.0), L.BODY_IOTA_I32: ((0, 0, 0), 0.0), L.BODY_COPY: ((0, 0, 0), 0.0),
          L.BODY_FILL_F32: ((0, 0, 0), R.bits_f32(R.QNAN)), L.BODY_CHECK_F32: ((0, 0, 0), -0.0),
          L.BODY_INCR_F32: ((0, 0, 0), -2.5), L.BODY_AXPY_F32: ((0, 0, 0), 1.3125),
          L.BODY_MEMSET_U8: ((0x1c3, 0, 0), 0.0), L.BODY_ADD_AT_I32: ((5, 11, 0), 0.0)}


@gpu
@pytest.mark.parametrize("n", LAUNCH_SIZES)
def test_body_launch_every_body(engine, n):
    rng = np.random.default_rng(n)
    launch_errors(reset=1)
    mismatches = 0
    for body, (ip, fp) in PARAMS.items():
        if body == L.BODY_AXPY_F32:
            _, _, fp = R.fma_pair_values(rng, 1)
        r = run_launch(engine, body, flows_for(rng, body, n), ip, float(fp))
        if body in R.CHECKS:
            mismatches += r >> 32
    assert mismatches > 0
    assert launch_errors(reset=0) == mismatches
    assert launch_errors(reset=1) == mismatches
    assert launch_errors(reset=0) == 0


@gpu
def test_body_launch_edges(engine):
    """ADD_AT at the first element, a 32 KiB boundary, the last element, the ragged tail and out of range; CHECK_F32 of
    -0.0 against +0.0; the float edge values under INCR_F32."""
    rng = np.random.default_rng(1)
    n = (40 << 10) + 3
    for at in (0, 8192, n // 4 - 1, n // 4, n // 4 + 100, -1, -(1 << 31)):
        run_launch(engine, L.BODY_ADD_AT_I32, [rng.integers(0, 256, n, dtype=np.uint8)], (at, 0x10001, 0))
    zeros = np.zeros(4096, np.float32)
    zeros[::3] = -0.0
    launch_errors(reset=1)
    r = run_launch(engine, L.BODY_CHECK_F32, [zeros.view(np.uint8)], fparam=0.0)
    assert r >> 32 == len(zeros[::3])
    assert launch_errors(reset=1) == r >> 32
    edge = np.array([0.0, -0.0, R.bits_f32(1), -R.bits_f32(0x7FFFFF), np.inf, -np.inf, 1.0], np.float32)
    for k in (0.0, -0.0, float(R.bits_f32(1)), -2.0):
        run_launch(engine, L.BODY_INCR_F32, [np.tile(edge, 1000).view(np.uint8)], fparam=k)


# ----------------------------------------------------------------------------------------------------------------------
# pb2_engine_copy_batch
# ----------------------------------------------------------------------------------------------------------------------
COPY_SIZES = [0, 1, 15, 16, 17, (1 << 20) + 3]
MISALIGN = [0, 4, 1]          # offset mod 16 of a region: 16-, 4- and 1-byte aligned


def regions(sizes, mis):
    """Offsets of regions of the given sizes at the given offsets mod 16, GUARD bytes or more apart; total bytes."""
    offs, o = [], GUARD
    for s, m in zip(sizes, mis):
        o = (o + 15) // 16 * 16 + m
        offs.append(o)
        o += s + GUARD
    return offs, o + GUARD


def copy_batch(engine, dst, src, nbytes):
    d, s, b = (np.array(v, np.uint64) for v in (dst, src, nbytes))
    rc = lib().pb2_engine_copy_batch(engine._h, d.ctypes.data, s.ctypes.data, b.ctypes.data, len(b))
    assert rc == L.PB2_SUCCESS
    engine.synchronize()


def check_batch(engine, direction, sizes, smis, dmis, seed):
    """One batch of copies from regions of a source image to regions of a destination image, each image on the device
    or in registered host memory as `direction` says; the destination must equal the expected image byte for byte."""
    rng = np.random.default_rng(seed)
    soffs, stotal = regions(sizes, smis)
    doffs, dtotal = regions(sizes, dmis)
    simg = rng.integers(0, 256, stotal, dtype=np.uint8)
    dimg = np.full(dtotal, SENTINEL, np.uint8)
    want = dimg.copy()
    for so, do, s in zip(soffs, doffs, sizes):
        want[do:do + s] = simg[so:so + s]
    hosted = []

    def place(img, on_host):
        if on_host:
            buf = img.copy()
            hosted.append(buf)
            return engine.host_register(buf), buf
        dev = engine.malloc(len(img))
        engine.h2d(dev, img)
        return dev, None

    sbase, _ = place(simg, direction == "h2d")
    dbase, dbuf = place(dimg, direction == "d2h")
    try:
        copy_batch(engine, [dbase + o for o in doffs], [sbase + o for o in soffs], sizes)
        got = dbuf.copy() if dbuf is not None else engine.d2h(np.empty_like(dimg), dbase)
        engine.synchronize()
    finally:
        for buf in hosted:
            engine.host_unregister(buf)
        for base, on_host in ((sbase, direction == "h2d"), (dbase, direction == "d2h")):
            if not on_host:
                engine.free(base)
    diff = np.flatnonzero(got != want)
    assert not len(diff), f"{direction}: {len(diff)} bytes differ, first at {diff[0]}"


@gpu
@pytest.mark.parametrize("direction", ["d2d", "h2d", "d2h"])
def test_copy_batch_alignments_and_sizes(engine, direction):
    """Every pair of source and destination alignments (16, 4, 1) at every size, in one batch smaller than the grid."""
    combos = list(itertools.product(MISALIGN, MISALIGN, COPY_SIZES))
    assert len(combos) < engine.info()["nworkers"]
    check_batch(engine, direction, [c[2] for c in combos], [c[0] for c in combos], [c[1] for c in combos], seed=len(direction))


@gpu
@pytest.mark.parametrize("direction", ["d2d", "h2d", "d2h"])
def test_copy_batch_larger_than_the_grid(engine, direction):
    """More copies than workers: the workers stride over the list."""
    n = engine.info()["nworkers"] * 2 + 37
    rng = np.random.default_rng(n)
    sizes = [int(v) for v in rng.integers(0, 300, n)]
    check_batch(engine, direction, sizes, [MISALIGN[i % 3] for i in range(n)], [MISALIGN[i // 3 % 3] for i in range(n)],
                seed=n)
