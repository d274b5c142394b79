"""The mixed DTD task pool of the stand-alone runtime's mixed-window tests and of tools/ab_mixed_windows.py.

For every C tile (i, j) of an NT x NT grid of T x T bf16 tiles, inserted in this order:
  FILL_I32  C(i,j) = pairs of bf16 1.0                                      (OUTPUT)
  GEMM      C(i,j) += A(i,k) B(k,j)^T, k = 0 .. NT-1, the last one pushed out (INOUT)
  CHECK_I32 C(i,j) against the FILL pattern                                 (INPUT)
  AXPY_F32  Y(i,j) += ALPHA * X(i,j), pushed out                            (X INPUT, Y INOUT)
X and Y are fp32 tiles of the same byte size as C.  The FILL and AXPY tasks have no predecessor; everything else is
released by a task of the pool.  A, B, C, X, Y are 2D block-cyclic collections over one host buffer (`Data.host`)."""
import ctypes as C

import numpy as np

from parsec_b200 import _lib as L
from parsec_b200 import runtime as R
from parsec_b200.bf16 import f32_to_bf16_bits

ONES = 0x3F803F80          # FILL_I32 pattern of the C tiles: two bf16 1.0
ALPHA = 2.0
NAMES = ("A", "B", "C", "X", "Y")


class Data:
    """The five matrices, tile after tile in one host buffer.  Tile (m, n) of a matrix sits at tile position n * NT + m
    (the block-cyclic layout of one rank)."""

    def __init__(self, NT, T, seed=0):
        self.NT, self.T = NT, T
        self.tile_bytes = T * T * 2
        self.mat_bytes = NT * NT * self.tile_bytes
        self.host = np.zeros(len(NAMES) * self.mat_bytes, np.uint8)
        rng = np.random.default_rng(seed)
        for name in ("A", "B"):
            vals = rng.uniform(-1.0, 1.0, NT * NT * T * T).astype(np.float32)
            self.view(name)[:] = f32_to_bf16_bits(vals).view(np.uint8)
        self.view("C")[:] = 0xFF                                  # overwritten by FILL before any GEMM reads it
        for name in ("X", "Y"):                                   # small integers: AXPY with ALPHA = 2 is exact
            self.view(name).view(np.float32)[:] = rng.integers(-1000, 1000, self.mat_bytes // 4).astype(np.float32)

    def view(self, name):
        i = NAMES.index(name)
        return self.host[i * self.mat_bytes:(i + 1) * self.mat_bytes]

    def tile(self, name, m, n):
        o = (n * self.NT + m) * self.tile_bytes
        return self.view(name)[o:o + self.tile_bytes]


def collections(ctx, data):
    """The five block-cyclic collections over `data` on `ctx`."""
    NT, T = data.NT, data.T
    dcs = {}
    for name in NAMES:
        elt = 4 if name in ("X", "Y") else 2
        cols = T * 2 // elt                                       # every tile holds tile_bytes bytes
        dcs[name] = ctx.block_cyclic(elt, T, cols, NT * T, NT * cols, mat=data.view(name))
    return dcs


def insert(ctx, data, dcs=None):
    """Builds the pool on `ctx` over `data` (over the collections `dcs` when given, so that a pool built again finds
    its tiles where the previous one left them); returns (taskpool, ids) with ids[(kind, i, j[, k])] = pool task id."""
    NT, T = data.NT, data.T
    dcs = dcs or collections(ctx, data)
    tp = C.c_void_p(ctx.l.pb2_dtd_taskpool_new(ctx.h))

    def klass(name, nf, body):
        ops = np.array([R.INOUT] * nf, np.int32)
        tc = C.c_void_p(ctx.l.pb2_dtd_create_task_class(tp, name, nf, ops.ctypes.data_as(C.c_void_p)))
        assert ctx.l.pb2_dtd_task_class_add_chore(tp, tc, R.DEV_CUDA, body, None) == 0
        return tc

    fill, gemm = klass(b"FILL", 1, L.BODY_FILL_I32), klass(b"GEMM", 3, L.BODY_GEMM_BF16)
    check, axpy = klass(b"CHECK", 1, L.BODY_CHECK_I32), klass(b"AXPY", 2, L.BODY_AXPY_F32)
    tile = lambda name, m, n: ctx.l.pb2_dtd_tile_of(tp, dcs[name], ctx.l.pb2_dc_data_key(dcs[name], m, n))
    i32 = lambda *v: np.array(v, np.int32)
    keep, ids = [], {}

    def put(key, tc, tiles, ops, iparam=(0, 0, 0), fparam=0.0):
        arr = (C.c_void_p * len(tiles))(*tiles)
        o, p = i32(*ops), i32(*iparam)
        keep.extend((arr, o, p))
        ids[key] = ctx.l.pb2_dtd_insert_task_with_task_class(tp, tc, 0, R.DEV_CUDA, arr, o.ctypes.data_as(C.c_void_p),
                                                             p.ctypes.data_as(C.c_void_p), fparam)
        assert ids[key] >= 0

    for i in range(NT):
        for j in range(NT):
            c = tile("C", i, j)
            put(("fill", i, j), fill, [c], [R.OUTPUT], (ONES, 0, 0))
            for k in range(NT):
                last = k == NT - 1
                put(("gemm", i, j, k), gemm, [tile("A", i, k), tile("B", k, j), c],
                    [R.INPUT, R.INPUT, (R.INOUT | R.PUSHOUT) if last else R.INOUT], (T, T, T))
            put(("check", i, j), check, [c], [R.INPUT], (ONES, 0, 0))
            put(("axpy", i, j), axpy, [tile("X", i, j), tile("Y", i, j)], [R.INPUT, R.INOUT | R.PUSHOUT], fparam=ALPHA)
    return tp, ids


def ntasks(NT):
    return NT * NT * (NT + 3)


def nready(NT):
    return 2 * NT * NT
