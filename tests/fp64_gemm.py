"""The fp64 DTD GEMM of the GEMM-worker body tests and of tools/ab_gemm_worker_bodies.py.

The DAG is the oracle's dtd_gemm (tests/dsl/dtd/dtd_test_simple_gemm.c: for i, j, k: C(i,j) += A(i,k) B(k,j)^T, the
last k pushed out) with its body rewritten to the DGEMM body of tests/cuda/gemm_worker_bodies.cu: fp64 tiles, A(i,k)
M x K, B(k,j) N x K and C(i,j) M x N, row-major, iparam = M, N, K.  The data is the reference's LCG (orc_lcg_tile,
seeds A 1789, B 1805, C 1901): tile (r, c) of a matrix is rows r.. and columns c.. of the generated global matrix."""
import ctypes as C
import os

import numpy as np

from oracle import orc
from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200 import runtime as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DGEMM, PROBE = L.BODY_LINKED_0, L.BODY_LINKED_0 + 1
GEMM_BODIES = 0x03                              # both fixture bodies are GEMM-worker bodies
SEEDS = {"A": 1789, "B": 1805, "C": 1901}
EPS = 2.0 ** -53                                # unit roundoff of float64


def image(fmt=L.IMAGE_CUBIN):
    ext = ".ptx" if fmt == L.IMAGE_PTX else ".cubin"
    path = os.path.join(ROOT, "tests", "cuda", "gemm_worker_bodies" + ext)
    assert os.path.exists(path), "build() makes " + path
    return open(path, "rb").read()


def lcg_tile(name, r0, c0, rows, cols, global_rows):
    """Rows r0 .. r0 + rows - 1 and columns c0 .. of the LCG matrix `name` (global_rows rows, column-major as the
    reference generates it), as a row-major float64 array."""
    buf = np.zeros((cols, rows), np.float32)
    orc.lib().orc_lcg_tile(buf.ctypes.data_as(C.c_void_p), r0, c0, rows, cols, global_rows, rows, SEEDS[name])
    return buf.T.astype(np.float64)


def dag(NT, M, N, K):
    """The fp64 dtd_gemm over NT x NT tiles of C; tile ids as dags.dtd_gemm.  Returns (dag, bytes of every tile)."""
    g = dags.dtd_gemm(NT, tile=M, elem_bytes=8)
    t = g.tasks.copy()
    t["body"] = DGEMM
    t["iparam"][:] = (M, N, K)
    sizes = np.array([M * K * 8] * NT * NT + [N * K * 8] * NT * NT + [M * N * 8] * NT * NT, np.int64)
    return dags.Dag(t, g.succ, g.ready, ntiles=3 * NT * NT, tile_bytes=0, kind=1, name="dtd_dgemm"), sizes


def tiles(NT, M, N, K):
    """Every tile's initial values, in tile-id order: A(i,k), B(k,j), C(i,j)."""
    a = [lcg_tile("A", i * M, k * K, M, K, NT * M) for i in range(NT) for k in range(NT)]
    b = [lcg_tile("B", j * N, k * K, N, K, NT * N) for k in range(NT) for j in range(NT)]
    c = [lcg_tile("C", i * M, j * N, M, N, NT * M) for i in range(NT) for j in range(NT)]
    return a + b + c


def reference(t, NT, i, j):
    """(C(i,j) after the chain, in float64 with NumPy, and the bound the GPU's C(i,j) must stay within).  Both sums
    are float64 sums of the same NT * K + 1 terms in different orders; each is within gamma_n (|C0| + sum |A| |B|^T)
    of the exact sum, gamma_n = n u / (1 - n u), n = NT * K + 1, so they differ by at most twice that."""
    c0 = t[2 * NT * NT + i * NT + j]
    acc, mag = c0.copy(), np.abs(c0)
    for k in range(NT):
        a, b = t[i * NT + k], t[NT * NT + k * NT + j]
        acc += a @ b.T
        mag += np.abs(a) @ np.abs(b).T
    n = NT * a.shape[1] + 1
    return acc, 2 * (n * EPS / (1 - n * EPS)) * mag


def insert(ctx, NT, M, N, K, t):
    """The pool on ctx as DTD tasks of one task class whose CUDA chore names DGEMM, over three block-cyclic collections
    on host buffers that hold the tiles of t (tile (m, n) at position n * NT + m).  Returns (taskpool, buffers)."""
    shapes = {"A": (M, K), "B": (N, K), "C": (M, N)}
    bufs, dcs = {}, {}
    for w, name in enumerate("ABC"):
        mb, nb = shapes[name]
        buf = np.zeros(NT * NT * mb * nb, np.float64)
        for m in range(NT):
            for n in range(NT):
                buf[(n * NT + m) * mb * nb:][:mb * nb] = t[w * NT * NT + m * NT + n].reshape(-1)
        bufs[name] = buf
        dcs[name] = ctx.block_cyclic(8, mb, nb, NT * mb, NT * nb, mat=buf)
    tp = C.c_void_p(ctx.l.pb2_dtd_taskpool_new(ctx.h))
    ops = np.array([R.INOUT] * 3, np.int32)
    tc = C.c_void_p(ctx.l.pb2_dtd_create_task_class(tp, b"DGEMM", 3, ops.ctypes.data_as(C.c_void_p)))
    assert ctx.l.pb2_dtd_task_class_add_chore(tp, tc, R.DEV_CUDA, DGEMM, None) == 0
    tile = lambda name, m, n: ctx.l.pb2_dtd_tile_of(tp, dcs[name], ctx.l.pb2_dc_data_key(dcs[name], m, n))
    keep = []
    for i in range(NT):
        for j in range(NT):
            for k in range(NT):
                last = k == NT - 1
                arr = (C.c_void_p * 3)(tile("A", i, k), tile("B", k, j), tile("C", i, j))
                o = np.array([R.INPUT, R.INPUT, (R.INOUT | R.PUSHOUT) if last else R.INOUT], np.int32)
                p = np.array([M, N, K], np.int32)
                keep.extend((arr, o, p))
                assert ctx.l.pb2_dtd_insert_task_with_task_class(tp, tc, 0, R.DEV_CUDA, arr, o.ctypes.data_as(C.c_void_p),
                                                                 p.ctypes.data_as(C.c_void_p), 0.0) >= 0
    return tp, bufs


def runtime_tile(bufs, name, m, n, NT, rows, cols):
    """Tile (m, n) of collection `name` in its host buffer, as a rows x cols array."""
    return bufs[name][(n * NT + m) * rows * cols:][:rows * cols].reshape(rows, cols)
