"""GPU tests of the tensor-core GEMM windows (BASELINE config 3 shape, reduced NT): fused k-chains (mode 0), every
task its own unit (mode 2) and its alias (mode 1)."""
import numpy as np
import pytest

from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200.bf16 import bf16_bits_to_f32, f32_to_bf16_bits, round_to_bf16
from parsec_b200.engine import Engine

pytestmark = pytest.mark.gpu


def chain_references(A, B, C, NT):
    """Per C(i,j): (a) the per-task semantics C <- bf16(f32(C) + A(i,k) B(k,j)^T) for k = 0..NT-1 (what the oracle and
    the unfused kernels compute), (b) the exact chain C0 + sum_k A B^T rounded once (what the fused kernel computes),
    (c) the largest magnitude along the chain (scale of the tolerance)."""
    per_task, exact, mag = np.empty_like(C), np.empty_like(C), np.empty_like(C)
    for i in range(NT):
        for j in range(NT):
            c = C[i, j].copy(); acc = C[i, j].astype(np.float64); m = np.abs(c)
            for k in range(NT):
                p = A[i, k].astype(np.float32) @ B[k, j].astype(np.float32).T
                c = round_to_bf16(c + p); acc = acc + p.astype(np.float64)
                m = np.maximum(m, np.maximum(np.abs(c), np.abs(acc).astype(np.float32)))
            per_task[i, j], exact[i, j], mag[i, j] = c, round_to_bf16(acc.astype(np.float32)), m
    return per_task, exact, mag


@pytest.mark.parametrize("mode", [0, 2, 1])
# 264: N % 16 == 8; 1152: 45 sub-tiles of 128 x 256 over 32 parts (13 parts run two); 1160: both
@pytest.mark.parametrize("NT,T", [(1, 128), (2, 256), (3, 512), (2, 320), (4, 512), (2, 768), (2, 1024),
                                  (2, 264), (2, 1152), (2, 1160)])
def test_dtd_gemm_chain(mode, NT, T):
    rng = np.random.default_rng(1789 + NT * 1000 + T)
    rnd = lambda shape: round_to_bf16(rng.uniform(-0.5, 0.5, shape).astype(np.float32))
    A, B, C = rnd((NT, NT, T, T)), rnd((NT, NT, T, T)), rnd((NT, NT, T, T))
    dag = dags.dtd_gemm(NT, T)
    tb = T * T * 2
    host = np.concatenate([f32_to_bf16_bits(A).ravel(), f32_to_bf16_bits(B).ravel(), f32_to_bf16_bits(C).ravel()])
    with Engine(0, gemm_mode=mode, timeout_ms=4000) as engine:
        slab = engine.malloc(dag.ntiles * tb)
        alias = engine.host_register(host)
        tiles = np.zeros(dag.ntiles, L.TILE_DTYPE)
        tiles["dev_ptr"] = slab + np.arange(dag.ntiles, dtype=np.uint64) * np.uint64(tb)
        tiles["src_ptr"] = alias + np.arange(dag.ntiles, dtype=np.uint64) * np.uint64(tb)
        tiles["bytes"] = tb
        w = engine.window(1, dag.tasks, dag.succ, tiles, dag.ready)
        st = w.run()
        res = w.results()
        w.close()
        engine.host_unregister(host)
    assert st["tasks_retired"] == NT ** 3
    assert all(v == 0 for v in dags.check_execution(dag, res).values())
    assert st["bytes_h2d"] == dag.ntiles * tb and st["bytes_d2h"] == NT * NT * tb
    # every C(i,j) chain ran in k order: task (i,j,k) saw version k of C
    assert np.array_equal(res["seen_version"][:, 2], np.tile(np.arange(NT), NT * NT))
    assert np.all(res["tiles"]["version"][2 * NT * NT:] == NT)
    got = bf16_bits_to_f32(host[2 * NT * NT * T * T:]).reshape(NT, NT, T, T)   # pushed out on the last k
    per_task, exact, mag = chain_references(A, B, C, NT)
    ref = exact if mode == 0 else per_task
    # tolerance: one bf16 ulp (at most 2^-7 relative) of the largest magnitude along the chain PER ROUNDING: the tensor
    # core's fp32 accumulation order differs from numpy's, which can flip a rounding to the neighbouring bf16 value.
    # Mode 0 keeps the accumulator in registers for the whole chain (one rounding, compared with the singly-rounded exact
    # sum); the per-task modes round once per task of the k-chain, so NT flips can add up.
    tol = (1 if mode == 0 else NT) * 2.0 ** -7 * np.maximum(mag, 1.0)
    bad = np.abs(got - ref) > tol
    assert not bad.any(), f"mode {mode}: {bad.sum()} / {bad.size} out of tolerance, max err {np.abs(got - ref).max()}"
