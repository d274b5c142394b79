"""DAGs that put a small GEMM k-chain beside element-wise tasks in one GEMM window, for the tests of read groups in GEMM
windows (tests/test_gemm_groups.py, tests/test_gemm_groups_gpu.py) and tools/ab_gemm_groups.py.  Plain numpy over
oracle/orc_dags.py and parsec_b200/_lib.py: no test framework."""
import numpy as np

from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200.bf16 import f32_to_bf16_bits

MNK = 128                                   # the chain's tiles: 128 x 128 bf16
# what two GEMMs of ones add to a zero C: 2 * 128 = 256.0, two bf16 per 32-bit word
C_WORD = int(np.array([256.0], np.float32).view(np.uint32)[0] >> 16) * 0x10001
C_READERS = (C_WORD, C_WORD, C_WORD + 1, C_WORD)


def with_gemm_chain(dag, nchain=2, readers=C_READERS, priority=0):
    """dag's tasks and tiles (ids unchanged), then a k-chain of nchain GEMMs C += A B^T on three new tiles A, B, C
    (ids dag.ntiles .. + 2, 128^3), then CHECK_I32 readers of C with the constants `readers`, released by the chain's
    last GEMM, as one kind-1 DAG.  The new tasks carry `priority`."""
    n0, T = dag.ntasks, dag.ntiles
    n = n0 + nchain + len(readers)
    t = np.zeros(n, L.TASK_DTYPE)
    t[:n0] = dag.tasks
    t["tile"][n0:] = -1
    src, dst, flow = [], [], []
    for u in range(n0):
        b, c = int(dag.tasks["succ_begin"][u]), int(dag.tasks["succ_count"][u])
        for s in dag.succ[b:b + c]:
            src.append(u); dst.append(int(s) & 0x07FFFFFF); flow.append(int(s) >> 27)
    for i in range(nchain):
        g = n0 + i
        t["body"][g], t["nb_flows"][g], t["iparam"][g] = L.BODY_GEMM_BF16, 3, (MNK, MNK, MNK)
        t["tile"][g, :3], t["access"][g, :3] = (T, T + 1, T + 2), (L.ACCESS_READ, L.ACCESS_READ, L.ACCESS_RW)
        t["dep_goal"][g], t["priority"][g] = (1 if i else 0), priority
        if i:
            src.append(g - 1); dst.append(g); flow.append(2)
    for j, k in enumerate(readers):
        r = n0 + nchain + j
        t["body"][r], t["nb_flows"][r], t["iparam"][r, 0] = L.BODY_CHECK_I32, 1, k
        t["tile"][r, 0], t["access"][r, 0], t["dep_goal"][r], t["priority"][r] = T + 2, L.ACCESS_READ, 1, priority
        src.append(n0 + nchain - 1); dst.append(r); flow.append(0)
    begin, count, succ = dags._csr_from_edges(n, np.array(src, np.int64), np.array(dst, np.int64), np.array(flow, np.int64))
    t["succ_begin"], t["succ_count"] = begin, count
    ready = np.concatenate([dag.ready, [n0]]).astype(np.int32)
    return dags.Dag(t, succ, ready, ntiles=T + 3, tile_bytes=dag.tile_bytes, kind=1, meta=dag.meta)


def ex05_beside_gemm(K, tile_bytes=256 * 1024, readers=C_READERS):
    """dags.ex05_broadcast(K) with with_gemm_chain's chain of two GEMMs and its readers.  Returns (dag, the Ex05 DAG
    alone, bytes per tile, the host image: the Ex05 tiles all -1, A and B bf16 ones, C zeros)."""
    ex = dags.ex05_broadcast(K, 14, tile_bytes)
    dag = with_gemm_chain(ex, readers=readers)
    ab = f32_to_bf16_bits(np.ones(MNK * MNK, np.float32)).view(np.uint8)
    sizes = [tile_bytes] * K + [MNK * MNK * 2] * 3
    host = np.concatenate([np.full(K * tile_bytes // 4, -1, np.int32).view(np.uint8), ab, ab,
                           np.zeros(MNK * MNK * 2, np.uint8)])
    return dag, ex, sizes, host
