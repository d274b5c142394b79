"""Fused units of HBM windows: a producer and the read group that checks the tile it writes run as one unit, chunk by
chunk.  Every per-task output must be what the same window computes with fusion off, and what the sequential oracle
computes; the dependency order must hold on every edge."""
import numpy as np
import pytest

from parsec_b200 import _lib as L
from oracle import orc
from oracle import orc_dags as dags
from parsec_b200.engine import Engine

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engines():
    on, off = Engine(0), Engine(0, fuse_readers=-1)
    yield on, off
    on.close()
    off.close()


def sizes_of(dag, sizes):
    return np.full(dag.ntiles, dag.tile_bytes, np.int64) if sizes is None else np.asarray(sizes, np.int64)


def run_on(e, dag, host, valid, sizes=None, pushout_home=False):
    """One run of dag on engine e, tile i of sizes[i] bytes (default dag.tile_bytes) in a fresh slab: resident copies of
    its bytes in host, or staged in from there.  Returns (stats, results, device bytes, host bytes after the run)."""
    sz = sizes_of(dag, sizes)
    offs = np.concatenate([[0], np.cumsum(sz)[:-1]]).astype(np.uint64)
    slots = (sz + 511) // 512 * 512
    soffs = np.concatenate([[0], np.cumsum(slots)[:-1]]).astype(np.uint64)
    host = host.copy()
    slab = e.malloc(max(int(slots.sum()), 16))
    alias = e.host_register(host)
    tiles = np.zeros(dag.ntiles, L.TILE_DTYPE)
    tiles["dev_ptr"] = slab + soffs
    tiles["src_ptr"] = alias + offs
    tiles["bytes"] = sz
    tiles["state"] = L.TILE_VALID if valid else L.TILE_INVALID
    hb = host.view(np.uint8)
    if valid:
        for i in range(dag.ntiles):
            e.h2d(int(tiles["dev_ptr"][i]), hb[int(offs[i]):int(offs[i]) + int(sz[i])])
    w = e.window(0, dag.tasks, dag.succ, tiles, dag.ready)
    st = w.run()
    res = w.results()
    w.close()
    data = np.empty(int(sz.sum()), np.uint8)
    for i in range(dag.ntiles):
        e.d2h(data[int(offs[i]):int(offs[i]) + int(sz[i])], int(tiles["dev_ptr"][i]))
    e.host_unregister(host)
    e.free(slab)
    return st, res, data, host


def oracle(dag, host, sizes=None):
    """The sequential oracle's run of dag (FIFO ready order), every tile staged in from host."""
    sz = sizes_of(dag, sizes)
    spec = np.zeros(dag.ntiles, orc.TILE_DTYPE)
    spec["bytes"] = sz
    spec["src_ptr"] = np.concatenate([[0], np.cumsum(sz)[:-1]]).astype(np.uint64)
    spec["state"] = orc.TILE_INVALID
    h = host.copy()
    ref = orc.run_window(dag.tasks, dag.succ, spec, dag.ready, h)
    assert ref["rc"] == 0
    ref["data"] = np.concatenate([ref["device"][i][:int(sz[i])] for i in range(dag.ntiles)]) if dag.ntiles else np.zeros(0, np.uint8)
    ref["host"] = h
    return ref


def assert_same(a, b):
    (st_a, res_a, data_a, host_a), (st_b, res_b, data_b, host_b) = a, b
    assert np.array_equal(res_a["result"], res_b["result"])
    assert np.array_equal(res_a["seen_version"], res_b["seen_version"])
    assert np.array_equal(res_a["tiles"]["version"], res_b["tiles"]["version"])
    assert np.array_equal(res_a["tiles"]["state"], res_b["tiles"]["state"])
    assert np.array_equal(data_a, data_b)
    assert np.array_equal(host_a, host_b)
    for k in ("tasks_retired", "bytes_h2d", "stage_ins", "body_errors"):
        assert st_a[k] == st_b[k], k


def assert_oracle(run, ref, dag):
    st, res, data, _ = run
    assert np.array_equal(res["result"], ref["result"])
    assert np.array_equal(res["seen_version"], ref["seen_version"])
    assert np.array_equal(data, ref["data"])
    assert st["body_errors"] == ref["stats"]["body_errors"]
    assert st["tasks_retired"] == dag.ntasks
    assert all(v == 0 for v in dags.check_execution(dag, res).values())


def fused(res, p, members):
    """The members ran in p's unit: on p's worker, started right after p ended, in member order."""
    ss, es = res["start_seq"].astype(np.int64), res["end_seq"].astype(np.int64)
    return all(res["worker"][m] == res["worker"][p] and ss[m] == es[p] + 1 + i for i, m in enumerate(members))


def not_fused(res, p, members):
    """The group ran as a task of its own.  (A group popped from the ring by p's own worker right after p, with no other
    event in between, would look fused; with every worker polling the ring that does not happen.)"""
    return not fused(res, p, members)


def check_both(engines, dag, host, valid=False, sizes=None):
    on, off = engines
    a = run_on(on, dag, host, valid, sizes)
    b = run_on(off, dag, host, valid, sizes)
    assert_same(a, b)
    ref = oracle(dag, host, sizes)
    assert_oracle(a, ref, dag)
    assert_oracle(b, ref, dag)
    return a[1], b[1]


@pytest.mark.parametrize("valid", [False, True], ids=["staged", "resident"])
@pytest.mark.parametrize("K,NB,tile_bytes", [(8, 6, 4), (64, 14, 256 * 256 * 4), (33, 4, 1000), (1, 0, 16), (512, 14, 256 * 256 * 4)])
def test_ex05_fused_on_off_identical(engines, K, NB, tile_bytes, valid):
    dag = dags.ex05_broadcast(K, NB, tile_bytes)
    F = dag.meta["F"]
    host = np.full(K * tile_bytes // 4, -7, np.int32)
    on, off = check_both(engines, dag, host, valid)
    assert np.array_equal(on["result"][K:], np.repeat(np.arange(K, dtype=np.uint64), F))   # 0 mismatches, first element k
    if F >= 2:
        units = [(k, list(range(K + k * F, K + (k + 1) * F))) for k in range(K)]
        assert all(fused(on, k, m) for k, m in units)
        assert not all(fused(off, k, m) for k, m in units)


def readers_dag(producer_body, producer_k, reader_ks, tile_bytes, access=L.ACCESS_WRITE):
    """Task 0 writes tile 0 (FILL k / IOTA), tasks 1.. read it with CHECK constants reader_ks (ints: CHECK_I32, floats:
    CHECK_F32 with those bits)."""
    n = 1 + len(reader_ks)
    t = np.zeros(n, L.TASK_DTYPE)
    t["tile"][:] = -1
    t["nb_flows"] = 1
    t["tile"][:, 0] = 0
    t["body"][0], t["iparam"][0, 0], t["access"][0, 0] = producer_body, producer_k, access
    for i, k in enumerate(reader_ks, start=1):
        t["access"][i, 0] = L.ACCESS_READ
        t["dep_goal"][i] = 1
        if isinstance(k, float):
            t["body"][i], t["fparam"][i] = L.BODY_CHECK_F32, np.float32(k)
        else:
            t["body"][i], t["iparam"][i, 0] = L.BODY_CHECK_I32, k
    t["succ_begin"][0], t["succ_count"][0] = 0, n - 1
    t["succ_begin"][1:] = n - 1
    succ = np.arange(1, n, dtype=np.uint32)
    return dags.Dag(t, succ, np.array([0], np.int32), ntiles=1, tile_bytes=tile_bytes, name="readers")


f5 = float(np.array([5], np.int32).view(np.float32)[0])     # a CHECK_F32 constant whose bits are the integer 5
KS = [5, 5, 6, f5, 0, 7, 1, 5]


@pytest.mark.parametrize("producer", ["fill5", "iota"])
@pytest.mark.parametrize("tile_bytes,part_bytes", [(4096 + 12, 0), (40000, 0), (1 << 20, 64 * 1024)],
                         ids=["ragged16", "ragged_chunk", "wide_parts"])
def test_mismatches_inside_a_fused_group(producer, tile_bytes, part_bytes):
    """Members with different constants, some of which fail, checking what FILL or IOTA writes: tiles that are not a
    multiple of 16 bytes, not a multiple of the chunk, or split into 16 parts."""
    body, k = (L.BODY_FILL_I32, 5) if producer == "fill5" else (L.BODY_IOTA_I32, 0)
    dag = readers_dag(body, k, KS, tile_bytes)
    host = np.zeros(tile_bytes // 4, np.int32)
    with Engine(0, part_bytes=part_bytes) as on, Engine(0, part_bytes=part_bytes, fuse_readers=-1) as off:
        a, b = check_both((on, off), dag, host)
    assert a["result"][1:].any() and (a["result"][1:] >> np.uint64(32)).any()
    assert fused(a, 0, list(range(1, 9)))
    assert not_fused(b, 0, list(range(1, 9)))


@pytest.mark.parametrize("chunk", [16, 4096 + 48])
def test_chunk_sizes(engines, monkeypatch, chunk):
    """A 16-byte chunk, and a chunk that does not divide the slice, give the same results."""
    monkeypatch.setenv("PB2_FUSE_CHUNK_BYTES", str(chunk))
    with Engine(0) as e:
        for body, k, tb in ((L.BODY_IOTA_I32, 0, 4096 + 12), (L.BODY_FILL_I32, 5, 40000)):
            dag = readers_dag(body, k, KS, tb)
            host = np.zeros(tb // 4, np.int32)
            a = run_on(e, dag, host, False)
            assert_same(a, run_on(engines[1], dag, host, False))
            assert_oracle(a, oracle(dag, host), dag)
            assert fused(a[1], 0, list(range(1, 9)))
        dag = dags.ex05_broadcast(16, 14, 4096 + 16)
        host = np.full(16 * (4096 + 16) // 4, -7, np.int32)
        a = run_on(e, dag, host, True)
        assert_same(a, run_on(engines[1], dag, host, True))
        assert_oracle(a, oracle(dag, host), dag)


def around_dag(mask):
    """P fills tile 0; its out-edges are [X0, R1, R2, X, R3, R4] with X0, X NOPs: {R1, R2} is fused with P, {R3, R4}
    (a second group on the same tile) runs on its own.  R2 has a successor of its own, S (INCR on tile 1), and so does
    R4 (T, INCR on tile 2).  Counter or mask dependency words."""
    P, X0, R1, R2, X, R3, R4, S, T = range(9)
    t = np.zeros(9, L.TASK_DTYPE)
    t["tile"][:] = -1
    t["nb_flows"] = 1
    t["tile"][:, 0] = 0
    t["body"][P], t["iparam"][P, 0], t["access"][P, 0] = L.BODY_FILL_I32, 9, L.ACCESS_WRITE
    for r, k in ((R1, 9), (R2, 8), (R3, 9), (R4, 8)):
        t["body"][r], t["iparam"][r, 0], t["access"][r, 0] = L.BODY_CHECK_I32, k, L.ACCESS_READ
    for x in (X0, X):
        t["body"][x], t["nb_flows"][x], t["tile"][x, 0] = L.BODY_NOP, 0, -1
    t["body"][S], t["iparam"][S, 0], t["tile"][S, 0], t["access"][S, 0] = L.BODY_INCR_I32, 3, 1, L.ACCESS_RW
    t["body"][T], t["iparam"][T, 0], t["tile"][T, 0], t["access"][T, 0] = L.BODY_INCR_I32, 4, 2, L.ACCESS_RW
    src = [P, P, P, P, P, P, R2, R4]
    dst = [X0, R1, R2, X, R3, R4, S, T]
    begin, count, succ = dags._csr_from_edges(9, src, dst, np.zeros(8, np.int64))
    t["succ_begin"], t["succ_count"] = begin, count
    if mask:
        t["flags"] = L.TASK_DEPS_MASK
        t["dep_goal"] = 0x1
    else:
        t["dep_goal"] = 1
    t["dep_goal"][P] = 0
    return dags.Dag(t, succ, np.array([P], np.int32), ntiles=3, tile_bytes=1024, name="around")


@pytest.mark.parametrize("mask", [False, True], ids=["counter", "mask"])
def test_other_successors_and_a_second_group(engines, mask):
    dag = around_dag(mask)
    host = np.arange(3 * 256, dtype=np.int32)
    on, off = check_both(engines, dag, host)
    assert fused(on, 0, [2, 3])
    assert not_fused(on, 0, [5, 6]) and on["worker"][5] == on["worker"][6]
    assert not_fused(off, 0, [2, 3])


def copy_dag(tile_bytes):
    """P copies tile 0 (read) into tile 1 (written, flow 1); eight readers check tile 1."""
    dag = readers_dag(L.BODY_COPY, 0, KS, tile_bytes)
    t = dag.tasks
    t["nb_flows"][0] = 2
    t["access"][0, 0], t["access"][0, 1] = L.ACCESS_READ, L.ACCESS_WRITE
    t["tile"][0, 1] = 1
    t["tile"][1:, 0] = 1
    return dags.Dag(t, dag.succ, dag.ready, ntiles=2, tile_bytes=tile_bytes, name="copy")


def test_two_flow_producer(engines):
    tb = 40000
    dag = copy_dag(tb)
    host = np.concatenate([np.full(tb // 4, 5, np.int32), np.zeros(tb // 4, np.int32)])
    host[17] = 6
    on, off = check_both(engines, dag, host)
    assert fused(on, 0, list(range(1, 9)))


def test_not_fused_when_the_read_tile_is_not_the_widest(engines):
    """P fills tile 1 while it also reads the wider tile 0: its parts follow tile 0, so its group runs on its own."""
    dag = copy_dag(4096)
    t = dag.tasks
    t["body"][0], t["iparam"][0, 0] = L.BODY_FILL_I32, 5
    t["tile"][0, 0], t["tile"][0, 1] = 1, 0
    t["access"][0, 0], t["access"][0, 1] = L.ACCESS_WRITE, L.ACCESS_READ
    sizes = [8192, 4096]
    host = np.zeros((8192 + 4096) // 4, np.int32)
    on, _ = check_both(engines, dag, host, sizes=sizes)
    assert not_fused(on, 0, list(range(1, 9)))


def test_not_fused_with_pushout(engines):
    dag = readers_dag(L.BODY_FILL_I32, 5, KS, 4096, access=L.ACCESS_WRITE | L.FLOW_PUSHOUT)
    host = np.zeros(1024, np.int32)
    on, _ = check_both(engines, dag, host)
    assert not_fused(on, 0, list(range(1, 9)))


def test_not_fused_without_read_groups():
    dag = readers_dag(L.BODY_FILL_I32, 5, KS, 4096)
    host = np.zeros(1024, np.int32)
    with Engine(0, read_groups=-1) as e:
        st, res, data, _ = run_on(e, dag, host, False)
    assert_oracle((st, res, data, None), oracle(dag, host), dag)
    assert not_fused(res, 0, list(range(1, 9)))


def test_single_worker_keeps_fifo_order():
    """With one worker nothing is fused: two producers retire before their readers, as the oracle's FIFO has it."""
    dag = dags.ex05_broadcast(8, 6, 4096)
    host = np.full(8 * 1024, -7, np.int32)
    ref = oracle(dag, host)
    with Engine(0, max_workers=1) as e:
        run = run_on(e, dag, host, False)
    assert_oracle(run, ref, dag)
    assert np.array_equal(run[1]["retire_order"], ref["retire_order"])
