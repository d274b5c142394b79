"""GPU parity tests of the L0 engine against known answers of the reference's own tests/examples."""
import numpy as np
import pytest

from parsec_b200 import _lib as L
from oracle import orc_dags as dags
from parsec_b200.engine import Engine
from window_harness import Layout, placed, run_engine

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("K,NB,tile_bytes", [(8, 6, 4), (64, 14, 256 * 256 * 4), (33, 4, 1000), (1, 0, 16)])
def test_ex05_broadcast(engine, K, NB, tile_bytes):
    """Ex05_Broadcast.jdf:33-39,53-57: every TaskRecv(k,n) observes k; each tile staged in exactly once."""
    dag = dags.ex05_broadcast(K, NB, tile_bytes)
    host = np.full(K * tile_bytes // 4, -7, np.int32)
    layout = Layout.packed(dag, host)
    st, res, dev, _, _, _ = run_engine(engine, dag, layout)
    assert st["tasks_retired"] == dag.ntasks
    assert st["body_errors"] == 0
    assert st["bytes_h2d"] == K * tile_bytes            # required_in == transferred: zero re-staging
    assert st["stage_ins"] == K
    assert all(v == 0 for v in dags.check_execution(dag, res).values())
    F = dag.meta["F"]
    recv = res["result"][K:]
    assert np.all((recv >> np.uint64(32)) == 0)
    assert np.array_equal((recv & np.uint64(0xFFFFFFFF)).astype(np.int64), np.repeat(np.arange(K), F))
    # versions: Bcast sees the staged-in v0 and writes v1; every Recv sees v1 (device_gpu.c:2148-2152)
    assert np.all(res["seen_version"][:K, 0] == 0)
    assert np.all(res["seen_version"][K:, 0] == 1)
    assert np.all(res["tiles"]["version"] == 1) and np.all(res["tiles"]["state"] == L.TILE_VALID)
    for k in (0, K - 1):
        assert np.all(layout.tile_bytes(dev, k).view(np.int32) == k)


@pytest.mark.parametrize("NB", [0, 1, 10, 999])
def test_ex02_chain(engine, NB):
    """Ex02_Chain.jdf:44-50: task k observes value k; final value NB (BASELINE config 1 known answer)."""
    dag = dags.ex02_chain(NB)
    layout = Layout.packed(dag)
    st, res, dev, _, _, _ = run_engine(engine, dag, layout)
    assert st["tasks_retired"] == NB + 1 and st["bytes_h2d"] == 0
    assert all(v == 0 for v in dags.check_execution(dag, res).values())
    assert np.array_equal(res["retire_order"], np.arange(NB + 1))      # strictly serial chain
    assert np.array_equal(res["seen_version"][:, 0], np.arange(NB + 1))
    assert layout.tile_bytes(dev, 0).view(np.int32)[0] == NB


def test_single_worker_is_fifo_deterministic():
    """With one worker the ring is a strict FIFO: execution order is exactly breadth-first."""
    with Engine(0, max_workers=1) as e:
        dag = dags.ex05_broadcast(16, 6, 64)
        res = run_engine(e, dag, Layout.packed(dag, np.zeros(16 * 16, np.int32))).res
        assert np.array_equal(res["retire_order"], np.arange(dag.ntasks))
        assert np.all(res["worker"] == 0)


def test_rtt_chain_pushout(engine):
    """rtt.jdf:26-47 on one GPU: T += 1 along NT hops per fragment, final tile written back home."""
    NT, FRAGS, tb = 50, 4, 4096 * 4
    dag = dags.rtt_chain(NT, FRAGS, tb)
    host = np.arange(FRAGS * tb // 4, dtype=np.float32)
    expect = host + NT
    st, res, _, got, _, _ = run_engine(engine, dag, Layout.packed(dag, host))
    assert all(v == 0 for v in dags.check_execution(dag, res).values())
    assert st["bytes_h2d"] == FRAGS * tb and st["bytes_d2h"] == FRAGS * tb
    assert np.array_equal(got.view(np.float32), expect)                   # pushout landed in host memory
    assert np.all(res["tiles"]["version"] == NT)


def test_ep_schedmicro_shape(engine):
    """ep.jdf (schedmicro): NT x DEPTH empty CTL-chained tasks all retire, order respected."""
    dag = dags.ep(512, 8)
    st, res, _, _, _, _ = run_engine(engine, dag, Layout.packed(dag))
    assert st["tasks_retired"] == 1 + 512 * 8
    assert all(v == 0 for v in dags.check_execution(dag, res).values())


def test_malformed_dag_trips_watchdog():
    """A dependency goal that can never be met must abort the window, not hang the GPU."""
    with Engine(0, timeout_ms=200) as e:
        dag = dags.ex02_chain(4)
        dag.tasks["dep_goal"][2] = 0x3          # waits for a flow bit nobody sets
        with placed(e, Layout.packed(dag)) as p:
            w = e.window(0, dag.tasks, dag.succ, p.tiles, dag.ready)
            w.launch()
            with pytest.raises(L.Pb2Error) as ei:
                w.wait()
            assert ei.value.rc == L.PB2_ERR_DEVICE
            assert w.stats["tasks_retired"] == 2
            w.close()


@pytest.mark.parametrize("tile_bytes,part_bytes", [(1 << 20, 64 * 1024), ((1 << 20) + 4, 100 * 1000), (4 << 20, 0), (40, 16)])
def test_wide_tasks_match_oracle(tile_bytes, part_bytes):
    """Tasks on large tiles run as parts (byte slices) on many workers: every body, the pushout, the versions and
    the CHECK results are bit-identical to the oracle's sequential run."""
    from oracle import orc
    n = tile_bytes // 4
    t = np.zeros(9, L.TASK_DTYPE)
    t["tile"][:] = -1
    t["nb_flows"] = 1
    t["tile"][:, 0] = 0
    t["access"][:, 0] = L.ACCESS_RW
    t["dep_goal"] = 1
    t["dep_goal"][0] = 0
    seq = [(L.BODY_IOTA_I32, 0, 0), (L.BODY_ADD_IOTA_I32, 0, 0), (L.BODY_SCALE_I32, 3, 0), (L.BODY_INCR_I32, -7, 0),
           (L.BODY_ADD_AT_I32, n - 1, 1000), (L.BODY_ADD_AT_I32, n // 2, 77), (L.BODY_CHECK_I32, 5, 0),
           (L.BODY_COPY, 0, 0), (L.BODY_CHECK_I32, 123, 0)]
    for i, (b, p0, p1) in enumerate(seq):
        t["body"][i], t["iparam"][i, 0], t["iparam"][i, 1] = b, p0, p1
    t["access"][0, 0] = L.ACCESS_WRITE
    t["access"][6, 0] = L.ACCESS_READ
    t["nb_flows"][7] = 2; t["tile"][7, 1] = 1; t["access"][7, 0] = L.ACCESS_READ; t["access"][7, 1] = L.ACCESS_WRITE | L.FLOW_PUSHOUT
    t["tile"][8, 0] = 1; t["access"][8, 0] = L.ACCESS_READ
    t["succ_begin"] = np.arange(9); t["succ_count"] = 1; t["succ_count"][8] = 0
    succ = np.arange(1, 9, dtype=np.uint32)
    host = np.full(2 * n, 123, np.int32)
    ohost = host.copy()
    spec = np.zeros(2, orc.TILE_DTYPE); spec["bytes"] = tile_bytes; spec["src_ptr"] = [0, tile_bytes]
    spec["state"] = [orc.TILE_VALID, orc.TILE_INVALID]
    ref = orc.run_window(t, succ, spec, np.array([0], np.int32), ohost)
    assert ref["rc"] == 0
    with Engine(0, part_bytes=part_bytes) as e:
        slab = e.malloc(2 * tile_bytes + 1024)
        alias = e.host_register(host)
        tiles = np.zeros(2, L.TILE_DTYPE)
        tiles["dev_ptr"] = [slab, slab + (tile_bytes + 511) // 512 * 512]
        tiles["src_ptr"] = [alias, alias + tile_bytes]
        tiles["bytes"] = tile_bytes
        tiles["state"] = [L.TILE_VALID, L.TILE_INVALID]
        w = e.window(0, t, succ, tiles, np.array([0], np.int32))
        st = w.run(); res = w.results(); w.close()
        got0 = np.empty(n, np.int32); e.d2h(got0, int(tiles["dev_ptr"][0]))
        e.host_unregister(host)
    assert np.array_equal(res["retire_order"], np.arange(9))
    assert np.array_equal(res["result"], ref["result"])
    assert np.array_equal(res["seen_version"], ref["seen_version"])
    assert np.array_equal(got0, ref["device"][0].view(np.int32)[:n])
    assert np.array_equal(host, ohost)                                   # pushout of tile 1, slice by slice
    assert st["body_errors"] == ref["stats"]["body_errors"] and st["bytes_d2h"] == tile_bytes
    assert st["bytes_h2d"] == ref["stats"]["bytes_h2d"]


@pytest.mark.parametrize("big,small,part_bytes", [(1 << 20, 1 << 20, 64 * 1024), ((1 << 20) + 20, 300 * 1000, 100 * 1000), (4 << 20, 64 * 1024, 0)])
def test_sliced_stage_in_of_wide_tiles(big, small, part_bytes):
    """Tiles larger than part_bytes that start INVALID are staged in slice by slice by the parts of their readers
    (each slice moved exactly once, also when two wide readers of the same version run at the same time and when a
    task is cut differently from the tile): bytes staged == tile bytes, values == oracle."""
    from oracle import orc
    nb, ns = big // 4, small // 4
    # tiles: 0 big (host, INVALID), 1 small (host, INVALID), 2 big scratch (VALID), 3 small scratch (VALID)
    t = np.zeros(6, L.TASK_DTYPE)
    t["tile"][:] = -1
    # 0: RW INCR on tile 0 (sliced stage-in by its own parts, then in-place update)
    t["body"][0], t["nb_flows"][0], t["iparam"][0, 0] = L.BODY_INCR_I32, 1, 5
    t["tile"][0, 0], t["access"][0, 0] = 0, L.ACCESS_RW
    # 1, 2: two concurrent readers of tile 1's first version... tile 1 is INVALID: COPY small -> big scratch (cut by the big tile)
    t["body"][1], t["nb_flows"][1] = L.BODY_COPY, 2
    t["tile"][1, 0], t["access"][1, 0], t["tile"][1, 1], t["access"][1, 1] = 1, L.ACCESS_READ, 2, L.ACCESS_WRITE
    t["body"][2], t["nb_flows"][2], t["iparam"][2, 0] = L.BODY_CHECK_I32, 1, 123
    t["tile"][2, 0], t["access"][2, 0] = 1, L.ACCESS_READ
    # 3: reader of tile 0 after the update; 4: COPY big -> small scratch (task cut by the big tile, small one whole)
    t["body"][3], t["nb_flows"][3], t["iparam"][3, 0], t["dep_goal"][3] = L.BODY_CHECK_I32, 1, 128, 1
    t["tile"][3, 0], t["access"][3, 0] = 0, L.ACCESS_READ
    t["body"][4], t["nb_flows"][4], t["dep_goal"][4] = L.BODY_COPY, 2, 1
    t["tile"][4, 0], t["access"][4, 0], t["tile"][4, 1], t["access"][4, 1] = 0, L.ACCESS_READ, 3, L.ACCESS_WRITE
    t["body"][5], t["nb_flows"][5], t["iparam"][5, 0], t["dep_goal"][5] = L.BODY_CHECK_I32, 1, 128, 1
    t["tile"][5, 0], t["access"][5, 0] = 3, L.ACCESS_READ
    t["succ_begin"] = [0, 2, 2, 2, 2, 3]; t["succ_count"] = [2, 0, 0, 0, 1, 0]
    succ = np.array([3, 4, 5], np.uint32)
    ready = np.array([0, 1, 2], np.int32)
    host = np.full(nb + ns, 123, np.int32)
    spec = np.zeros(4, orc.TILE_DTYPE)
    spec["bytes"] = [big, small, big, small]
    spec["src_ptr"] = [0, big, 0, 0]
    spec["state"] = [orc.TILE_INVALID, orc.TILE_INVALID, orc.TILE_VALID, orc.TILE_VALID]
    ref = orc.run_window(t, succ, spec, ready, host.copy())
    assert ref["rc"] == 0
    with Engine(0, part_bytes=part_bytes) as e:
        offs = np.cumsum([0] + [(b + 511) // 512 * 512 for b in (big, small, big, small)])
        slab = e.malloc(int(offs[-1]))
        e.h2d(slab, np.zeros(int(offs[-1]), np.uint8))
        alias = e.host_register(host)
        tiles = np.zeros(4, L.TILE_DTYPE)
        tiles["dev_ptr"] = slab + offs[:4].astype(np.uint64)
        tiles["src_ptr"] = [alias, alias + big, 0, 0]
        tiles["bytes"] = [big, small, big, small]
        tiles["state"] = [L.TILE_INVALID, L.TILE_INVALID, L.TILE_VALID, L.TILE_VALID]
        w = e.window(0, t, succ, tiles, ready)
        for _ in range(3):                                    # re-armed windows stage again
            st = w.run(); res = w.results()
            assert np.array_equal(res["result"], ref["result"])
            assert st["bytes_h2d"] == big + small == ref["stats"]["bytes_h2d"]
            assert st["body_errors"] == ref["stats"]["body_errors"]
        got = [np.empty(b // 4, np.int32) for b in (big, small, big, small)]
        for i in range(4):
            e.d2h(got[i], int(tiles["dev_ptr"][i]))
        w.close()
        e.host_unregister(host)
    for i in range(4):
        assert np.array_equal(got[i], ref["device"][i].view(np.int32)[:len(got[i])]), i


def test_big_tile_chain_uses_the_whole_gpu():
    """Config-4 body on one GPU: a serial chain of 4 MiB tiles; with parts one hop is spread over up to 32 workers."""
    NT, tb = 64, 4 << 20
    dag = dags.rtt_chain(NT, 1, tb)
    host = np.zeros(tb // 4, np.float32)
    times = {}
    for pb in (-1, 0):
        with Engine(0, part_bytes=pb) as e, placed(e, Layout.packed(dag, host)) as p:
            w = e.window(0, dag.tasks, dag.succ, p.tiles, dag.ready)
            w.run(); p.host[:] = 0
            st = w.run(); res = w.results(); w.close()
            assert all(v == 0 for v in dags.check_execution(dag, res).values())
            assert np.all(p.host.view(np.float32) == NT)
            times[pb] = st["kernel_ms"]
    assert times[0] < times[-1] / 4, times


def test_hbm_window_larger_than_the_ring_entry_id_is_rejected(engine):
    """Ready-ring entries of the HBM kernel carry the task id in 22 bits: a kind-0 window of 2^22 tasks must be refused
    at creation, loudly, not run with truncated ids."""
    n = 1 << 22
    tasks = np.zeros(n, L.TASK_DTYPE)
    tasks["tile"][:] = -1
    tasks["body"] = L.BODY_NOP
    tiles = np.zeros(1, L.TILE_DTYPE)
    tiles["bytes"], tiles["state"] = 64, L.TILE_VALID
    with pytest.raises(L.Pb2Error) as ei:
        engine.window(0, tasks, np.zeros(0, np.uint32), tiles, np.arange(n, dtype=np.int32))
    assert ei.value.rc == L.PB2_ERR_VALUE_OUT_OF_BOUNDS


def test_unknown_window_kind_is_rejected(engine):
    """Kinds other than 0 (HBM bodies) and 1 (GEMM bodies) name no kernel: refused at creation."""
    tasks = np.zeros(1, L.TASK_DTYPE)
    tasks["tile"][:] = -1
    tiles = np.zeros(1, L.TILE_DTYPE)
    tiles["bytes"], tiles["state"] = 64, L.TILE_VALID
    with pytest.raises(L.Pb2Error) as ei:
        engine.window(2, tasks, np.zeros(0, np.uint32), tiles, np.zeros(1, np.int32))
    assert ei.value.rc == L.PB2_ERR_BAD_PARAM
