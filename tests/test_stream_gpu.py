"""GPU parity tests of the streaming ring + persistent kernel (pb2_stream.cu) against the oracle: the same DAGs the
window tests use, driven (a) with device-side release of look-ahead edges and (b) with one host round trip per edge."""
import numpy as np
import pytest

from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200.stream import Stream, run_dag
from window_harness import Layout, placed, run_oracle

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode", ["lookahead", "host"])
@pytest.mark.parametrize("name,maker", [
    ("ex05", lambda: dags.ex05_broadcast(64, 14, 256 * 256 * 4)),
    ("ex05_ragged", lambda: dags.ex05_broadcast(33, 4, 1000)),
    ("ex02", lambda: dags.ex02_chain(200)),
    ("rtt_wide", lambda: dags.rtt_chain(8, 2, 1024 * 1024 * 4)),
    ("ep", lambda: dags.ep(64, 8)),
])
def test_stream_matches_oracle(engine, mode, name, maker):
    dag = maker()
    words = max(dag.ntiles * dag.tile_bytes // 4, 1)
    host = (np.arange(words, dtype=np.int64) % 1000).astype(np.int32) if name.startswith("rtt") else np.full(words, -7, np.int32)
    if name.startswith("rtt"):
        host = host.view(np.float32).copy(); host[:] = 1.0; host = host.view(np.int32)
    layout = Layout.packed(dag, host)
    ref = run_oracle(dag, layout)
    with placed(engine, layout) as p, Stream(engine, cmd_slots=4096, max_tiles=max(dag.ntiles, 1), idle_us=500) as s:
        out = run_dag(s, dag, p.tiles, mode=mode)
        s.quiesce()
        st = s.stats()
    n = len(dag.tasks)
    assert sorted(out["retire_order"].tolist()) == list(range(n))
    pos = np.empty(n, np.int64)
    pos[out["retire_order"]] = np.arange(n)
    for u in range(n):
        t = dag.tasks[u]
        for e in dag.succ[t["succ_begin"]:t["succ_begin"] + t["succ_count"]]:
            assert pos[u] < pos[int(e) & 0x07FFFFFF], "retire order is not a linear extension of the DAG"
    assert np.array_equal(out["result"], ref.res["result"]), "body results differ from the oracle"
    assert np.array_equal(out["seen_version"], ref.res["seen_version"]), "flow versions differ from the oracle"
    for k in ("body_errors", "bytes_h2d", "bytes_d2h"):
        assert st[k] == ref.stats[k], k
    assert np.array_equal(p.host, ref.host), "pushed-out tiles differ from the oracle"
    for i in (0, dag.ntiles - 1):
        if dag.tile_bytes >= 4:
            nb = dag.tile_bytes // 4 * 4
            assert np.array_equal(layout.tile_bytes(p.dev, i)[:nb], layout.tile_bytes(ref.dev, i)[:nb]), "final tile bytes differ"
    if mode == "lookahead" and any(t["succ_count"] for t in dag.tasks):
        assert st["released_on_device"] + st["edges_late"] > 0


def test_stream_parks_and_restarts(engine):
    """The persistent kernel exits when idle and is relaunched by the next submission; tickets survive the gap."""
    import time
    dag = dags.ex02_chain(20)
    layout = Layout.packed(dag, np.zeros(1, np.int32), valid=True)
    with placed(engine, layout) as p, Stream(engine, cmd_slots=1024, max_tiles=1, idle_us=200) as s:
        for rnd in range(3):
            out = run_dag(s, dag, p.tiles, mode="lookahead")
            assert out["retire_order"].tolist() == list(range(21))
            time.sleep(0.05)                     # >> idle_us: the kernel parks
        st = s.stats()
        assert st["kernel_launches"] >= 3
        assert st["retired"] == 63


def test_stream_unknown_body_is_reported(engine):
    with Stream(engine, cmd_slots=1024, max_tiles=1, idle_us=200, timeout_ms=2000) as s:
        row = np.zeros(1, L.TASK_DTYPE)
        row["tile"] = -1
        row["body"] = 15                         # below PB2_BODY_MAX, not a body the kernel knows
        s.submit(row, cookie=1)
        s.kick()
        import time
        t0 = time.time()
        recs = []
        with pytest.raises(L.Pb2Error):
            while time.time() - t0 < 10:
                recs += s.poll()
                if recs:
                    assert recs[0][4] != 0
                    raise L.Pb2Error(recs[0][4], "bad body")


def test_submit_and_poll_from_two_threads(engine):
    """The submit side and the poll side of a stream on two threads at once (what the device module's starter and manager
    do): 50 000 empty tasks through a 1024-slot ring, every cookie retired exactly once."""
    from test_stream_host import _two_sided
    with Stream(engine, cmd_slots=1024) as s:
        _two_sided(s, 50000)
