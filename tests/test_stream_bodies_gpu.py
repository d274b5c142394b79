"""Every element-wise body on the streaming kernel (pb2_stream.cu) against the NumPy reference (body_ref.py): random DTD
programs over ragged tiles whose slots sit at 16 mod 128 and whose host homes are 16-, 4- and 1-byte aligned, with
sentinel gaps between them, through both submission modes, three part sizes and both tile movers; ticket recycling; a
tile described again between two DAGs; a staged tile whose trailing stage-in slices are empty; and the window tests' DAGs
compared with the oracle over every tile and every statistic."""
import numpy as np
import pytest

import body_ref as R
from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200.engine import Engine
from parsec_b200.stream import Stream, run_dag
from window_harness import Layout, assert_like_oracle, placed, run_engine, run_oracle

pytestmark = pytest.mark.gpu

SIZES = [0, 1, 3, 4, 15, 16, 17, 4096 + 12, 65536 + 4, (1 << 20) + 20]


@pytest.fixture(scope="module")
def movers(engine):
    """The session's engine (TMA bulk tile mover) and one with the SIMT mover (stage_mode 1)."""
    with Engine(0, stage_mode=1) as simt:
        yield {0: engine, 1: simt}


def run_stream(eng, dag, layout, mode="lookahead", **kw):
    """dag through a fresh stream on eng over layout: (run_dag's output, stats, slab image, host image)."""
    with placed(eng, layout) as p:
        assert p.alias % 16 == 0 and p.host.ctypes.data % 16 == 0
        with Stream(eng, max_tiles=max(dag.ntiles, 1), idle_us=500, **kw) as s:
            out = run_dag(s, dag, p.tiles, mode=mode)
            s.quiesce()
            st = s.stats()
    return out, st, p.dev, p.host


def assert_like_ref(out, st, dev, host, ref, dag=None):
    n = len(ref["result"])
    assert sorted(out["retire_order"].tolist()) == list(range(n))
    if dag is not None:
        pos = np.empty(n, np.int64)
        pos[out["retire_order"]] = np.arange(n)
        src, dst, _ = dag.edges()
        assert np.all(pos[src] < pos[dst]), "retire order is not a linear extension of the DAG"
    bad = np.flatnonzero(out["result"] != ref["result"])
    assert not len(bad), f"{len(bad)} results differ, first task {bad[0]}"
    assert np.array_equal(out["seen_version"], ref["seen_version"]), "seen versions"
    for k in ("bytes_h2d", "bytes_d2h", "stage_ins", "body_errors"):
        assert st[k] == ref["stats"][k], (k, st[k], ref["stats"][k])
    diff = np.flatnonzero(dev != ref["dev"])
    assert not len(diff), f"{len(diff)} slab bytes differ, first at {diff[0]}"
    diff = np.flatnonzero(host != ref["host"])
    assert not len(diff), f"{len(diff)} host bytes differ, first at {diff[0]}"


_CASE = {}


def every_body_case():
    """About 300 tasks over 40 tiles, every body; built once per module."""
    if not _CASE:
        rng = np.random.default_rng(2024)
        nt = 40
        sizes = SIZES + [int(v) for v in rng.integers(0, 70000, nt - len(SIZES))]
        rng.shuffle(sizes)
        kinds = ["int"] * nt
        pairs = [i for i in range(nt - 1) if 64 <= sizes[i] and 64 <= sizes[i + 1]][:7:3]
        for i in pairs:
            kinds[i], kinds[i + 1] = "fx", "fy"
        for i in [i for i in range(nt) if kinds[i] == "int"][1::3]:
            kinds[i] = "float"
        layout = R.scattered_layout(rng, sizes, rng.random(nt) < 0.4)
        R.fill_kinds(rng, layout, kinds)
        prog = R.random_program(rng, sizes, 300, kinds)
        dag = prog.dag()
        ref = R.run_program(prog, layout)
        orc = run_oracle(dag, layout)
        assert np.array_equal(ref["seen_version"], orc.res["seen_version"])
        assert np.array_equal(ref["result"], orc.res["result"])
        _CASE.update(prog=prog, layout=layout, dag=dag, ref=ref)
    return _CASE


@pytest.mark.parametrize("stage_mode", [0, 1])
@pytest.mark.parametrize("part_bytes", [0, 16384, 100])
@pytest.mark.parametrize("mode", ["lookahead", "host"])
def test_every_body_on_the_streaming_kernel(movers, stage_mode, part_bytes, mode):
    """part_bytes 0: the default (256 KiB); 100: tiles of 4 KiB and more are cut into parts of which the last ones are
    empty, and staged in 100-byte slices."""
    c = every_body_case()
    out, st, dev, host = run_stream(movers[stage_mode], c["dag"], c["layout"], mode, part_bytes=part_bytes)
    assert_like_ref(out, st, dev, host, c["ref"], c["dag"])


def test_ticket_recycling(engine):
    """6 000 tasks through 1 024 tickets, each with a constant of its own: INCR by distinct steps, ADD_AT at distinct
    indices, CHECKs over five parts whose counts differ.  A descriptor, result or part count left over from the ticket's
    last task would change a result or the final image."""
    rng = np.random.default_rng(5)
    sizes = [65536 + 4] * 4 + [4096, 20]
    layout = R.scattered_layout(rng, sizes, [True, False, True, False, True, True])
    for i in range(5):
        # value v (< 128) in about 2v + 1 elements: CHECKs of different values count different mismatches
        R.put_words(layout, i, np.sqrt(np.arange(sizes[i] // 4)).astype(np.uint32) % 128)
    prog = R.Program(len(sizes))
    shift = [0] * 5                              # what the INCRs added to tile i so far
    for j in range(6000):
        i = j % 5
        kind = (j // 5) % 3
        if kind == 0:
            prog.task(L.BODY_INCR_I32, [(i, L.ACCESS_RW)], (j + 1, 0, 0))
            shift[i] += j + 1
        elif kind == 1:
            n = sizes[i] // 4
            prog.task(L.BODY_ADD_AT_I32, [(i, L.ACCESS_RW | (L.FLOW_PUSHOUT if j % 7 == 0 else 0))], ((j * 7919) % n, j, 0))
        else:
            k = (shift[i] + int(rng.integers(0, 128))) & 0xFFFFFFFF
            prog.task(L.BODY_CHECK_I32, [(i, L.ACCESS_READ)], (k - (1 << 32) if k >= 1 << 31 else k, 0, 0))
    dag = prog.dag()
    ref = R.run_program(prog, layout)
    checks = np.array([int(r) >> 32 for (b, *_), r in zip(prog.tasks, ref["result"]) if b == L.BODY_CHECK_I32])
    assert len(set(checks.tolist())) > 100
    out, st, dev, host = run_stream(engine, dag, layout, "lookahead", cmd_slots=1024, part_bytes=16384)
    assert_like_ref(out, st, dev, host, ref)


def test_tile_described_again_is_staged_again(engine):
    """A wide tile staged in slices by one DAG, then described again as INVALID with another home: the next DAG's
    stage-in pulls the new home's bytes (the dispatcher clears the tile's slice claims)."""
    rng = np.random.default_rng(9)
    n = (256 << 10) + 20
    layout = R.scattered_layout(rng, [n, n, n], [False, True, False])
    prog = R.Program(3)
    prog.task(L.BODY_COPY, [(0, L.ACCESS_READ), (1, L.ACCESS_WRITE | L.FLOW_PUSHOUT)])
    dag = prog.dag()
    home = lambda img, i: img[int(layout.hoff[i]):int(layout.hoff[i]) + n]
    with placed(engine, layout) as p, Stream(engine, max_tiles=3, idle_us=500, part_bytes=4096) as s:
        run_dag(s, dag, p.tiles)
        s.quiesce()
        assert np.array_equal(home(p.host, 1), home(layout.host, 0))
        again = p.tiles.copy()
        again["src_ptr"][0] = p.tiles["src_ptr"][2]
        run_dag(s, dag, again)
        s.quiesce()
        st = s.stats()
        assert np.array_equal(home(p.host, 1), home(layout.host, 2)), "the second DAG read the old bytes"
    assert st["stage_ins"] == 2 and st["bytes_h2d"] == 2 * n and st["bytes_d2h"] == 2 * n


def empty_slices_case():
    """A staged tile of 512 x 4097 bytes read by a 512-part INCR with part_bytes 4096: its stage-in slices are 4112 bytes,
    so the last one is empty."""
    rng = np.random.default_rng(4097)
    layout = R.scattered_layout(rng, [512 * 4097, 64], [False, True])
    prog = R.Program(2)
    prog.task(L.BODY_INCR_I32, [(0, L.ACCESS_RW)], (3, 0, 0))
    prog.task(L.BODY_CHECK_I32, [(0, L.ACCESS_READ)], (3, 0, 0))
    prog.task(L.BODY_COPY, [(0, L.ACCESS_READ), (1, L.ACCESS_RW | L.FLOW_PUSHOUT)])
    return prog, layout


def test_empty_trailing_slices_on_the_streaming_kernel(engine):
    prog, layout = empty_slices_case()
    ref = R.run_program(prog, layout)
    out, st, dev, host = run_stream(engine, prog.dag(), layout, "lookahead", part_bytes=4096)
    assert st["stage_ins"] == 1
    assert_like_ref(out, st, dev, host, ref)


def test_empty_trailing_slices_in_an_hbm_window():
    prog, layout = empty_slices_case()
    dag = prog.dag()
    with Engine(0, part_bytes=4096) as eng:
        run = run_engine(eng, dag, layout)
    ref = run_oracle(dag, layout)
    assert run.res["tiles"]["state"][0] == L.TILE_VALID
    assert_like_oracle(run, ref, dag)
    assert ref.stats["stage_ins"] == 1


@pytest.mark.parametrize("mode", ["lookahead", "host"])
@pytest.mark.parametrize("name,maker", [
    ("ex05", lambda: dags.ex05_broadcast(64, 14, 256 * 256 * 4)),
    ("ex05_ragged", lambda: dags.ex05_broadcast(33, 4, 1000)),
    ("ex02", lambda: dags.ex02_chain(200)),
    ("rtt_wide", lambda: dags.rtt_chain(8, 2, 1024 * 1024 * 4)),
    ("ep", lambda: dags.ep(64, 8)),
])
def test_oracle_dags_every_tile_and_stage_in(engine, mode, name, maker):
    """The DAGs of test_stream_matches_oracle, compared with the oracle on every tile's final bytes (not only the first
    and the last tile's whole elements), the host image, the results, and every statistic including stage_ins."""
    dag = maker()
    words = max(dag.ntiles * dag.tile_bytes // 4, 1)
    host = np.full(words, -7, np.int32)
    if name.startswith("rtt"):
        host = np.ones(words, np.float32).view(np.int32)
    layout = Layout.packed(dag, host)
    ref = run_oracle(dag, layout)
    out, st, dev, host_after = run_stream(engine, dag, layout, mode, cmd_slots=4096)
    assert np.array_equal(out["result"], ref.res["result"]), "results"
    assert np.array_equal(out["seen_version"], ref.res["seen_version"]), "seen versions"
    for k in ("body_errors", "bytes_h2d", "bytes_d2h", "stage_ins"):
        assert st[k] == ref.stats[k], (k, st[k], ref.stats[k])
    assert np.array_equal(host_after, ref.host), "host image"
    for i in range(dag.ntiles):
        assert np.array_equal(layout.tile_bytes(dev, i), layout.tile_bytes(ref.dev, i)), f"final bytes of tile {i}"
