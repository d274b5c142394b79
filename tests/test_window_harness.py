"""The window harness of the GPU tests, without a GPU: its layouts are the ones the tests have always built by hand, its
oracle run is orc.run_window's, and each comparison fails on a single byte of what it compares."""
import numpy as np
import pytest

from oracle import orc
from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from window_harness import KS, Layout, Run, assert_like_oracle, assert_same_run, readers_dag, run_oracle

SLAB, ALIAS = 0x7F0000000000, 0x200000000


def hand_table(n, slot_offsets, host_offsets, sizes, state, host=True):
    t = np.zeros(n, L.TILE_DTYPE)
    t["dev_ptr"] = SLAB + np.asarray(slot_offsets, np.uint64)
    t["src_ptr"] = (ALIAS + np.asarray(host_offsets, np.uint64)) if host else 0
    t["bytes"] = sizes
    t["state"] = state
    return t


def packed_by_hand(dag, host=True, valid=False):
    """One 512-byte-rounded slot per tile, host copies back to back."""
    nt, tb = dag.ntiles, dag.tile_bytes
    slot = (tb + 511) // 512 * 512
    return hand_table(nt, np.arange(nt) * slot, np.arange(nt) * tb, tb, L.TILE_VALID if valid else L.TILE_INVALID, host)


@pytest.mark.parametrize("valid", [False, True])
def test_packed_layout_of_ragged_ex05(valid):
    dag = dags.ex05_broadcast(33, 4, 1000)
    host = np.arange(33 * 250, dtype=np.int32)
    layout = Layout.packed(dag, host, valid)
    assert layout.table(SLAB, ALIAS).tobytes() == packed_by_hand(dag, valid=valid).tobytes()
    assert len(layout.dev) == 33 * 1024
    for i in (0, 17, 32):                         # resident tiles hold their host bytes, the rest of the slab is zero
        want = host.view(np.uint8)[i * 1000:(i + 1) * 1000] if valid else np.zeros(1000, np.uint8)
        assert np.array_equal(layout.tile_bytes(layout.dev, i), want)
    assert not layout.dev[1000:1024].any()


def test_packed_layout_without_host():
    dag = dags.ex02_chain(10)
    layout = Layout.packed(dag)
    assert layout.table(SLAB, ALIAS).tobytes() == packed_by_hand(dag, host=False).tobytes()
    assert len(layout.dev) == 512 and len(layout.host) == 0


def test_packed_layout_with_sizes():
    """The fused tests' two-tile case: tiles of 8192 and 4096 bytes, host copies back to back."""
    dag = readers_dag(L.BODY_FILL_I32, 5, KS, 4096)
    dag = dags.Dag(dag.tasks, dag.succ, dag.ready, ntiles=2, tile_bytes=4096)
    for sizes, slots in (([8192, 4096], [0, 8192]), ([4096 + 13, 13], [0, 4608])):
        layout = Layout.packed(dag, np.zeros(sum(sizes) // 4 + 1, np.int32), True, sizes=sizes)
        want = hand_table(2, slots, [0, sizes[0]], sizes, L.TILE_VALID)
        assert layout.table(SLAB, ALIAS).tobytes() == want.tobytes()


def test_contiguous_layouts():
    dag = dags.ex05_broadcast(8, 6, 4096)
    init = np.arange(8 * 1024, dtype=np.int32)
    resident = Layout.contiguous(dag, dev=init)
    want = hand_table(8, np.arange(8) * 4096, np.zeros(8), 4096, L.TILE_VALID, host=False)
    assert resident.table(SLAB, ALIAS).tobytes() == want.tobytes()
    assert np.array_equal(resident.dev, init.view(np.uint8))
    staged = Layout.contiguous(dag, host=init, valid=False)
    want = hand_table(8, np.arange(8) * 4096, np.arange(8) * 4096, 4096, L.TILE_INVALID)
    assert staged.table(SLAB, ALIAS).tobytes() == want.tobytes()
    assert len(staged.dev) == 8 * 4096 and not staged.dev.any()


def direct(dag, layout, host):
    """orc.run_window of dag over the layout's offsets: a zeroed device, a home in host (modified in place)."""
    ref = orc.run_window(dag.tasks, dag.succ, layout.offsets(), dag.ready, host)
    assert ref["rc"] == 0
    return ref


@pytest.mark.parametrize("name,dag,sizes", [
    ("ex05_ragged", dags.ex05_broadcast(33, 4, 1000), None),
    ("rtt_pushout", dags.rtt_chain(10, 3, 4096), None),
    ("readers_sized", readers_dag(L.BODY_IOTA_I32, 0, KS, 4096 + 12), [4096 + 12]),
])
def test_run_oracle_is_run_window_on_staged_tiles(name, dag, sizes):
    host = np.random.default_rng(1).integers(-9, 9, dag.ntiles * dag.tile_bytes // 4).astype(np.int32)
    layout = Layout.packed(dag, host, sizes=sizes)
    run = run_oracle(dag, layout)
    h = host.copy()
    ref = direct(dag, layout, h)
    for k in ("retire_order", "start_seq", "end_seq", "seen_version", "result"):
        assert np.array_equal(run.res[k], ref[k]), k
    assert run.stats == ref["stats"]
    assert np.array_equal(run.host, h.view(np.uint8))
    for i in range(dag.ntiles):
        assert np.array_equal(layout.tile_bytes(run.dev, i), ref["device"][i][:layout.nbytes[i]]), i
    assert np.array_equal(run.res["tiles"]["version"], ref["tiles"]["version"])
    assert np.array_equal(run.res["tiles"]["state"], ref["tiles"]["state"])
    assert np.array_equal(layout.host, host.view(np.uint8))            # the layout's images are not touched


def test_run_oracle_is_run_window_on_resident_tiles():
    """Resident tiles: orc.run_window's device starts zeroed, so both get a zeroed slab."""
    dag = dags.ex05_broadcast(16, 6, 4096)
    layout = Layout.contiguous(dag)
    run = run_oracle(dag, layout)
    ref = direct(dag, layout, None)
    for k in ("retire_order", "seen_version", "result"):
        assert np.array_equal(run.res[k], ref[k]), k
    assert run.stats == ref["stats"]
    assert np.array_equal(run.dev, np.concatenate(ref["device"]))


def synthetic_run():
    rng = np.random.default_rng(3)
    tiles = np.zeros(3, L.TILE_DTYPE)
    tiles["dev_ptr"], tiles["bytes"], tiles["version"], tiles["state"] = [0, 512, 1024], 64, [1, 2, 3], L.TILE_VALID
    res = {"result": rng.integers(0, 99, 4).astype(np.uint64), "seen_version": np.zeros((4, 4), np.uint32),
           "retire_order": np.arange(4, dtype=np.int32), "start_seq": np.arange(0, 8, 2, dtype=np.uint32),
           "end_seq": np.arange(1, 8, 2, dtype=np.uint32), "tiles": tiles}
    stats = {k: int(rng.integers(1, 99)) for k in ("tasks_retired", "bytes_h2d", "bytes_d2d", "bytes_d2h", "stage_ins",
                                                     "body_errors")}
    stats["tasks_retired"] = 4
    return Run(stats, res, rng.integers(0, 255, 1536).astype(np.uint8), rng.integers(0, 255, 192).astype(np.uint8), [],
               tiles.copy())


def one_byte_off(run, what):
    """A copy of run with one byte (or one count) of `what` changed."""
    res = {k: v.copy() for k, v in run.res.items()}
    stats, dev, host, table = dict(run.stats), run.dev.copy(), run.host.copy(), run.table.copy()
    if what in ("result", "seen_version"):
        res[what].reshape(-1).view(np.uint8)[5] ^= 1
    elif what in ("version", "state"):
        res["tiles"][what][1] += 1
        table[what][1] += 1
    elif what == "table":
        table["src_ptr"][2] += 1
    elif what == "dev":
        dev[700] ^= 0x80
    elif what == "host":
        host[191] ^= 1
    else:
        stats[what] += 1
    return Run(stats, res, dev, host, [], table)


CHANGES = ["result", "seen_version", "version", "state", "table", "dev", "host", "tasks_retired", "bytes_h2d",
           "bytes_d2d", "bytes_d2h", "stage_ins", "body_errors"]


@pytest.mark.parametrize("what", CHANGES)
def test_assert_same_run_sees_one_byte(what):
    a = synthetic_run()
    assert_same_run(a, a)
    with pytest.raises(AssertionError):
        assert_same_run(a, one_byte_off(a, what))


@pytest.mark.parametrize("what", [c for c in CHANGES if c != "table"] + ["order"])
def test_assert_like_oracle_sees_one_byte(what):
    dag = dags.ex02_chain(3)
    a = synthetic_run()
    assert_like_oracle(a, a, dag)
    if what == "order":                              # a task that starts before its predecessor ended
        b = one_byte_off(a, "result")
        b.res["result"][:] = a.res["result"]
        b.res["start_seq"][2] = 2
    else:
        b = one_byte_off(a, what)
    with pytest.raises(AssertionError):
        assert_like_oracle(b, a, dag)
