"""Fused units stage each chunk of the producer's output in shared memory: the members check it there, and a bulk store
writes it to the tile.  These cases cover what only the staged form does: producers that read what they write, a
written flow other than flow 0, a byte tail that the bulk store cannot take, a producer whose tile is staged in first,
and a producer body without a staged form.  Every per-task output must be what the same window computes with fusion
off, and what the sequential oracle computes."""
import numpy as np
import pytest

from parsec_b200 import _lib as L
from oracle import orc_dags as dags
from window_harness import KS, Layout, check_pair, engines, fused, not_fused, readers_dag  # noqa: F401

pytestmark = pytest.mark.gpu


def bits(x):
    return int(np.array([x], np.float32).view(np.int32)[0])


@pytest.mark.parametrize("valid", [False, True], ids=["staged_in", "resident"])
@pytest.mark.parametrize("tile_bytes", [4096 + 12, 40000])
@pytest.mark.parametrize("producer", ["incr", "add_iota"])
def test_read_modify_write_producer(engines, producer, tile_bytes, valid):
    """INCR or ADD_IOTA reads the tile it writes, from a tile with nonzero contents, and the members mismatch.
    staged_in: the producer's tile is first staged in from host memory, so the bulk ring is reused right after."""
    host = np.full(tile_bytes // 4, 2, np.int32)
    host[17] = 9
    if producer == "incr":
        dag = readers_dag(L.BODY_INCR_I32, 3, KS, tile_bytes, access=L.ACCESS_RW)
    else:
        dag = readers_dag(L.BODY_ADD_IOTA_I32, 0, KS, tile_bytes, access=L.ACCESS_RW)
        host[:] = 5 - np.arange(tile_bytes // 4, dtype=np.int32)     # element i becomes 5, the members' constant
        host[1000] = 0
    on, off = check_pair(engines, dag, Layout.packed(dag, host, valid))
    assert (on["result"][1:] >> np.uint64(32)).all()                 # every member counts a mismatch
    assert fused(on, 0, list(range(1, 9)))
    assert not_fused(off, 0, list(range(1, 9)))


def test_axpy_producer_writes_flow_1(engines):
    """AXPY reads x (flow 0) and writes y (flow 1): the members check y."""
    tb = 40000 + 16
    f5, f6 = bits(5.0), bits(6.0)
    ks = [5.0, f5, 5.0, f6, 0, 6.0, 1, f5]
    dag = readers_dag(L.BODY_AXPY_F32, 0, ks, tb)
    t = dag.tasks
    t["nb_flows"][0] = 2
    t["fparam"][0] = 2.0
    t["access"][0, 0], t["access"][0, 1] = L.ACCESS_READ, L.ACCESS_RW
    t["tile"][0, 1] = 1
    t["tile"][1:, 0] = 1
    dag = dags.Dag(t, dag.succ, dag.ready, ntiles=2, tile_bytes=tb, name="axpy")
    x = np.full(tb // 4, 1.5, np.float32)
    y = np.full(tb // 4, 2.0, np.float32)
    y[4099] = 3.0
    host = np.concatenate([x, y]).view(np.int32)
    on, _ = check_pair(engines, dag, Layout.packed(dag, host))
    assert (on["result"][1:] >> np.uint64(32)).all()
    assert fused(on, 0, list(range(1, 9)))


@pytest.mark.parametrize("tile_bytes", [4096 + 13, 13])
def test_memset_producer_ragged_tail(engines, tile_bytes):
    """MEMSET_U8 writes every byte, so the last chunk ends with a tail of < 16 bytes written from the slot by SIMT
    stores; the members check the whole 4-byte elements."""
    k = 0x05050505
    dag = readers_dag(L.BODY_MEMSET_U8, 5, [k, k, 5, 0, k, 7, 1, k], tile_bytes)
    host = np.full((tile_bytes + 3) // 4, -1, np.int32)
    on, _ = check_pair(engines, dag, Layout.packed(dag, host))
    assert fused(on, 0, list(range(1, 9)))


def test_add_at_producer_is_not_fused(engines):
    """ADD_AT updates one element and has no staged form: its readers still run as one read group, apart from it."""
    tb = 40000
    dag = readers_dag(L.BODY_ADD_AT_I32, 123, KS, tb, access=L.ACCESS_RW)
    dag.tasks["iparam"][0, 1] = 4
    host = np.full(tb // 4, 1, np.int32)
    on, off = check_pair(engines, dag, Layout.packed(dag, host))
    members = list(range(1, 9))
    assert not_fused(on, 0, members)
    assert all(on["worker"][m] == on["worker"][1] for m in members)
    assert np.array_equal(on["result"], off["result"])
