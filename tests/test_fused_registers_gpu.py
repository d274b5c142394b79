"""A fused unit checks the producer's output in registers: every body with a checked form writes its output flow as it
would alone, and each thread compares every value it stores with the leader's constant before it stores it.  Every
such body runs here with members that pass and members that fail, with a leader whose own constant fails, and with one
bad element in what the producer reads, over tiles of 13 bytes, 4096 + 12 bytes, 40000 bytes and 1 MiB (16 parts of
64 KiB), staged in from host memory or already resident.  Results, seen versions, event order and tile bytes must be
what the same window computes with fusion off and what the sequential oracle computes, and the unit must have been
fused."""
import numpy as np
import pytest

from parsec_b200 import _lib as L
from oracle import orc_dags as dags
from parsec_b200.engine import Engine
from window_harness import Layout, check_pair, fused, not_fused, readers_dag

pytestmark = pytest.mark.gpu

PART = 64 * 1024
MEMBERS = list(range(1, 9))


@pytest.fixture(scope="module")
def engines():
    with Engine(0, part_bytes=PART) as on, Engine(0, part_bytes=PART, fuse_readers=-1) as off:
        yield on, off


def u32(x):
    """The bits of float32 x."""
    return int(np.array([x], np.float32).view(np.uint32)[0])


def f32(bits):
    """The float32 whose bits are `bits` (a CHECK_F32 constant that compares like the integer)."""
    return float(np.array([bits], np.uint32).view(np.float32)[0])


def i32(bits):
    return int(np.array([bits], np.uint32).view(np.int32)[0])


# body -> (producer's int param, float param, what it reads (None: nothing) as float32 / int32 elements, the value it
# writes everywhere (None: no single value), whether it writes flow 1)
BODIES = {
    "fill_i32": (L.BODY_FILL_I32, 5, 0.0, None, 5, False),
    "fill_f32": (L.BODY_FILL_F32, 0, 2.5, None, u32(2.5), False),
    "memset_u8": (L.BODY_MEMSET_U8, 5, 0.0, None, 0x05050505, False),
    "iota": (L.BODY_IOTA_I32, 0, 0.0, None, None, False),
    "incr_i32": (L.BODY_INCR_I32, 3, 0.0, ("i", 2), 5, False),
    "incr_f32": (L.BODY_INCR_F32, 0, 0.5, ("f", 1.5), u32(2.0), False),
    "scale_i32": (L.BODY_SCALE_I32, 3, 0.0, ("i", 2), 6, False),
    "add_iota": (L.BODY_ADD_IOTA_I32, 0, 0.0, ("iota", 5), 5, False),
    "copy": (L.BODY_COPY, 0, 0.0, ("i", 5), 5, True),
    "axpy": (L.BODY_AXPY_F32, 0, 2.0, ("f", 2.0), u32(5.0), True),     # y = 2 * 1.5 + 2
}
READS = [b for b, v in BODIES.items() if v[3] is not None]
CASES = [(b, c) for b in BODIES for c in ("pass", "leader_fails")] + [(b, "bad_element") for b in READS]


def member_ks(v, case):
    """Eight CHECK constants: integers are CHECK_I32, floats CHECK_F32 with those bits.  With a single written value v,
    "pass" has the leader and three others pass; "leader_fails" has the leader and two others on one failing constant."""
    if v is None:
        v = 0                                  # IOTA: element 0 is 0 in part 0, every other element differs
    good, bad = i32(v), i32((v + 1) & 0xffffffff)
    if case == "leader_fails":
        return [bad, good, bad, f32(v), 0, good, 1, bad]
    return [good, good, bad, f32(v), 0, good, 1, good]


def tile_of(kind, tb, bad):
    """tb bytes of what the producer reads: int32 / float32 elements, or 5 - i (ADD_IOTA makes element i 5)."""
    n = (tb + 3) // 4
    if kind[0] == "f":
        e = np.full(n, kind[1], np.float32).view(np.int32)
        if bad: e[n // 2] = np.array([3.0], np.float32).view(np.int32)[0]
    elif kind[0] == "iota":
        e = (kind[1] - np.arange(n)).astype(np.int32)
        if bad: e[n // 2] = 0
    else:
        e = np.full(n, kind[1], np.int32)
        if bad: e[n // 2] = 9
    return e.view(np.uint8)[:tb]


def unit_dag(body, tb, case):
    code, ip, fp, reads, v, flow1 = BODIES[body]
    ks = member_ks(v, case)
    # the written tile is read too, so that it is staged in (or resident) like the others: the bytes of a 13-byte tile
    # beyond the last whole element are not written by every body, and they must be defined
    dag = readers_dag(code, ip, ks, tb, access=L.ACCESS_RW)
    t = dag.tasks
    t["fparam"][0] = fp
    fill = np.full(tb, 0xff, np.uint8)         # what the written tile holds before the producer runs
    if not flow1:
        tiles = [tile_of(reads, tb, case == "bad_element") if reads is not None else fill]
    else:
        # flow 0 is read (COPY's source, AXPY's x), flow 1 is written and checked
        t["nb_flows"][0] = 2
        t["access"][0, 0], t["access"][0, 1] = L.ACCESS_READ, L.ACCESS_RW
        t["tile"][0, 1] = 1
        t["tile"][1:, 0] = 1
        dag = dags.Dag(t, dag.succ, dag.ready, ntiles=2, tile_bytes=tb, name=body)
        bad = case == "bad_element"
        if code == L.BODY_AXPY_F32:
            tiles = [tile_of(("f", 1.5), tb, False), tile_of(reads, tb, bad)]
        else:
            tiles = [tile_of(reads, tb, bad), fill]
    raw = np.concatenate(tiles)
    host = np.zeros((raw.size + 3) // 4 * 4, np.uint8)
    host[:raw.size] = raw
    return dag, host.view(np.int32)


@pytest.mark.parametrize("valid", [False, True], ids=["staged_in", "resident"])
@pytest.mark.parametrize("tile_bytes", [13, 4096 + 12, 40000, 1 << 20], ids=["b13", "b4108", "b40000", "mib_16parts"])
@pytest.mark.parametrize("body,case", CASES, ids=["%s-%s" % c for c in CASES])
def test_checked_bodies(engines, body, case, tile_bytes, valid):
    dag, host = unit_dag(body, tile_bytes, case)
    on, off = check_pair(engines, dag, Layout.packed(dag, host, valid))
    assert fused(on, 0, MEMBERS)
    assert not_fused(off, 0, MEMBERS)
    mism = on["result"][1:] >> np.uint64(32)
    if tile_bytes >= 4:
        assert mism.any()                                                   # some member fails in every case
    if case == "leader_fails" or (case == "bad_element" and tile_bytes >= 4):
        assert mism[0] > 0
    if case == "pass" and BODIES[body][4] is not None:
        assert mism[0] == 0 and mism[1] == 0 and mism[5] == 0 and mism[7] == 0
