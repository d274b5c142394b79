"""Tile slots the bodies cannot access are refused on the host, before anything is launched.  Every body but NOP loads and
stores its flows with 16-byte vectors, so a window (pb2_window_create's plan), a stream (pb2_stream_set_tile) and a
stand-alone launch (pb2_body_launch) refuse a non-empty slot that is not 16-byte aligned with PB2_ERR_BAD_PARAM; host
homes keep any alignment.  No GPU: the plan is host code, the stream is a dry run and the launch is refused before it
reaches the device."""
import ctypes as C

import numpy as np
import pytest

from oracle import orc_dags as dags
from parsec_b200 import _lib as L
from parsec_b200.stream import Stream
from test_window_plan import plan_of, planner, refused, tiles_for  # noqa: F401  (planner is a fixture)


def test_windows_refuse_unaligned_body_slots(planner):
    dag = dags.ex05_broadcast(2)
    for skew in (8, 4, 1):
        tiles = tiles_for(dag.ntiles, dag.tile_bytes)
        tiles["dev_ptr"][1] += skew
        assert refused(planner, dag, tiles) == (L.PB2_ERR_BAD_PARAM, "tile of a task body not 16-byte aligned")
    # a NOP never touches its tiles, and an empty tile is never accessed
    nop = dags.ex05_broadcast(2)
    nop.tasks["body"][:] = L.BODY_NOP
    assert plan_of(planner, nop.tasks, nop.succ, tiles, nop.ready)[2] is not None
    tiles["bytes"][1] = 0
    assert plan_of(planner, dag.tasks, dag.succ, tiles, dag.ready)[2] is not None
    # host homes may have any alignment (the stage-in and pushout copies take the narrow loops)
    tiles = tiles_for(dag.ntiles, dag.tile_bytes)
    tiles["src_ptr"] = 0x20003
    assert plan_of(planner, dag.tasks, dag.succ, tiles, dag.ready)[2] is not None


def test_gemm_windows_refuse_an_unaligned_c_tile(planner):
    dag = dags.dtd_gemm(2)
    tiles = tiles_for(dag.ntiles, dag.tile_bytes)
    tiles["dev_ptr"][-1] += 1
    assert refused(planner, dag, tiles, kind=1) == (L.PB2_ERR_BAD_PARAM, "GEMM tile not 16-byte aligned")


def test_stream_refuses_unaligned_slots():
    with Stream(None, dry_run=1, cmd_slots=1024, max_tiles=4) as s:
        tile = np.zeros(1, L.TILE_DTYPE)
        tile["bytes"] = 64
        tile["src_ptr"] = 0x30001
        for addr in (0x10008, 0x10004, 0x10001):
            tile["dev_ptr"] = addr
            with pytest.raises(L.Pb2Error) as e:
                s.set_tile(0, tile)
            assert e.value.rc == L.PB2_ERR_BAD_PARAM and "16-byte aligned" in str(e.value)
        tile["dev_ptr"] = 0x10010
        s.set_tile(0, tile)                # aligned slot, 1-byte aligned home
        tile["dev_ptr"] = 0x10001
        tile["bytes"] = 0
        s.set_tile(1, tile)                # an empty tile is never accessed


def body_launch(body, ptrs, nbytes, iparam=(1, 0, 0)):
    p = (C.c_void_p * len(ptrs))(*ptrs)
    b = (C.c_uint64 * len(nbytes))(*nbytes)
    ip = (C.c_int32 * 3)(*iparam)
    return L.load().pb2_body_launch(None, body, len(ptrs), C.cast(p, C.c_void_p), C.cast(b, C.c_void_p),
                                    C.cast(ip, C.c_void_p), C.c_float(0.0))


def test_body_launch_refuses_flows_it_cannot_run():
    ok = 0x7f0000000000
    for ptrs, nbytes in [([ok + 8], [64]), ([ok + 4], [4]), ([ok + 1], [1]), ([None], [16]),
                         ([ok, ok + 0x1000 + 4], [64, 64]), ([ok, None], [64, 8])]:
        assert body_launch(L.BODY_INCR_I32, ptrs, nbytes) == L.PB2_ERR_BAD_PARAM, (ptrs, nbytes)
    assert body_launch(L.BODY_FILL_I32, [ok], [1 << 32]) == L.PB2_ERR_VALUE_OUT_OF_BOUNDS
    # NOP launches nothing; its empty flows may be unaligned or NULL
    assert body_launch(L.BODY_NOP, [ok + 3, None], [0, 0]) == L.PB2_SUCCESS
