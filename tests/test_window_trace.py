"""Window trace without a GPU: the Chrome-trace writer on synthetic intervals, the C ABI's argument checks, the
device_engine_trace MCA parameter, and the per-task device trace of a dry-run pool (no window ran: zeros)."""
import ctypes as C
import json

import numpy as np

from parsec_b200 import _lib as L
from parsec_b200 import runtime as R
from parsec_b200.engine import chrome_trace


def test_chrome_trace_synthetic():
    rng = np.random.default_rng(7)
    n = 200
    t0 = (10_000_000 + rng.integers(0, 50_000, n)).astype(np.uint64)
    t1 = t0 + rng.integers(0, 20_000, n).astype(np.uint64)
    sm = rng.integers(0, 132, n).astype(np.uint32)
    cls = rng.integers(0, 2, n).astype(np.int32)
    loc = rng.integers(0, 100, (n, 2)).astype(np.int32)
    unit = np.arange(n, dtype=np.int32) // 3 * 3
    doc = json.loads(json.dumps(chrome_trace(t0, t1, sm, class_id=cls, locals=loc, class_names={0: "TaskBcast"},
                                             unit=unit, pid=3, process_name="cuda:0")))
    ev = doc["traceEvents"]
    x = [e for e in ev if e["ph"] == "X"]
    assert len(x) == n
    assert sorted(e["args"]["task"] for e in x) == list(range(n))
    base = int(t0.min())
    for e in x:
        i = e["args"]["task"]
        assert e["pid"] == 3 and e["tid"] == int(sm[i])
        assert e["dur"] == int(t1[i] - t0[i]) / 1000.0          # microseconds, exact to the nanosecond
        assert e["ts"] == (int(t0[i]) - base) / 1000.0
        assert e["args"]["unit"] == int(unit[i])
        want = ("TaskBcast" if cls[i] == 0 else "class 1") + "(%d, %d)" % tuple(loc[i])
        assert e["name"] == want
    # one named row per SM that retired something, and nothing else
    rows = {e["tid"]: e["args"]["name"] for e in ev if e["ph"] == "M" and e["name"] == "thread_name"}
    assert rows == {int(s): "SM %d" % int(s) for s in np.unique(sm)}
    assert min(e["ts"] for e in x) == 0.0


def test_chrome_trace_skips_unrecorded_tasks():
    t0 = np.array([5, 0, 7], np.uint64)
    t1 = np.array([9, 0, 7], np.uint64)
    doc = chrome_trace(t0, t1, np.array([1, 0, 2], np.uint32))
    x = [e for e in doc["traceEvents"] if e["ph"] == "X"]
    assert [e["args"]["task"] for e in x] == [0, 2]
    assert [e["name"] for e in x] == ["task 0", "task 2"]
    assert x[1]["dur"] == 0.0 and x[1]["ts"] == 0.002


def test_window_trace_abi_argument_checks():
    lib = L.load()
    assert lib.pb2_engine_set_window_trace(None, 1) == L.PB2_ERR_BAD_PARAM
    assert lib.pb2_engine_set_window_trace(None, 0) == L.PB2_ERR_BAD_PARAM
    assert lib.pb2_window_trace(None, None, None, None, None) == L.PB2_ERR_BAD_PARAM


def test_device_engine_trace_mca_parameter():
    with R.Context(cuda_devices=(), dry_run=True) as ctx:
        v = C.c_int64(-1)
        assert ctx.l.pb2_mca_param_get_int(ctx.h, b"device_engine_trace", C.byref(v)) == 0 and v.value == 0
        assert ctx.l.pb2_mca_param_set_int(ctx.h, b"device_engine_trace", 1) == 0
        assert ctx.l.pb2_mca_param_get_int(ctx.h, b"device_engine_trace", C.byref(v)) == 0 and v.value == 1
    assert R.lib().pb2_taskpool_device_trace(None, None, None, None, None) == L.PB2_ERR_BAD_PARAM


def test_dry_run_pool_device_trace_is_zero():
    K, NB, tb = 16, 6, 4096
    host = np.zeros(K * tb // 4, np.int32)
    with R.Context(cuda_devices=(0,), dry_run=True, mca={"device_engine_trace": 1}) as ctx:
        dc = ctx.block_cyclic(4, tb // 4, 1, K * tb // 4, 1, mat=host)
        tp = C.c_void_p(ctx.l.pb2_ptg_ex05_broadcast_new(ctx.h, dc, K, NB))
        n = ctx.l.pb2_taskpool_nb_tasks(tp)
        before = ctx.device_trace(tp)
        assert np.all(before["device"] == -1)          # nothing ran yet
        ctx.wait()
        tr = ctx.device_trace(tp)
        _, dev = ctx.trace(tp)
        gpu = ctx.l.pb2_device_index(ctx.devices[0])
    assert n == K * (1 + NB // 2 + 1)
    assert len(dev) == n and np.all(dev == gpu)
    assert np.all(tr["device"] == gpu)
    for k in ("t_start_ns", "t_end_ns", "smid"):
        assert len(tr[k]) == n and np.all(tr[k] == 0), k
