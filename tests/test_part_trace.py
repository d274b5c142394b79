"""Part records without a GPU: the C layout of pb2_part_trace_t against PART_TRACE_DTYPE, the Chrome-trace writer on
synthetic records, the C ABI's argument checks and the records of a dry-run pool (no window ran: none)."""
import ctypes as C
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

from parsec_b200 import _lib as L
from parsec_b200 import runtime as R
from parsec_b200.engine import chrome_trace_parts

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

LAYOUT_C = r"""
#include <stddef.h>
#include <stdio.h>
#include "pb2_engine.h"
#define F(m) printf(#m " %zu\n", offsetof(pb2_part_trace_t, m))
int main(void) {
    printf("size %zu\n", sizeof(pb2_part_trace_t));
    F(t_pop_ns); F(t_in_ns); F(t_exec_ns); F(t_out_ns); F(in_bytes); F(out_bytes);
    F(task); F(part); F(nparts); F(smid); F(flags);
    printf("waited %u retired %u\n", PB2_PART_WAITED_INPUT, PB2_PART_RETIRED);
    return 0;
}
"""


@pytest.mark.skipif(shutil.which("gcc") is None, reason="needs gcc")
def test_part_trace_layout_matches_c(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text(LAYOUT_C)
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src),
                           "-o", str(exe)])
    got = dict(line.rsplit(" ", 1) for line in subprocess.check_output([str(exe)], text=True).splitlines()[:-1])
    assert int(got.pop("size")) == L.PART_TRACE_DTYPE.itemsize == 64
    assert {k: int(v) for k, v in got.items()} == {k: L.PART_TRACE_DTYPE.fields[k][1] for k in L.PART_TRACE_DTYPE.names}
    last = subprocess.check_output([str(exe)], text=True).splitlines()[-1].split()
    assert (int(last[1]), int(last[3])) == (L.PART_WAITED_INPUT, L.PART_RETIRED)


def _records(rows):
    rec = np.zeros(len(rows), L.PART_TRACE_DTYPE)
    for i, r in enumerate(rows):
        for k, v in r.items():
            rec[i][k] = v
    return rec


def test_chrome_trace_parts_phases():
    base = 1_000_000
    rec = _records([
        # a host-fed part: movein, body and moveout
        dict(t_pop_ns=base, t_in_ns=base + 3000, t_exec_ns=base + 5000, t_out_ns=base + 5500, in_bytes=65536,
             out_bytes=4096, task=4, part=1, nparts=3, smid=7, flags=L.PART_WAITED_INPUT),
        # a resident part that pushes nothing: its empty movein and moveout are dropped
        dict(t_pop_ns=base + 100, t_in_ns=base + 100, t_exec_ns=base + 2100, t_out_ns=base + 2100, task=2, part=0,
             nparts=1, smid=3, flags=L.PART_RETIRED),
        # never ran (a failed run): no event
        dict(task=9, part=0, nparts=1),
    ])
    cls = np.array([0, 0, 1, 0, 2, 0, 0, 0, 0, 0], np.int32)
    doc = json.loads(json.dumps(chrome_trace_parts(rec, class_id=cls, class_names={2: "TaskBcast"}, pid=1,
                                                   process_name="cuda:0")))
    ev = doc["traceEvents"]
    x = [e for e in ev if e["ph"] == "X"]
    assert [(e["name"], e["tid"], e["ts"], e["dur"]) for e in x] == [
        ("movein", 7, 0.0, 3.0), ("TaskBcast", 7, 3.0, 2.0), ("moveout", 7, 5.0, 0.5),
        ("class 1", 3, 0.1, 2.0)]
    assert all(e["pid"] == 1 for e in ev)
    assert x[0]["args"] == {"task": 4, "part": 1, "nparts": 3, "bytes": 65536}
    assert x[1]["args"] == {"task": 4, "part": 1, "nparts": 3}
    assert x[2]["args"]["bytes"] == 4096
    assert x[3]["args"] == {"task": 2, "part": 0, "nparts": 1}
    rows = {e["tid"]: e["args"]["name"] for e in ev if e["ph"] == "M" and e["name"] == "thread_name"}
    assert rows == {3: "SM 3", 7: "SM 7"}
    names = [e for e in ev if e["ph"] == "M" and e["name"] == "process_name"]
    assert names == [{"ph": "M", "name": "process_name", "pid": 1, "tid": 0, "args": {"name": "cuda:0"}}]


def test_chrome_trace_parts_without_classes():
    rec = _records([dict(t_pop_ns=10, t_in_ns=10, t_exec_ns=30, t_out_ns=30, task=0, part=0, nparts=1, smid=5)])
    x = [e for e in chrome_trace_parts(rec)["traceEvents"] if e["ph"] == "X"]
    assert [(e["name"], e["ts"], e["dur"]) for e in x] == [("exec", 0.0, 0.02)]
    assert chrome_trace_parts(np.zeros(0, L.PART_TRACE_DTYPE))["traceEvents"] == []


def test_part_trace_abi_argument_checks():
    lib = L.load()
    n = C.c_int32(-1)
    assert lib.pb2_window_part_trace(None, None, 0, C.byref(n)) == L.PB2_ERR_BAD_PARAM
    rl = R.lib()
    assert rl.pb2_taskpool_device_part_trace(None, None, None, 0, C.byref(n)) == L.PB2_ERR_BAD_PARAM


def test_dry_run_pool_has_no_part_records():
    K, NB, tb = 16, 6, 4096
    host = np.zeros(K * tb // 4, np.int32)
    with R.Context(cuda_devices=(0,), dry_run=True, mca={"device_engine_trace": 1}) as ctx:
        dc = ctx.block_cyclic(4, tb // 4, 1, K * tb // 4, 1, mat=host)
        tp = C.c_void_p(ctx.l.pb2_ptg_ex05_broadcast_new(ctx.h, dc, K, NB))
        ctx.wait()
        rec, dev = ctx.device_part_trace(tp)
        n = C.c_int32(-1)
        assert ctx.l.pb2_taskpool_device_part_trace(tp, None, None, 0, C.byref(n)) == 0 and n.value == 0
    assert rec.dtype == L.PART_TRACE_DTYPE and len(rec) == 0 and len(dev) == 0
