"""Thin Python mirror of the L0 engine C ABI (include/pb2_engine.h).

Everything here is plumbing around ``libparsec_b200.so``: arrays are numpy structured arrays with
the exact C layouts, pointers are plain integers.  No compute happens in Python.
"""
import ctypes as C

import numpy as np

from . import _lib as L


def _check(rc, what, engine=None):
    if rc != L.PB2_SUCCESS:
        detail = ""
        if engine is not None and engine._h:
            detail = (L.load().pb2_engine_last_error(engine._h) or b"").decode()
        raise L.Pb2Error(rc, what, detail)


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def chrome_trace(t_start_ns, t_end_ns, smid, class_id=None, locals=None, class_names=None, unit=None, pid=0,
                 process_name=None):
    """Per-task device intervals (Window.trace, Context.device_trace) as a Chrome trace: {"traceEvents": [...]}, one
    complete ("X") event per recorded task on the row of its SM, times in microseconds from the earliest start.
    A task is named from class_id (through class_names when given) and locals; unit, when given, goes into each event's
    args.  Tasks with t_end_ns == 0 were not recorded and get no event.  pid: the trace process (one per device: every
    device has its own clock)."""
    t0 = np.asarray(t_start_ns, np.uint64)
    t1 = np.asarray(t_end_ns, np.uint64)
    sm = np.asarray(smid, np.uint32)
    rec = np.nonzero(t1 != 0)[0]
    base = int(t0[rec].min()) if len(rec) else 0
    events = []
    if process_name is not None:
        events.append({"ph": "M", "name": "process_name", "pid": pid, "tid": 0, "args": {"name": process_name}})
    for s in sorted({int(x) for x in sm[rec]}):
        events.append({"ph": "M", "name": "thread_name", "pid": pid, "tid": s, "args": {"name": "SM %d" % s}})
        events.append({"ph": "M", "name": "thread_sort_index", "pid": pid, "tid": s, "args": {"sort_index": s}})
    for i in rec:
        i = int(i)
        if class_id is None:
            name = "task %d" % i
        else:
            c = int(class_id[i])
            name = class_names.get(c, "class %d" % c) if class_names else "class %d" % c
        if locals is not None:
            name += "(%s)" % ", ".join(str(int(v)) for v in np.atleast_1d(locals[i]))
        args = {"task": i}
        if unit is not None:
            args["unit"] = int(unit[i])
        events.append({"ph": "X", "name": name, "pid": pid, "tid": int(sm[i]),
                       "ts": (int(t0[i]) - base) / 1000.0, "dur": (int(t1[i]) - int(t0[i])) / 1000.0, "args": args})
    return {"traceEvents": events, "displayTimeUnit": "ns"}


def chrome_trace_parts(records, class_id=None, class_names=None, pid=0, process_name=None):
    """Part records (Window.part_trace, Context.device_part_trace; PART_TRACE_DTYPE) as a Chrome trace: one row per SM,
    and per part up to three complete ("X") events -- "movein" from its pop to the end of its stage-in, the body (named
    from class_id[task] through class_names when given, else "exec") and "moveout" for its pushout.  Phases of zero
    length get no event, nor do records that were never stamped.  Times in microseconds from the earliest pop; args:
    task, part, nparts and, for movein and moveout, the bytes moved.  pid: the trace process (one per device)."""
    rec = np.asarray(records)
    rec = rec[rec["t_pop_ns"] != 0]
    base = int(rec["t_pop_ns"].min()) if len(rec) else 0
    events = []
    if process_name is not None:
        events.append({"ph": "M", "name": "process_name", "pid": pid, "tid": 0, "args": {"name": process_name}})
    for s in sorted({int(x) for x in rec["smid"]}):
        events.append({"ph": "M", "name": "thread_name", "pid": pid, "tid": s, "args": {"name": "SM %d" % s}})
        events.append({"ph": "M", "name": "thread_sort_index", "pid": pid, "tid": s, "args": {"sort_index": s}})
    for r in rec:
        task = int(r["task"])
        if class_id is None:
            body = "exec"
        else:
            c = int(class_id[task])
            body = class_names.get(c, "class %d" % c) if class_names else "class %d" % c
        args = {"task": task, "part": int(r["part"]), "nparts": int(r["nparts"])}
        t = [int(r["t_pop_ns"]), int(r["t_in_ns"]), int(r["t_exec_ns"]), int(r["t_out_ns"])]
        for (name, t0, t1, nbytes) in (("movein", t[0], t[1], int(r["in_bytes"])), (body, t[1], t[2], None),
                                       ("moveout", t[2], t[3], int(r["out_bytes"]))):
            if t1 <= t0:
                continue
            a = dict(args) if nbytes is None else dict(args, bytes=nbytes)
            events.append({"ph": "X", "name": name, "pid": pid, "tid": int(r["smid"]),
                           "ts": (t0 - base) / 1000.0, "dur": (t1 - t0) / 1000.0, "args": a})
    return {"traceEvents": events, "displayTimeUnit": "ns"}


class Engine:
    """One engine per GPU (the reference's parsec_device_cuda_module_t, device_cuda.h:43-48).

    queue_policy: 0 (default) pops ready tasks in FIFO order; 1 pops higher ``priority`` first, FIFO among equal
    priorities, through 16 priority lanes (exact with at most 16 distinct priorities in a window; see
    pb2_engine_params_t::queue_policy in include/pb2_engine.h).  Policy 1 is refused for shared windows."""

    def __init__(self, cuda_device=0, workers_per_sm=0, threads=0, max_workers=0, stage_mode=0,
                 queue_policy=0, timeout_ms=0, gemm_mode=0, part_bytes=0, read_groups=0,
                 fuse_readers=0, window_trace=False):
        self._lib = L.load()
        self._h = C.c_void_p()
        p = L.EngineParams(workers_per_sm, threads, max_workers, stage_mode, queue_policy, timeout_ms, gemm_mode, part_bytes,
                           read_groups, fuse_readers)
        rc = self._lib.pb2_engine_create(C.byref(self._h), cuda_device, C.byref(p))
        if rc != L.PB2_SUCCESS:
            self._h = C.c_void_p()
            raise L.Pb2Error(rc, "pb2_engine_create")
        self._allocs = []
        if window_trace:
            self.set_window_trace(True)

    def info(self):
        i = L.EngineInfo()
        _check(self._lib.pb2_engine_info(self._h, C.byref(i)), "pb2_engine_info", self)
        return {f[0]: getattr(i, f[0]) for f in L.EngineInfo._fields_ if f[0] != "reserved"}

    def malloc(self, nbytes, ipc=False):
        """Device memory, compressible where the device supports it and nbytes is one granule or more (info()'s
        slab_compressible tells which); ipc=True gives cudaMalloc memory, which ipc_export can export."""
        p = C.c_void_p()
        _check(self._lib.pb2_engine_malloc_ex(self._h, nbytes, L.MALLOC_IPC if ipc else 0, C.byref(p)), "pb2_engine_malloc_ex", self)
        self._allocs.append(p.value)
        return p.value

    def free(self, ptr):
        _check(self._lib.pb2_engine_free(self._h, C.c_void_p(ptr)), "pb2_engine_free", self)
        if ptr in self._allocs:
            self._allocs.remove(ptr)

    def host_register(self, arr):
        """cudaHostRegister a numpy array (memory_register, device_cuda_module.c:183); returns the device alias."""
        alias = C.c_void_p()
        _check(self._lib.pb2_engine_host_register(self._h, _ptr(arr), arr.nbytes, C.byref(alias)),
               "pb2_engine_host_register", self)
        return alias.value

    def host_unregister(self, arr):
        _check(self._lib.pb2_engine_host_unregister(self._h, _ptr(arr)), "pb2_engine_host_unregister", self)

    def h2d(self, dev_ptr, arr):
        arr = np.ascontiguousarray(arr)
        _check(self._lib.pb2_engine_memcpy_h2d(self._h, C.c_void_p(dev_ptr), _ptr(arr), arr.nbytes), "h2d", self)
        self.synchronize()

    def d2h(self, arr, dev_ptr):
        assert arr.flags["C_CONTIGUOUS"]
        _check(self._lib.pb2_engine_memcpy_d2h(self._h, _ptr(arr), C.c_void_p(dev_ptr), arr.nbytes), "d2h", self)
        return arr

    def use_stream(self, cuda_stream):
        """Enqueue engine work on a caller-owned stream (int cudaStream_t, e.g. torch.cuda.current_stream().cuda_stream)."""
        if not cuda_stream:
            raise ValueError("use_stream needs a real stream handle (the legacy default stream is 0: create a torch.cuda.Stream)")
        _check(self._lib.pb2_engine_set_stream(self._h, C.c_void_p(cuda_stream)), "pb2_engine_set_stream", self)

    def set_shared_windows(self, on=True, next_rs_begin=None):
        """next_rs_begin: int32 remote out-edge CSR of the NEXT window (kept alive by the caller until it is created)."""
        self._rs_keep = None if next_rs_begin is None else np.ascontiguousarray(next_rs_begin, np.int32)
        _check(self._lib.pb2_engine_set_shared_windows(self._h, 1 if on else 0, _ptr(self._rs_keep)), "set_shared_windows", self)

    def set_part_bytes(self, part_bytes):
        _check(self._lib.pb2_engine_set_part_bytes(self._h, part_bytes), "set_part_bytes", self)

    def set_window_trace(self, on=True):
        """Windows created from now on record per-task device time stamps (Window.trace)."""
        _check(self._lib.pb2_engine_set_window_trace(self._h, 1 if on else 0), "set_window_trace", self)

    def link_bodies(self, image, format, sliceable=0, checked=0, gemm_windows=False, readers=0, reader_groups=0,
                    gemm_bodies=0, gemm_body_entry=False):
        """Link the application's device bodies (include/pb2_device_body.h) into this engine's HBM window kernel, once:
        image is PTX text (format L.IMAGE_PTX) or a relocatable sm_90a cubin (L.IMAGE_CUBIN), as bytes; bit i of
        sliceable lets tasks of body L.BODY_LINKED_0 + i be cut into byte-slice parts, and bit i of checked (a subset
        of sliceable) declares that body's checked form, so that it runs fused with its read group.  gemm_windows
        (L.LINK_GEMM_WINDOWS) links the GEMM window kernel too, so that GEMM windows may hold linked tasks.  Bit i of
        readers (L.LINK_READERS, a subset of sliceable) declares that body a reader, so that its tasks run in read
        groups and their results add up over parts.  Bit i of reader_groups (L.LINK_READER_GROUPS, a subset of
        readers) declares that reader's group form, which the image then defines: a read group calls it once per chunk
        for all such members.  Bit i of gemm_bodies (L.LINK_GEMM_BODIES, with gemm_windows, disjoint from sliceable)
        declares that body a GEMM-worker body: it runs in GEMM windows only, as one part, with the GEMM worker's
        operand ring (PB2_GEMM_BODY_SMEM_BYTES) as its scratch.  gemm_body_entry (L.LINK_GEMM_BODY_ENTRY, with a nonzero
        gemm_bodies) calls those bodies through the image's pb2_linked_gemm_body, which only the GEMM window kernels
        reach, so it has their 168 registers per thread instead of the HBM kernels' 80."""
        image = bytes(image)
        flags = ((L.LINK_GEMM_WINDOWS if gemm_windows else 0) | L.LINK_READERS(readers) | L.LINK_READER_GROUPS(reader_groups)
                 | L.LINK_GEMM_BODIES(gemm_bodies) | (L.LINK_GEMM_BODY_ENTRY if gemm_body_entry else 0))
        _check(self._lib.pb2_engine_link_bodies_ex(self._h, image, len(image), format, sliceable, checked, flags),
               "pb2_engine_link_bodies_ex", self)

    def set_gemm_body_parts(self, body, nparts):
        """Run every task of GEMM-worker body `body` (a bit of link_bodies' gemm_bodies) as nparts parts, 1 ..
        L.GEMM_BODY_MAX_PARTS, in the GEMM windows created from now on.  Each part gets the task's whole tiles and its
        part index, and the body splits the work by it (include/pb2_device_body.h).  The default is 1."""
        _check(self._lib.pb2_engine_set_gemm_body_parts(self._h, body, nparts), "set_gemm_body_parts", self)

    def linked_info(self):
        """What the linker made of the linked kernel: registers and local bytes per thread, static shared memory per
        CTA, and the workers a linked window runs."""
        v = [C.c_int32() for _ in range(4)]
        _check(self._lib.pb2_engine_linked_info(self._h, *[C.byref(x) for x in v]), "pb2_engine_linked_info", self)
        return dict(zip(("regs", "local_bytes", "static_smem", "nworkers"), (x.value for x in v)))

    def linked_gemm_info(self):
        """linked_info for the linked GEMM window kernel (link_bodies(..., gemm_windows=True))."""
        v = [C.c_int32() for _ in range(4)]
        _check(self._lib.pb2_engine_linked_gemm_info(self._h, *[C.byref(x) for x in v]), "pb2_engine_linked_gemm_info", self)
        return dict(zip(("regs", "local_bytes", "static_smem", "nworkers"), (x.value for x in v)))

    def ipc_export(self, dev_ptr):
        h = (C.c_ubyte * 64)()
        _check(self._lib.pb2_engine_ipc_export(self._h, C.c_void_p(dev_ptr), h), "ipc_export", self)
        return bytes(h)

    def ipc_open(self, handle):
        h = (C.c_ubyte * 64).from_buffer_copy(handle)
        p = C.c_void_p()
        _check(self._lib.pb2_engine_ipc_open(self._h, h, C.byref(p)), "ipc_open", self)
        return p.value

    def synchronize(self):
        _check(self._lib.pb2_engine_synchronize(self._h), "pb2_engine_synchronize", self)

    def window(self, kind, tasks, succ, tiles, ready):
        return Window(self, kind, tasks, succ, tiles, ready)

    def close(self):
        if self._h:
            for p in list(self._allocs):
                self._lib.pb2_engine_free(self._h, C.c_void_p(p))
            self._allocs = []
            self._lib.pb2_engine_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Window:
    """One DAG window resident on the GPU: create once, launch/wait any number of times."""

    def __init__(self, engine, kind, tasks, succ, tiles, ready):
        self.engine = engine
        self._lib = engine._lib
        tasks = np.ascontiguousarray(tasks, dtype=L.TASK_DTYPE)
        succ = np.ascontiguousarray(succ, dtype=np.uint32)
        tiles = np.ascontiguousarray(tiles, dtype=L.TILE_DTYPE)
        ready = np.ascontiguousarray(ready, dtype=np.int32)
        self.ntasks, self.ntiles = len(tasks), len(tiles)
        self._h = C.c_void_p()
        rc = self._lib.pb2_window_create(engine._h, C.byref(self._h), kind,
                                         _ptr(tasks), len(tasks), _ptr(succ), len(succ),
                                         _ptr(tiles), len(tiles), _ptr(ready), len(ready))
        if rc != L.PB2_SUCCESS:
            self._h = C.c_void_p()
        _check(rc, "pb2_window_create", engine)

    def launch(self):
        _check(self._lib.pb2_window_launch(self._h), "pb2_window_launch", self.engine)

    def arm(self):
        _check(self._lib.pb2_window_arm(self._h), "pb2_window_arm", self.engine)

    def start(self):
        _check(self._lib.pb2_window_start(self._h), "pb2_window_start", self.engine)

    def export(self):
        h = L.WindowHandle()
        _check(self._lib.pb2_window_export(self._h, C.byref(h)), "pb2_window_export", self.engine)
        return bytes(h)

    def task_entries(self):
        out = np.empty(self.ntasks, np.int32)
        _check(self._lib.pb2_window_task_entries(self._h, _ptr(out)), "pb2_window_task_entries", self.engine)
        return out

    def set_push(self, ps_begin, push):
        """Producer-side pushes (pb2_window_set_push): call after set_remote."""
        ps_begin = np.ascontiguousarray(ps_begin, np.int32)
        push = np.ascontiguousarray(push, L.PUSH_DTYPE)
        _check(self._lib.pb2_window_set_push(self._h, _ptr(ps_begin), _ptr(push), len(push)), "pb2_window_set_push", self.engine)

    def set_remote(self, my_rank, handles, rs_begin, rs_rank, rs_target):
        """handles: list of bytes (one exported WindowHandle per rank)."""
        arr = (L.WindowHandle * len(handles))(*[L.WindowHandle.from_buffer_copy(h) for h in handles])
        rs_begin = np.ascontiguousarray(rs_begin, np.int32)
        rs_rank = np.ascontiguousarray(rs_rank, np.int32)
        rs_target = np.ascontiguousarray(rs_target, np.uint32)
        _check(self._lib.pb2_window_set_remote(self._h, my_rank, len(handles), arr, _ptr(rs_begin), _ptr(rs_rank),
                                               _ptr(rs_target), len(rs_rank)), "pb2_window_set_remote", self.engine)

    def wait(self):
        st = L.WindowStats()
        rc = self._lib.pb2_window_wait(self._h, C.byref(st))
        self.stats = {f[0]: getattr(st, f[0]) for f in L.WindowStats._fields_}
        _check(rc, "pb2_window_wait", self.engine)
        return self.stats

    def run(self):
        self.launch()
        return self.wait()

    def results(self):
        n = self.ntasks
        out = {
            "retire_order": np.empty(n, np.int32), "start_seq": np.empty(n, np.uint32),
            "end_seq": np.empty(n, np.uint32), "seen_version": np.empty((n, L.MAX_FLOWS), np.uint32),
            "result": np.empty(n, np.uint64), "worker": np.empty(n, np.int32),
            "tiles": np.empty(self.ntiles, L.TILE_DTYPE),
        }
        _check(self._lib.pb2_window_results(self._h, _ptr(out["retire_order"]), _ptr(out["start_seq"]),
                                            _ptr(out["end_seq"]), _ptr(out["seen_version"]),
                                            _ptr(out["result"]), _ptr(out["worker"]), _ptr(out["tiles"])),
               "pb2_window_results", self.engine)
        return out

    def trace(self):
        """Device time stamps of the last launch (a window created with trace on; pb2_window_trace): per task the
        interval of its scheduling entity in %globaltimer ns, the SM that retired it and the task leading the entity."""
        n = self.ntasks
        out = {"t_start_ns": np.empty(n, np.uint64), "t_end_ns": np.empty(n, np.uint64),
               "smid": np.empty(n, np.uint32), "unit": np.empty(n, np.int32)}
        _check(self._lib.pb2_window_trace(self._h, _ptr(out["t_start_ns"]), _ptr(out["t_end_ns"]), _ptr(out["smid"]),
                                          _ptr(out["unit"])), "pb2_window_trace", self.engine)
        return out

    def part_trace(self):
        """Part records of the last launch (a window created with trace on; pb2_window_part_trace): one PART_TRACE_DTYPE
        record per ring entry, by leading task, then part."""
        n = C.c_int32(0)
        _check(self._lib.pb2_window_part_trace(self._h, None, 0, C.byref(n)), "pb2_window_part_trace", self.engine)
        out = np.zeros(n.value, L.PART_TRACE_DTYPE)
        _check(self._lib.pb2_window_part_trace(self._h, _ptr(out), n.value, C.byref(n)), "pb2_window_part_trace",
               self.engine)
        return out

    def close(self):
        if self._h:
            self._lib.pb2_window_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
