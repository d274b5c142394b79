"""ctypes mirror of include/pb2_parsec.h: the reference-shaped host API (context, device modules, data,
2D block-cyclic collections, DTD and PTG task pools).  Thin plumbing; every call lands in libparsec_b200.so."""
import ctypes as C

import numpy as np

from . import _lib as L

HOOK_RETURN_DONE, HOOK_RETURN_AGAIN, HOOK_RETURN_NEXT, HOOK_RETURN_DISABLE, HOOK_RETURN_ASYNC, HOOK_RETURN_ERROR = 0, -1, -2, -3, -4, -5
DEV_CPU, DEV_RECURSIVE, DEV_CUDA = 0x01, 0x02, 0x04
ADVICE_PREFETCH, ADVICE_PREFERRED_DEVICE, ADVICE_WARMUP = 1, 2, 3
COHERENCY_INVALID, COHERENCY_OWNED, COHERENCY_EXCLUSIVE, COHERENCY_SHARED = 0, 1, 2, 4
INPUT, OUTPUT, INOUT = 0x100000, 0x200000, 0x300000
AFFINITY, DONT_TRACK, PUSHOUT = 1 << 16, 1 << 17, 1 << 18
MAX_DEVICES = 16


class DeviceStats(C.Structure):
    _fields_ = [("executed_tasks", C.c_uint64), ("required_data_in", C.c_uint64), ("required_data_out", C.c_uint64),
                ("data_out_to_host", C.c_uint64), ("nb_data_faults", C.c_uint64), ("nb_evictions", C.c_uint64),
                ("data_in_from_device", C.c_uint64 * MAX_DEVICES), ("device_load", C.c_int64),
                ("time_estimate_default", C.c_int64), ("gflops_fp16", C.c_int64), ("gflops_fp32", C.c_int64),
                ("gflops_fp64", C.c_int64), ("gflops_tf32", C.c_int64), ("windows_launched", C.c_uint64),
                ("tasks_released_on_device", C.c_uint64), ("kernel_ms_total", C.c_double)]


# every extern "C" symbol include/pb2_parsec.h declares
PARSEC_SYMBOLS = [
    "pb2_init", "pb2_fini", "pb2_mca_param_set_int", "pb2_mca_param_get_int", "pb2_device_cuda_module_init",
    "pb2_mca_device_registration_complete", "pb2_nb_devices", "pb2_mca_device_get", "pb2_device_get_stats",
    "pb2_devices_statistics_string", "pb2_device_link_bodies", "pb2_device_link_bodies_checked",
    "pb2_device_link_bodies_ex", "pb2_device_set_gemm_body_parts", "pb2_device_gemm_body_parts",
    "pb2_device_index", "pb2_device_type", "pb2_device_memory_register", "pb2_device_memory_unregister",
    "pb2_device_memory_release", "pb2_device_data_advise", "pb2_device_taskpool_register",
    "pb2_device_taskpool_unregister", "pb2_device_kernel_scheduler", "pb2_device_zone_malloc", "pb2_device_zone_free",
    "pb2_device_zone_in_use", "pb2_device_lru_sizes", "pb2_select_best_device", "pb2_data_create",
    "pb2_data_new_temporary", "pb2_data_start_transfer_ownership_to_copy", "pb2_data_end_transfer_ownership_to_copy",
    "pb2_data_get_copy", "pb2_data_copy_attach", "pb2_data_copy_state", "pb2_data_owner_device", "pb2_data_preferred_device",
    "pb2_matrix_block_cyclic_new", "pb2_data_collection_free", "pb2_data_collection_set_mat", "pb2_dc_rank_of",
    "pb2_dc_data_of", "pb2_dc_data_key", "pb2_dc_position", "pb2_dc_info", "pb2_dc_register_memory",
    "pb2_dc_distribute_on_devices", "pb2_dc_host_write_all", "pb2_context_add_taskpool", "pb2_context_start", "pb2_context_wait",
    "pb2_taskpool_wait", "pb2_taskpool_free", "pb2_taskpool_nb_tasks", "pb2_taskpool_set_device_types",
    "pb2_taskpool_completion_trace", "pb2_taskpool_device_trace", "pb2_taskpool_device_part_trace", "pb2_taskpool_task_info", "pb2_taskpool_export_window", "pb2_dtd_taskpool_new",
    "pb2_dtd_tile_of", "pb2_dtd_tile_new", "pb2_dtd_tile_data", "pb2_dtd_create_task_class",
    "pb2_dtd_task_class_add_chore", "pb2_dtd_insert_task_with_task_class", "pb2_dtd_data_flush_all",
    "pb2_dtd_task_class_add_submit", "pb2_gpu_task_flow_ptr", "pb2_gpu_task_flow_bytes", "pb2_gpu_task_iparam",
    "pb2_dtd_data_flush", "pb2_ptg_ex02_chain_new", "pb2_ptg_ex05_broadcast_new", "pb2_ptg_rtt_new",
    "pb2_ptg_ep_new", "pb2_ptg_pingpong_new", "pb2_ptg_get_best_device_new", "pb2_ptg_cholesky_shape_new",
    "pb2_app_dtd_simple_gemm",
]

_bound = False


def lib():
    global _bound
    l = L.load()
    if _bound:
        return l
    vp, i32, P = C.c_void_p, C.c_int32, C.POINTER
    sig = {
        "pb2_init": (C.c_int, [P(vp), C.c_int]), "pb2_fini": (C.c_int, [P(vp)]),
        "pb2_mca_param_set_int": (C.c_int, [vp, C.c_char_p, C.c_int64]),
        "pb2_mca_param_get_int": (C.c_int, [vp, C.c_char_p, P(C.c_int64)]),
        "pb2_device_cuda_module_init": (C.c_int, [vp, C.c_int, C.c_int, P(vp)]),
        "pb2_mca_device_registration_complete": (C.c_int, [vp]), "pb2_nb_devices": (C.c_int, [vp]),
        "pb2_mca_device_get": (vp, [vp, C.c_int]), "pb2_device_get_stats": (C.c_int, [vp, P(DeviceStats)]),
        "pb2_devices_statistics_string": (C.c_int, [vp, C.c_char_p, C.c_size_t]),
        "pb2_device_index": (C.c_int, [vp]), "pb2_device_type": (C.c_int, [vp]),
        "pb2_device_link_bodies": (C.c_int, [vp, C.c_char_p, C.c_size_t, C.c_int, C.c_uint32]),
        "pb2_device_link_bodies_checked": (C.c_int, [vp, C.c_char_p, C.c_size_t, C.c_int, C.c_uint32, C.c_uint32]),
        "pb2_device_link_bodies_ex": (C.c_int, [vp, C.c_char_p, C.c_size_t, C.c_int, C.c_uint32, C.c_uint32, C.c_uint32]),
        "pb2_device_set_gemm_body_parts": (C.c_int, [vp, C.c_int, C.c_int32]),
        "pb2_device_gemm_body_parts": (C.c_int, [vp, C.c_int]),
        "pb2_device_memory_register": (C.c_int, [vp, vp, vp, C.c_size_t]),
        "pb2_device_memory_unregister": (C.c_int, [vp, vp, vp]), "pb2_device_memory_release": (C.c_int, [vp]),
        "pb2_device_data_advise": (C.c_int, [vp, vp, C.c_int]),
        "pb2_device_taskpool_register": (C.c_int, [vp, vp]), "pb2_device_taskpool_unregister": (C.c_int, [vp, vp]),
        "pb2_device_kernel_scheduler": (C.c_int, [vp, vp, vp]),
        "pb2_device_zone_malloc": (vp, [vp, C.c_size_t]), "pb2_device_zone_free": (C.c_int, [vp, vp]),
        "pb2_device_zone_in_use": (C.c_size_t, [vp]), "pb2_device_lru_sizes": (C.c_int, [vp, P(C.c_int), P(C.c_int)]),
        "pb2_select_best_device": (C.c_int, [vp, vp]),
        "pb2_data_create": (vp, [vp, C.c_uint64, vp, C.c_size_t]), "pb2_data_new_temporary": (vp, [vp, C.c_size_t]),
        "pb2_data_start_transfer_ownership_to_copy": (C.c_int, [vp, vp, C.c_uint8, C.c_uint8]),
        "pb2_data_end_transfer_ownership_to_copy": (None, [vp, C.c_uint8, C.c_uint8]),
        "pb2_data_get_copy": (vp, [vp, C.c_int]), "pb2_data_copy_attach": (vp, [vp, C.c_int]), "pb2_data_copy_state": (C.c_int, [vp, C.c_int, P(i32)]),
        "pb2_data_owner_device": (C.c_int, [vp]), "pb2_data_preferred_device": (C.c_int, [vp]),
        "pb2_matrix_block_cyclic_new": (vp, [vp] + [C.c_int] * 16),
        "pb2_data_collection_free": (C.c_int, [vp]), "pb2_data_collection_set_mat": (C.c_int, [vp, vp]),
        "pb2_dc_rank_of": (C.c_uint32, [vp, C.c_int, C.c_int]), "pb2_dc_data_of": (vp, [vp, C.c_int, C.c_int]),
        "pb2_dc_data_key": (C.c_uint64, [vp, C.c_int, C.c_int]), "pb2_dc_position": (C.c_int, [vp, C.c_int, C.c_int]),
        "pb2_dc_info": (C.c_int, [vp, P(C.c_int64)]), "pb2_dc_register_memory": (C.c_int, [vp, vp]),
        "pb2_dc_distribute_on_devices": (C.c_int, [vp]), "pb2_dc_host_write_all": (C.c_int, [vp]),
        "pb2_context_add_taskpool": (C.c_int, [vp, vp]), "pb2_context_start": (C.c_int, [vp]),
        "pb2_context_wait": (C.c_int, [vp]), "pb2_taskpool_wait": (C.c_int, [vp]), "pb2_taskpool_free": (C.c_int, [vp]),
        "pb2_taskpool_nb_tasks": (C.c_int, [vp]), "pb2_taskpool_set_device_types": (C.c_int, [vp, C.c_int]),
        "pb2_taskpool_completion_trace": (C.c_int, [vp, vp, vp, i32]),
        "pb2_taskpool_device_trace": (C.c_int, [vp, vp, vp, vp, vp]),
        "pb2_taskpool_device_part_trace": (C.c_int, [vp, vp, vp, i32, P(i32)]),
        "pb2_taskpool_task_info": (C.c_int, [vp, vp, vp, vp, vp]),
        "pb2_taskpool_export_window": (C.c_int, [vp, vp, vp, P(i32), vp, P(i32), vp, P(i32), vp, P(i32), vp]),
        "pb2_dtd_taskpool_new": (vp, [vp]), "pb2_dtd_tile_of": (vp, [vp, vp, C.c_uint64]),
        "pb2_dtd_tile_new": (vp, [vp, C.c_size_t]), "pb2_dtd_tile_data": (vp, [vp]),
        "pb2_dtd_create_task_class": (vp, [vp, C.c_char_p, C.c_int, vp]),
        "pb2_dtd_task_class_add_chore": (C.c_int, [vp, vp, C.c_int, C.c_int, vp]),
        "pb2_dtd_insert_task_with_task_class": (C.c_int, [vp, vp, C.c_int, C.c_int, vp, vp, vp, C.c_float]),
        "pb2_dtd_task_class_add_submit": (C.c_int, [vp, vp, GPU_SUBMIT]),
        "pb2_gpu_task_flow_ptr": (vp, [vp, vp, C.c_int]), "pb2_gpu_task_flow_bytes": (C.c_size_t, [vp, C.c_int]),
        "pb2_gpu_task_iparam": (P(i32), [vp]),
        "pb2_dtd_data_flush_all": (C.c_int, [vp, vp]), "pb2_dtd_data_flush": (C.c_int, [vp, vp]),
        "pb2_ptg_ex02_chain_new": (vp, [vp, C.c_int]), "pb2_ptg_ex05_broadcast_new": (vp, [vp, vp, C.c_int, C.c_int]),
        "pb2_ptg_rtt_new": (vp, [vp, vp, C.c_int, C.c_int, C.c_int]), "pb2_ptg_ep_new": (vp, [vp, vp, C.c_int, C.c_int]),
        "pb2_ptg_pingpong_new": (vp, [vp, vp, C.c_int, P(i32)]), "pb2_ptg_get_best_device_new": (vp, [vp, vp, vp]),
        "pb2_ptg_cholesky_shape_new": (vp, [vp, vp, C.c_int]),
        "pb2_app_dtd_simple_gemm": (C.c_int, [vp, vp, vp, vp, C.c_int, P(C.c_double), P(vp)]),
    }
    for name, (res, args) in sig.items():
        f = getattr(l, name)
        f.restype, f.argtypes = res, args
    _bound = True
    return l


# pb2_gpu_submit_t: int submit(pb2_device_module_t* dev, pb2_gpu_task_t* gpu_task, void* cuda_stream)
GPU_SUBMIT = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p)
# pb2_cpu_hook_t: int hook(pb2_htask_t* task, void** flow_ptrs, const int32_t* iparam, float fparam)
CPU_HOOK = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int32), C.c_float)


def _chk(rc, what):
    if rc != L.PB2_SUCCESS:
        raise L.Pb2Error(rc, what)


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class Context:
    """parsec_context_t: devices 0 (cpu), 1 (recursive), then one module per GPU given in `cuda_devices`."""

    def __init__(self, nb_cores=1, cuda_devices=(0,), dry_run=False, mca=None):
        self.l = lib()
        self.h = C.c_void_p()
        _chk(self.l.pb2_init(C.byref(self.h), nb_cores), "pb2_init")
        for k, v in (mca or {}).items():
            _chk(self.l.pb2_mca_param_set_int(self.h, k.encode(), int(v)), f"mca {k}")
        self.devices = []
        for ci in cuda_devices:
            m = C.c_void_p()
            rc = self.l.pb2_device_cuda_module_init(self.h, ci, 1 if dry_run else 0, C.byref(m))
            if rc != L.PB2_SUCCESS:
                self.l.pb2_fini(C.byref(self.h))
                raise L.Pb2Error(rc, "pb2_device_cuda_module_init")
            self.devices.append(m)
        _chk(self.l.pb2_mca_device_registration_complete(self.h), "registration_complete")
        self._keep = []

    def device(self, index):
        return C.c_void_p(self.l.pb2_mca_device_get(self.h, index))

    def statistics_table(self):
        n = self.l.pb2_devices_statistics_string(self.h, None, 0)
        buf = C.create_string_buffer(n)
        self.l.pb2_devices_statistics_string(self.h, buf, n)
        return buf.value.decode()

    def link_bodies(self, dev, image, format, sliceable=0, checked=0, gemm_windows=False, readers=0, reader_groups=0,
                    gemm_bodies=0, gemm_body_entry=False):
        """Link the application's device bodies into module dev's engine before its first window (Engine.link_bodies;
        a dry-run module checks the arguments and records the link).  gemm_windows: GEMM chains and linked tasks may
        then share a window.  readers, reader_groups: the bodies declared readers, and the readers declared with the
        group form (Engine.link_bodies).  gemm_bodies: the GEMM-worker bodies (Engine.link_bodies), whose tasks then
        always run in GEMM windows.  gemm_body_entry: call them through pb2_linked_gemm_body (Engine.link_bodies)."""
        image = bytes(image)
        flags = ((L.LINK_GEMM_WINDOWS if gemm_windows else 0) | L.LINK_READERS(readers) | L.LINK_READER_GROUPS(reader_groups)
                 | L.LINK_GEMM_BODIES(gemm_bodies) | (L.LINK_GEMM_BODY_ENTRY if gemm_body_entry else 0))
        _chk(self.l.pb2_device_link_bodies_ex(dev, image, len(image), format, sliceable, checked, flags),
             "pb2_device_link_bodies_ex")

    def set_gemm_body_parts(self, dev, body, nparts):
        """Run every task of GEMM-worker body `body` as nparts parts in the windows module dev builds afterwards
        (Engine.set_gemm_body_parts; a dry-run module checks the arguments and records the count)."""
        _chk(self.l.pb2_device_set_gemm_body_parts(dev, body, nparts), "pb2_device_set_gemm_body_parts")

    def gemm_body_parts(self, dev, body):
        """The part count module dev holds for GEMM-worker body `body` (1 unless set)."""
        n = self.l.pb2_device_gemm_body_parts(dev, body)
        _chk(min(n, 0), "pb2_device_gemm_body_parts")
        return n

    def stats(self, dev):
        st = DeviceStats()
        _chk(self.l.pb2_device_get_stats(dev, C.byref(st)), "stats")
        d = {f[0]: getattr(st, f[0]) for f in DeviceStats._fields_}
        d["data_in_from_device"] = list(st.data_in_from_device)
        return d

    def block_cyclic(self, elt_bytes, mb, nb, lm, ln, P=1, Q=1, myrank=0, kp=1, kq=1, ip=0, jq=0, mat=None):
        dc = C.c_void_p(self.l.pb2_matrix_block_cyclic_new(self.h, elt_bytes, myrank, mb, nb, lm, ln, 0, 0, lm, ln, P, Q, kp, kq, ip, jq))
        if not dc:
            raise L.Pb2Error(L.PB2_ERR_BAD_PARAM, "pb2_matrix_block_cyclic_new")
        if mat is not None:
            self._keep.append(mat)
            _chk(self.l.pb2_data_collection_set_mat(dc, _p(mat)), "set_mat")
        return dc

    def wait(self):
        _chk(self.l.pb2_context_wait(self.h), "pb2_context_wait")

    def copy_state(self, data, device):
        out = (C.c_int32 * 6)()
        self.l.pb2_data_copy_state(data, device, out)
        return dict(present=out[0], coherency=out[1], status=out[2], readers=out[3], version=out[4], flags=out[5])

    def trace(self, tp):
        n = self.l.pb2_taskpool_nb_tasks(tp)
        t, d = np.full(n, -1, np.int32), np.full(n, -1, np.int32)
        k = self.l.pb2_taskpool_completion_trace(tp, _p(t), _p(d), n)
        return t[:k], d[:k]

    def device_trace(self, tp):
        """Per task id: the device time stamps of its window run (MCA parameter device_engine_trace; 0 for tasks that
        ran elsewhere), the device index that ran it and the SM.  Each device has its own clock."""
        n = self.l.pb2_taskpool_nb_tasks(tp)
        t0, t1 = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
        dev, sm = np.zeros(n, np.int32), np.zeros(n, np.uint32)
        _chk(self.l.pb2_taskpool_device_trace(tp, _p(t0), _p(t1), _p(dev), _p(sm)), "device_trace")
        return dict(t_start_ns=t0, t_end_ns=t1, device=dev, smid=sm)

    def device_part_trace(self, tp):
        """The part records (PART_TRACE_DTYPE) of the entities the pool's tasks led in GPU windows (MCA parameter
        device_engine_trace), window by window; task is the pool task id.  Returns (records, device index per record)."""
        n = C.c_int32(0)
        _chk(self.l.pb2_taskpool_device_part_trace(tp, None, None, 0, C.byref(n)), "device_part_trace")
        rec, dev = np.zeros(n.value, L.PART_TRACE_DTYPE), np.zeros(n.value, np.int32)
        _chk(self.l.pb2_taskpool_device_part_trace(tp, _p(rec), _p(dev), n.value, C.byref(n)), "device_part_trace")
        return rec, dev

    def task_info(self, tp):
        n = self.l.pb2_taskpool_nb_tasks(tp)
        cls, loc = np.zeros(n, np.int32), np.zeros((n, 2), np.int32)
        seen, res = np.zeros((n, 4), np.uint32), np.zeros(n, np.uint64)
        _chk(self.l.pb2_taskpool_task_info(tp, _p(cls), _p(loc), _p(seen), _p(res)), "task_info")
        return dict(class_id=cls, locals=loc, seen_version=seen, result=res)

    def export_window(self, tp, dev):
        nt, ns, nl, nr = C.c_int32(0), C.c_int32(0), C.c_int32(0), C.c_int32(0)
        _chk(self.l.pb2_taskpool_export_window(tp, dev, None, C.byref(nt), None, C.byref(ns), None, C.byref(nl), None, C.byref(nr), None), "export(size)")
        tasks, succ = np.zeros(nt.value, L.TASK_DTYPE), np.zeros(ns.value, np.uint32)
        tiles, ready, ids = np.zeros(nl.value, L.TILE_DTYPE), np.zeros(nr.value, np.int32), np.zeros(nt.value, np.int32)
        _chk(self.l.pb2_taskpool_export_window(tp, dev, _p(tasks), C.byref(nt), _p(succ), C.byref(ns), _p(tiles), C.byref(nl), _p(ready), C.byref(nr), _p(ids)), "export")
        return dict(tasks=tasks, succ=succ, tiles=tiles, ready=ready, task_ids=ids)

    def close(self):
        if self.h:
            self.l.pb2_fini(C.byref(self.h))
            self.h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()
