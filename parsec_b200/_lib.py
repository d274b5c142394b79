"""ctypes loader for the in-tree native library ``libparsec_b200.so``.

The library is built by ``make`` / ``__graft_entry__.build()`` with nvcc for sm_90a only.
There is no Python or CPU fallback: if the shared object is missing, or the machine has no
H100-class GPU, the product path fails loudly (``pb2_engine_create`` returns PB2_ERR_DEVICE).
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# PB2_LIB_PATH: development aid (sweeps over build variants); the default is the in-tree library
LIB_PATH = os.environ.get("PB2_LIB_PATH") or os.path.join(_HERE, "libparsec_b200.so")

PB2_SUCCESS = 0
PB2_ERROR = -1
PB2_ERR_OUT_OF_RESOURCE = -2
PB2_ERR_NOT_FOUND = -3
PB2_ERR_BAD_PARAM = -4
PB2_ERR_EXISTS = -5
PB2_ERR_NOT_IMPLEMENTED = -6
PB2_ERR_NOT_SUPPORTED = -7
PB2_ERR_VALUE_OUT_OF_BOUNDS = -8
PB2_ERR_TRUNCATE = -9
PB2_ERR_DEVICE = -10

ERR_NAMES = {
    0: "PB2_SUCCESS", -1: "PB2_ERROR", -2: "PB2_ERR_OUT_OF_RESOURCE", -3: "PB2_ERR_NOT_FOUND",
    -4: "PB2_ERR_BAD_PARAM", -5: "PB2_ERR_EXISTS", -6: "PB2_ERR_NOT_IMPLEMENTED",
    -7: "PB2_ERR_NOT_SUPPORTED", -8: "PB2_ERR_VALUE_OUT_OF_BOUNDS", -9: "PB2_ERR_TRUNCATE",
    -10: "PB2_ERR_DEVICE",
}

# flow access bits (parsec_description_structures.h:62-67)
ACCESS_NONE, ACCESS_READ, ACCESS_WRITE, ACCESS_RW, FLOW_PUSHOUT = 0x00, 0x04, 0x08, 0x0C, 0x40

# bodies (enum pb2_body_e)
BODY_NOP, BODY_FILL_I32, BODY_CHECK_I32, BODY_INCR_I32, BODY_ADD_IOTA_I32 = 0, 1, 2, 3, 4
BODY_SCALE_I32, BODY_IOTA_I32, BODY_COPY, BODY_FILL_F32, BODY_CHECK_F32 = 5, 6, 7, 8, 9
BODY_INCR_F32, BODY_AXPY_F32, BODY_MEMSET_U8, BODY_ADD_AT_I32, BODY_GEMM_BF16 = 10, 11, 12, 13, 16
# application device bodies linked into HBM windows (pb2_engine_link_bodies): BODY_LINKED_0 + i, i < 8
BODY_LINKED_0, BODY_LINKED_7 = 20, 27
IMAGE_PTX, IMAGE_CUBIN = 1, 2
# pb2_engine_link_bodies_ex flags: also link the GEMM window kernel, so linked bodies run in GEMM windows too
LINK_GEMM_WINDOWS = 0x1
# ... and call the GEMM-worker bodies (LINK_GEMM_BODIES) through the image's pb2_linked_gemm_body, at the GEMM kernels'
# register budget (needs a nonzero GEMM-worker mask)
LINK_GEMM_BODY_ENTRY = 0x2
# the most parts a task of a GEMM-worker body runs as (pb2_engine_set_gemm_body_parts): a GEMM ring entry's part field
GEMM_BODY_MAX_PARTS = 32
# pb2_engine_malloc_ex flags: cudaMalloc memory, which ipc_export can export (compressible memory cannot be)
MALLOC_IPC = 0x1


def LINK_READERS(mask):
    """pb2_engine_link_bodies_ex flags: bit i of mask declares body BODY_LINKED_0 + i a reader (bits 8..15)."""
    return mask << 8


def LINK_READER_GROUPS(mask):
    """pb2_engine_link_bodies_ex flags: bit i of mask declares that reader BODY_LINKED_0 + i has the group form,
    pb2_linked_reader_group (bits 16..23, a subset of the readers mask)."""
    return mask << 16


def LINK_GEMM_BODIES(mask):
    """pb2_engine_link_bodies_ex flags: bit i of mask declares body BODY_LINKED_0 + i a GEMM-worker body, which gets the
    GEMM worker's operand ring as shared memory (bits 24..31; needs LINK_GEMM_WINDOWS, disjoint from sliceable)."""
    return mask << 24

TASK_DEPS_MASK = 0x01
TILE_INVALID, TILE_STAGING, TILE_VALID = 0, 1, 2
SRC_HOST, SRC_PEER = 0, 1
MAX_FLOWS = 4

# numpy mirrors of the 64-byte pb2_task_t and 32-byte pb2_tile_t (include/pb2_engine.h)
TASK_DTYPE = np.dtype([
    ("dep_goal", "<i4"), ("succ_begin", "<i4"), ("succ_count", "<i4"), ("priority", "<i4"),
    ("body", "u1"), ("nb_flows", "u1"), ("flags", "u1"), ("class_id", "u1"),
    ("tile", "<i4", (4,)), ("access", "u1", (4,)),
    ("iparam", "<i4", (3,)), ("fparam", "<f4"), ("locals", "<i4", (2,)),
], align=False)
assert TASK_DTYPE.itemsize == 64

TILE_DTYPE = np.dtype([
    ("dev_ptr", "<u8"), ("src_ptr", "<u8"), ("bytes", "<u4"), ("state", "<i4"),
    ("version", "<u4"), ("src_kind", "<i4"),
], align=False)
assert TILE_DTYPE.itemsize == 32

# numpy mirror of the 64-byte pb2_part_trace_t (pb2_window_part_trace)
PART_WAITED_INPUT, PART_RETIRED = 1, 2
PART_TRACE_DTYPE = np.dtype([
    ("t_pop_ns", "<u8"), ("t_in_ns", "<u8"), ("t_exec_ns", "<u8"), ("t_out_ns", "<u8"),
    ("in_bytes", "<u8"), ("out_bytes", "<u8"), ("task", "<i4"), ("part", "<u2"), ("nparts", "<u2"),
    ("smid", "<u4"), ("flags", "<u4"),
], align=False)
assert PART_TRACE_DTYPE.itemsize == 64

# numpy mirror of pb2_body_args_t (include/pb2_device_body.h), what a linked body is handed: 72 bytes
BODY_ARGS_DTYPE = np.dtype([
    ("flow", "<u8", (4,)), ("bytes", "<u4", (4,)), ("elem0", "<u4"), ("part", "<u4"),
    ("iparam", "<i4", (3,)), ("fparam", "<f4"),
], align=True)
assert BODY_ARGS_DTYPE.itemsize == 72


def succ_make(task, flow=0):
    return (np.uint32(flow) << np.uint32(27)) | np.uint32(task)


class EngineParams(C.Structure):
    _fields_ = [("workers_per_sm", C.c_int32), ("threads", C.c_int32), ("max_workers", C.c_int32),
                ("stage_mode", C.c_int32), ("queue_policy", C.c_int32), ("timeout_ms", C.c_int32),
                ("gemm_mode", C.c_int32), ("part_bytes", C.c_int32), ("read_groups", C.c_int32),
                ("fuse_readers", C.c_int32)]


class EngineInfo(C.Structure):
    _fields_ = [("cuda_device", C.c_int32), ("sm_count", C.c_int32), ("cc_major", C.c_int32),
                ("cc_minor", C.c_int32), ("nworkers", C.c_int32), ("nworkers_gemm", C.c_int32),
                ("can_map_host", C.c_int32), ("reserved", C.c_int32),
                ("total_mem", C.c_uint64), ("free_mem", C.c_uint64),
                ("compression_supported", C.c_int32), ("slab_compressible", C.c_int32)]


class WindowStats(C.Structure):
    _fields_ = [("tasks_retired", C.c_uint64), ("bytes_h2d", C.c_uint64), ("bytes_d2d", C.c_uint64),
                ("bytes_d2h", C.c_uint64), ("stage_ins", C.c_uint64), ("body_errors", C.c_uint64),
                ("kernel_ms", C.c_float), ("reset_ms", C.c_float)]


class WindowHandle(C.Structure):
    _fields_ = [("dep", C.c_ubyte * 64), ("ring", C.c_ubyte * 64), ("ctl", C.c_ubyte * 64), ("tiles", C.c_ubyte * 64),
                ("cap_mask", C.c_uint32), ("ntasks", C.c_int32), ("entry_kind", C.c_int32), ("ntiles", C.c_int32)]


PUSH_DTYPE = np.dtype([("dst", np.uint64), ("bytes", np.uint32), ("src_tile", np.int32), ("rank", np.int32), ("desc", np.int32),
                       ("pad", np.int32, (2,))])
assert PUSH_DTYPE.itemsize == 32


class PartitionSizes(C.Structure):
    _fields_ = [("ntasks", C.c_int32), ("nsucc", C.c_int32), ("ntiles", C.c_int32), ("nready", C.c_int32),
                ("nremote", C.c_int32), ("nslots", C.c_int32), ("slab_bytes", C.c_uint64)]


class Pb2Error(RuntimeError):
    def __init__(self, rc, what, detail=""):
        self.rc = rc
        super().__init__(f"{what}: {ERR_NAMES.get(rc, rc)} {detail}".strip())


_lib = None

# every extern "C" symbol include/pb2_engine.h declares
ENGINE_SYMBOLS = [
    "pb2_engine_create", "pb2_engine_destroy", "pb2_engine_info", "pb2_engine_last_error",
    "pb2_engine_malloc", "pb2_engine_malloc_ex", "pb2_engine_free", "pb2_engine_host_register", "pb2_engine_host_unregister",
    "pb2_engine_memcpy_h2d", "pb2_engine_prefetch_h2d", "pb2_engine_memcpy_d2h", "pb2_engine_synchronize", "pb2_engine_set_stream", "pb2_engine_get_stream", "pb2_engine_copy_batch", "pb2_engine_ipc_export", "pb2_engine_ipc_open",
    "pb2_engine_ipc_close", "pb2_engine_enable_peer", "pb2_body_launch", "pb2_body_launch_errors", "pb2_engine_set_shared_windows", "pb2_engine_set_part_bytes", "pb2_engine_set_gemm_body_parts", "pb2_engine_set_window_trace", "pb2_engine_set_stage_slice_bytes", "pb2_window_export", "pb2_window_set_remote", "pb2_window_task_entries",
    "pb2_window_arm", "pb2_window_start",
    "pb2_window_create", "pb2_window_destroy", "pb2_window_launch", "pb2_window_wait",
    "pb2_window_results", "pb2_window_trace", "pb2_window_part_trace",
    "pb2_partition_create", "pb2_partition_sizes", "pb2_partition_get", "pb2_partition_destroy", "pb2_partition_error",
    "pb2_partition_set_push", "pb2_partition_push_count", "pb2_partition_get_push", "pb2_window_set_push",
    "pb2_engine_link_bodies", "pb2_engine_link_bodies_checked", "pb2_engine_linked_info",
    "pb2_engine_link_bodies_ex", "pb2_engine_linked_gemm_info",
]


def load():
    """Load libparsec_b200.so (no compute happens here; safe without a GPU)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: run `make` (or __graft_entry__.build()) first. "
            "parsec_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    vp, i32, u64 = C.c_void_p, C.c_int32, C.c_uint64
    P = C.POINTER
    lib.pb2_engine_create.argtypes = [P(vp), C.c_int, P(EngineParams)]
    lib.pb2_engine_destroy.argtypes = [vp]
    lib.pb2_engine_info.argtypes = [vp, P(EngineInfo)]
    lib.pb2_engine_last_error.argtypes = [vp]
    lib.pb2_engine_last_error.restype = C.c_char_p
    lib.pb2_engine_malloc.argtypes = [vp, C.c_size_t, P(vp)]
    lib.pb2_engine_malloc_ex.argtypes = [vp, C.c_size_t, C.c_uint32, P(vp)]
    lib.pb2_engine_free.argtypes = [vp, vp]
    lib.pb2_engine_host_register.argtypes = [vp, vp, C.c_size_t, P(vp)]
    lib.pb2_engine_host_unregister.argtypes = [vp, vp]
    lib.pb2_engine_memcpy_h2d.argtypes = [vp, vp, vp, C.c_size_t]
    lib.pb2_engine_memcpy_d2h.argtypes = [vp, vp, vp, C.c_size_t]
    lib.pb2_engine_synchronize.argtypes = [vp]
    lib.pb2_engine_set_stream.argtypes = [vp, vp]
    lib.pb2_engine_copy_batch.argtypes = [vp, vp, vp, vp, i32]
    lib.pb2_engine_ipc_export.argtypes = [vp, vp, vp]
    lib.pb2_engine_ipc_open.argtypes = [vp, vp, P(vp)]
    lib.pb2_engine_ipc_close.argtypes = [vp, vp]
    lib.pb2_engine_enable_peer.argtypes = [vp, C.c_int]
    lib.pb2_body_launch.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, C.c_float]
    lib.pb2_body_launch_errors.argtypes = [vp, C.c_int]
    lib.pb2_engine_set_shared_windows.argtypes = [vp, C.c_int, vp]
    lib.pb2_window_task_entries.argtypes = [vp, vp]
    lib.pb2_engine_set_part_bytes.argtypes = [vp, i32]
    lib.pb2_engine_set_gemm_body_parts.argtypes = [vp, C.c_int, i32]
    lib.pb2_engine_set_window_trace.argtypes = [vp, C.c_int]
    lib.pb2_window_trace.argtypes = [vp, vp, vp, vp, vp]
    lib.pb2_window_part_trace.argtypes = [vp, vp, i32, P(i32)]
    lib.pb2_engine_set_stage_slice_bytes.argtypes = [vp, i32]
    lib.pb2_engine_link_bodies.argtypes = [vp, C.c_char_p, C.c_size_t, C.c_int, C.c_uint32]
    lib.pb2_engine_link_bodies_checked.argtypes = [vp, C.c_char_p, C.c_size_t, C.c_int, C.c_uint32, C.c_uint32]
    lib.pb2_engine_linked_info.argtypes = [vp, P(i32), P(i32), P(i32), P(i32)]
    lib.pb2_engine_link_bodies_ex.argtypes = [vp, C.c_char_p, C.c_size_t, C.c_int, C.c_uint32, C.c_uint32, C.c_uint32]
    lib.pb2_engine_linked_gemm_info.argtypes = [vp, P(i32), P(i32), P(i32), P(i32)]
    lib.pb2_window_export.argtypes = [vp, vp]
    lib.pb2_window_set_remote.argtypes = [vp, i32, i32, vp, vp, vp, vp, i32]
    lib.pb2_partition_set_push.argtypes = [vp, C.c_int]
    lib.pb2_partition_push_count.argtypes = [vp, i32, vp]
    lib.pb2_partition_get_push.argtypes = [vp, i32, vp, vp, vp]
    lib.pb2_window_set_push.argtypes = [vp, vp, vp, i32]
    lib.pb2_window_arm.argtypes = [vp]
    lib.pb2_window_start.argtypes = [vp]
    lib.pb2_window_create.argtypes = [vp, P(vp), C.c_int, vp, i32, vp, i32, vp, i32, vp, i32]
    lib.pb2_window_destroy.argtypes = [vp]
    lib.pb2_window_launch.argtypes = [vp]
    lib.pb2_window_wait.argtypes = [vp, P(WindowStats)]
    lib.pb2_window_results.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp]
    lib.pb2_partition_create.argtypes = [P(vp), vp, i32, vp, i32, vp, i32, vp, i32, vp, vp, i32, i32]
    lib.pb2_partition_sizes.argtypes = [vp, i32, P(PartitionSizes)]
    lib.pb2_partition_get.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.pb2_partition_destroy.argtypes = [vp]
    for name in ENGINE_SYMBOLS:
        if name not in ("pb2_engine_last_error", "pb2_partition_error", "pb2_partition_destroy", "pb2_engine_get_stream"):
            getattr(lib, name).restype = C.c_int
    lib.pb2_engine_get_stream.argtypes = [vp]
    lib.pb2_engine_get_stream.restype = vp
    lib.pb2_partition_error.restype = C.c_char_p
    lib.pb2_partition_destroy.restype = None
    _lib = lib
    return lib
