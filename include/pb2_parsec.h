/*
 * pb2_parsec.h -- C ABI of the host side that sits above the engine (layers L1 + L2).
 *
 * It mirrors, name for name (prefix pb2_ instead of parsec_), the slice of PaRSEC's interfaces that lies on
 * the GPU-task hot path, so that the parity tests read like the reference's own tests and a PaRSEC maintainer
 * can map every entry point to the reference symbol it replaces (INTEGRATION.md shows the MCA-component
 * binding).  Citations are file:line in /root/reference.
 *
 *   device registry + selection   parsec/mca/device/device.{h,c}      (module struct device.h:145-189)
 *   GPU device module             parsec/mca/device/device_gpu.{h,c}, cuda/device_cuda_module.c
 *   data + coherency              parsec/data.{h,c}, parsec/data_internal.h:30-85
 *   device heap                   parsec/utils/zone_malloc.{h,c}
 *   task completion / release     parsec/scheduling.c:126-206,469-505 ; parsec/parsec.c:1609-1975
 *   2D block cyclic collection    parsec/data_dist/matrix/two_dim_rectangle_cyclic.{h,c}
 *   DTD front end                 parsec/interfaces/dtd/insert_function.{h,c}
 *   PTG front end                 what parsec-ptgpp generates for a .jdf (interfaces/ptg/ptg-compiler/jdf2c.c)
 *
 * Plain C: pointers, integers, no C++ / torch types.
 */
#ifndef PB2_PARSEC_H
#define PB2_PARSEC_H

#include <stddef.h>
#include <stdint.h>
#include "pb2_engine.h"

#ifdef __cplusplus
extern "C" {
#endif

/* parsec/runtime.h:141-147 */
typedef enum pb2_hook_return_e {
    PB2_HOOK_RETURN_DONE    =  0,
    PB2_HOOK_RETURN_AGAIN   = -1,
    PB2_HOOK_RETURN_NEXT    = -2,
    PB2_HOOK_RETURN_DISABLE = -3,
    PB2_HOOK_RETURN_ASYNC   = -4,
    PB2_HOOK_RETURN_ERROR   = -5
} pb2_hook_return_t;

/* device.h:60-75 */
#define PB2_DEV_NONE       0x00
#define PB2_DEV_CPU        0x01
#define PB2_DEV_RECURSIVE  0x02
#define PB2_DEV_CUDA       0x04
#define PB2_DEV_ANY_TYPE   0x3f
#define PB2_DEV_IS_GPU(t)  (0 != ((t) & PB2_DEV_CUDA))
/* device.h:79-81 */
#define PB2_DEV_DATA_ADVICE_PREFETCH          0x01
#define PB2_DEV_DATA_ADVICE_PREFERRED_DEVICE  0x02
#define PB2_DEV_DATA_ADVICE_WARMUP            0x03

/* data.h:33-43 */
#define PB2_DATA_COHERENCY_INVALID   0x0
#define PB2_DATA_COHERENCY_OWNED     0x1
#define PB2_DATA_COHERENCY_EXCLUSIVE 0x2
#define PB2_DATA_COHERENCY_SHARED    0x4
#define PB2_DATA_STATUS_NOT_TRANSFER      0x0
#define PB2_DATA_STATUS_UNDER_TRANSFER    0x1
#define PB2_DATA_STATUS_COMPLETE_TRANSFER 0x2
/* data.h:64-71 */
#define PB2_DATA_FLAG_EVICTED        (1 << 5)
#define PB2_DATA_FLAG_PARSEC_MANAGED (1 << 6)
#define PB2_DATA_FLAG_PARSEC_OWNED   (1 << 7)

/* insert_function.h:54-65 */
#define PB2_INPUT        0x100000
#define PB2_OUTPUT       0x200000
#define PB2_INOUT        0x300000
#define PB2_VALUE        0x600000
#define PB2_GET_OP_TYPE  0xf00000
#define PB2_AFFINITY     (1 << 16)
#define PB2_DONT_TRACK   (1 << 17)
#define PB2_PUSHOUT      (1 << 18)

#define PB2_MAX_DEVICES 16

typedef struct pb2_context_s          pb2_context_t;
typedef struct pb2_taskpool_s         pb2_taskpool_t;
typedef struct pb2_device_module_s    pb2_device_module_t;
typedef struct pb2_data_s             pb2_data_t;
typedef struct pb2_data_copy_s        pb2_data_copy_t;
typedef struct pb2_data_collection_s  pb2_data_collection_t;
typedef struct pb2_dtd_tile_s         pb2_dtd_tile_t;
typedef struct pb2_task_class_s       pb2_task_class_t;
typedef struct pb2_htask_s            pb2_htask_t;        /* parsec_task_t */
typedef struct pb2_gpu_task_s         pb2_gpu_task_t;     /* parsec_gpu_task_t */

/* data_internal.h:54-85: one replica of a datum on one device; fields are host-visible state, part of the API */
struct pb2_data_copy_s {
    int8_t    device_index;
    uint8_t   flags;
    uint8_t   coherency_state;
    uint8_t   data_transfer_status;
    int32_t   readers;
    uint32_t  version;
    pb2_data_t* original;
    void*     device_private;      /* host pointer (device 0) or HBM slot */
    /* engine private */
    pb2_data_copy_t *lru_prev, *lru_next;
    int32_t   lru_list;            /* 0 none, 1 gpu_mem_lru (clean), 2 gpu_mem_owned_lru (dirty) */
    int32_t   window_tile;         /* tile id inside the window being built/run, -1 otherwise */
    const void* window_owner;      /* which in-flight window window_tile refers to */
};

/* data_internal.h:30-49 */
struct pb2_data_s {
    int8_t    owner_device;
    int8_t    preferred_device;
    int32_t   nb_copies;
    uint64_t  key;
    pb2_data_collection_t* dc;
    size_t    span;
    pb2_data_copy_t* device_copies[PB2_MAX_DEVICES];
};

/* device.h:145-189 statistics, as an array-friendly struct */
typedef struct pb2_device_stats_s {
    uint64_t executed_tasks;
    uint64_t required_data_in, required_data_out;
    uint64_t data_out_to_host;
    uint64_t nb_data_faults, nb_evictions;
    uint64_t data_in_from_device[PB2_MAX_DEVICES];
    int64_t  device_load;
    int64_t  time_estimate_default;
    int64_t  gflops_fp16, gflops_fp32, gflops_fp64, gflops_tf32;
    uint64_t windows_launched;       /* engine extension: persistent-kernel launches                           */
    uint64_t tasks_released_on_device; /* engine extension: tasks made ready by a device atomic, no host trip  */
    double   kernel_ms_total;
} pb2_device_stats_t;

/* ---------------------------------------------------------------- context + device registry (device.c) */
/* parsec_init (parsec.c:405) restricted to what the device path needs; adds the CPU (index 0) and the
 * recursive pseudo device (index 1) like parsec_mca_device_attach, device.c:1041-1110. */
int  pb2_init(pb2_context_t** ctx, int nb_cores);
int  pb2_fini(pb2_context_t** ctx);
/* MCA parameters of device.c:342-363 / device_cuda_component.c:135-178 by name ("device_load_balance_skew",
 * "device_cuda_memory_use", "device_cuda_memory_block_size", "device_cuda_memory_number_of_blocks",
 * "device_load_balance_allow_cpu", "device_cuda_max_number_of_ejected_data", "device_show_statistics") */
int  pb2_mca_param_set_int(pb2_context_t* ctx, const char* name, int64_t value);
int  pb2_mca_param_get_int(pb2_context_t* ctx, const char* name, int64_t* value);
/* parsec_cuda_module_init (device_cuda_module.c:406) + parsec_mca_device_add (device.c:1112): opens an engine on
 * CUDA device cuda_index and registers a module; GPUs get device_index 2, 3, ...  dry_run != 0 builds the
 * module without touching CUDA (host-logic tests: windows are built and exported, never launched). */
int  pb2_device_cuda_module_init(pb2_context_t* ctx, int cuda_index, int dry_run, pb2_device_module_t** module);
/* parsec_mca_device_registration_complete (device.c:792): peer-access matrix, time_estimate_default, freeze */
int  pb2_mca_device_registration_complete(pb2_context_t* ctx);
int  pb2_nb_devices(pb2_context_t* ctx);
pb2_device_module_t* pb2_mca_device_get(pb2_context_t* ctx, int device_index);
int  pb2_device_get_stats(pb2_device_module_t* dev, pb2_device_stats_t* stats);
/* Link the application's device bodies into the module's engine (pb2_engine_link_bodies: image, format, sliceable as
 * there), before the module's first window.  Afterwards DTD chores may name PB2_BODY_LINKED_0 .. _7 once every GPU
 * module of the context has linked an image, and the module's windows run those tasks in the linked HBM kernel; a window
 * never holds both GEMM tasks and linked-body tasks unless the link set PB2_LINK_GEMM_WINDOWS (pb2_device_link_bodies_ex).  A dry-run module checks the arguments and records the link.
 * PB2_ERR_EXISTS for a second image, PB2_ERR_NOT_SUPPORTED after the module's first window. */
int  pb2_device_link_bodies(pb2_device_module_t* dev, const void* image, size_t bytes, int format, uint32_t sliceable);
/* pb2_device_link_bodies with the `checked` mask of pb2_engine_link_bodies_checked (pb2_device_link_bodies is this call
 * with checked = 0). */
int  pb2_device_link_bodies_checked(pb2_device_module_t* dev, const void* image, size_t bytes, int format, uint32_t sliceable,
                                    uint32_t checked);
/* pb2_device_link_bodies_checked with the link flags of pb2_engine_link_bodies_ex (pb2_device_link_bodies_checked is this
 * call with flags = 0).  With PB2_LINK_GEMM_WINDOWS a window may hold GEMM tasks and linked-body tasks together: GEMM
 * chains and the application's bodies around them run in one GEMM window.  PB2_LINK_READERS(mask) and
 * PB2_LINK_READER_GROUPS(mask) declare readers and the readers with the group form (pb2_linked_reader_group) as there.
 * PB2_LINK_GEMM_BODIES(mask) declares GEMM-worker bodies as there: a window that holds a task of one is a GEMM window,
 * as one that holds a GEMM task is, so those tasks never reach an HBM window.  PB2_LINK_GEMM_BODY_ENTRY (with such a
 * mask) calls them through pb2_linked_gemm_body, at the GEMM kernels' 168 registers, as there.  A dry-run module checks
 * the flags and records the link. */
int  pb2_device_link_bodies_ex(pb2_device_module_t* dev, const void* image, size_t bytes, int format, uint32_t sliceable,
                               uint32_t checked, uint32_t flags);
/* pb2_engine_set_gemm_body_parts for the module's engine: the tasks of GEMM-worker body `body` run as `nparts` parts in
 * the windows the module builds afterwards.  The same refusals, with PB2_ERR_NOT_FOUND before
 * pb2_device_link_bodies_ex; the message is in the context's last error.  A dry-run module checks the arguments and
 * records the count (pb2_device_gemm_body_parts). */
int  pb2_device_set_gemm_body_parts(pb2_device_module_t* dev, int body, int32_t nparts);
/* The part count the module holds for GEMM-worker body `body` (1 unless set), or a negative error code. */
int  pb2_device_gemm_body_parts(pb2_device_module_t* dev, int body);
/* parsec_devices_print_statistics (device.c:499-590): one row per device -- kernels run and their share, bytes
 * required in / moved H2D and D2D (with the percentage of "required"), bytes required out / written back, evictions --
 * plus the engine's own columns (windows launched, successors released by the device).  Writes a NUL-terminated
 * table into buf (truncated to cap) and returns the length it would need.  pb2_fini prints it to stdout when the MCA
 * parameter device_show_statistics is set, like parsec_mca_device_fini does. */
int  pb2_devices_statistics_string(pb2_context_t* ctx, char* buf, size_t cap);
int  pb2_device_index(pb2_device_module_t* dev);
int  pb2_device_type(pb2_device_module_t* dev);
/* the module entry points, device.h:154-166 (called through the module like the reference does) */
int  pb2_device_memory_register(pb2_device_module_t* dev, pb2_data_collection_t* dc, void* ptr, size_t len);
int  pb2_device_memory_unregister(pb2_device_module_t* dev, pb2_data_collection_t* dc, void* ptr);
int  pb2_device_memory_release(pb2_device_module_t* dev);               /* flush LRUs, device_gpu.c:1059 */
int  pb2_device_data_advise(pb2_device_module_t* dev, pb2_data_t* data, int advice);   /* device_gpu.c:713 */
int  pb2_device_taskpool_register(pb2_device_module_t* dev, pb2_taskpool_t* tp);
int  pb2_device_taskpool_unregister(pb2_device_module_t* dev, pb2_taskpool_t* tp);
/* THE hot call, device.h:133 / device_gpu.c:3375: takes ownership of gpu_task, returns PB2_HOOK_RETURN_ASYNC */
pb2_hook_return_t pb2_device_kernel_scheduler(pb2_device_module_t* dev, void* es, void* gpu_task);
/* the device heap: zone_malloc.c:62,130,215,335 on this module's slab; offsets are returned as pointers */
void*  pb2_device_zone_malloc(pb2_device_module_t* dev, size_t size);
int    pb2_device_zone_free(pb2_device_module_t* dev, void* ptr);
size_t pb2_device_zone_in_use(pb2_device_module_t* dev);
int    pb2_device_lru_sizes(pb2_device_module_t* dev, int* clean, int* owned);

/* parsec_select_best_device, device.c:100-310 (exposed for the placement tests) */
int  pb2_select_best_device(pb2_context_t* ctx, pb2_htask_t* task);

/* ---------------------------------------------------------------- data (data.c) */
pb2_data_t* pb2_data_create(pb2_data_collection_t* dc, uint64_t key, void* ptr, size_t size);   /* data.c:524 */
pb2_data_t* pb2_data_new_temporary(pb2_context_t* ctx, size_t size);   /* arena NEW datum (arena.c:194)            */
int  pb2_data_start_transfer_ownership_to_copy(pb2_context_t* ctx, pb2_data_t* data, uint8_t device, uint8_t access);
void pb2_data_end_transfer_ownership_to_copy(pb2_data_t* data, uint8_t device, uint8_t access);
pb2_data_copy_t* pb2_data_get_copy(pb2_data_t* data, int device);
/* parsec_data_copy_attach, data.c:174-196: a fresh INVALID replica on `device` (NULL when the datum already has one) */
pb2_data_copy_t* pb2_data_copy_attach(pb2_data_t* data, int device);
/* out[6] = present, coherency_state, data_transfer_status, readers, version, flags */
int  pb2_data_copy_state(pb2_data_t* data, int device, int32_t* out);
int  pb2_data_owner_device(pb2_data_t* data);
int  pb2_data_preferred_device(pb2_data_t* data);

/* ---------------------------------------------------------------- 2D block cyclic collection */
/* parsec_matrix_block_cyclic_init, two_dim_rectangle_cyclic.c:109-230 (TILE storage, element size elt_bytes) */
pb2_data_collection_t* pb2_matrix_block_cyclic_new(pb2_context_t* ctx, int elt_bytes, int myrank,
                                                   int mb, int nb, int lm, int ln, int i, int j, int m, int n,
                                                   int P, int Q, int kp, int kq, int ip, int jq);
int   pb2_data_collection_free(pb2_data_collection_t* dc);
int   pb2_data_collection_set_mat(pb2_data_collection_t* dc, void* mat);   /* dc->mat = user memory for local tiles */
uint32_t pb2_dc_rank_of(pb2_data_collection_t* dc, int m, int n);          /* :258-286 / :531-567 */
pb2_data_t* pb2_dc_data_of(pb2_data_collection_t* dc, int m, int n);       /* :368-412 */
uint64_t pb2_dc_data_key(pb2_data_collection_t* dc, int m, int n);         /* matrix.c:235 */
int   pb2_dc_position(pb2_data_collection_t* dc, int m, int n);            /* :351-366, -1 if not local */
/* out[8] = lmt, lnt, mt, nt, nb_elem_r, nb_elem_c, nb_local_tiles, bytes per tile */
int   pb2_dc_info(pb2_data_collection_t* dc, int64_t* out);
int   pb2_dc_register_memory(pb2_data_collection_t* dc, pb2_device_module_t* dev);   /* twoDBC_memory_register :39-49 */
/* map the P x Q "process" grid onto the GPUs of this process: owner rank r -> device 2 + r % ngpu, by setting
 * preferred_device on every local datum (dtd_test_simple_gemm.c:241-251 does this by hand with data_advise) */
int   pb2_dc_distribute_on_devices(pb2_data_collection_t* dc);
/* the application rewrote every local tile in host memory (== a CPU task with WRITE access per tile): host copies
 * take ownership with a new version, GPU replicas become stale and are staged in again on next use */
int   pb2_dc_host_write_all(pb2_data_collection_t* dc);

/* ---------------------------------------------------------------- task pools, generic */
int  pb2_context_add_taskpool(pb2_context_t* ctx, pb2_taskpool_t* tp);     /* scheduling.c:865 */
int  pb2_context_start(pb2_context_t* ctx);                                 /* scheduling.c:968 */
int  pb2_context_wait(pb2_context_t* ctx);                                  /* scheduling.c:994 */
int  pb2_taskpool_wait(pb2_taskpool_t* tp);
int  pb2_taskpool_free(pb2_taskpool_t* tp);
int  pb2_taskpool_nb_tasks(pb2_taskpool_t* tp);
/* restrict the incarnations the tasks of this pool may use (tests/CMakeLists.txt:62-91 runs everything with
 * PARSEC_MCA_device_cuda_enabled=0 unless a test opts in): PB2_DEV_CPU, PB2_DEV_CUDA or both */
int  pb2_taskpool_set_device_types(pb2_taskpool_t* tp, int types);
/* completion trace, one entry per task in the order the host ran __parsec_complete_execution:
 * out_task[i] = task id (insertion / enumeration order), out_device[i] = device_index that ran it */
int  pb2_taskpool_completion_trace(pb2_taskpool_t* tp, int32_t* out_task, int32_t* out_device, int32_t cap);
/* device time stamps, indexed by task id (arrays sized nb_tasks, may be NULL): with the MCA parameter
 * device_engine_trace set, a task that ran in a GPU window gets that window's interval for it (%globaltimer ns of
 * ITS device's clock: devices are not on one time axis) and the SM; every other task (CPU incarnations, user submit
 * bodies, dry runs) gets 0, 0 and 0.  device[i] = device_index that ran task i (-1: not run) */
int  pb2_taskpool_device_trace(pb2_taskpool_t* tp, uint64_t* t_start_ns, uint64_t* t_end_ns, int32_t* device, uint32_t* smid);
/* device part records (pb2_window_part_trace), with the MCA parameter device_engine_trace: every part of every entity
 * the pool's tasks led in a GPU window, window by window as the windows retired; task is the pool task id of the
 * leading task, device[i] the device_index that ran record i (its clock).  *n gets the number of records; at most cap
 * are written (out and device may be NULL). */
int  pb2_taskpool_device_part_trace(pb2_taskpool_t* tp, pb2_part_trace_t* out, int32_t* device, int32_t cap, int32_t* n);
/* per task: locals[0..1], class id, flow versions seen (4), body result; arrays sized nb_tasks (may be NULL) */
int  pb2_taskpool_task_info(pb2_taskpool_t* tp, int32_t* class_id, int32_t* locals2, uint32_t* seen_version4,
                            uint64_t* result);
/* export the device window the module would build for the currently ready tasks on `dev` WITHOUT running it
 * (host-logic tests, works in dry_run mode): sizes first (NULL arrays), then the arrays */
int  pb2_taskpool_export_window(pb2_taskpool_t* tp, pb2_device_module_t* dev,
                                pb2_task_t* tasks, int32_t* ntasks, uint32_t* succ, int32_t* nsucc,
                                pb2_tile_t* tiles, int32_t* ntiles, int32_t* ready, int32_t* nready,
                                int32_t* task_ids /* window task -> taskpool task id */);

/* ---------------------------------------------------------------- DTD (insert_function.h) */
pb2_taskpool_t* pb2_dtd_taskpool_new(pb2_context_t* ctx);                                       /* :1441 */
pb2_dtd_tile_t* pb2_dtd_tile_of(pb2_taskpool_t* tp, pb2_data_collection_t* dc, uint64_t key);   /* PARSEC_DTD_TILE_OF_KEY */
pb2_dtd_tile_t* pb2_dtd_tile_new(pb2_taskpool_t* tp, size_t bytes);                             /* parsec_dtd_tile_new_dev */
pb2_data_t*     pb2_dtd_tile_data(pb2_dtd_tile_t* tile);
/* parsec_dtd_create_task_class: flow_ops[i] = PB2_INPUT / PB2_INOUT / PB2_OUTPUT (| PB2_AFFINITY) */
pb2_task_class_t* pb2_dtd_create_task_class(pb2_taskpool_t* tp, const char* name, int nb_flows, const int32_t* flow_ops);
/* parsec_dtd_task_class_add_chore (:2503).  GPU chores name an in-engine body (enum pb2_body_e); CPU chores a host fn */
typedef int (*pb2_cpu_hook_t)(pb2_htask_t* task, void** flow_ptrs, const int32_t* iparam, float fparam);
int  pb2_dtd_task_class_add_chore(pb2_taskpool_t* tp, pb2_task_class_t* tc, int device_type, int body, pb2_cpu_hook_t cpu_hook);
/* A GPU chore that is an opaque user function, the reference's own kind of CUDA body: parsec_advance_task_function_t
 * submit(gpu_device, gpu_task, gpu_stream) (device_gpu.h:49-51; dtd_test_simple_gemm.c:470-540).  It is called on the
 * host once every flow is resident on `dev`, enqueues its work on `cuda_stream` and returns PB2_HOOK_RETURN_DONE
 * (AGAIN: call me again after the stream has drained; anything negative else is fatal).  Such tasks run on a
 * host-driven stream lane, in dependency order, between engine windows; pb2_gpu_task_flow_ptr gives the device
 * address of a flow (parsec_dtd_get_dev_ptr, insert_function.c:3714-3726). */
typedef int (*pb2_gpu_submit_t)(pb2_device_module_t* dev, pb2_gpu_task_t* gpu_task, void* cuda_stream);
int  pb2_dtd_task_class_add_submit(pb2_taskpool_t* tp, pb2_task_class_t* tc, pb2_gpu_submit_t submit);
void* pb2_gpu_task_flow_ptr(pb2_device_module_t* dev, pb2_gpu_task_t* gpu_task, int flow);
size_t pb2_gpu_task_flow_bytes(pb2_gpu_task_t* gpu_task, int flow);
const int32_t* pb2_gpu_task_iparam(pb2_gpu_task_t* gpu_task);
/* parsec_dtd_insert_task_with_task_class (:3333): flow_ops may add PB2_PUSHOUT per call, like the reference */
int  pb2_dtd_insert_task_with_task_class(pb2_taskpool_t* tp, pb2_task_class_t* tc, int priority, int device_type,
                                         pb2_dtd_tile_t* const* tiles, const int32_t* flow_ops,
                                         const int32_t* iparam3, float fparam);
int  pb2_dtd_data_flush_all(pb2_taskpool_t* tp, pb2_data_collection_t* dc);                     /* :3555 */
int  pb2_dtd_data_flush(pb2_taskpool_t* tp, pb2_dtd_tile_t* tile);

/* ---------------------------------------------------------------- PTG: the task pools ptgpp would generate */
/* examples/Ex02_Chain.jdf */
pb2_taskpool_t* pb2_ptg_ex02_chain_new(pb2_context_t* ctx, int NB);
/* examples/Ex05_Broadcast.jdf with tile-sized data: mydata is a 1-D collection of `nodes` tiles */
pb2_taskpool_t* pb2_ptg_ex05_broadcast_new(pb2_context_t* ctx, pb2_data_collection_t* mydata, int nodes, int NB);
/* tests/apps/pingpong/rtt.jdf (body: T[:] += 1.0f) */
pb2_taskpool_t* pb2_ptg_rtt_new(pb2_context_t* ctx, pb2_data_collection_t* A, int NT, int FRAGS, int WS);
/* tests/runtime/scheduling/ep.jdf */
pb2_taskpool_t* pb2_ptg_ep_new(pb2_context_t* ctx, pb2_data_collection_t* A, int NT, int DEPTH);
/* tests/runtime/cuda/ptg_pingpong.jdf (CPU and GPU incarnations alternate) */
pb2_taskpool_t* pb2_ptg_pingpong_new(pb2_context_t* ctx, pb2_data_collection_t* dist, int NB_TOKEN, int32_t* nb_err);
/* tests/runtime/cuda/get_best_device_check.jdf */
pb2_taskpool_t* pb2_ptg_get_best_device_new(pb2_context_t* ctx, pb2_data_collection_t* A, int32_t* info /* mt*nt device ids */);
/* right-looking tile Cholesky shape (SURVEY 8d config 5): POTRF/TRSM/SYRK/GEMM with GEMM-class bodies */
pb2_taskpool_t* pb2_ptg_cholesky_shape_new(pb2_context_t* ctx, pb2_data_collection_t* A, int NT);

/* ---------------------------------------------------------------- applications (the reference's test mains) */
/* tests/dsl/dtd/dtd_test_simple_gemm.c: simple_gemm() :640-720; inserts NT^3 tasks, waits, returns seconds */
int  pb2_app_dtd_simple_gemm(pb2_context_t* ctx, pb2_data_collection_t* A, pb2_data_collection_t* B,
                             pb2_data_collection_t* C, int device_type, double* seconds, pb2_taskpool_t** keep_tp);

#ifdef __cplusplus
}
#endif
#endif /* PB2_PARSEC_H */
