/*
 * pb2_engine.h -- C ABI of the H100 device-side DAG execution engine (layer L0).
 *
 * One engine instance drives one GPU.  It replaces, for tasks whose incarnation
 * is GPU, the host-driven stream pipeline of the reference
 *   parsec/mca/device/device_gpu.c:3375 (parsec_device_kernel_scheduler)
 *   parsec/mca/device/device_gpu.c:2592 (parsec_device_progress_stream)
 *   parsec/mca/device/device_gpu.c:2745/2873/2943 (kernel_push / _exec / _pop)
 * and the host dependency release of
 *   parsec/parsec.c:1609/1656/1749/1836 (update_deps_with_counter / _with_mask,
 *   release_local_OUT_dependencies, release_dep_fct)
 * by ONE persistent sm_90a kernel per "window" of the DAG: workers (CTAs) pop
 * ready task descriptors from a device-resident ring, stage tiles in from
 * host-pinned / peer memory, run the body, release successors with device
 * atomics and append to a retire log.  No host round trip per task or per edge.
 *
 * Plain C, plain pointers and sizes; no torch / C++ types cross this boundary.
 * The reference-shaped module API (parsec_device_module_t, parsec_gpu_task_t,
 * kernel_scheduler, ...) is layered on top of this file in pb2_parsec.h.
 */
#ifndef PB2_ENGINE_H
#define PB2_ENGINE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Error codes: same values as parsec/include/parsec/constants.h:14-26 */
#define PB2_SUCCESS                   0
#define PB2_ERROR                    -1
#define PB2_ERR_OUT_OF_RESOURCE      -2
#define PB2_ERR_NOT_FOUND            -3
#define PB2_ERR_BAD_PARAM            -4
#define PB2_ERR_EXISTS               -5
#define PB2_ERR_NOT_IMPLEMENTED      -6
#define PB2_ERR_NOT_SUPPORTED        -7
#define PB2_ERR_VALUE_OUT_OF_BOUNDS  -8
#define PB2_ERR_TRUNCATE             -9
#define PB2_ERR_DEVICE              -10

/* Flow access bits: same values as
 * parsec/include/parsec/parsec_description_structures.h:62-67 */
#define PB2_FLOW_ACCESS_NONE   0x00
#define PB2_FLOW_ACCESS_READ   0x04
#define PB2_FLOW_ACCESS_WRITE  0x08
#define PB2_FLOW_ACCESS_RW     0x0c
#define PB2_FLOW_PUSHOUT       0x40   /* engine-private: D2H the flow after the body (gpu_task->pushout bit) */

/* Task bodies the persistent kernel can run in place (the "incarnations").
 * HBM-bound bodies are coalesced 16-byte vector loops; GEMM is wgmma. */
enum pb2_body_e {
    PB2_BODY_NOP        = 0,  /* empty body: tests/runtime/scheduling/ep.jdf:36-40                       */
    PB2_BODY_FILL_I32   = 1,  /* flow0[:] = iparam[0]          (Ex05 TaskBcast: "*Aint = k", tile-wide)   */
    PB2_BODY_CHECK_I32  = 2,  /* result = #elements of flow0 != iparam[0]; sum   (Ex05 TaskRecv)           */
    PB2_BODY_INCR_I32   = 3,  /* flow0[:] += iparam[0]         (Ex02 "*Aint += 1"; rtt.jdf PING)           */
    PB2_BODY_ADD_IOTA_I32 = 4,/* flow0[i] += i                 (tests/runtime/cuda/ping_kernel.cu:15)      */
    PB2_BODY_SCALE_I32  = 5,  /* flow0[:] *= iparam[0]         (dtd_test_new_tile_cuda_kernels.cu:30)      */
    PB2_BODY_IOTA_I32   = 6,  /* flow0[i] = i                  (dtd_test_new_tile_cuda_kernels.cu:17)      */
    PB2_BODY_COPY       = 7,  /* flow1[:] = flow0[:]           (write_check.cu "A3=A2")                    */
    PB2_BODY_FILL_F32   = 8,  /* flow0[:] = fparam                                                         */
    PB2_BODY_CHECK_F32  = 9,  /* result = #elements of flow0 != fparam                                     */
    PB2_BODY_INCR_F32   = 10, /* flow0[:] += fparam            (config 4: "T[:] += 1")                     */
    PB2_BODY_AXPY_F32   = 11, /* flow1[:] += fparam*flow0[:]                                               */
    PB2_BODY_MEMSET_U8  = 12, /* flow0 bytes = iparam[0]&0xff  (get_best_device_check.jdf:82 cudaMemset)   */
    PB2_BODY_ADD_AT_I32 = 13, /* flow0[iparam[0]] += iparam[1]  (ping_kernel.cu:13-21 pong_kernel <<<1,1>>>,
                               *                                 ptg_pingpong.jdf:72-73 TOKEN_CPU)          */
    PB2_BODY_GEMM_BF16  = 16, /* flow2 (C, M x N row-major bf16) += flow0 (A, M x K row-major) *
                               * flow1 (B, N x K row-major == K x N column-major), fp32 accumulate in registers
                               * iparam[0]=M, iparam[1]=N, iparam[2]=K (each tile edge)                     */
    PB2_BODY_LINKED_0   = 20, /* .. PB2_BODY_LINKED_7: the application's device body, linked into the HBM window
                               * kernel by pb2_engine_link_bodies (include/pb2_device_body.h); HBM windows, and
                               * GEMM windows when linked with PB2_LINK_GEMM_WINDOWS                              */
    PB2_BODY_LINKED_7   = 27,
    PB2_BODY_USER       = 31, /* host-side only: the chore is a user `submit` callback that enqueues its own CUDA work
                               * on a stream (device_gpu.h:49-51); such tasks never enter an engine window           */
    PB2_BODY_MAX        = 32
};

#define PB2_MAX_FLOWS 4

/* One task, 64 bytes, read-only on the device.  Mirrors what the reference keeps
 * in parsec_task_t (parsec_internal.h:551-563: task_class, locals[], data[], priority)
 * plus parsec_gpu_task_t (device_gpu.h:117-143: pushout, nb_flows, flow_info[]). */
typedef struct pb2_task_s {
    int32_t  dep_goal;      /* counter mode: #task-sourced input deps (parsec.c:1471-1556);
                             * mask mode: tc->dependencies_goal (parsec.c:1656-1720)                        */
    int32_t  succ_begin;    /* first entry in succ[]                                                         */
    int32_t  succ_count;    /* number of out-edges (iterate_successors fan-out)                              */
    int32_t  priority;      /* task priority: with queue_policy 1 a larger value is popped first (see
                             * pb2_engine_params_t::queue_policy); ignored with the default FIFO policy        */
    uint8_t  body;          /* enum pb2_body_e                                                                */
    uint8_t  nb_flows;
    uint8_t  flags;         /* PB2_TASK_* */
    uint8_t  class_id;      /* task_class_id, for traces                                                      */
    int32_t  tile[PB2_MAX_FLOWS];    /* tile ids, -1 = CTL / unused                                           */
    uint8_t  access[PB2_MAX_FLOWS];  /* PB2_FLOW_ACCESS_* | PB2_FLOW_PUSHOUT                                  */
    int32_t  iparam[3];     /* body immediates                                                               */
    float    fparam;
    int32_t  locals[2];     /* first two locals of the task (k, n / m, n) for traces                          */
} pb2_task_t;                /* sizeof == 64 */

#define PB2_TASK_DEPS_MASK  0x01   /* dep word is a bit mask (PARSEC_USE_DEPS_MASK) instead of a counter     */

/* succ[] entry: low 27 bits = successor task id, high 5 bits = destination flow index */
#define PB2_SUCC_MAKE(task, flow)  (((uint32_t)(flow) << 27) | (uint32_t)(task))
#define PB2_SUCC_TASK(s)           ((int32_t)((s) & 0x07ffffffu))
#define PB2_SUCC_FLOW(s)           ((int32_t)((s) >> 27))

/* Device-side replica of one parsec_data_t on this GPU (data_internal.h:30-85), 32 bytes. */
typedef struct pb2_tile_s {
    void*    dev_ptr;   /* slot in this GPU's HBM (parsec_data_copy_t::device_private of the GPU copy)       */
    void*    src_ptr;   /* device-visible address of the source/home copy: cudaHostRegister'ed host
                         * memory (device_cuda_module.c:183-212) or a peer GPU's slot                        */
    uint32_t bytes;     /* span to move: min(src span, dst span), device_gpu.c:1639-1644                     */
    int32_t  state;     /* PB2_TILE_*                                                                        */
    uint32_t version;   /* parsec_data_copy_t::version of the GPU copy                                       */
    int32_t  src_kind;  /* PB2_SRC_HOST / PB2_SRC_PEER: which statistic the stage-in is charged to
                         * (data_in_from_device[src], device_gpu.c:2133)                                    */
} pb2_tile_t;

#define PB2_SRC_HOST 0
#define PB2_SRC_PEER 1
#define PB2_SRC_PUSH 2      /* the producer's worker writes the bytes into this slot over NVLink and publishes the state:
                             * a local task never pulls it, it finds it VALID (pb2_window_set_push) */

#define PB2_TILE_INVALID   0   /* PARSEC_DATA_COHERENCY_INVALID, must be staged in before a READ             */
#define PB2_TILE_STAGING   1   /* PARSEC_DATA_STATUS_UNDER_TRANSFER                                          */
#define PB2_TILE_VALID     2   /* SHARED/OWNED + COMPLETE_TRANSFER                                           */

typedef struct pb2_engine_params_s {
    int32_t  workers_per_sm;   /* CTAs per SM for HBM-body windows (default 8, at most what the kernel's occupancy allows: 12) */
    int32_t  threads;          /* threads per CTA for HBM-body windows (default and maximum 64)               */
    int32_t  max_workers;      /* 0 = all; 1 = single worker => deterministic FIFO order (tests)             */
    int32_t  stage_mode;       /* tile mover of the HBM-body kernels: 0 = TMA bulk copy (cp.async.bulk through a
                                * shared-memory ring, default), 1 = SIMT 16-byte LDG/STG loops                      */
    int32_t  queue_policy;     /* order in which the workers of HBM and GEMM windows pop ready tasks:
                                *   0 = one FIFO ready ring (default);
                                *   1 = priority, the reference's rule (device_gpu.c:2169-2174): higher
                                *       pb2_task_t::priority first, FIFO among equal priorities.  The ring is cut into
                                *       16 FIFO lanes; the distinct priorities of a window's tasks are ranked highest
                                *       first and rank r goes to lane r when there are at most 16 of them (exact
                                *       order), to lane floor(r * 16 / ndistinct) otherwise.  A read group or a fused
                                *       unit runs in its leader's / producer's lane, a GEMM unit in its first task's.
                                *       Not with shared windows (pb2_window_create: PB2_ERR_NOT_SUPPORTED).
                                * pb2_engine_create refuses any other value (PB2_ERR_BAD_PARAM).  The streaming kernel
                                * (pb2_stream.h) always pops in submission order.                                 */
    int32_t  timeout_ms;       /* device-side watchdog: a window that makes no progress for this long aborts
                                * (default 20000); a malformed DAG must never hang the GPU                   */
    int32_t  gemm_mode;        /* 0 = fused k-chains (default), 2 = every task is its own unit and flushes C
                                * (per-task bf16 rounding, as the oracle); 1 is accepted as an alias of 2        */
    int32_t  part_bytes;       /* HBM bodies: a task whose largest tile exceeds this many bytes is run as up to 512
                                * parts (byte slices) by different workers (default 256 KiB, <0 = never split);
                                * pb2_engine_set_part_bytes changes it for the windows created afterwards       */
    int32_t  read_groups;      /* windows that are not shared: 0 = a run of consecutive out-edges of one task into
                                * CHECK readers of the same tile (that edge their only input) is executed as one
                                * group that streams the tile once for all its members (default); < 0 = every task
                                * alone.  A GEMM task never joins a group; a GEMM window with queue_policy 1 and one
                                * worker forms none                                                              */
    int32_t  fuse_readers;     /* windows that are not shared, with read groups on and more than one worker of the
                                * window's kind (nworkers, nworkers_gemm):
                                * 0 = a producer that writes the tile its first read group checks runs with that
                                * group as one unit, each chunk written and then checked while it is still in L2
                                * (default); < 0 = the producer and the group run one after the other            */
} pb2_engine_params_t;

typedef struct pb2_engine_info_s {
    int32_t  cuda_device;
    int32_t  sm_count;
    int32_t  cc_major, cc_minor;
    int32_t  nworkers;         /* grid size used for HBM-body windows                                        */
    int32_t  nworkers_gemm;    /* grid size used for GEMM windows                                            */
    int32_t  can_map_host;
    int32_t  reserved;
    uint64_t total_mem;
    uint64_t free_mem;
    int32_t  compression_supported;  /* the device and the driver offer compressible memory (cuMemCreate with
                                      * CU_MEM_ALLOCATION_COMP_GENERIC)                                            */
    int32_t  slab_compressible;      /* the engine's last allocation of one granule or more was granted compression */
} pb2_engine_info_t;

/* What one window run produced; device counters mirror device.h:165-171 statistics. */
typedef struct pb2_window_stats_s {
    uint64_t tasks_retired;
    uint64_t bytes_h2d;        /* data_in_from_device[host]: bytes staged in by the kernel                   */
    uint64_t bytes_d2d;        /* bytes staged in from a peer GPU slot                                       */
    uint64_t bytes_d2h;        /* data_out_to_host: pushout bytes                                            */
    uint64_t stage_ins;        /* nb_data_faults (count)                                                     */
    uint64_t body_errors;      /* sum of CHECK body mismatches                                               */
    float    kernel_ms;        /* CUDA-event time of the window kernel on its launch stream                  */
    float    reset_ms;
} pb2_window_stats_t;

typedef struct pb2_engine_s pb2_engine_t;
typedef struct pb2_window_s pb2_window_t;

/* --- engine life cycle (parsec_cuda_module_init / _fini, device_cuda_module.c:406,660) --- */
int  pb2_engine_create(pb2_engine_t** engine, int cuda_device, const pb2_engine_params_t* params);
int  pb2_engine_destroy(pb2_engine_t* engine);
int  pb2_engine_info(pb2_engine_t* engine, pb2_engine_info_t* info);
const char* pb2_engine_last_error(pb2_engine_t* engine);

/* --- device memory (parsec_device_memory_reserve device_gpu.c:866; cuda memory_allocate/free) --- */
/* Tile memory.  Where the device supports it, an allocation of one granule (typically 2 MiB) or more is compressible
 * memory, rounded up to whole granules: the L2 compresses lines on their way to DRAM, so uniform or zero-heavy tiles
 * cost fewer DRAM bytes, and loads, stores, TMA and copies see ordinary memory.  The device and every peer that
 * cudaDeviceCanAccessPeer reports may access it.  Smaller requests, and any the driver cannot back with compressed
 * memory, are cudaMalloc'ed.  pb2_engine_malloc is pb2_engine_malloc_ex with flags 0. */
#define PB2_MALLOC_IPC 0x1u   /* cudaMalloc memory, which pb2_engine_ipc_export can export to another process */
int  pb2_engine_malloc(pb2_engine_t* engine, size_t bytes, void** dev_ptr);
int  pb2_engine_malloc_ex(pb2_engine_t* engine, size_t bytes, uint32_t flags, void** dev_ptr);
int  pb2_engine_free(pb2_engine_t* engine, void* dev_ptr);
/* cudaHostRegister(Portable|Mapped) of a whole collection + its device-visible alias
 * (parsec_cuda_memory_register device_cuda_module.c:183-212). Idempotent per ptr. */
int  pb2_engine_host_register(pb2_engine_t* engine, void* host_ptr, size_t bytes, void** dev_alias);
int  pb2_engine_host_unregister(pb2_engine_t* engine, void* host_ptr);
int  pb2_engine_memcpy_h2d(pb2_engine_t* engine, void* dev, const void* host, size_t bytes);
/* Copy-engine prefetch for the NEXT window that is armed: queued on a DMA stream that runs beside the window in
 * flight; pb2_window_arm makes the engine stream wait for everything queued here.  `host` must be pinned
 * (pb2_engine_host_register).  One call moves `rows` equally spaced tiles (cudaMemcpy2DAsync; a zone heap with
 * 512 KiB units holds 256 KiB tiles at a 512 KiB pitch).  Large runs reach the PCIe DMA rate (54 GB/s on this box) where worker
 * CTAs reading host memory reach 46 GB/s; the caller marks the tiles it prefetched PB2_TILE_VALID. */
int  pb2_engine_prefetch_h2d(pb2_engine_t* engine, void* dev, size_t dev_pitch, const void* host, size_t host_pitch,
                             size_t width_bytes, size_t rows);   /* rows tiles of width_bytes, constant strides */
int  pb2_engine_memcpy_d2h(pb2_engine_t* engine, void* host, const void* dev, size_t bytes);
int  pb2_engine_synchronize(pb2_engine_t* engine);
/* Enqueue all engine work on a caller-owned CUDA stream (cudaStream_t passed as void*), e.g. the stream NCCL
 * collectives are ordered against; NULL restores the engine's own non-blocking stream. */
int  pb2_engine_set_stream(pb2_engine_t* engine, void* cuda_stream);
void* pb2_engine_get_stream(pb2_engine_t* engine);       /* the cudaStream_t engine work is enqueued on */

/* n independent copies dst[i][0:bytes[i]] = src[i][..] in ONE kernel launch (workers grid-stride over the list);
 * either side may be HBM, a peer GPU or cudaHostRegister'ed host memory (device-visible alias).  This is what the
 * module uses to write a batch of dirty tiles home (parsec_gpu_create_w2r_task batches <= 20 copies per
 * pseudo-task and pays one cudaMemcpyAsync + event per tile, transfer_gpu.c:224-304).  Stream-ordered.  Any alignment;
 * PB2_ERR_VALUE_OUT_OF_BOUNDS, with nothing launched, when a copy is 4 GiB or larger. */
int  pb2_engine_copy_batch(pb2_engine_t* engine, void* const* dst, const void* const* src, const uint64_t* bytes, int32_t n);

/* --- multi-GPU (one process per GPU): peer-visible memory ---
 * 64-byte CUDA IPC handles of cudaMalloc'ed memory (PB2_MALLOC_IPC; compressible memory is refused with
 * PB2_ERR_NOT_SUPPORTED); a peer process opens them to get a pointer its kernels can
 * load from / store to over NVLink (parsec_cuda_all_devices_attached enables the same peer access inside one
 * process, device_cuda_module.c:144-181). */
int  pb2_engine_ipc_export(pb2_engine_t* engine, void* dev_ptr, unsigned char handle[64]);
int  pb2_engine_ipc_open(pb2_engine_t* engine, const unsigned char handle[64], void** dev_ptr);
int  pb2_engine_ipc_close(pb2_engine_t* engine, void* dev_ptr);
/* cudaDeviceEnablePeerAccess towards another GPU of this process (parsec_cuda_all_devices_attached,
 * device_cuda_module.c:144-181): afterwards tile sources may point into that GPU's memory. */
int  pb2_engine_enable_peer(pb2_engine_t* engine, int peer_cuda_device);
/* The in-kernel bodies as ONE stand-alone kernel launch on a caller-owned stream: what a BODY [type=CUDA] that names
 * an engine body enqueues when it runs under a device module that is not the engine's (the reference's stream
 * engine drives it then, device_gpu.c:2873-2934).  ptrs/bytes: device address and span of each body argument.
 * CHECK bodies add their mismatch count to a device counter read (and optionally cleared) by
 * pb2_body_launch_errors.  PB2_ERR_BAD_PARAM for an argument of bytes > 0 whose pointer is NULL or not 16-byte aligned
 * (the bodies move 16-byte vectors), PB2_ERR_VALUE_OUT_OF_BOUNDS for one of 4 GiB or more. */
int  pb2_body_launch(void* cuda_stream, int body, int nb_args, void* const* ptrs, const uint64_t* bytes,
                     const int32_t* iparam3, float fparam);
int  pb2_body_launch_errors(uint64_t* errors, int reset);
/* all windows created after this call keep their scheduling arrays in IPC-exportable memory and treat their tasks'
 * dependency goals as counting in-edges from other GPUs too.  next_rs_begin (may be NULL; ntasks+1 entries, must stay
 * valid until the next pb2_window_create returns) is the remote out-edge CSR of the next window: a task with remote
 * successors is never fused into the middle of a GEMM k-chain unit. */
int  pb2_engine_set_shared_windows(pb2_engine_t* engine, int on, const int32_t* next_rs_begin);
/* part size for the windows created from now on (a serial chain of large tiles wants small parts: a 64-thread
 * worker keeps only 4 KiB in flight; wide DAGs want one part per tile) */
int  pb2_engine_set_part_bytes(pb2_engine_t* engine, int32_t part_bytes);
/* on != 0: the windows created from now on record when and on which SM each task ran (pb2_window_trace), through
 * traced builds of the window kernels; off (the default) they run the untraced kernels */
int  pb2_engine_set_window_trace(pb2_engine_t* engine, int on);
/* granularity of cooperative stage-in (default 64 KiB, <= 0: whole tiles): a tile that has to be staged in is cut into
 * slices of this size and every worker that needs the tile pulls the slices nobody has claimed yet */
int  pb2_engine_set_stage_slice_bytes(pb2_engine_t* engine, int32_t bytes);

/* --- application device bodies (include/pb2_device_body.h) ---
 * Link `image` -- PTX (PB2_IMAGE_PTX, text, compiled with -rdc=true) or a relocatable sm_90a cubin (PB2_IMAGE_CUBIN) that
 * defines pb2_linked_body -- into the engine's relocatable build of the HBM window kernel, with the driver's JIT linker.
 * Afterwards HBM windows (kind 0) whose tasks name PB2_BODY_LINKED_0 .. _7 run the linked kernel; every other window runs
 * the built-in kernels as before.  Bit i of `sliceable` lets the engine cut the tasks of body PB2_BODY_LINKED_0 + i into
 * byte-slice parts (pb2_engine_params_t::part_bytes); a clear bit runs them as one part over whole tiles.
 * PB2_ERR_BAD_PARAM for a NULL or empty image, an unknown format, mask bits above bit 7, or a link error (the linker's
 * log is in pb2_engine_last_error); PB2_ERR_EXISTS when the engine has linked an image already (once per engine). */
#define PB2_IMAGE_PTX   1
#define PB2_IMAGE_CUBIN 2
int  pb2_engine_link_bodies(pb2_engine_t* engine, const void* image, size_t bytes, int format, uint32_t sliceable);
/* pb2_engine_link_bodies (which is this call with checked = 0), where bit i of `checked` declares that body
 * PB2_BODY_LINKED_0 + i has a checked form (include/pb2_device_body.h).  Such a task that writes exactly one tile, does
 * not push it out, has no wider tile, and releases a read group of that tile (CHECK readers) runs fused with the group
 * as a built-in producer does (pb2_engine_params_t::fuse_readers): its readers never stream the tile from DRAM again.
 * `checked` must be a subset of `sliceable`, without bits above bit 7: PB2_ERR_BAD_PARAM otherwise. */
int  pb2_engine_link_bodies_checked(pb2_engine_t* engine, const void* image, size_t bytes, int format, uint32_t sliceable,
                                    uint32_t checked);
/* pb2_engine_link_bodies_checked (which is this call with flags = 0) with link flags:
 *   PB2_LINK_GEMM_WINDOWS  also link the engine's relocatable build of the GEMM window kernel.  GEMM windows (kind 1)
 *                          whose tasks name a linked body then run it beside their GEMM units, and GEMM windows without
 *                          one keep the built-in kernel.  In a GEMM window a body runs on the 384 threads of the GEMM
 *                          worker, in check mode too when its bit is set in `checked`.  Its static shared memory comes on top of the GEMM kernel's
 *                          dynamic shared memory: PB2_ERR_NOT_SUPPORTED, and the engine stays unlinked, when the two do
 *                          not fit on one SM.  The flag costs link time (four more kernels), so it is opt-in.
 *   PB2_LINK_READERS(mask) bits 8..15: bit i of `mask` declares that body PB2_BODY_LINKED_0 + i is a reader
 *                          (include/pb2_device_body.h): it only loads from its flows, and its task's result is the sum
 *                          of what it returns over all calls.  Consecutive readers of one tile that a task releases run
 *                          as one read group on one worker, fused with that task when it writes the tile
 *                          (pb2_engine_params_t::read_groups, fuse_readers), in windows of both kinds.  `mask` must be a
 *                          subset of `sliceable`: PB2_ERR_BAD_PARAM otherwise.
 *   PB2_LINK_READER_GROUPS(mask) bits 16..23: bit i of `mask` declares that reader PB2_BODY_LINKED_0 + i has the group
 *                          form (pb2_linked_reader_group, include/pb2_device_body.h): a read group makes one call of it per
 *                          chunk for all such members, which then share one pass over the chunk.  `mask` must be a subset
 *                          of the readers mask (PB2_ERR_BAD_PARAM otherwise).  A nonzero mask links a second build of
 *                          the window kernels, which makes the call: the image must then define pb2_linked_reader_group
 *                          (else the link fails as any link error does).  With a zero mask the kernels never call it.
 *   PB2_LINK_GEMM_BODIES(mask) bits 24..31: bit i of `mask` declares that body PB2_BODY_LINKED_0 + i is a GEMM-worker
 *                          body (include/pb2_device_body.h): in GEMM windows it gets the worker's 192 KiB operand ring
 *                          as `scratch` and runs as one part, never grouped or fused; HBM windows refuse its tasks
 *                          (PB2_ERR_NOT_SUPPORTED).  A nonzero mask needs PB2_LINK_GEMM_WINDOWS and must not overlap
 *                          `sliceable` (so neither `checked` nor the readers masks): PB2_ERR_BAD_PARAM otherwise.
 *   PB2_LINK_GEMM_BODY_ENTRY bit 1: the GEMM window kernels call every body of the GEMM-worker mask through
 *                          pb2_linked_gemm_body, declared in include/pb2_device_body.h, which only they reach: it has
 *                          their budget of 168 registers per thread and not the HBM kernels' 80; every other call still
 *                          goes through pb2_linked_body.  Needs a nonzero PB2_LINK_GEMM_BODIES mask (PB2_ERR_BAD_PARAM
 *                          otherwise, and nothing is recorded).  The flag links another build of the GEMM window
 *                          kernels, which makes the call: the image must then define pb2_linked_gemm_body, or the link
 *                          fails as any link error does and the engine stays unlinked.  Without the flag the kernels
 *                          never call it.
 * PB2_ERR_BAD_PARAM for any other bit. */
#define PB2_LINK_GEMM_WINDOWS 0x1u
#define PB2_LINK_GEMM_BODY_ENTRY 0x2u
#define PB2_LINK_READERS(mask) ((uint32_t)(mask) << 8)
#define PB2_LINK_READER_GROUPS(mask) ((uint32_t)(mask) << 16)
#define PB2_LINK_GEMM_BODIES(mask) ((uint32_t)(mask) << 24)
int  pb2_engine_link_bodies_ex(pb2_engine_t* engine, const void* image, size_t bytes, int format, uint32_t sliceable,
                               uint32_t checked, uint32_t flags);
/* What the linker made of the untraced linked kernel of the engine's queue policy: registers per thread, local (spill
 * and stack) bytes per thread, static shared memory per CTA, and the workers a linked window runs (the engine's HBM
 * worker count, or fewer when the linked kernel's occupancy allows fewer).  Any pointer may be NULL.
 * PB2_ERR_NOT_FOUND before pb2_engine_link_bodies. */
int  pb2_engine_linked_info(pb2_engine_t* engine, int32_t* regs, int32_t* local_bytes, int32_t* static_smem, int32_t* nworkers);
/* The same for the untraced linked GEMM window kernel of the engine's queue policy; nworkers: the workers a GEMM window
 * with linked tasks runs (the engine's GEMM worker count, or fewer when the kernel's occupancy allows fewer).
 * PB2_ERR_NOT_FOUND unless the engine linked with PB2_LINK_GEMM_WINDOWS. */
int  pb2_engine_linked_gemm_info(pb2_engine_t* engine, int32_t* regs, int32_t* local_bytes, int32_t* static_smem,
                                 int32_t* nworkers);
/* Parts per task of GEMM-worker body `body` (PB2_BODY_LINKED_0 .. _7, its bit set in the link's PB2_LINK_GEMM_BODIES
 * mask) in the GEMM windows created from now on: every task of the body then runs as `nparts` parts, each on a worker of
 * its own where workers are free, each handed the task's whole tiles and its part index (include/pb2_device_body.h,
 * pb2_gemm_body_args_t); the body splits the work by part itself.  The default is 1 for every body: one part on one
 * worker.  PB2_ERR_NOT_FOUND before pb2_engine_link_bodies_ex; PB2_ERR_BAD_PARAM for any other id, or one that is not a
 * GEMM-worker body of the link; PB2_ERR_VALUE_OUT_OF_BOUNDS for nparts < 1 or > PB2_GEMM_BODY_MAX_PARTS.  Every refusal
 * leaves the counts as they were and says why in pb2_engine_last_error. */
#define PB2_GEMM_BODY_MAX_PARTS 32             /* the 5-bit part field of a GEMM window's ring entry */
int  pb2_engine_set_gemm_body_parts(pb2_engine_t* engine, int body, int32_t nparts);

/* --- one window of the DAG ---
 * tasks[ntasks], succ[nsucc] (CSR via succ_begin/succ_count), tiles[ntiles] and the ids of
 * the tasks that are ready at submission (startup tasks, parsec.c:1724-1740).
 * 'kind' selects the kernel instantiation: 0 = HBM bodies, 1 = tensor-core GEMM bodies.  An HBM window with a task of
 * a linked body (PB2_BODY_LINKED_0 .. _7) runs the engine's linked kernel (pb2_engine_link_bodies), and so does a GEMM
 * window with one when the engine linked with PB2_LINK_GEMM_WINDOWS; such a task in any other GEMM window, in a shared
 * window or on an engine without an image is refused (PB2_ERR_NOT_SUPPORTED).  The slot (dev_ptr) of a non-empty tile
 * that a task of any body but NOP names must be 16-byte aligned (PB2_ERR_BAD_PARAM otherwise); host homes (src_ptr) may
 * have any alignment. */
int  pb2_window_create(pb2_engine_t* engine, pb2_window_t** window, int kind,
                       const pb2_task_t* tasks, int32_t ntasks,
                       const uint32_t* succ, int32_t nsucc,
                       const pb2_tile_t* tiles, int32_t ntiles,
                       const int32_t* ready, int32_t nready);
int  pb2_window_destroy(pb2_window_t* window);
/* (re)arm the window's per-run state (dependency words, ring, counters, tile states, cleared outputs); then launch; both
 * are stream-ordered.  A non-shared HBM window keeps two copies of that state and alternates between them: each launch
 * queues the reset of the other copy, for the next launch, on a stream of its own beside the run, so from a window's
 * third launch on the arm launches nothing (its reset_ms reads about 0).  Waits, stats and results are those of the
 * last launch. */
int  pb2_window_launch(pb2_window_t* window);
/* block until the window retired all its tasks (or the watchdog tripped); fills stats */
int  pb2_window_wait(pb2_window_t* window, pb2_window_stats_t* stats);
/* per-task outputs, valid after wait; any pointer may be NULL */
int  pb2_window_results(pb2_window_t* window,
                        int32_t*  retire_order,  /* [ntasks] task ids in completion order               */
                        uint32_t* start_seq,     /* [ntasks] global event number when the task started  */
                        uint32_t* end_seq,       /* [ntasks] global event number when it retired        */
                        uint32_t* seen_version,  /* [ntasks*PB2_MAX_FLOWS] tile version seen per flow   */
                        uint64_t* result,        /* [ntasks] body result (CHECK: mismatches<<40 | sum)   */
                        int32_t*  worker,        /* [ntasks] CTA that ran the task                       */
                        pb2_tile_t* tiles_out);  /* [ntiles] final tile table (state, version)           */
/* Per-task device time stamps of the last launch of a window created with trace on (pb2_engine_set_window_trace),
 * valid after wait; any pointer may be NULL.  Times are %globaltimer nanoseconds of this GPU's clock.  A task gets the
 * interval of its scheduling entity, derived from the entity's part records (pb2_window_part_trace): from the earliest
 * t_pop of its parts to the latest t_out, so the retirement bookkeeping after the last part's pushout (the epilog, a
 * few atomics, a fused unit's member stores) is not part of it.  The members of a read group, of a fused producer unit
 * or of a GEMM unit share one interval and SM.  A task whose entity was never popped reads 0; one whose entity did not
 * retire (a failed run) reads 0 as t_end and SM.  PB2_ERR_NOT_SUPPORTED for a window created without trace. */
int  pb2_window_trace(pb2_window_t* window,
                      uint64_t* t_start_ns,      /* [ntasks] earliest pop of a part of the task's entity  */
                      uint64_t* t_end_ns,        /* [ntasks] latest pushout end of one of its parts       */
                      uint32_t* smid,            /* [ntasks] SM of the part that retired it               */
                      int32_t*  unit);           /* [ntasks] the task that leads the entity (host side):
                                                  * read-group leader, fused producer, GEMM unit's first
                                                  * task, or the task itself                              */
/* One part of a scheduling entity as a worker ran it (a window created with trace on): the entity's parts are its ring
 * entries -- the byte slices of a wide task, of a read group or of a fused producer unit, the sub-tile sets of a GEMM
 * unit.  The four stamps are %globaltimer nanoseconds taken by one thread on one SM, so they are ordered:
 *   t_pop   the pop of the entry (the value the entity's t_start is the minimum of)
 *   t_in    stage-in done (the tiles the part found INVALID are in HBM); t_pop..t_in is "movein"
 *   t_exec  body done (a read group's members, a fused unit's check, a GEMM unit's TMA operand stream and MMAs)
 *   t_out   pushout done (= t_exec when the part pushes nothing out); t_exec..t_out is "moveout"
 * in_bytes: bytes this worker staged in itself (from the host or a peer); out_bytes: bytes it pushed out. */
#define PB2_PART_WAITED_INPUT 1u    /* the part found an input tile not VALID                                    */
#define PB2_PART_RETIRED      2u    /* the part retired its entity (the SM of pb2_window_trace)                  */
typedef struct pb2_part_trace_s {
    uint64_t t_pop_ns, t_in_ns, t_exec_ns, t_out_ns;   /* %globaltimer of this GPU                                  */
    uint64_t in_bytes, out_bytes;
    int32_t  task;                                     /* the task leading the entity: pb2_window_trace's unit[]    */
    uint16_t part, nparts;
    uint32_t smid;
    uint32_t flags;                                    /* PB2_PART_WAITED_INPUT | PB2_PART_RETIRED                   */
} pb2_part_trace_t;                                    /* 64 bytes */
/* The part records of the last launch of a window created with trace on, valid after wait: one per ring entry, ordered
 * by leading task id, then by part.  *n gets the number of records; at most cap of them are written to out (out may be
 * NULL).  A part that never ran (a failed run) has zero stamps.  PB2_ERR_NOT_SUPPORTED for a window created without
 * trace. */
int  pb2_window_part_trace(pb2_window_t* window, pb2_part_trace_t* out, int32_t cap, int32_t* n);

/* --- windows that release dependencies of tasks living in OTHER GPUs' windows (remote_dep edges, remote_dep.h:42-58,
 * without the host: the activation is a device atomic on the peer's dependency word plus a ring write over NVLink).
 * Handle of this window's scheduling arrays, to be given to the peers: */
typedef struct pb2_window_handle_s {
    unsigned char dep[64], ring[64], ctl[64], tiles[64];
    uint32_t cap_mask;
    int32_t  ntasks;
    int32_t  entry_kind;   /* 0: dep words and ring entries are per task, 1: per fused GEMM unit */
    int32_t  ntiles;       /* entries of the exported tile table (producer-side pushes publish tile states in it) */
} pb2_window_handle_t;
/* entry[t] = what a remote producer must put in rs_target to release task t of THIS window (index of the
 * dependency word + number of ring entries, in this window's own encoding).  Exchange it with the peers. */
int  pb2_window_task_entries(pb2_window_t* window, int32_t* entry);
int  pb2_window_export(pb2_window_t* window, pb2_window_handle_t* handle);
/* remote out-edges of this window: for task t, entries rs_begin[t] .. rs_begin[t+1]-1 of (rank[], target[]) where
 * target = the destination window's pb2_window_task_entries value of the destination task; remote successors are
 * counter-mode.
 * peers[r] is rank r's exported handle (peers[my_rank] is ignored). */
int  pb2_window_set_remote(pb2_window_t* window, int32_t my_rank, int32_t nranks, const pb2_window_handle_t* peers,
                           const int32_t* rs_begin, const int32_t* rs_rank, const uint32_t* rs_target, int32_t nrs);
/* two-phase launch for windows that are released into by peers: every rank arms, all ranks synchronise, every
 * rank starts.  pb2_window_launch == arm + start.  arm picks the copy of the per-run state the next start runs on (the
 * other one than the last start's, in a non-shared HBM window) and runs the reset kernel on it unless the last start
 * queued that reset already (then the engine stream waits for it); shared windows and GEMM windows have one copy,
 * which every arm resets. */
int  pb2_window_arm(pb2_window_t* window);
int  pb2_window_start(pb2_window_t* window);

/* --- splitting one window over the GPUs of a box (host logic, no device work) ------------------------------------
 * What remote_dep.c does per task at run time (parsec_remote_dep_activate, remote_dep.c:451: which ranks own the
 * successors of this task, per output flow) is done once per window: every edge whose end points live on different
 * ranks becomes a remote edge of the producer's window, and the consumer's flow gets a tile descriptor that pulls the
 * producer's copy over NVLink (src_kind PEER) the first time a local task needs that version.
 *   task_rank[t] : rank that runs task t (rank_of of its affinity datum, two_dim_rectangle_cyclic.c:258-286)
 *   tile_rank[i] : rank whose slab holds the initial / final copy of tile i
 * A rank that overwrites a tile it has sent is held back by a write-after-read edge from the remote readers, the
 * rule parsec_dtd_ordering_correctly applies to local readers (insert_function.c:2603). */
typedef struct pb2_partition_s pb2_partition_t;
typedef struct pb2_partition_sizes_s {
    int32_t  ntasks, nsucc, ntiles, nready, nremote, nslots;
    uint64_t slab_bytes;           /* bytes of the rank's tile slab (every slot 256-byte aligned) */
} pb2_partition_sizes_t;
int  pb2_partition_create(pb2_partition_t** partition, const pb2_task_t* tasks, int32_t ntasks,
                          const uint32_t* succ, int32_t nsucc, const pb2_tile_t* tiles, int32_t ntiles,
                          const int32_t* ready, int32_t nready, const int32_t* task_rank, const int32_t* tile_rank,
                          int32_t nranks, int32_t part_bytes);
int  pb2_partition_sizes(const pb2_partition_t* partition, int32_t rank, pb2_partition_sizes_t* sizes);
/* slab_base[r]: address of rank r's slab as seen from `rank` (own allocation / IPC mapping).  Arrays sized by
 * pb2_partition_sizes; rs_begin has ntasks+1 entries; rs_target[e] is the LOCAL TASK ID in rank rs_rank[e]'s part
 * (translate it with that rank's pb2_window_task_entries before pb2_window_set_remote); global_id[t] is the id the
 * local task had in the input; part_bytes of pb2_partition_create is reserved (pass 0);
 * slot_tile / slot_offset describe the slab (global tile id and byte offset of each slot). */
int  pb2_partition_get(const pb2_partition_t* partition, int32_t rank, const uint64_t* slab_base,
                       pb2_task_t* tasks, uint32_t* succ, pb2_tile_t* tiles, int32_t* ready,
                       int32_t* rs_begin, int32_t* rs_rank, uint32_t* rs_target, int32_t* global_id,
                       int32_t* slot_tile, uint64_t* slot_offset);
/* Producer-side push.  A version a rank reads out of another rank's slot can be written into the reader's slot by the
 * PRODUCER, right after its body, when nothing on the reader's rank used that slot before (no write-after-read hazard):
 * posted stores over NVLink instead of a pull whose every chunk pays a round trip.  pb2_partition_set_push(p, 1) makes
 * pb2_partition_get describe such tiles with src_kind PB2_SRC_PUSH; pb2_partition_get_push returns, for the tasks of
 * `rank`, what each has to push (CSR ps_begin[ntasks+1]); give it to the window with pb2_window_set_push AFTER
 * pb2_window_set_remote (the destination tile tables come from the peers' handles). */
typedef struct pb2_push_s {
    uint64_t dst;          /* destination slot, as seen from the pushing rank (slab_base[rank] + offset)             */
    uint32_t bytes;
    int32_t  src_tile;     /* the pushing task's own descriptor of the tile                                           */
    int32_t  rank;         /* destination rank                                                                        */
    int32_t  desc;         /* destination descriptor (index in that rank's tile table)                                */
    int32_t  pad[2];
} pb2_push_t;
int  pb2_partition_set_push(pb2_partition_t* partition, int on);
int  pb2_partition_push_count(const pb2_partition_t* partition, int32_t rank, int32_t* npush);
int  pb2_partition_get_push(const pb2_partition_t* partition, int32_t rank, const uint64_t* slab_base,
                            int32_t* ps_begin, pb2_push_t* push);
int  pb2_window_set_push(pb2_window_t* window, const int32_t* ps_begin, const pb2_push_t* push, int32_t npush);
void pb2_partition_destroy(pb2_partition_t* partition);
const char* pb2_partition_error(void);

#ifdef __cplusplus
}
#endif
#endif /* PB2_ENGINE_H */
