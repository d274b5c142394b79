/*
 * pb2_stream.h -- C ABI of the STREAMING side of the engine: a host-written descriptor ring and ONE persistent
 * sm_90a kernel per GPU that pulls task descriptors from it (BASELINE north_star; SURVEY.md 7 step 4).
 *
 * What it replaces in the reference, for one GPU:
 *   - the three stream rings (H2D / exec / D2H) with four CUDA events each that parsec_device_progress_stream
 *     polls (parsec/mca/device/device_gpu.c:2592-2731, device_gpu.h:283-298) and the per-task
 *     cudaMemcpyAsync + cudaEventRecord + cudaEventQuery traffic behind them:
 *       host  -> device : a ring of 64-byte COMMANDS in pinned, device-mapped host memory.  The host only stores;
 *                         a dispatcher warp of the persistent kernel reads it over PCIe and feeds the device-resident
 *                         ready ring the worker CTAs pop from;
 *       device -> host  : a ring of 32-byte RETIRE records the workers write into pinned host memory with posted
 *                         PCIe writes; the host polls its own memory, never the device;
 *   - parsec_release_dep_fct for edges between two tasks that are both in flight on this GPU (parsec/parsec.c:1836):
 *     pb2_stream_add_edge links a successor that was submitted BEFORE its predecessor finished; the worker that
 *     retires the predecessor decrements the successor's dependency word on the device and pushes it on the ready
 *     ring, no host round trip;
 *   - parsec_device_data_stage_in / parsec_default_gpu_stage_in/_stage_out (device_gpu.c:1799, :1623, :1673): a task
 *     whose tile descriptor says INVALID stages the tile in itself (TMA bulk copy from pinned host memory or a
 *     peer GPU), pushout flows are copied home by the worker.
 *
 * The kernel is launched when the first command arrives and PARKS itself (exits) after `idle_us` without work,
 * so that a quiet device never holds SMs and blocking CUDA calls (cudaFree, cudaHostUnregister, ...) cannot
 * deadlock against it; the next submission relaunches it.
 *
 * Threading: a stream has a SUBMIT side (pb2_stream_set_tile / _submit / _add_edge / _kick) and a POLL side
 * (pb2_stream_poll).  One thread at a time may be on each side, and the two sides may run at the same time on
 * different threads: tickets travel back through a single-producer single-consumer ring, each side keeps its own
 * counters on its own cache line, either side may find the kernel parked and relaunch it.  The caller's record
 * (`*ticket`, whatever `cookie` points to) must be final BEFORE pb2_stream_submit: the task may retire, and be polled
 * by the other thread, before the call returns.  Election of the two threads happens above this layer (the starter
 * and the manager of the device module; gpu_device->mutex in device_gpu.c:3408-3424).  pb2_stream_quiesce, _stats,
 * _destroy: with both sides idle.
 *
 * dry_run streams touch no CUDA API: tasks "retire" in dependency order without running their bodies.  They exist
 * for host-logic tests in GPU-less containers and are never a fallback: a stream is dry-run only when its creator
 * asked for it explicitly.
 */
#ifndef PB2_STREAM_H
#define PB2_STREAM_H

#include "pb2_engine.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct pb2_stream_s pb2_stream_t;

typedef struct pb2_stream_params_s {
    int32_t cmd_slots;     /* capacity of the command ring == max commands whose task has not retired; power of two,
                            * 1024 .. 2^21 (default 65536)                                                          */
    int32_t max_tiles;     /* entries of the device-resident tile table (default 65536)                              */
    int32_t idle_us;       /* the kernel parks after this long without commands or tasks in flight (default 2000)    */
    int32_t dry_run;       /* != 0: no CUDA at all, see above                                                        */
    int32_t timeout_ms;    /* device watchdog: tasks in flight and no retirement for this long -> abort (20000)      */
    int32_t part_bytes;    /* tasks whose widest tile exceeds this are run as byte-slice parts by several workers
                            * (default 256 KiB; < 0: never split)                                                    */
    int32_t max_workers;   /* 0 = every resident CTA; 1 = one worker (deterministic FIFO order, tests)                */
    int32_t trace;         /* != 0: workers time-stamp every task with the device clock (pb2_retire_t.t_start_ns / t_end_ns) */
} pb2_stream_params_t;

/* One retired task, as the host reads it from the retire ring. */
typedef struct pb2_retire_s {
    uint64_t cookie;            /* the value given to pb2_stream_submit (the gpu_task pointer in the MCA component)   */
    uint64_t result;            /* body result (CHECK bodies: mismatches << 32 | first element)                       */
    uint32_t seen_version[PB2_MAX_FLOWS];   /* tile version each flow saw when the task started                        */
    int32_t  ticket;
    int32_t  status;            /* PB2_SUCCESS, or PB2_ERR_BAD_PARAM for an unknown body id                           */
    uint64_t t_start_ns;        /* params.trace: %globaltimer when a worker popped the task (its last part), ...      */
    uint64_t t_end_ns;          /* ... and when its body, pushout and successor release were done; else 0             */
    uint32_t smid;              /* params.trace: the SM that ran it                                                    */
    uint32_t pad;
} pb2_retire_t;

typedef struct pb2_stream_stats_s {
    uint64_t submitted, retired;
    uint64_t bytes_h2d, bytes_d2d, bytes_d2h, stage_ins, body_errors;
    uint64_t kernel_launches;       /* how often the persistent kernel was (re)started                                */
    uint64_t edges, edges_late;     /* look-ahead edges given to the device / found already satisfied by the dispatcher */
    uint64_t released_on_device;    /* tasks made ready by a device-side decrement                                     */
} pb2_stream_stats_t;

int  pb2_stream_create(pb2_engine_t* engine, const pb2_stream_params_t* params, pb2_stream_t** stream);
/* engine may be NULL only for dry_run streams */
int  pb2_stream_destroy(pb2_stream_t* stream);
const char* pb2_stream_last_error(pb2_stream_t* stream);

/* (Re)describe tile `tile` of the device tile table: where the replica lives in HBM, where its source/home copy is,
 * how many bytes, whether it is valid or has to be staged in, and its version.  Takes effect before any task
 * submitted later; the caller must not redescribe a tile that an unretired task uses unless nothing but `src_ptr`
 * of a VALID tile changes.  PB2_ERR_BAD_PARAM for a non-empty tile whose dev_ptr is not 16-byte aligned (the bodies
 * access slots with 16-byte vectors; src_ptr may have any alignment). */
int  pb2_stream_set_tile(pb2_stream_t* stream, int32_t tile, const pb2_tile_t* desc);

/* Submit one task.  task->tile[] index the tile table; task->dep_goal is the number of pb2_stream_add_edge calls
 * that will name this task as successor (0: ready now); succ_begin / succ_count are ignored.  *ticket identifies the
 * task until its retire record has been polled.  PB2_ERR_OUT_OF_RESOURCE: ring full -- poll and retry. */
int  pb2_stream_submit(pb2_stream_t* stream, const pb2_task_t* task, uint64_t cookie, int32_t* ticket);

/* The successor (already submitted, with this edge counted in its dep_goal) must wait for `pred_ticket`, a task whose
 * retire record the caller has NOT polled yet. */
int  pb2_stream_add_edge(pb2_stream_t* stream, int32_t pred_ticket, int32_t succ_ticket);

/* Make everything submitted so far visible to the device and make sure the persistent kernel is running. */
int  pb2_stream_kick(pb2_stream_t* stream);

/* Non-blocking: copy up to `max` retire records, oldest first; returns how many, or a negative PB2_ERR_* when the
 * device reported a failure (watchdog, bad body). */
int  pb2_stream_poll(pb2_stream_t* stream, pb2_retire_t* out, int32_t max);

/* Block until every submitted task has retired (records stay queued for pb2_stream_poll) and the kernel has parked;
 * after this no kernel of the stream is resident.  */
int  pb2_stream_quiesce(pb2_stream_t* stream);
int  pb2_stream_stats(pb2_stream_t* stream, pb2_stream_stats_t* stats);
int  pb2_stream_inflight(pb2_stream_t* stream);     /* submitted and not yet polled                                    */

#ifdef __cplusplus
}
#endif
#endif /* PB2_STREAM_H */
