/*
 * device_b200.h -- public interface of the b200 device component (parsec/mca/device/b200).
 *
 * The component fills the reference's own plug-in contract: one parsec_device_module_t (parsec/mca/device/device.h:145-189)
 * per GPU, type PARSEC_DEV_CUDA so that BODY [type=CUDA] chores emitted by parsec-ptgpp (jdf2c.c:6832-6969) and DTD
 * chores added with PARSEC_DEV_CUDA (insert_function.c:2393-2425) are scheduled on it unchanged, and a
 * kernel_scheduler (device.h:133) that takes the parsec_gpu_task_t those hooks build (device_gpu.h:117-155).
 *
 * What a body can do differently on this device: instead of enqueueing a CUDA kernel on the stream it is given, it
 * may NAME one of the engine's in-kernel bodies with parsec_b200_task_body().  The task then runs inside the
 * persistent kernel (stage-in, body, pushout and successor release on the device, no launch, no event).  The same
 * call made under any other device module (the reference's cuda component for instance) launches an equivalent
 * stand-alone kernel on the stream, so one .jdf serves both.
 */
#ifndef PARSEC_DEVICE_B200_H
#define PARSEC_DEVICE_B200_H

#include "parsec/mca/device/device_gpu.h"

BEGIN_C_DECLS

extern parsec_device_base_component_t parsec_device_b200_component;

/* bodies: enum pb2_body_e of include/pb2_engine.h (PB2_BODY_FILL_I32, PB2_BODY_CHECK_I32, PB2_BODY_INCR_F32, ...) */

/**
 * To be called from the body of a GPU incarnation (the submit function, device_gpu.h:49-51).
 * @param gpu_device, gpu_task, gpu_stream  the three arguments of the submit function
 * @param body        enum pb2_body_e
 * @param nb_args     how many task flows the body uses (1..4)
 * @param flow_index  flow_index[i] = index of the task flow bound to body argument i
 * @param iparam      three integer immediates (may be NULL)
 * @param fparam      one float immediate
 * @return PARSEC_HOOK_RETURN_DONE, or PARSEC_HOOK_RETURN_ERROR for a bad argument
 */
int parsec_b200_task_body(parsec_device_gpu_module_t *gpu_device, parsec_gpu_task_t *gpu_task,
                          parsec_gpu_exec_stream_t *gpu_stream,
                          int body, int nb_args, const int *flow_index, const int32_t *iparam, float fparam);

/* the body result of a finished task that named a CHECK body: mismatches << 32 | first element (valid inside a
 * complete_stage callback and until the gpu_task is released) */
uint64_t parsec_b200_task_result(const parsec_gpu_task_t *gpu_task);

/* 1 when `device` is a module of this component */
int parsec_b200_is_b200_device(const parsec_device_module_t *device);

/* counters of one b200 device (engine extension of the statistics of device.h:165-171) */
typedef struct parsec_b200_stats_s {
    uint64_t tasks_engine;          /* ran inside the persistent kernel                                             */
    uint64_t tasks_lane;            /* opaque submit bodies run on the stream lane                                   */
    uint64_t kernel_launches;       /* (re)starts of the persistent kernel                                           */
    uint64_t released_on_device;    /* successors made ready by a device-side decrement (look-ahead)                 */
    uint64_t bytes_h2d_kernel, bytes_d2d_kernel, bytes_d2h_kernel;  /* moved by the persistent kernel               */
    uint64_t bytes_h2d_dma, bytes_d2h_dma;                          /* moved by the copy engine (unregistered memory)*/
    uint64_t evictions, w2r_copies;
    uint64_t registration_hits;             /* memory_register calls served by the registration cache */
    uint64_t first_entry_ns, first_task_ns, last_done_ns;   /* CLOCK_MONOTONIC of the first hand-over / last completion since the last memory_release */
    uint64_t peer_pulls;            /* stage-ins whose source was another GPU's replica, read over NVLink           */
    uint64_t peer_detours;          /* GPU sources that could not be read in place (no peer access): copy engine      */
    uint64_t check_mismatches;      /* elements the CHECK bodies found different from what they expected             */
    uint64_t manager_entries;       /* how often a worker thread became the manager                                  */
    uint64_t lane_batched;          /* lane tasks a batching body took along (parsec_gpu_task_collect_batch)          */
    uint64_t forwarded;             /* tasks short of memory here that were handed to the peer device holding their inputs */
    uint64_t max_concurrent_callers;
} parsec_b200_stats_t;
int parsec_b200_get_stats(const parsec_device_module_t *device, parsec_b200_stats_t *stats);

END_C_DECLS
#endif
