/*
 * pb2_device_body.h -- device ABI of the bodies an application links into HBM engine windows
 * (pb2_engine_link_bodies).
 *
 * The application compiles ONE device function against this header, to a relocatable sm_90a cubin
 * (nvcc -rdc=true -cubin -gencode arch=compute_90a,code=sm_90a) or to PTX (nvcc -rdc=true -ptx, or NVRTC with
 * -rdc=true), and hands the image to pb2_engine_link_bodies.  The engine links it into its own build of the HBM window
 * kernel; windows whose tasks name a body id PB2_BODY_LINKED_0 .. PB2_BODY_LINKED_7 (20..27) run that kernel, and it
 * calls
 *
 *     extern "C" __device__ unsigned long long pb2_linked_body(int body, const pb2_body_args_t* a, unsigned int* scratch);
 *
 * with the task's body id unchanged.  Contract:
 *   - All 64 threads of the worker CTA call it together (uniform control flow), so __syncthreads() is allowed.
 *   - a: this part's slice of every flow (flow[f] / bytes[f]; NULL / 0 for a flow without a tile), the slice's first
 *     4-byte element inside the tile (elem0), the part index and the task's immediates.  A body whose bit is clear in
 *     the `sliceable` mask of the link call always runs as one part over whole tiles (part 0, elem0 0); a body whose bit
 *     is set may be cut into byte-slice parts like the built-in element-wise bodies, each part run by another worker.
 *   - scratch: 32 words of the worker's shared memory, free for the body's use.
 *   - The result is taken from thread 0.  A multi-part task keeps the result of part 0.
 *   - Returning ~0ull aborts the window as a bad body (pb2_window_wait: PB2_ERR_BAD_PARAM).
 *   - Static __shared__ variables are allowed; they count against the linked kernel's occupancy, which
 *     pb2_engine_linked_info reports.
 *   - Stores to the flows are made visible to successor tasks by the engine (barrier + fence after the body).
 *
 * Plain C types only: the header compiles under gcc, nvcc and NVRTC without any other header.
 */
#ifndef PB2_DEVICE_BODY_H
#define PB2_DEVICE_BODY_H

#define PB2_BODY_ARGS_FLOWS 4

typedef struct pb2_body_args_s {
    void*        flow[PB2_BODY_ARGS_FLOWS];    /* device pointer of this part's slice of each flow's tile          */
    unsigned int bytes[PB2_BODY_ARGS_FLOWS];   /* bytes of the slice                                               */
    unsigned int elem0;                        /* index of the slice's first 4-byte element inside the tile        */
    unsigned int part;                         /* part index (0 for a body that is not sliceable)                  */
    int          iparam[3];                    /* pb2_task_t::iparam                                               */
    float        fparam;                       /* pb2_task_t::fparam                                               */
} pb2_body_args_t;                             /* 72 bytes on LP64 */

#if defined(__CUDACC__)
extern "C" __device__ unsigned long long pb2_linked_body(int body, const pb2_body_args_t* a, unsigned int* scratch);
#endif

#endif /* PB2_DEVICE_BODY_H */
