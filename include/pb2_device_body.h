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
 * with the task's body id unchanged.  Linked with PB2_LINK_GEMM_WINDOWS (pb2_engine_link_bodies_ex), GEMM windows run
 * it too.  Contract:
 *   - All threads of the worker CTA call it together (uniform control flow), so __syncthreads() is allowed: 64 in HBM
 *     windows, 384 in GEMM windows; use blockDim.x.
 *   - a: this part's slice of every flow (flow[f] / bytes[f]; NULL / 0 for a flow without a tile), the slice's first
 *     4-byte element inside the tile (elem0), the part index and the task's immediates.  A body whose bit is clear in
 *     the `sliceable` mask of the link call always runs as one part over whole tiles (part 0, elem0 0); a body whose bit
 *     is set may be cut into byte-slice parts like the built-in element-wise bodies, each part run by another worker.
 *   - scratch: 32 words of the worker's shared memory, free for the body's use (32 in GEMM windows too; a GEMM-worker
 *     body, below, gets the worker's whole operand ring).
 *   - The result is taken from thread 0.  A multi-part task keeps the result of part 0 (a reader's add up, below).
 *   - Returning ~0ull aborts the window as a bad body (pb2_window_wait: PB2_ERR_BAD_PARAM).
 *   - Static __shared__ variables are allowed; they count against the linked kernel's occupancy, which
 *     pb2_engine_linked_info reports (pb2_engine_linked_gemm_info for GEMM windows, where they come on top of the
 *     kernel's 193 KiB of dynamic shared memory).
 *   - Stores to the flows are made visible to successor tasks by the engine (barrier + fence after the body).
 *
 * Checked bodies (pb2_engine_link_bodies_checked): `a` always points at the `args` member of a pb2_body_check_t, whose
 * `check` and `k0` follow the 72 bytes of pb2_body_args_t; an image compiled against a header without them never reads
 * them, and `check` is 1 only for a body id whose bit is set in the link's `checked` mask (in HBM windows, and in GEMM windows
 * linked with PB2_LINK_GEMM_WINDOWS, on their 384 threads).  The engine then runs the
 * task fused with the CHECK tasks that read its output tile (one read group), on the same worker, and calls the body in
 * check mode.  A body in check mode
 *   - writes its slice of the output flow (the one flow it writes) exactly as it does with check 0, and stores every
 *     whole 4-byte element of that slice (bytes past the last whole element are stored but not checked);
 *   - returns, from EVERY thread, a value whose low 32 bits are nonzero if and only if some element that thread stored
 *     differs from k0, and whose high 32 bits are zero.
 * Thread 0 returning ~0ull still aborts the window as a bad body.  A fused producer's own result is recorded as 0.  The
 * engine decides the readers' results from one barrier over these values, and counts their mismatches exactly from the
 * tile only when some thread reported one.  The body's stores carry whatever cache policy the body gives them.
 *
 * Readers (PB2_LINK_READERS(mask) in the flags of pb2_engine_link_bodies_ex, a subset of `sliceable`): a body whose bit
 * is set in `mask`
 *   - only loads from its flows, and stores nothing to them;
 *   - may be called on any 16-byte-aligned sub-slice of a part (flow, bytes and elem0 describe that sub-slice), and
 *     several times in a row on one worker, with a barrier between calls; scratch does not survive from one call to
 *     the next;
 *   - has its task's result defined as the sum, modulo 2^64, of the values thread 0 returns over all calls and parts.
 *     ~0ull from any call still aborts the window, and is not added.  A task that runs as one call keeps its value.
 * The result is then the same whether the engine runs the task alone, cuts it into parts, runs it with the other
 * readers of the same tile on one worker (a read group, which calls every member on one chunk of the part before the
 * next), or fuses that group with the task that writes the tile (which then writes each chunk before the members read it
 * back, with check 0: it needs no checked form).  Reductions that must not depend on that order are integer ones.
 *
 * Reader groups (PB2_LINK_READER_GROUPS(mask), bits 16..23 of the same flags, a subset of the readers mask): the image
 * also defines
 *
 *     extern "C" __device__ unsigned long long pb2_linked_reader_group(const pb2_reader_group_t* g,
 *                                                                      unsigned long long* results, unsigned int* scratch);
 *
 * and a read group calls it once per chunk for all of its members whose bit is set in `mask`, instead of calling
 * pb2_linked_body once per member; the group's other members are still called one by one.  Contract:
 *   - All threads of the worker call it together, as pb2_linked_body: 64 in HBM windows, 384 in GEMM windows.
 *   - g: one chunk of the group's tile (flow, bytes, elem0 and part mean what flow[0], bytes[0], elem0 and part of
 *     pb2_body_args_t mean for a reader) and the n members of the call, each with its body id and its task's immediates.
 *   - results[0 .. n): shared memory that the engine zeroes before the call; any thread may atomicAdd into it.  After the
 *     call results[m] must equal what pb2_linked_body(g->body[m], <the same chunk>) returns from thread 0, so a task's
 *     result is the same integer on every path: alone, in parts, in a read group called per member or in one call.
 *     A results[m] of ~0ull marks member m as a bad body, as pb2_linked_body returning ~0 does.
 *   - scratch: the same 32 words of shared memory as pb2_linked_body gets.
 *   - ~0ull returned from thread 0 aborts the window as a bad body: every member of the call is then bad, and none of
 *     their results of the call is added.  Any other return value is ignored.
 *   - pb2_linked_body must still cover every id: readers that run alone, ungrouped windows (read_groups = -1) and
 *     members whose bit is clear use it.
 * An image linked with a nonzero mask must define pb2_linked_reader_group (the link fails otherwise, as any link error
 * does); with a zero mask the engine links kernels that never call it.  The call runs inside the HBM window kernel's
 * 80-register budget, which the link enforces: a form that keeps a value per member in registers may need
 * -maxrregcount=80 (tests/cuda/reader_group_bodies.cu is built so).
 *
 * GEMM-worker bodies (PB2_LINK_GEMM_BODIES(mask), bits 24..31 of the same flags, with PB2_LINK_GEMM_WINDOWS; disjoint
 * from `sliceable`, and so from `checked` and the readers masks): a body whose bit is set in `mask` runs in GEMM windows
 * only, and there `scratch` points at the GEMM worker's operand ring instead of the 32 words, so that the application
 * can stage tensor-core operands (fp64 DMMA, other layouts and precisions) in shared memory.  Contract, on top of the
 * one above:
 *   - The ring is PB2_GEMM_BODY_SMEM_BYTES bytes, 1024-byte aligned; its contents are undefined on entry, and the body
 *     may use all of it.  Nothing of it survives to the next task.
 *   - The body is called on all 384 threads of the worker (blockDim.x), once per task, over whole tiles (one part,
 *     elem0 0): such a task is never cut into byte slices, grouped with readers or fused with a producer.  It runs as
 *     several parts only when the application declares so (below, "in parts").
 *   - No TMA or bulk copy the body issues may still be in flight when it returns (cp.async copies must be waited on).
 *   - The engine executes fence.proxy.async before the call and after it, so the body's generic stores to the ring never
 *     race the wgmma reads and TMA writes of the GEMM units that run on the worker before or after it.
 *   - scratch is a generic pointer; __cvta_generic_to_shared(scratch) gives its shared-window address, for ld.shared,
 *     cp.async and ldmatrix.
 *   - Linked without PB2_LINK_GEMM_BODY_ENTRY, the body is reached through pb2_linked_body, which the engine links into
 *     its HBM window kernels too: the image must then fit their 80 registers per thread, as every image must
 *     (-maxrregcount=80; the link fails otherwise).  tests/cuda/gemm_worker_bodies.cu runs an fp64 DMMA tile GEMM within
 *     that budget.
 * The 32-word contract is a subset of this one: an image compiled against a header without the mask keeps working.
 * A task of such a body in an HBM window is refused (PB2_ERR_NOT_SUPPORTED).
 *
 * The GEMM-worker entry point (PB2_LINK_GEMM_BODY_ENTRY, bit 1 of the same flags, with a nonzero GEMM-worker mask): the
 * image also defines
 *
 *     extern "C" __device__ unsigned long long pb2_linked_gemm_body(int body, const pb2_body_args_t* a,
 *                                                                   unsigned int* scratch);
 *
 * and the GEMM window kernels call it, instead of pb2_linked_body, for every task of a body in the GEMM-worker mask.
 * Its contract is the GEMM-worker contract above (384 threads, once per task over whole tiles, scratch the ring, no bulk
 * copy in flight on return, the engine's fences around the call, the result from thread 0, ~0ull aborts the window),
 * with one difference: only the GEMM window kernels reach it, so its budget is theirs, PB2_GEMM_BODY_MAX_REGS (168)
 * registers per thread, and not the HBM kernels' 80.  Both budgets are enforced when the engine links the image: a
 * callee that needs more registers than a kernel that reaches it fails the link (PB2_ERR_BAD_PARAM, with the linker's
 * message), and the engine stays unlinked.  One image holds both entry points, so it is compiled with
 * -maxrregcount=168; its pb2_linked_body still reaches the HBM kernels and must still fit their 80 registers, which the
 * HBM link checks: keep the large bodies behind pb2_linked_gemm_body, and pb2_linked_body small.  Other linked
 * bodies in GEMM windows, and everything in HBM windows, still go through pb2_linked_body.  An image that defines both
 * and is linked without the flag runs its GEMM-worker bodies through pb2_linked_body; an image linked with the flag
 * must define pb2_linked_gemm_body (the link fails otherwise, as any link error does).  A PTX image is compiled by the
 * driver's JIT without any register cap, whatever -maxrregcount it was generated with: a function that then needs more
 * than a kernel's budget fails the link.  tests/cuda/gemm_entry_bodies.cu runs an fp64 DMMA tile GEMM with 32 x 32 of
 * C per warp through this entry.
 *
 * GEMM-worker bodies in parts (pb2_engine_set_gemm_body_parts(engine, body, nparts), pb2_device_set_gemm_body_parts):
 * every task of a body declared with nparts > 1 runs as nparts parts, through either entry point.  The default, 1, is
 * the contract above unchanged.  With nparts > 1:
 *   - The body is called once per part, on all 384 threads of a worker.  Parts may run at the same time on different
 *     workers, or one after another on one worker.
 *   - Every part gets the task's whole tiles: flow / bytes as for one part, elem0 0, and args.part = its part index p.
 *     `a` points at the `args` member of a pb2_gemm_body_args_t, whose `nparts` gives the count (1 for a task that
 *     runs as one part; check and k0 are 0).  An image compiled against a header without it never reads it.
 *   - The body splits the work by (p, nparts) itself: the parts store disjoint bytes of the flows the task writes, and
 *     no part reads bytes that another part of the same task writes.
 *   - Every part gets its own worker's ring as scratch, with the fences above; nothing passes from one part to another.
 *   - The task's result is part 0's; ~0ull from any part aborts the window.
 *   - The part that finishes last retires the task: successors are released and versions bumped once, after every
 *     part's stores.
 *   - A written flow marked PB2_FLOW_PUSHOUT is copied home whole and once, by the worker that retires the task, after
 *     the last part's stores; bytes_d2h and that part's record count it once.  The parts push nothing themselves:
 *     they are not byte slices of the tile.
 * Parts of a task that runs alone on a wide machine put more SMs on it; when the window has more independent tasks than
 * workers they only add operand traffic, so the count is the application's choice.
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

/* The block `a` of pb2_linked_body points into (at args): a body declared checked reads check and k0 through
 * ((const pb2_body_check_t*)a).  The layout of pb2_body_args_t is fixed by the images already compiled against it, so
 * the two words follow it rather than grow it. */
typedef struct pb2_body_check_s {
    pb2_body_args_t args;
    unsigned int    check;                     /* 1: check mode (only for ids in the link's `checked` mask), else 0 */
    unsigned int    k0;                        /* check mode: the constant every stored element is compared with    */
} pb2_body_check_t;                            /* 80 bytes on LP64 */

/* The block a GEMM-worker body's `a` points into (at args) in GEMM windows: pb2_body_check_t's words, then the parts
 * its task runs as (pb2_engine_set_gemm_body_parts).  Read it through ((const pb2_gemm_body_args_t*)a). */
typedef struct pb2_gemm_body_args_s {
    pb2_body_args_t args;
    unsigned int    check;                     /* 0                                                                 */
    unsigned int    k0;                        /* 0                                                                 */
    unsigned int    nparts;                    /* the task's parts (args.part is this part's index, 0 .. nparts - 1) */
    unsigned int    reserved;                  /* 0                                                                 */
} pb2_gemm_body_args_t;                        /* 88 bytes on LP64 */

#define PB2_GROUP_MAX 8                        /* members of a read group */

/* The shared memory a GEMM-worker body gets as `scratch`: the GEMM worker's operand ring, 1024-byte aligned. */
#define PB2_GEMM_BODY_SMEM_BYTES 196608
#define PB2_GEMM_BODY_SMEM_ALIGN 1024
/* The register budget of pb2_linked_gemm_body (PB2_LINK_GEMM_BODY_ENTRY): that of the GEMM window kernels, which alone
 * call it (__launch_bounds__(384, 1)); enforced when the engine links the image.  pb2_linked_body's budget is 80. */
#define PB2_GEMM_BODY_MAX_REGS 168

/* What pb2_linked_reader_group is handed: one chunk of the group's tile and the members of the call, in member order. */
typedef struct pb2_reader_group_s {
    const void*  flow;                         /* the chunk: device pointer, 16-byte aligned                       */
    unsigned int bytes;                        /* bytes of the chunk                                               */
    unsigned int elem0;                        /* index of the chunk's first 4-byte element inside the tile        */
    unsigned int part;                         /* part index                                                       */
    unsigned int n;                            /* members in this call, 1 .. PB2_GROUP_MAX                         */
    int          body[PB2_GROUP_MAX];          /* member m's body id                                               */
    int          iparam[PB2_GROUP_MAX][3];     /* member m's pb2_task_t::iparam                                    */
    float        fparam[PB2_GROUP_MAX];        /* member m's pb2_task_t::fparam                                    */
} pb2_reader_group_t;                          /* 184 bytes on LP64 */

#if defined(__CUDACC__)
extern "C" __device__ unsigned long long pb2_linked_body(int body, const pb2_body_args_t* a, unsigned int* scratch);
extern "C" __device__ unsigned long long pb2_linked_reader_group(const pb2_reader_group_t* g, unsigned long long* results,
                                                                 unsigned int* scratch);
extern "C" __device__ unsigned long long pb2_linked_gemm_body(int body, const pb2_body_args_t* a, unsigned int* scratch);
#endif

#endif /* PB2_DEVICE_BODY_H */
