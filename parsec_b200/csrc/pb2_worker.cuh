// pb2_worker.cuh -- what one worker CTA does with one (part of a) task: push (stage-in), exec (body), pop (pushout).
// Shared by the HBM window kernel (pb2_hbm.cuh), the streaming kernel (pb2_stream.cu) and the HBM-body units of the
// GEMM window kernel (pb2_gemm.cuh); they differ only in where ready tasks come from, in what runs as the body and in
// how a finished task is retired and its successors are released.
//
// Reference: parsec_device_kernel_push / _exec / _pop, parsec/mca/device/device_gpu.c:2745, :2873, :2943.
//
// Register discipline: the HBM and streaming kernels are built for 12 CTAs of 64 threads per SM (<= 80 registers per
// thread).  Everything that is indexed by a run-time flow number lives in shared memory (TaskSmem), filled by one thread
// per flow, so that no array is demoted to local memory; tile payloads move through TMA (no payload registers) or
// 4 x 16-byte loads.  The GEMM kernel (384 threads, no bulk ring) runs the same code with BULK = false.
#pragma once
#include "pb2_sched.cuh"

namespace pb2 {

struct alignas(16) TaskSmem {
    pb2_task_t task;                 // four 16-byte loads
    BodyArgs   args;                 // this part's slice of every flow
    uint32_t   off[PB2_MAX_FLOWS];   // byte offset of the slice inside its tile
    uint32_t   tbytes[PB2_MAX_FLOWS];// whole-tile byte counts
    int32_t    entry;                // ring entry popped (kEmpty: leave)
    int32_t    need;                 // bit f: flow f has to be staged in
    int32_t    decide;               // scratch of the stage-in helpers
    int32_t    last;                 // this part retired the task
    int32_t    window_done;          // this task was the last of the window
    uint32_t   red[32];
};

// All threads (uniform): stage in every flow whose bit is set in s.need.  One CTA-wide call per task at most.
// BULK: the calling kernel has a TMA bulk ring (without one the copies take the SIMT loops).  Each instantiation has
// one caller kernel per translation unit: a second caller kernel makes ptxas give this helper the standard call ABI,
// which costs the HBM kernels a stack frame and spills at their 80-register budget (see pb2_hbm.cuh).  COUNT (traced
// kernels): add the bytes this CTA moved to *moved.
template <bool BULK, bool COUNT>
static __device__ __noinline__ void stage_in_needed_flows(const StageCtx c, TaskSmem* sp, BulkSmem* bulk, unsigned long long* moved) {
    TaskSmem& s = *sp;
    const int need = s.need;
#pragma unroll 1
    for (int f = 0; f < PB2_MAX_FLOWS; ++f) {
        if (!((need >> f) & 1)) continue;
        const int32_t tid = s.task.tile[f];
        const uint32_t bytes = s.tbytes[f];
        const int ns = tile_slices_of(c.part_bytes, c.slice_claim, bytes);
        if (ns == 1) {
            stage_in_flow<COUNT>(c, &c.tiles[tid], s.task.access[f], &s.decide, BULK ? bulk : nullptr, moved);
        } else {
            int s0, s1;
            slices_over(bytes, ns, s.off[f], s.args.bytes[f], s0, s1);     // the slices under this part's bytes
            stage_in_slices<COUNT>(c, tid, ns, s0, s1, &s.decide, BULK ? bulk : nullptr, moved);
        }
    }
}

// All threads.  On entry s.task holds the descriptor (published by a barrier).  exec() runs the body over s.args (all
// threads) and returns its result in thread 0.  Returns the body result (thread 0).  BULK as for
// stage_in_needed_flows; without it `bulk` is not used.  TRACE (traced window kernels): thread 0 stamps the end of the
// stage-in, of the body and of the pushout into *rec, and counts the bytes this CTA moved in and pushed out there.
template <bool BULK, bool TRACE = false, class Exec>
__device__ __forceinline__ unsigned long long
run_task_part(const WinDev& w, TaskSmem& s, BulkSmem* bulk, int32_t id, int part, int nparts, Exec exec,
              PartSmem* rec = nullptr) {
    const pb2_task_t& t = s.task;
    // ---- push: one thread per flow works out its slice and whether the tile has to be staged in -----------------
    if (threadIdx.x < 32) {
        const int f = (int)threadIdx.x;
        const bool mine = f < PB2_MAX_FLOWS && f < (int)t.nb_flows && t.tile[f < PB2_MAX_FLOWS ? f : 0] >= 0;
        pb2_tile_t* tile = mine ? &w.tiles[t.tile[f]] : nullptr;
        const uint32_t bytes = mine ? tile->bytes : 0u;
        // every flow is cut at the offsets of the task's widest tile (part_slice)
        uint32_t widest = bytes;
        for (int o = 1; o < PB2_MAX_FLOWS; o <<= 1) {
            const uint32_t v = __shfl_xor_sync(0xffffffffu, widest, o);
            widest = v > widest ? v : widest;
        }
        uint32_t off, len;
        part_slice(widest, (uint32_t)nparts, (uint32_t)part, bytes, off, len);
        const bool need = mine && (t.access[f] & PB2_FLOW_ACCESS_READ) && ld_acquire_gpu(&tile->state) != PB2_TILE_VALID;
        const unsigned needmask = __ballot_sync(0xffffffffu, need);
        if (f < PB2_MAX_FLOWS) {
            s.args.flow[f] = mine ? reinterpret_cast<uint8_t*>(tile->dev_ptr) + off : nullptr;
            s.args.bytes[f] = len; s.off[f] = off; s.tbytes[f] = bytes;
            if (mine && part == 0)
                w.seen_version[(size_t)id * PB2_MAX_FLOWS + f] = *reinterpret_cast<volatile uint32_t*>(&tile->version);
        }
        if (f == 0) {
            s.need = (int32_t)needmask;
            s.args.part = (uint32_t)part; s.args.elem0 = off >> 2;
            s.args.iparam[0] = t.iparam[0]; s.args.iparam[1] = t.iparam[1]; s.args.iparam[2] = t.iparam[2];
            s.args.fparam = t.fparam;
        }
    }
    __syncthreads();
    // the cold path, out of line and called once: everything it needs is in shared memory, nothing of the caller's
    // has to survive the call in registers
    if (s.need) stage_in_needed_flows<BULK, TRACE>(stage_ctx(w), &s, bulk, TRACE ? &rec->in_bytes : nullptr);
    if (TRACE && threadIdx.x == 0) { if (s.need) rec->flags |= PB2_PART_WAITED_INPUT; rec->t_in = globaltimer_ns(); }

    // ---- exec: the body (parsec_device_kernel_exec -> submit) ----
    const unsigned long long r = exec();
    __syncthreads();
    if (TRACE && threadIdx.x == 0) rec->t_exec = globaltimer_ns();

    // ---- pop: pushout of written flows to their home copy (parsec_device_kernel_pop stage_out) ----
#pragma unroll
    for (int f = 0; f < PB2_MAX_FLOWS; ++f) {
        if (f < (int)t.nb_flows && t.tile[f] >= 0 && (t.access[f] & PB2_FLOW_PUSHOUT) && (t.access[f] & PB2_FLOW_ACCESS_WRITE)) {
            const pb2_tile_t* tile = &w.tiles[t.tile[f]];
            cta_copy<false>(reinterpret_cast<uint8_t*>(tile->src_ptr) + s.off[f], s.args.flow[f], s.args.bytes[f],
                            BULK ? bulk : nullptr);
            if (threadIdx.x == 0) atomicAdd(&w.ctl->bytes_d2h.v, (unsigned long long)s.args.bytes[f]);
            if (TRACE && threadIdx.x == 0) rec->out_bytes += s.args.bytes[f];
        }
    }
    __syncthreads();
    if (TRACE && threadIdx.x == 0) rec->t_out = globaltimer_ns();     // trace_part reports t_exec if nothing went out
    return r;
}

// Thread 0 of the part that finished last: version / coherency epilog of the written flows
// (version = candidate->version + 1 for WRITE flows, device_gpu.c:2148-2152).  Returns the version it gave tile x
// (0: t does not write x).
__device__ __forceinline__ uint32_t epilog_written_flows(const WinDev& w, const pb2_task_t& t, int32_t x = -1) {
    uint32_t vx = 0;
    for (int f = 0; f < (int)t.nb_flows; ++f) {
        if (t.tile[f] < 0 || !(t.access[f] & PB2_FLOW_ACCESS_WRITE)) continue;
        pb2_tile_t* tile = &w.tiles[t.tile[f]];
        const uint32_t v = *reinterpret_cast<volatile uint32_t*>(&tile->version) + 1;
        *reinterpret_cast<volatile uint32_t*>(&tile->version) = v;
        if (t.tile[f] == x) vx = v;
        if (!(t.access[f] & PB2_FLOW_ACCESS_READ)) st_relaxed_gpu(&tile->state, PB2_TILE_VALID);
    }
    return vx;
}

// Thread 0: store a CHECK body's result of this part (the mismatch counts of the parts add up).
__device__ __forceinline__ void store_check_result(const WinDev& w, int32_t id, int nparts, unsigned long long r) {
    if (nparts == 1) w.result[id] = r; else if (r) atomicAdd(&w.result[id], r);
    if (r >> 32) atomicAdd(&w.ctl->body_errors.v, r >> 32);
}

// Thread 0: store the body result of this part.
__device__ __forceinline__ void store_result(const WinDev& w, const pb2_task_t& t, int32_t id, int part, int nparts,
                                             unsigned long long r) {
    if (r == ~0ull) st_relaxed_gpu(reinterpret_cast<int32_t*>(&w.ctl->done.v), kDoneBadBody);
    if (t.body == PB2_BODY_CHECK_I32 || t.body == PB2_BODY_CHECK_F32) store_check_result(w, id, nparts, r);
    else if (part == 0) w.result[id] = r;
}

}  // namespace pb2
