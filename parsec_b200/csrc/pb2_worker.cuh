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
// GEMM_BODY_PARTS (the linked GEMM window kernels): a part of a GEMM-worker task that runs in parts
// (pb2_engine_set_gemm_body_parts) covers the task's whole tiles, whose stage-in the parts share through the slice
// claims, and pushes nothing out: the part that retires the task pushes its flows out whole (pb2_gemm.cuh).
template <bool BULK, bool TRACE = false, bool GEMM_BODY_PARTS = false, class Exec>
__device__ __forceinline__ unsigned long long
run_task_part(const WinDev& w, TaskSmem& s, BulkSmem* bulk, int32_t id, int part, int nparts, Exec exec,
              PartSmem* rec = nullptr) {
    const pb2_task_t& t = s.task;
    const bool whole = GEMM_BODY_PARTS && nparts > 1 && (t.flags & PB2_TASK_GEMM_BODY);
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
        part_slice(widest, whole ? 1u : (uint32_t)nparts, whole ? 0u : (uint32_t)part, bytes, off, len);
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
        if (!whole && f < (int)t.nb_flows && t.tile[f] >= 0 && (t.access[f] & PB2_FLOW_PUSHOUT) && (t.access[f] & PB2_FLOW_ACCESS_WRITE)) {
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

// Thread 0: store a linked reader's result of this part (the sum of its calls): the parts' results add up, modulo 2^64;
// ~0 aborts the window and is not added.
__device__ __forceinline__ void store_reader_result(const WinDev& w, int32_t id, int nparts, unsigned long long r) {
    if (r == ~0ull) st_relaxed_gpu(reinterpret_cast<int32_t*>(&w.ctl->done.v), kDoneBadBody);
    else if (nparts == 1) w.result[id] = r;
    else if (r) atomicAdd(&w.result[id], r);
}

// Thread 0: store the body result of this part.  LINKED (the linked kernels): a task marked PB2_TASK_READER adds it.
template <bool LINKED = false>
__device__ __forceinline__ void store_result(const WinDev& w, const pb2_task_t& t, int32_t id, int part, int nparts,
                                             unsigned long long r) {
    if (LINKED && (t.flags & PB2_TASK_READER)) { store_reader_result(w, id, nparts, r); return; }
    if (r == ~0ull) st_relaxed_gpu(reinterpret_cast<int32_t*>(&w.ctl->done.v), kDoneBadBody);
    if (t.body == PB2_BODY_CHECK_I32 || t.body == PB2_BODY_CHECK_F32) store_check_result(w, id, nparts, r);
    else if (part == 0) w.result[id] = r;
}

// ---------------------------------------------------------------------------------------------
// read groups and fused producer units (form_read_groups, pb2_window_plan.cpp), in the HBM window kernel and in the
// HBM-body units of the GEMM window kernel
// ---------------------------------------------------------------------------------------------
// The out-of-line helpers below take NT, the threads of the calling kernel's CTA (PB2_HBM_THREADS or gemm::kThreads):
// their loops use blockDim.x, and NT gives each kernel its own instantiation, so that no helper has two caller kernels
// in one translation unit (see stage_in_needed_flows).

// A read group in flight on one worker: its members (the leader first), their CHECK constants and out-edges, this
// part's results.  The retire path takes what it needs of a member from here, not from its descriptor.
struct GroupSmem {
    int32_t n;                              // members; 0: the popped task runs alone
    int32_t fused;                          // the popped task is a producer that runs with this group as one unit
    int32_t tile;                           // the tile the members read
    int32_t mem[PB2_GROUP_MAX];
    uint32_t k[PB2_GROUP_MAX];
    int32_t succ_begin[PB2_GROUP_MAX];
    int32_t succ_count[PB2_GROUP_MAX];
    unsigned long long res[PB2_GROUP_MAX];  // res[0]: the leader's result, set before group_results
};

// All threads: the members of the group that task id leads or runs with (w.group) into g, published by the caller's
// barrier.  Returns id's group word (0: id runs alone); thread 0 of the caller sets g.n and g.fused from it.
__device__ __forceinline__ uint32_t load_group_members(const WinDev& w, int32_t id, GroupSmem& g) {
    const uint32_t gd = w.group ? __ldg(&w.group[id]) : 0u;
    const int gn = (int)(gd & 15u);
    const uint32_t gb = (gd & ~PB2_GROUP_FUSED) >> 4;
    if ((int)threadIdx.x < gn) {
        const int32_t m = __ldg(&w.group_mem[gb + threadIdx.x]);
        const pb2_task_t& mt = w.tasks[m];
        g.mem[threadIdx.x] = m;
        g.k[threadIdx.x] = mt.body == PB2_BODY_CHECK_F32 ? __float_as_uint(__ldg(&mt.fparam)) : (uint32_t)__ldg(&mt.iparam[0]);
        g.succ_begin[threadIdx.x] = __ldg(&mt.succ_begin);
        g.succ_count[threadIdx.x] = __ldg(&mt.succ_count);
        if (threadIdx.x == 0) g.tile = __ldg(&mt.tile[0]);
    }
    return gd;
}

// Whether g, published, is a read group of linked readers (run_linked_group_part): its members are marked
// PB2_TASK_READER, a CHECK group's never.
__device__ __forceinline__ bool linked_reader_group(const WinDev& w, const GroupSmem& g) {
    return g.n && (__ldg(&w.tasks[g.mem[0]].flags) & PB2_TASK_READER);
}

// All threads, after run_task_part ran the leader's CHECK over this part's slice.  Every member compares the same
// bytes with its own constant k (CHECK_F32 compares the bits of fparam, so both bodies are CHECK_I32 on the bits):
//  - k equal to the leader's: the leader's result;
//  - the slice held nothing but the leader's constant: every element mismatches (the first element is the same);
//  - otherwise the member's slice is counted again, exactly, as a failing CHECK counts it.
template <int NT>
static __device__ __noinline__ void group_results(TaskSmem* sp, GroupSmem* gp) {
    TaskSmem& s = *sp;
    GroupSmem& g = *gp;
    const unsigned long long r0 = g.res[0];
#pragma unroll 1
    for (int i = 1; i < g.n; ++i) {
        const uint32_t k = g.k[i];
        if (k == g.k[0] || !(r0 >> 32)) {
            if (threadIdx.x == 0) g.res[i] = k == g.k[0] ? r0 : ((unsigned long long)(s.args.bytes[0] >> 2) << 32) | (uint32_t)r0;
            continue;
        }
        if (threadIdx.x == 0) s.args.iparam[0] = (int32_t)k;
        __syncthreads();
        const unsigned long long r = run_hbm_body(PB2_BODY_CHECK_I32, s.args, s.red);
        if (threadIdx.x == 0) g.res[i] = r;
        __syncthreads();
    }
    __syncthreads();
}

// All threads, after run_task_part ran the leader of a read group (not fused) over this part with result r (thread 0):
// the members' results of the part.  TRACE: the members' results are part of the body; the readers push nothing out.
template <int NT, bool TRACE>
__device__ __forceinline__ void group_part_results(const WinDev& w, TaskSmem& s, GroupSmem& g, int32_t id, int part,
                                                   unsigned long long r, PartSmem* rec) {
    // the leader's part stored the version it saw; every member saw the same one
    if (threadIdx.x == 0) {
        g.res[0] = r;
        if (part == 0) {
            const uint32_t v = *reinterpret_cast<volatile uint32_t*>(&w.seen_version[(size_t)id * PB2_MAX_FLOWS]);
            for (int i = 1; i < g.n; ++i) w.seen_version[(size_t)g.mem[i] * PB2_MAX_FLOWS] = v;
        }
    }
    __syncthreads();
    group_results<NT>(&s, &g);
    if (TRACE && threadIdx.x == 0) rec->t_exec = rec->t_out = globaltimer_ns();
}

// Thread 0, after a part of task id ran with result r: the part's results, the members' of a group first (CHECK bodies,
// or in the LINKED kernels linked readers), then id's own unless id is a group's leader (members[0] has it).
template <bool LINKED = false>
__device__ __forceinline__ void store_part_results(const WinDev& w, const pb2_task_t& t, int32_t id, int part, int nparts,
                                                   unsigned long long r, const GroupSmem& g) {
    const int gn = g.n;
    if (LINKED && linked_reader_group(w, g))
        for (int i = 0; i < gn; ++i) store_reader_result(w, g.mem[i], nparts, g.res[i]);
    else
        for (int i = 0; i < gn; ++i) store_check_result(w, g.mem[i], nparts, g.res[i]);
    if (!gn || g.fused) store_result<LINKED>(w, t, id, part, nparts, r);
}

// All threads, after the producer of a fused unit stored its slice of output flow fx and one barrier told them whether
// any element it stored differed from the leader's constant k0: the members' results (run_fused_part).
static __device__ __forceinline__ void fused_member_results(TaskSmem& s, GroupSmem& g, uint32_t k0, bool mismatch, int fx) {
    const uint32_t len = s.args.bytes[fx];
    const uint32_t* const out = static_cast<const uint32_t*>(s.args.flow[fx]);
    // the slice's first element: k0 if nothing mismatched, else what thread 0 stored there
    const uint32_t first = threadIdx.x == 0 && s.args.part == 0 && len >= 4 ? (mismatch ? __ldcg(out) : k0) : 0u;
    if (!mismatch) {
        if (threadIdx.x == 0)
            for (int m = 0; m < g.n; ++m) g.res[m] = g.k[m] == k0 ? first : ((unsigned long long)(len >> 2) << 32) | first;
        return;
    }
    unsigned long long r0 = 0;
#pragma unroll 1
    for (int m = 0; m < g.n; ++m) {
        const uint32_t k = g.k[m];
        unsigned long long rm = r0;
        if (m == 0 || k != k0) rm = ((unsigned long long)cta_count_ne(out, len, k, s.red) << 32) | first;
        if (threadIdx.x == 0) { if (m == 0) r0 = rm; g.res[m] = rm; }
    }
}

// All threads, in place of the body of a producer fused with its read group (fuse_readers).  s.args holds the
// producer's slice of every flow for this part.  Run as separate tasks, the readers of a tile come long after its
// writer: every other worker writes its own tile in between, far more than L2 holds.  Here the members check the bytes
// before they leave the SM: the producer's checked body (run_hbm_body<true>) writes its output flow as it would alone,
// and every thread ORs (element ^ the leader's constant) of each value it stores while the value is still in registers.
// Its stores carry an L2 evict-first policy: nobody reads the tile back here (the resident Ex05 step is about 3 %
// shorter than with the default policy, DESIGN.md §8).  One barrier then tells every thread whether the slice held
// anything but the leader's constant, and the members get group_results' rules:
//  - nothing else: a member with the leader's constant counts no mismatch, any other member counts every element;
//  - otherwise the slice is counted again, exactly, from the tile (the barrier made the CTA's stores visible to its
//    threads, and the loads go through L2), for the leader and every member whose constant differs from the leader's.
// Returns the producer's result (thread 0); the caller's barrier and __threadfence() order the stores before the release.
template <int NT>
static __device__ __noinline__ unsigned long long run_fused_part(TaskSmem* sp, GroupSmem* gp) {
    TaskSmem& s = *sp;
    GroupSmem& g = *gp;
    const int body = s.task.body;
    const uint32_t k0 = g.k[0];
    Checked ck{k0, 0u, l2_evict_first()};
    const unsigned long long r = run_hbm_body<true>(body, s.args, s.red, &ck);
    const bool mismatch = __syncthreads_or(ck.diff != 0u) != 0;
    const int fx = (body == PB2_BODY_COPY || body == PB2_BODY_AXPY_F32) ? 1 : 0;     // see fusable() in form_read_groups
    fused_member_results(s, g, k0, mismatch, fx);
    return r;
}

// All threads, in place of a linked body (LINKED instantiations).  The body gets its slice in the 80-byte block *lp
// (include/pb2_device_body.h), with check 0, unless the task is a checked linked producer fused with its read group:
// then it runs in check mode against the leader's constant, its threads' return values stand for run_fused_part's
// Checked::diff, and the members get their results as there.  Its output flow is the flow whose tile is the group's
// (the one flow it writes, fusable() in form_read_groups).  Its stores carry the body's own cache policy: unlike the
// built-in producers it writes without the evict-first hint.  A fused producer's own result is 0 (~0 still aborts).
template <int NT>
static __device__ __noinline__ unsigned long long run_linked_part(TaskSmem* sp, GroupSmem* gp, pb2_body_check_t* lp) {
    TaskSmem& s = *sp;
    GroupSmem& g = *gp;
    const bool fused = g.fused != 0;
    static_assert(sizeof(BodyArgs) % 4 == 0 && sizeof(BodyArgs) / 4 <= NT, "one word of BodyArgs per thread");
    if (threadIdx.x < sizeof(BodyArgs) / 4)
        reinterpret_cast<uint32_t*>(&lp->args)[threadIdx.x] = reinterpret_cast<const uint32_t*>(&s.args)[threadIdx.x];
    if (threadIdx.x == 0) { lp->check = fused ? 1u : 0u; lp->k0 = fused ? g.k[0] : 0u; }
    __syncthreads();
    const unsigned long long r = pb2_linked_body(s.task.body, &lp->args, s.red);
    if (!fused) return r;
    const bool mismatch = __syncthreads_or((uint32_t)r != 0u) != 0;
    int fx = 0;
    while (fx + 1 < (int)s.task.nb_flows && !(s.task.tile[fx] == g.tile && (s.task.access[fx] & PB2_FLOW_ACCESS_WRITE))) ++fx;
    fused_member_results(s, g, lp->k0, mismatch, fx);
    return threadIdx.x == 0 && r == ~0ull ? ~0ull : 0ull;
}

// The bytes a read group of linked readers walks its part in (run_linked_group_part): half of H100's 50 MB L2 (sm_90a
// is the only target) over the kernel's workers, in whole 4 KiB, at least 4 KiB.  Every worker keeps one chunk in
// flight, so the chunks of all workers stay inside L2 while the members re-read them: 24 KiB with the HBM window's
// 1 056 workers, 192 KiB with the GEMM window's 132.  Chunks that overflow L2 send the re-reads to DRAM, and small
// ones pay the per-call barriers more often (the sweep is in DESIGN.md §8, *Linked readers*).
constexpr uint32_t kL2Bytes = 50u << 20;
__device__ __forceinline__ uint32_t reader_chunk_bytes() {
    const uint32_t c = (kL2Bytes / 2u / gridDim.x) & ~4095u;
    return c < 4096u ? 4096u : c;
}

// Thread 0: a reader's results over its calls, ~0 kept once any call returned it.
__device__ __forceinline__ unsigned long long add_call_result(unsigned long long acc, unsigned long long r) {
    return acc == ~0ull || r == ~0ull ? ~0ull : acc + r;
}

#ifdef PB2_LINKED_READER_GROUPS
static_assert(sizeof(((pb2_reader_group_t*)0)->body) == PB2_GROUP_MAX * sizeof(int), "one group block entry per member");

// Thread 0, before the first chunk of run_linked_group_part: the members of g marked PB2_TASK_READER_GROUP into the
// group block rg, in member order, their results zeroed, and their bits in mask.
__device__ __forceinline__ void fill_reader_group(const pb2_task_t* tasks, const GroupSmem& g, pb2_reader_group_t& rg,
                                                  unsigned long long* res, uint32_t& mask) {
    uint32_t m = 0, n = 0;
    for (int i = 0; i < g.n; ++i) {
        const pb2_task_t& mt = tasks[g.mem[i]];
        if (!(__ldg(&mt.flags) & PB2_TASK_READER_GROUP)) continue;
        m |= 1u << i;
        rg.body[n] = __ldg(&mt.body);
        rg.iparam[n][0] = __ldg(&mt.iparam[0]); rg.iparam[n][1] = __ldg(&mt.iparam[1]); rg.iparam[n][2] = __ldg(&mt.iparam[2]);
        rg.fparam[n] = __ldg(&mt.fparam);
        res[n++] = 0;
    }
    rg.n = n;
    mask = m;
}

// Thread 0, after a call of pb2_linked_reader_group that returned r: each member of the call adds its result (all of
// them ~0 when r is), and its result word is zeroed for the next call.
__device__ __forceinline__ void fold_reader_group(GroupSmem& g, uint32_t mask, unsigned long long r, unsigned long long* res) {
    for (int i = 0, j = 0; i < g.n; ++i) {
        if (!((mask >> i) & 1u)) continue;
        g.res[i] = add_call_result(g.res[i], r == ~0ull ? ~0ull : res[j]);
        res[j++] = 0;
    }
}
#endif

// All threads (LINKED instantiations), in place of the body of a task that leads a read group of linked readers, or
// of a producer that runs with one (form_read_groups).  Called one after the other over a whole part, the members would
// each stream it from DRAM: with every worker doing so, far more than L2 holds passes through it between two members'
// passes.  So the part is walked in chunks of reader_chunk_bytes() (16-byte multiples; the last chunk takes the rest),
// and every member is called on one chunk before the next: the producer first when one runs with the group (its stores
// carry the default cache policy, as the members read them back), then each member over the chunk's slice of the tile,
// a barrier between calls.  Each member's results add up over its calls into g.res (include/pb2_device_body.h); the
// members of a group led by its first member saw the version the leader saw (as in group_part_results).  Returns the
// producer's result (thread 0): the sum of its calls when it is itself a reader, else its first chunk's (~0 if any
// call returned ~0); without a producer, the leader's.
// Built with PB2_LINKED_READER_GROUPS (the kernels linked with PB2_LINK_READER_GROUPS), the members marked
// PB2_TASK_READER_GROUP are not called one by one: one call of pb2_linked_reader_group per chunk gives them all their
// results, in one pass over the chunk, before the other members are called as above.  Its block and results live in the
// linked kernels' static shared memory, like *lp.
template <int NT>
static __device__ __noinline__ unsigned long long run_linked_group_part(TaskSmem* sp, GroupSmem* gp, pb2_body_check_t* lp,
                                                                        const pb2_task_t* tasks, uint32_t* seen_version) {
    TaskSmem& s = *sp;
    GroupSmem& g = *gp;
    const bool fused = g.fused != 0;
    const int body = s.task.body;
    int fx = 0;
    if (fused)
        while (fx + 1 < (int)s.task.nb_flows && !(s.task.tile[fx] == g.tile && (s.task.access[fx] & PB2_FLOW_ACCESS_WRITE))) ++fx;
    const uint32_t len = s.args.bytes[fx], cmax = reader_chunk_bytes();
    const uint32_t nc = len > cmax ? len / cmax : 1u;
    uint8_t* const x = static_cast<uint8_t*>(s.args.flow[fx]);
    // the members' body ids go where a CHECK group keeps its constants
    if ((int)threadIdx.x < g.n) { g.k[threadIdx.x] = __ldg(&tasks[g.mem[threadIdx.x]].body); g.res[threadIdx.x] = 0; }
    if (threadIdx.x == 0) { lp->check = 0; lp->k0 = 0; }
#ifdef PB2_LINKED_READER_GROUPS
    __shared__ pb2_reader_group_t rg;
    __shared__ unsigned long long rg_res[PB2_GROUP_MAX];
    __shared__ uint32_t rg_mask;
    if (threadIdx.x == 0) fill_reader_group(tasks, g, rg, rg_res, rg_mask);
#endif
    const bool psum = (s.task.flags & PB2_TASK_READER) != 0;
    unsigned long long rp = 0;
    __syncthreads();
#ifdef PB2_LINKED_READER_GROUPS
    const uint32_t gmask = rg_mask;
#endif
#pragma unroll 1
    for (uint32_t c = 0; c < nc; ++c) {
        const uint32_t off = c * cmax;
        const bool lastc = c + 1 == nc;
        if (fused) {
            if (threadIdx.x < PB2_MAX_FLOWS) {
                const int f = (int)threadIdx.x;
                const uint32_t b = s.args.bytes[f], o = off < b ? off : b;
                lp->args.flow[f] = s.args.flow[f] ? static_cast<uint8_t*>(s.args.flow[f]) + o : nullptr;
                lp->args.bytes[f] = lastc || b - o < cmax ? b - o : cmax;
                if (f == 0) {
                    lp->args.elem0 = s.args.elem0 + (off >> 2); lp->args.part = s.args.part;
                    lp->args.iparam[0] = s.args.iparam[0]; lp->args.iparam[1] = s.args.iparam[1];
                    lp->args.iparam[2] = s.args.iparam[2]; lp->args.fparam = s.args.fparam;
                }
            }
            __syncthreads();
            const unsigned long long r = is_linked_body(body) ? pb2_linked_body(body, &lp->args, s.red)
                                                              : run_hbm_body(body, *reinterpret_cast<const BodyArgs*>(&lp->args), s.red);
            if (threadIdx.x == 0) rp = psum ? add_call_result(rp, r) : c == 0 || r == ~0ull ? r : rp;
            __syncthreads();
        }
        const uint32_t cb = lastc ? len - off : cmax;
#ifdef PB2_LINKED_READER_GROUPS
        if (gmask) {
            if (threadIdx.x == 0) { rg.flow = x + off; rg.bytes = cb; rg.elem0 = s.args.elem0 + (off >> 2); rg.part = s.args.part; }
            __syncthreads();
            const unsigned long long r = pb2_linked_reader_group(&rg, rg_res, s.red);
            __syncthreads();
            if (threadIdx.x == 0) fold_reader_group(g, gmask, r, rg_res);
        }
#endif
#pragma unroll 1
        for (int i = 0; i < g.n; ++i) {
#ifdef PB2_LINKED_READER_GROUPS
            if ((gmask >> i) & 1u) continue;
#endif
            if (threadIdx.x == 0) {
                const pb2_task_t& mt = tasks[g.mem[i]];
                pb2_body_args_t& a = lp->args;
                a.flow[0] = x + off; a.bytes[0] = cb;
                for (int f = 1; f < PB2_MAX_FLOWS; ++f) { a.flow[f] = nullptr; a.bytes[f] = 0; }
                a.elem0 = s.args.elem0 + (off >> 2); a.part = s.args.part;
                a.iparam[0] = __ldg(&mt.iparam[0]); a.iparam[1] = __ldg(&mt.iparam[1]); a.iparam[2] = __ldg(&mt.iparam[2]);
                a.fparam = __ldg(&mt.fparam);
            }
            __syncthreads();
            const unsigned long long r = pb2_linked_body((int)g.k[i], &lp->args, s.red);
            if (threadIdx.x == 0) g.res[i] = add_call_result(g.res[i], r);
            __syncthreads();
        }
    }
    if (threadIdx.x == 0 && !fused && s.args.part == 0) {
        const uint32_t v = *reinterpret_cast<volatile uint32_t*>(&seen_version[(size_t)g.mem[0] * PB2_MAX_FLOWS]);
        for (int i = 1; i < g.n; ++i) seen_version[(size_t)g.mem[i] * PB2_MAX_FLOWS] = v;
    }
    return fused ? rp : g.res[0];
}

}  // namespace pb2
