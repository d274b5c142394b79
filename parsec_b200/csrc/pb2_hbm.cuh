// pb2_hbm.cuh -- the persistent engine kernel of HBM-body windows (pb2_engine_hbm_kernel); what one worker does with a
// task, a read group or a fused producer unit is the shared worker code of pb2_worker.cuh.  Instantiated for the FIFO ready
// ring and for priority lanes (queue_policy 1), untraced and traced (window trace), by pb2_window_kernels.cu, one object
// per variant: each translation unit holds one instantiation, because a second kernel calling the same __noinline__
// helpers makes ptxas give them the standard call ABI, which costs the kernel a stack frame and spills at its
// 80-register budget.
#pragma once
#include "pb2_sched.cuh"
#include "pb2_worker.cuh"

namespace pb2 {

// ---------------------------------------------------------------------------------------------
// the persistent engine kernel, HBM-bound bodies
// ---------------------------------------------------------------------------------------------
// 64-thread workers, up to 12 per SM (<= 80 registers, no spills; 8 by default, kHbmWorkersPerSm): a worker keeps PB2_CHECK_UNROLL = 16 (read-only bodies) or
// PB2_UNROLL = 4 (read-modify-write bodies) 16-byte requests per thread in flight -- bytes in flight per SM are what
// a window that streams tiles through L2 responds to (r02 sweep in DESIGN.md: 20 x 4 requests 0.76 ms, 20 x 6 0.62 ms,
// 12 x 16 0.60 ms), while many small workers still overlap the serial pop / release sections of one task with the
// streaming of the others.  The Ex05 window is no longer L2-bound: its eight readers of a tile run as one read group
// (form_read_groups, pb2_window_plan.cpp), so each tile crosses L2 -> SM twice (FILL, one grouped CHECK) instead of nine times.  And the
// producer runs with its group as one unit (run_fused_part) that checks every value in registers before it stores it:
// the tile goes SM -> L2 -> DRAM once and never comes back to the SM (DESIGN.md §5, §8).
// What one worker does with a task is in pb2_worker.cuh (shared with the streaming kernel of pb2_stream.cu and the
// HBM-body units of the GEMM kernel).
#ifndef PB2_HBM_MINB
#define PB2_HBM_MINB 12
#endif
// Workers per SM of an HBM window unless pb2_engine_params_t::workers_per_sm says otherwise.  The kernel keeps the
// 80-register budget of PB2_HBM_MINB = 12, but a fused unit is a plain streaming write loop, and the resident Ex05 step
// is about 3.5 % shorter at 8 (or 6) workers per SM than at 12, with the fusion-off window unchanged (DESIGN.md §8).
constexpr int kHbmWorkersPerSm = 8;
#ifndef PB2_HBM_THREADS
#define PB2_HBM_THREADS 64
#endif
// PRIO: queue_policy 1 (priority lanes, pop_prio); the FIFO instantiation is the kernel as it was without them.
// TRACE: write a record of every part into tr (PartSmem, then trace_part); the untraced instantiations never touch tr.
// LINKED: body ids PB2_BODY_LINKED_0 .. _7 call the application's pb2_linked_body (include/pb2_device_body.h); built
// only in pb2_engine_linked.cu, as relocatable device code that pb2_engine_link_bodies links with the application's
// image.  The other instantiations compile as if the flag did not exist.
template <bool PRIO, bool TRACE, bool LINKED = false>
__global__ void __launch_bounds__(PB2_HBM_THREADS, PB2_HBM_MINB)
pb2_engine_hbm_kernel(WinDev w, TraceDev tr) {
    __shared__ TaskSmem s;
    __shared__ BulkSmem bulk;
    __shared__ GroupSmem g;
    __shared__ unsigned long long t_start;   // the watchdog's earliest reference (pop_idle)
    PartSmem* rec = nullptr;
    if constexpr (TRACE) { __shared__ PartSmem part_rec; rec = &part_rec; }
    pb2_body_check_t* lk = nullptr;          // LINKED: what a linked body is handed (run_linked_part)
    if constexpr (LINKED) { __shared__ pb2_body_check_t linked_args; lk = &linked_args; }
    if (threadIdx.x == 0) { bulk_init(bulk); t_start = globaltimer_ns(); }
    __syncthreads();

    for (;;) {
        if (threadIdx.x == 0) {
            const int32_t e = pop_entry<PRIO>(w, &t_start);
            if (e != kEmpty) __threadfence();   // acquire side: order the tile reads below after the slot read
            if (TRACE && e != kEmpty) *rec = PartSmem{globaltimer_ns(), 0, 0, 0, 0, 0, 0};
            s.entry = e;
        }
        __syncthreads();
        const int32_t entry = s.entry;
        if (entry == kEmpty) break;
        const int32_t id = w.nparts ? PB2_ENT_TASK(entry) : entry;
        const int part = w.nparts ? PB2_ENT_PART(entry) : 0;
        if (threadIdx.x < 4) reinterpret_cast<uint4*>(&s.task)[threadIdx.x] =
            __ldg(reinterpret_cast<const uint4*>(&w.tasks[id]) + threadIdx.x);
        {
            // load_group_members, written out: called, it costs this kernel spills at its 80-register budget
            const uint32_t gd = w.group ? __ldg(&w.group[id]) : 0u;
            const int gn = (int)(gd & 15u);
            const uint32_t gb = (gd & ~PB2_GROUP_FUSED) >> 4;
            const bool fused = (gd & PB2_GROUP_FUSED) != 0;
            if ((int)threadIdx.x < gn) {
                const int32_t m = __ldg(&w.group_mem[gb + threadIdx.x]);
                const pb2_task_t& mt = w.tasks[m];
                g.mem[threadIdx.x] = m;
                g.k[threadIdx.x] = mt.body == PB2_BODY_CHECK_F32 ? __float_as_uint(__ldg(&mt.fparam)) : (uint32_t)__ldg(&mt.iparam[0]);
                g.succ_begin[threadIdx.x] = __ldg(&mt.succ_begin);
                g.succ_count[threadIdx.x] = __ldg(&mt.succ_count);
                if (threadIdx.x == 0) g.tile = __ldg(&mt.tile[0]);
            }
            if (threadIdx.x == 0) {
                g.n = gn; g.fused = fused;
                if (part == 0 && gn && !fused) {
                    // the members start together: consecutive event numbers, one worker
                    const uint32_t seq = (uint32_t)atomicAdd(&w.ctl->evt.v, (unsigned long long)gn);
                    for (int i = 0; i < gn; ++i) {
                        const int32_t m = __ldg(&w.group_mem[gb + i]);
                        w.start_seq[m] = seq + (uint32_t)i;
                        w.worker[m] = (int32_t)blockIdx.x;
                    }
                } else if (part == 0) {
                    w.start_seq[id] = (uint32_t)atomicAdd(&w.ctl->evt.v, 1ull);
                    w.worker[id] = (int32_t)blockIdx.x;
                    // a fused unit's members start when it retires (below); they run on the producer's worker
                    for (int i = 0; i < gn; ++i) w.worker[__ldg(&w.group_mem[gb + i])] = (int32_t)blockIdx.x;
                }
            }
        }
        __syncthreads();
        const int nparts = task_nparts(w, id);
        const unsigned long long r = run_task_part<true, TRACE>(w, s, &bulk, id, part, nparts, [&] {
            if constexpr (LINKED) {
                if (linked_reader_group(w, g)) return run_linked_group_part<PB2_HBM_THREADS>(&s, &g, lk, w.tasks, w.seen_version);
                if (is_linked_body(s.task.body)) return run_linked_part<PB2_HBM_THREADS>(&s, &g, lk);
            }
            return g.fused ? run_fused_part<PB2_HBM_THREADS>(&s, &g) : run_hbm_body(s.task.body, s.args, s.red);
        }, rec);
        // the leader of a group of linked readers is a reader; run_linked_group_part gave its members their results
        if (g.n && !g.fused && !(LINKED && (s.task.flags & PB2_TASK_READER)))
            group_part_results<PB2_HBM_THREADS, TRACE>(w, s, g, id, part, r, rec);

        if (threadIdx.x < 32) {
            __threadfence();   // release side: the body's stores (all threads, ordered by the barrier) become
                               // visible before any successor can observe its dependency word / ring slot
            if (threadIdx.x == 0) {
                const pb2_task_t& t = s.task;
                const int gn = g.n;
                store_part_results<LINKED>(w, t, id, part, nparts, r, g);
                // the last part to finish retires the task (fence / RMW chain orders every part's stores before it)
                int last = 1;
                if (nparts > 1) { last = atomicSub(&w.parts_left[id], 1) == 1; __threadfence(); }
                s.window_done = 0; s.last = last;
                if (last && gn && g.fused) {
                    // the producer, then its members as if they had run right after it: they saw the version it
                    // wrote; its end, their starts, their ends are consecutive events (end before start on every
                    // edge); they retire right after it, in member order
                    const uint32_t v = epilog_written_flows(w, t, g.tile);
                    const uint32_t ev = (uint32_t)atomicAdd(&w.ctl->evt.v, (unsigned long long)(1 + 2 * gn));
                    const uint32_t seq = (uint32_t)atomicAdd(&w.ctl->retired.v, (unsigned long long)(1 + gn));
                    w.end_seq[id] = ev;
                    w.retire_log[seq] = id;
                    for (int i = 0; i < gn; ++i) {
                        const int32_t m = g.mem[i];
                        w.seen_version[(size_t)m * PB2_MAX_FLOWS] = v;
                        w.start_seq[m] = ev + 1u + (uint32_t)i;
                        w.end_seq[m] = ev + 1u + (uint32_t)(gn + i);
                        w.retire_log[seq + 1u + (uint32_t)i] = m;
                    }
                    *reinterpret_cast<volatile unsigned long long*>(&w.ctl->progress_ns.v) = globaltimer_ns();
                    s.window_done = (int32_t)(seq + 1u + (uint32_t)gn) == w.ntasks ? 1 : 0;
                    __threadfence();
                } else if (last && gn) {
                    // members only read their tile: no written flows; they retire back to back, in member order
                    const uint32_t ev = (uint32_t)atomicAdd(&w.ctl->evt.v, (unsigned long long)gn);
                    const uint32_t seq = (uint32_t)atomicAdd(&w.ctl->retired.v, (unsigned long long)gn);
                    for (int i = 0; i < gn; ++i) { w.end_seq[g.mem[i]] = ev + (uint32_t)i; w.retire_log[seq + (uint32_t)i] = g.mem[i]; }
                    *reinterpret_cast<volatile unsigned long long*>(&w.ctl->progress_ns.v) = globaltimer_ns();
                    s.window_done = (int32_t)(seq + (uint32_t)gn) == w.ntasks ? 1 : 0;
                    __threadfence();
                } else if (last) {
                    epilog_written_flows(w, t);
                    w.end_seq[id] = (uint32_t)atomicAdd(&w.ctl->evt.v, 1ull);
                    // the retire log is written before the out-edges are released, so that it is a linear
                    // extension of the DAG's partial order (a successor can only retire after us)
                    s.window_done = retire_task(w, id) ? 1 : 0;
                    __threadfence();
                }
            }
            __syncwarp();
        }
        if (w.ps_begin != nullptr) {
            // tiles this task wrote for readers on other GPUs go out before those readers are released
            __syncthreads();
            if (s.last && w.ps_begin[id + 1] > w.ps_begin[id]) push_written_tiles(w.tiles, w.ctl, w.ps_begin, w.ps, id, &bulk);
        }
        if (threadIdx.x < 32) {
            if (s.last) {
                // a fused producer's own successors first (its edge to the group is not among them), then the members'
                if (!g.n || g.fused) { release_successors_warp<PRIO>(w, s.task.succ_begin, s.task.succ_count); release_remote_warp(w, id); }
                for (int i = 0; i < g.n; ++i) release_successors_warp<PRIO>(w, g.succ_begin[i], g.succ_count[i]);
            }
            if (threadIdx.x == 0 && s.window_done) {
                __threadfence();
                st_release_gpu(reinterpret_cast<int32_t*>(&w.ctl->done.v), kDoneOK);
            }
        }
        if (TRACE && threadIdx.x == 0) {
            // the part's record, off the retire path (its stamps were taken before it); owner and part from shared
            // memory: nothing of the part has to stay in registers until here
            const int32_t e = s.entry;
            trace_part(tr, w.nparts ? PB2_ENT_TASK(e) : e, w.nparts ? PB2_ENT_PART(e) : 0, *rec, s.last != 0);
        }
        __syncthreads();
    }
}

}  // namespace pb2
