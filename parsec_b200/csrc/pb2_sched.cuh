// pb2_sched.cuh -- device-resident scheduling state and primitives shared by the engine kernels
// (HBM-body kernel in pb2_hbm.cuh, tensor-core kernel in pb2_gemm.cuh).
#pragma once
#include "../../include/pb2_engine.h"
#include "pb2_dev_utils.cuh"
#include "pb2_bodies.cuh"
#include "pb2_window_layout.h"

namespace pb2 {

constexpr int32_t kDoneOK = 1;
constexpr int32_t kDoneTimeout = 2;
constexpr int32_t kDoneBadBody = 3;

struct Ctl {
    Line head;       // pop tickets handed out
    Line tail;       // push tickets handed out
    Line evt;        // global event counter (start/end sequence numbers)
    Line retired;    // tasks retired
    Line done;       // 0 running, kDone*
    Line progress_ns;// globaltimer of the last retirement (watchdog)
    Line bytes_h2d, bytes_d2d, bytes_d2h, stage_ins, body_errors;
};

struct WinDev {
    const pb2_task_t* tasks;
    const uint32_t*   succ;
    pb2_tile_t*       tiles;
    int32_t*          dep;
    int32_t*          ring;
    Ctl*              ctl;
    int32_t*          retire_log;
    uint32_t*         start_seq;
    uint32_t*         end_seq;
    uint32_t*         seen_version;
    unsigned long long* result;
    int32_t*          worker;
    uint32_t          cap_mask;
    int32_t           ntasks;
    int32_t           ntiles;
    int32_t           stage_mode;
    unsigned long long timeout_ns;
    int32_t*          parts_left;     // HBM windows: parts of a task still running (wide tasks)
    // remote out-edges (other GPUs' windows), see pb2_window_set_remote
    const int32_t*    rs_begin;
    const int32_t*    rs_rank;
    const uint32_t*   rs_target;
    const struct PeerWin* peers;
    // producer-side pushes (pb2_window_set_push): task t writes ps[ps_begin[t] .. ps_begin[t+1]) into its readers' slots
    const int32_t*    ps_begin;
    const struct PushDev* ps;
    int32_t           shared;         // scheduling arrays are written by peers: poll / publish at system scope
    // sliced stage-in of tiles larger than part_bytes (HBM windows): which slices are claimed / staged
    uint32_t*         slice_claim;
    uint32_t*         slice_done;
    int32_t           part_bytes;
    const uint16_t*   nparts;         // HBM windows with wide tasks: parts per task (null: every task is one part)
    int32_t           remote_units;   // remote targets are (parts-1) << 27 | unit of a fused-GEMM window, not << 22 | task
    // read groups (form_read_groups in pb2_window_plan.cpp; null: none): task id leads the members
    // group_mem[group[id] >> 4 .. + (group[id] & 15)), itself first; a count of 0 means the task runs alone.  The other
    // members are never released or popped on their own.  A producer fused with a group (PB2_GROUP_FUSED set in its
    // group word) names that group's members, the leader included, and its edge to the leader is gone from succ[].
    const uint32_t*   group;
    const int32_t*    group_mem;
    // queue_policy 1 (null / 0 otherwise): the ready ring is cut into priority lanes, see Lanes (pb2_window_layout.h)
    int32_t           nlanes;         // lanes in use (1 .. PB2_PRIO_LANES)
    struct Lanes*     lanes;
    const uint8_t*    lane;           // lane of each ring-entry owner: a task (HBM windows) or a unit (GEMM windows)
};

struct PeerWin { int32_t* dep; int32_t* ring; Ctl* ctl; uint32_t cap_mask; int32_t pad; pb2_tile_t* tiles; };
struct alignas(32) PushDev { void* dst; int32_t* dst_state; uint32_t bytes; int32_t src_tile; int32_t pad[2]; };

__device__ __forceinline__ int task_nparts(const WinDev& w, int32_t id) { return w.nparts ? (int)w.nparts[id] : 1; }

// The byte slice [off, off + len) of a flow of `bytes` bytes that part `part` of `nparts` runs.  Every flow of a task is
// cut at the offsets of its widest flow (16-byte aligned, the last part takes the remainder), so two-flow bodies pair
// equal offsets.  Both engine kernels cut their wide HBM bodies with it.
__device__ __forceinline__ void part_slice(uint32_t widest, uint32_t nparts, uint32_t part, uint32_t bytes,
                                           uint32_t& off, uint32_t& len) {
    const uint32_t per = ((widest / nparts) + 15u) & ~15u;
    off = per * part < bytes ? per * part : bytes;
    len = (part == nparts - 1) ? bytes - off : (off + per <= bytes ? per : bytes - off);
}

// The stage-in slices [s0, s1) that cover the bytes [off, off + len) of a tile of `bytes` bytes cut into ns slices
// (stage_in_slices cuts the same way).  A part may be cut differently from the tile when its widest flow is another tile.
__device__ __forceinline__ void slices_over(uint32_t bytes, int ns, uint32_t off, uint32_t len, int& s0, int& s1) {
    const uint32_t sper = ((bytes / (uint32_t)ns) + 15u) & ~15u;
    s0 = (int)(off / sper);
    s1 = (int)((off + len + sper - 1) / sper);
    if (s0 > ns - 1) s0 = ns - 1;
    if (s1 > ns) s1 = ns;
    if (len == 0) s1 = s0;
}

// Whole warp: lanes with np > 0 own a ready task `sid` whose entries go to ring[first .. first + np).  Tasks with
// hundreds of parts are written by all 32 lanes together.
template <bool SYS>
__device__ __forceinline__ void push_entries_warp(int32_t* ring, uint32_t cap_mask, int32_t sid, int np, uint32_t first) {
    const int lane = threadIdx.x & 31;
    const unsigned many = __ballot_sync(0xffffffffu, np > 4);
    if (np > 0 && np <= 4)
        for (int p = 0; p < np; ++p) {
            if (SYS) st_release_sys(&ring[(first + (uint32_t)p) & cap_mask], PB2_ENT_MAKE(sid, p));
            else st_release_gpu(&ring[(first + (uint32_t)p) & cap_mask], PB2_ENT_MAKE(sid, p));
        }
    for (unsigned m = many; m; m &= m - 1) {
        const int src = __ffs(m) - 1;
        const int32_t s2 = __shfl_sync(0xffffffffu, sid, src);
        const int n2 = __shfl_sync(0xffffffffu, np, src);
        const uint32_t f2 = __shfl_sync(0xffffffffu, first, src);
        for (int p = lane; p < n2; p += 32) {
            if (SYS) st_release_sys(&ring[(f2 + (uint32_t)p) & cap_mask], PB2_ENT_MAKE(s2, p));
            else st_release_gpu(&ring[(f2 + (uint32_t)p) & cap_mask], PB2_ENT_MAKE(s2, p));
        }
    }
}

// ---------------------------------------------------------------------------------------------
// scheduling primitives shared by the HBM and the GEMM engine kernels
// ---------------------------------------------------------------------------------------------

// One thread, while it finds nothing to pop: true when the window is finished (or aborted, or the watchdog trips),
// otherwise back off.  since (null: none): the globaltimer at which the calling CTA started; the watchdog counts from
// the later of it and the last retirement, because an HBM window's next run is armed during the run before it
// (pb2_window_start), which can be long before the host starts it.
__device__ __forceinline__ bool pop_idle(const WinDev& w, uint32_t& spins, const unsigned long long* since) {
    if (ld_relaxed_gpu(reinterpret_cast<const int32_t*>(&w.ctl->done.v)) != 0) return true;
    if ((++spins & 1023u) == 0) {
        // watchdog: a DAG whose dependency counts are wrong would spin forever
        unsigned long long last = *reinterpret_cast<volatile unsigned long long*>(&w.ctl->progress_ns.v);
        if (since && *since > last) last = *since;
        // signed: %globaltimer read on another SM can be slightly behind the value a retiring SM just stored
        if ((long long)(globaltimer_ns() - last) > (long long)w.timeout_ns) {
            st_relaxed_gpu(reinterpret_cast<int32_t*>(&w.ctl->done.v), kDoneTimeout);
            return true;
        }
    }
    __nanosleep(spins < 64 ? 32 : 256);
    return false;
}

// One thread: take the next pop ticket and wait for its slot.  Returns a task id, or kEmpty when the
// window is finished (or aborted).  Ticket order == push order, i.e. a strict FIFO ready queue.
__device__ __forceinline__ int32_t pop_task(const WinDev& w, const unsigned long long* since) {
    const uint32_t ticket = (uint32_t)atomicAdd(&w.ctl->head.v, 1ull);
    int32_t* slot = &w.ring[ticket & w.cap_mask];
    uint32_t spins = 0;
    int32_t id;
#ifdef PB2_EXPERIMENT_GPU_SCOPE_POLL
    while ((id = ld_acquire_gpu(slot)) == kEmpty) {
#else
    while ((id = (w.shared ? ld_acquire_sys(slot) : ld_acquire_gpu(slot))) == kEmpty) {
#endif
        if (pop_idle(w, spins, since)) return kEmpty;
    }
    return id;
}

// One thread, queue_policy 1: claim the head entry of the first non-empty lane.  The claim is a decrement of the
// lane's avail count that found it positive (a decrement that did not is given back), then a head ticket: the number
// of tickets never exceeds the entries pushers have reserved, so the ticket's slot is below the tail.  The pusher
// reserves before it stores the entry, so the slot may still have to be waited for.  (A CAS on the head while it is
// below the tail claims the same slots, but a thousand workers polling one lane make it a retry round trip per claim:
// 7x the FIFO time of the resident Ex05 window.)  Shared windows never get here: their peers push into one remote
// ring (pb2_window_create refuses the combination).
__device__ __forceinline__ int32_t pop_prio(const WinDev& w, const unsigned long long* since) {
    uint32_t spins = 0;
    for (;;) {
        for (int l = 0; l < w.nlanes; ++l) {
            unsigned long long* avail = &w.lanes->avail[l].v;
            if (*reinterpret_cast<volatile long long*>(avail) <= 0) continue;
            if ((long long)atomicAdd(avail, ~0ull) > 0) {
                const unsigned long long h = atomicAdd(&w.lanes->head[l].v, 1ull);
                int32_t id;
                while ((id = ld_acquire_gpu(&w.ring[h])) == kEmpty) __nanosleep(32);
                return id;
            }
            atomicAdd(avail, 1ull);
        }
        if (pop_idle(w, spins, since)) return kEmpty;
    }
}

template <bool PRIO>
__device__ __forceinline__ int32_t pop_entry(const WinDev& w, const unsigned long long* since = nullptr) {
    return PRIO ? pop_prio(w, since) : pop_task(w, since);
}

// Whole warp, queue_policy 1: lanes with np > 0 push np entries into priority lane `ln`.  One tail reservation per
// lane in use (the lanes of the warp that push into the same one are aggregated); returns this lane's first slot.
// Out of line: inlined, it costs the HBM kernel spills at its 80-register budget.
static __device__ __noinline__ uint32_t reserve_lane_slots(Lanes* lanes, int ln, int np) {
    const int lane = threadIdx.x & 31;
    const unsigned grp = __match_any_sync(0xffffffffu, np > 0 ? ln : -1);
    const unsigned act = __ballot_sync(0xffffffffu, np > 0);
    int pre = 0, tot = 0;
    for (unsigned m = act; m; m &= m - 1) {
        const int j = __ffs(m) - 1;
        const int v = __shfl_sync(0xffffffffu, np, j);
        if ((grp >> j) & 1u) { tot += v; if (j < lane) pre += v; }
    }
    const int leader = __ffs(grp) - 1;
    unsigned long long base = 0;
    if (np > 0 && lane == leader) {
        base = atomicAdd(&lanes->tail[ln].v, (unsigned long long)tot);
        atomicAdd(&lanes->avail[ln].v, (unsigned long long)tot);
    }
    base = __shfl_sync(0xffffffffu, base, leader);
    return (uint32_t)base + (uint32_t)pre;
}

// Whole warp: release the out-edges succ[succ_begin .. + succ_count) of a task (parsec_release_dep_fct semantics), push
// the newly ready successors.  Must be called after a __threadfence() that follows the body's stores.
template <bool PRIO>
__device__ __forceinline__ void release_successors_warp(const WinDev& w, int32_t succ_begin, int32_t succ_count) {
    const int lane = threadIdx.x & 31;
    for (int e0 = 0; e0 < succ_count; e0 += 32) {
        const int e = e0 + lane;
        bool ready = false;
        int32_t sid = -1;
        if (e < succ_count) {
            const uint32_t s = w.succ[succ_begin + e];
            sid = PB2_SUCC_TASK(s);
            const pb2_task_t& st = w.tasks[sid];
            if (st.flags & PB2_TASK_DEPS_MASK) {
                // parsec_update_deps_with_mask, parsec.c:1656-1720: OR the destination flow bit, the
                // task is ready when (word & goal) == goal; each bit is set exactly once (:1688 assert)
                const int32_t bit = 1 << PB2_SUCC_FLOW(s);
                const int32_t old = atomicOr(&w.dep[sid], bit);
                ready = (((old | bit) & st.dep_goal) == st.dep_goal) && ((old & st.dep_goal) != st.dep_goal);
            } else {
                // parsec_update_deps_with_counter, parsec.c:1609-1654: fetch_dec, ready at 0
                ready = (atomicSub(&w.dep[sid], 1) == 1);
            }
        }
        // a ready successor contributes one ring entry per part: exclusive scan of the part counts over the warp
        const int nparts = ready ? task_nparts(w, sid) : 0;
        int incl = nparts;
        for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
        const int total = __shfl_sync(0xffffffffu, incl, 31);
        if (total && PRIO) {
            const uint32_t first = reserve_lane_slots(w.lanes, nparts ? (int)w.lane[sid] : 0, nparts);
            push_entries_warp<false>(w.ring, 0xffffffffu, sid, nparts, first);     // lanes never wrap
        } else if (total) {
            unsigned long long base = 0;
            if (lane == 0) base = atomicAdd(&w.ctl->tail.v, (unsigned long long)total);
            base = __shfl_sync(0xffffffffu, base, 0);
            push_entries_warp<false>(w.ring, w.cap_mask, sid, nparts, (uint32_t)base + (uint32_t)(incl - nparts));
        }
    }
}

// Whole warp: release the out-edges that lead into other GPUs' windows.  The activation message of the reference
// (remote_dep_mpi.c:1860 remote_dep_mpi_recv_activate -> release of the local successors) becomes a system-scope
// atomic on the peer's dependency word and, when it reaches zero, ring entries written into the peer's HBM over
// NVLink.  The tile itself is pulled by the peer's worker from this GPU's slot when the task runs (stage_in_flow).
__device__ __forceinline__ void release_remote_warp(const WinDev& w, int32_t id) {
    if (!w.rs_begin) return;
    const int lane = threadIdx.x & 31;
    const int32_t b = w.rs_begin[id], e1 = w.rs_begin[id + 1];
    if (b == e1) return;
    __threadfence_system();            // our tile bytes are visible to the peers before they can see the release
    for (int32_t e0 = b; e0 < e1; e0 += 32) {
        const int32_t e = e0 + lane;
        int np = 0;
        int32_t sid = 0;
        uint32_t first = 0;
        PeerWin pw = w.peers[w.rs_rank[e < e1 ? e : b]];
        if (e < e1) {
            const uint32_t tgt = w.rs_target[e];
            sid = w.remote_units ? (int32_t)PB2_SUCC_TASK(tgt) : PB2_ENT_TASK(tgt);
            if (atomicSub_system(&pw.dep[sid], 1) == 1) {
                np = (w.remote_units ? (int)PB2_SUCC_FLOW(tgt) : PB2_ENT_PART(tgt)) + 1;
                first = (uint32_t)atomicAdd_system(&pw.ctl->tail.v, (unsigned long long)np);
            }
        }
        // entries of one ready task go to ONE peer: lanes cooperate per ready lane, the ring pointer travels with it
        const unsigned many = __ballot_sync(0xffffffffu, np > 0);
        for (unsigned m = many; m; m &= m - 1) {
            const int src = __ffs(m) - 1;
            const int32_t s2 = __shfl_sync(0xffffffffu, sid, src);
            const int n2 = __shfl_sync(0xffffffffu, np, src);
            const uint32_t f2 = __shfl_sync(0xffffffffu, first, src);
            const unsigned long long rp = __shfl_sync(0xffffffffu, (unsigned long long)(uintptr_t)pw.ring, src);
            const uint32_t cm = __shfl_sync(0xffffffffu, pw.cap_mask, src);
            int32_t* ring = reinterpret_cast<int32_t*>((uintptr_t)rp);
            for (int p = lane; p < n2; p += 32)
                st_release_sys(&ring[(f2 + (uint32_t)p) & cm], w.remote_units ? (int32_t)PB2_SUCC_MAKE(s2, p) : PB2_ENT_MAKE(s2, p));
        }
    }
}

// Whole CTA, after the body of a task whose written tile other GPUs read: write the tile into every reader rank's slot
// (posted stores over NVLink through the bulk mover: local reads, remote writes, no round trip per chunk), then publish
// the slot's state at system scope.  The release of the remote successors follows (release_remote_warp): they find
// the tile VALID.  This is the PUT of remote_dep_mpi.c:2120 issued by the producer instead of a GET by each consumer.
static __device__ __noinline__ void push_written_tiles(const pb2_tile_t* tiles, Ctl* ctl, const int32_t* ps_begin, const PushDev* ps,
                                                       int32_t id, BulkSmem* bulk) {
    const int32_t b = ps_begin[id], e = ps_begin[id + 1];
    for (int32_t i = b; i < e; ++i) {
        const PushDev p = ps[i];
        cta_copy<false>(p.dst, tiles[p.src_tile].dev_ptr, p.bytes, bulk);
        __syncthreads();
        if (threadIdx.x == 0) {
            __threadfence_system();
            st_release_sys(p.dst_state, PB2_TILE_VALID);
            atomicAdd(&ctl->bytes_d2d.v, (unsigned long long)p.bytes);
        }
    }
    __syncthreads();
}

// One thread: append to the retire log and store the watchdog's progress; returns true when this was the last task of
// the window.
__device__ __forceinline__ bool retire_task(const WinDev& w, int32_t id) {
    const uint32_t seq = (uint32_t)atomicAdd(&w.ctl->retired.v, 1ull);
    w.retire_log[seq] = id;
    *reinterpret_cast<volatile unsigned long long*>(&w.ctl->progress_ns.v) = globaltimer_ns();
    return (int32_t)(seq + 1) == w.ntasks;
}

// ---------------------------------------------------------------------------------------------
// device time stamps of a traced window (pb2_engine_set_window_trace)
// ---------------------------------------------------------------------------------------------
// Per ring entry of the run, the part record (pb2_part_trace_t) of the worker that ran it, at part_base[owner] + part;
// the owner is the popped task of an HBM window, the unit of a GEMM window.  The host fills task, part and nparts, and
// derives each entity's interval and SM from its parts' records (pb2_window_trace).  Only the TRACE instantiations of
// the window kernels touch the records (null in an untraced window).
struct TraceDev {
    pb2_part_trace_t* parts;          // nparts records, cleared by the reset kernel
    const int32_t* part_base;         // per ring-entry owner: its first record
    int32_t nparts;
};
static_assert(sizeof(pb2_part_trace_t) == 64, "pb2_part_trace_t is a 64-byte public record");

// A traced worker's record of the part it runs, in shared memory: nothing of it is held in registers across the body.
// Thread 0 writes it.
struct PartSmem { unsigned long long t_pop, t_in, t_exec, t_out, in_bytes, out_bytes; uint32_t flags; };

// Thread 0, after the part's pushout, once it knows whether the part retired its entity: the record of part `part` of
// ring-entry owner `owner`.  A part that pushed nothing out ends at t_exec (deciding that here, not where t_out is
// stamped, keeps the HBM kernels' pushout path free of spills at their 80-register budget).
__device__ __forceinline__ void trace_part(const TraceDev& tr, int32_t owner, int part, const PartSmem& r, bool retired) {
    pb2_part_trace_t* p = &tr.parts[tr.part_base[owner] + part];
    p->t_pop_ns = r.t_pop; p->t_in_ns = r.t_in; p->t_exec_ns = r.t_exec; p->t_out_ns = r.out_bytes ? r.t_out : r.t_exec;
    p->in_bytes = r.in_bytes; p->out_bytes = r.out_bytes;
    p->smid = smid(); p->flags = r.flags | (retired ? PB2_PART_RETIRED : 0u);
}

// ---------------------------------------------------------------------------------------------
// (re)arm the per-run state of a window
// ---------------------------------------------------------------------------------------------
// Thread gid of gsz: its grid-stride share of what a run starts from -- dependency words, ring, Ctl, tile table, part
// counts, stage-in claims, priority lanes and the cleared per-task outputs.  `ready` is the window's image of its first
// nready ring slots.  pb2_window_reset_kernel runs it over its grid.
__device__ __forceinline__ void rearm_run(const WinDev& w, const pb2_tile_t* tiles_init, const int32_t* ready, int32_t nready,
                                          size_t gid, size_t gsz) {
    for (size_t i = gid; i < (size_t)w.ntasks; i += gsz) {
        const pb2_task_t& t = w.tasks[i];
        // counter mode counts down from the goal (parsec.c:1625-1633); mask mode ORs up from 0 (:1693-1703)
        w.dep[i] = (t.flags & PB2_TASK_DEPS_MASK) ? 0 : t.dep_goal;
        if (w.parts_left) w.parts_left[i] = task_nparts(w, (int32_t)i);
        w.start_seq[i] = 0; w.end_seq[i] = 0; w.result[i] = 0; w.worker[i] = -1; w.retire_log[i] = -1;
        for (int f = 0; f < PB2_MAX_FLOWS; ++f) w.seen_version[i * PB2_MAX_FLOWS + f] = 0;
    }
    for (size_t i = gid; i <= (size_t)w.cap_mask; i += gsz)
        w.ring[i] = (i < (size_t)nready) ? ready[i] : kEmpty;
    for (size_t i = gid; i < (size_t)w.ntiles; i += gsz) {
        w.tiles[i] = tiles_init[i];
        if (w.slice_claim) {
            for (int k = 0; k < PB2_SLICE_WORDS; ++k) w.slice_claim[i * PB2_SLICE_WORDS + k] = 0;
            for (int k = 0; k <= PB2_SLICE_WORDS; ++k) w.slice_done[i * (PB2_SLICE_WORDS + 1) + k] = 0;
        }
    }
    // queue_policy 1: every lane starts with its initial entries, which `ready` holds at the start of the lane's
    // segment (empty slots kEmpty)
    if (w.lanes && gid < PB2_PRIO_LANES) {
        w.lanes->head[gid].v = w.lanes->begin[gid];
        w.lanes->tail[gid].v = (unsigned long long)w.lanes->begin[gid] + w.lanes->ninit[gid];
        w.lanes->avail[gid].v = w.lanes->ninit[gid];
    }
    if (gid == 0) {
        w.ctl->head.v = 0; w.ctl->tail.v = (unsigned long long)nready; w.ctl->evt.v = 0;
        w.ctl->retired.v = 0; w.ctl->done.v = (w.ntasks == 0) ? kDoneOK : 0;
        w.ctl->progress_ns.v = globaltimer_ns();
        w.ctl->bytes_h2d.v = 0; w.ctl->bytes_d2d.v = 0; w.ctl->bytes_d2h.v = 0;
        w.ctl->stage_ins.v = 0; w.ctl->body_errors.v = 0;
    }
}

// ---------------------------------------------------------------------------------------------
// stage-in / stage-out of one flow by the whole CTA
// ---------------------------------------------------------------------------------------------
// What the out-of-line stage-in helpers need from the window, passed BY VALUE in registers: a reference to the
// kernel-parameter struct would force a 300-byte local-memory copy of it in every caller.
struct StageCtx {
    pb2_tile_t* tiles; Ctl* ctl; uint32_t* slice_claim; uint32_t* slice_done; int32_t use_bulk; int32_t part_bytes;
};
__device__ __forceinline__ StageCtx stage_ctx(const WinDev& w) {
    return StageCtx{w.tiles, w.ctl, w.slice_claim, w.slice_done, w.stage_mode == 0 ? 1 : 0, w.part_bytes};
}

// The stage-in helpers below are out of line.  COUNT (the traced window kernels): thread 0 also adds the bytes the
// calling CTA moved to *moved (its PartSmem::in_bytes); without it `moved` is not used.

// Thread 0 decides (s_decide[0]): 1 = this CTA moves the tile, 0 = already valid (possibly after waiting)
template <bool COUNT>
static __device__ __noinline__ void stage_in_flow(const StageCtx w, pb2_tile_t* tile, uint8_t access, int* s_decide, BulkSmem* bulk,
                                                  unsigned long long* moved) {
    if (threadIdx.x == 0) {
        int decide = 0;
        if ((access & PB2_FLOW_ACCESS_READ) && tile->src_kind == PB2_SRC_PUSH) {
            // the producer writes this slot and publishes its state before it releases us: nothing to move
            while (ld_acquire_sys(&tile->state) != PB2_TILE_VALID) __nanosleep(64);
        } else if (access & PB2_FLOW_ACCESS_READ) {
            // parsec_device_data_stage_in, device_gpu.c:1799-2165: only a READ access needs the bytes;
            // "finally we'll just overwrite w/o read" (data.c:427) for WRITE-only flows.
            int32_t st = atomicCAS(&tile->state, PB2_TILE_INVALID, PB2_TILE_STAGING);
            if (st == PB2_TILE_INVALID) {
                decide = 1;
            } else {
                // another worker is moving it: "data copy is already under transfer" (:1873-1884)
                while (st != PB2_TILE_VALID) { __nanosleep(64); st = ld_acquire_gpu(&tile->state); }
            }
        }
        *s_decide = decide;
    }
    __syncthreads();
    if (*s_decide) {
        cta_copy<true>(tile->dev_ptr, tile->src_ptr, tile->bytes, w.use_bulk ? bulk : nullptr);
        __syncthreads();
        if (threadIdx.x == 0) {
            __threadfence();
            st_release_gpu(&tile->state, PB2_TILE_VALID);   // COMPLETE_TRANSFER (:2358-2573)
            atomicAdd(tile->src_kind == PB2_SRC_PEER ? &w.ctl->bytes_d2d.v : &w.ctl->bytes_h2d.v,
                      (unsigned long long)tile->bytes);
            atomicAdd(&w.ctl->stage_ins.v, 1ull);
            if (COUNT) *moved += tile->bytes;
        }
    }
    __syncthreads();
}

// Number of stage-in slices of a tile: the same rule pb2_window_create uses for the parts of a wide task.
__device__ __forceinline__ int tile_slices_of(int32_t part_bytes, const uint32_t* slice_claim, uint32_t bytes) {
    if (part_bytes <= 0 || !slice_claim) return 1;
    const uint32_t n = (bytes + (uint32_t)part_bytes - 1) / (uint32_t)part_bytes;
    return n > PB2_MAX_PARTS ? PB2_MAX_PARTS : (n < 1 ? 1 : (int)n);
}
__device__ __forceinline__ int tile_slices(const WinDev& w, uint32_t bytes) { return tile_slices_of(w.part_bytes, w.slice_claim, bytes); }

// How many of the ns slices of a tile of `bytes` bytes hold bytes.  Slices are ceil16(bytes / ns) long, so when
// (ns - 1) slices already reach `bytes` the trailing ones are empty (512 x 4097 bytes in 512 slices of 4112: slice 511).  No
// part's bytes lie in an empty slice (slices_over), so nobody would claim it: the tile is complete once the slices
// that hold bytes are in.
__device__ __forceinline__ int live_slices(uint32_t bytes, int ns) {
    const uint32_t sper = ((bytes / (uint32_t)ns) + 15u) & ~15u;
    if (sper == 0) return ns;
    const uint32_t n = bytes / sper + (bytes % sper != 0u);
    return n < (uint32_t)ns ? (int)n : ns;
}

// Stage in the slices [s0, s1) of a tile larger than part_bytes, the empty ones (live_slices) left out.  Every slice is
// moved by exactly one CTA (claim bit), so the parts of a wide task -- and the parts of other readers of the same
// version -- pull the tile in parallel instead of one CTA moving 4 MiB alone; a CTA that finds a slice claimed by
// someone else only waits for it.  The worker whose slice completes the tile publishes PB2_TILE_VALID.
template <bool COUNT>
static __device__ __noinline__ void stage_in_slices(const StageCtx w, int32_t tile_id, int nslices, int s0, int s1, int* s_decide,
                                                    BulkSmem* bulk, unsigned long long* moved) {
    pb2_tile_t* tile = &w.tiles[tile_id];
    if (tile->src_kind == PB2_SRC_PUSH) {       // written by its producer (see stage_in_flow)
        if (threadIdx.x == 0) while (ld_acquire_sys(&tile->state) != PB2_TILE_VALID) __nanosleep(64);
        __syncthreads();
        return;
    }
    const uint32_t bytes = tile->bytes;
    const uint32_t sper = ((bytes / (uint32_t)nslices) + 15u) & ~15u;
    const int live = live_slices(bytes, nslices);
    if (s1 > live) s1 = live;
    uint32_t* claim = w.slice_claim + (size_t)tile_id * PB2_SLICE_WORDS;
    uint32_t* done = w.slice_done + (size_t)tile_id * (PB2_SLICE_WORDS + 1);     // last word: number of staged slices
    for (int sl = s0; sl < s1; ++sl) {
        const uint32_t bit = 1u << (sl & 31);
        if (threadIdx.x == 0) *s_decide = (atomicOr(&claim[sl >> 5], bit) & bit) ? 0 : 1;
        __syncthreads();
        if (*s_decide) {
            const uint32_t off = sper * (uint32_t)sl < bytes ? sper * (uint32_t)sl : bytes;
            const uint32_t len = (sl == nslices - 1) ? bytes - off : (off + sper <= bytes ? sper : bytes - off);
            cta_copy<true>(reinterpret_cast<uint8_t*>(tile->dev_ptr) + off, reinterpret_cast<const uint8_t*>(tile->src_ptr) + off, len, w.use_bulk ? bulk : nullptr);
            __syncthreads();
            if (threadIdx.x == 0) {
                __threadfence();
                atomicOr(&done[sl >> 5], bit);
                atomicAdd(tile->src_kind == PB2_SRC_PEER ? &w.ctl->bytes_d2d.v : &w.ctl->bytes_h2d.v, (unsigned long long)len);
                if (COUNT) *moved += len;
                if ((int)atomicAdd(&done[PB2_SLICE_WORDS], 1u) + 1 == live) {
                    __threadfence();
                    st_release_gpu(&tile->state, PB2_TILE_VALID);
                    atomicAdd(&w.ctl->stage_ins.v, 1ull);
                }
            }
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        for (int sl = s0; sl < s1; ++sl) {
            const uint32_t bit = 1u << (sl & 31);
            while (!(ld_acquire_gpu(reinterpret_cast<const int32_t*>(&done[sl >> 5])) & bit)) __nanosleep(64);
        }
        __threadfence();
    }
    __syncthreads();
}

}  // namespace pb2
