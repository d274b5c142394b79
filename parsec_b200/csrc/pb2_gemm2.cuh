// pb2_gemm2.cuh -- tensor-core engine kernel v2 for PB2_BODY_GEMM_BF16 windows: fused k-chains.
//
// What changes against v1 (pb2_gemm.cuh):
//   * the host groups GEMM tasks into UNITS: a maximal chain of tasks that accumulate into the same C tile and whose
//     only missing dependency is the previous link (the C(i,j) k-chain of dtd_test_simple_gemm.c:675-696, the k-chains
//     of a tile Cholesky).  A unit is executed by `nparts` independent parts of 128 rows x 256 columns of C; the
//     worker that runs a part keeps its 128 x 256 fp32 accumulator in the registers of its two consumer warpgroups
//     across ALL the members of the chain and touches C once: C_out = bf16(C_in + sum_k A_k B_k^T).  This is the
//     reference's "keep the released successor for the same execution stream" (es->next_task,
//     scheduling.c:517-530) taken to its conclusion: 32 dependent tasks become one accumulation.  Members still
//     retire one by one, in chain order, with their own sequence numbers, versions and out-edges (the dependency
//     trace is unchanged); only the intermediate bf16 roundings of C disappear.
//   * scheduling entities on the device are units (counter-mode dependency words), ring entries are (part, unit).
// The worker is the v1 CTA (one per SM, three warpgroups, the same TMA ring and wgmma consumers).
#pragma once
#include <cuda.h>
#include "pb2_sched.cuh"
#include "pb2_gemm.cuh"

namespace pb2 {

struct GUnit {                  // 48 bytes, read-only
    int32_t seg_begin, seg_count;   // members, in chain order
    int32_t succ_begin, succ_count; // out-edges of all members (chain links removed): target unit ids
    int32_t dep_goal;               // in-edges from other units
    int32_t nparts;
    int32_t tileC;                  // GEMM units: the C tile; -1 otherwise
    int32_t M, N, K;
    int32_t flags;                  // bit0 is_gemm, bit1 pushout C
    int32_t pad;
};
struct GSeg { int32_t task, tileA, tileB, pad; };

struct Win2Dev {
    WinDev w;                       // task-level arrays (descriptors, tiles, outputs, ctl, ring)
    const GUnit* units;
    const GSeg*  segs;
    const int32_t* usucc;
    int32_t* udep;
    int32_t* parts_left;
    const CUtensorMap* tmaps;
    int32_t nunits;
    int32_t debug;                  // development only (PB2_GEMM_DEBUG): 1 = no TMA loads, 2 = no MMAs, 4 = no epilogue
};

namespace gemm2 {
using namespace gemm;

constexpr int kPartRows = BM;      // a part is one 128 x 256 accumulator sub-tile of C
constexpr int kPartCols = BN;
constexpr int kMaxParts = 32;      // the part index travels in the 5-bit flow field of a ring entry

struct Job {
    int32_t unit, part, stop, is_gemm;
    int32_t seg_begin, seg_count, tileC, m0;
    int32_t M, N, K, pushout;
    int32_t n0, Nj, pad0, pad1;     // this part's columns [n0, n0 + Nj) of the N-wide tile
};

struct Shared2 {
    alignas(16) Job job;
    alignas(16) pb2_task_t task;    // non-GEMM units: the single member's descriptor
    uint64_t full[kStages];
    uint64_t empty[kStages];
    int32_t  need, decide;
    uint32_t red[32];
};

// one thread: pop a (part, unit) entry; same ticket ring as the task-level kernels
__device__ __forceinline__ int32_t pop_entry(const WinDev& w) { return pop_task(w); }

// whole warp: the unit is complete (all parts): retire its members in chain order, release its out-edges
__device__ __forceinline__ void retire_unit_warp(const Win2Dev& g, const GUnit& u, int unit_id) {
    const WinDev& w = g.w;
    const int lane = threadIdx.x & 31;
    const int L = u.seg_count;
    unsigned long long ebase = 0, rbase = 0;
    if (lane == 0) {
        ebase = atomicAdd(&w.ctl->evt.v, (unsigned long long)(2 * L));
        rbase = atomicAdd(&w.ctl->retired.v, (unsigned long long)L);
        *reinterpret_cast<volatile unsigned long long*>(&w.ctl->progress_ns.v) = globaltimer_ns();
    }
    ebase = __shfl_sync(0xffffffffu, ebase, 0);
    rbase = __shfl_sync(0xffffffffu, rbase, 0);
    const uint32_t cver = (u.flags & 1) ? *reinterpret_cast<volatile uint32_t*>(&w.tiles[u.tileC].version) : 0u;
    for (int i = lane; i < L; i += 32) {
        const GSeg s = g.segs[u.seg_begin + i];
        const pb2_task_t& t = w.tasks[s.task];
        w.start_seq[s.task] = (uint32_t)(ebase + 2 * i);
        w.end_seq[s.task] = (uint32_t)(ebase + 2 * i + 1);
        w.retire_log[rbase + i] = s.task;
        w.worker[s.task] = (int32_t)blockIdx.x;
        if (u.flags & 1) {
            w.seen_version[s.task * PB2_MAX_FLOWS + 0] = *reinterpret_cast<volatile uint32_t*>(&w.tiles[s.tileA].version);
            w.seen_version[s.task * PB2_MAX_FLOWS + 1] = *reinterpret_cast<volatile uint32_t*>(&w.tiles[s.tileB].version);
            w.seen_version[s.task * PB2_MAX_FLOWS + 2] = cver + (uint32_t)i;
            w.result[s.task] = 0;
        } else {
            for (int f = 0; f < t.nb_flows; ++f)
                if (t.tile[f] >= 0) {
                    pb2_tile_t* tile = &w.tiles[t.tile[f]];
                    const uint32_t v = *reinterpret_cast<volatile uint32_t*>(&tile->version);
                    w.seen_version[s.task * PB2_MAX_FLOWS + f] = v;
                    if (t.access[f] & PB2_FLOW_ACCESS_WRITE) {
                        *reinterpret_cast<volatile uint32_t*>(&tile->version) = v + 1;
                        st_relaxed_gpu(&tile->state, PB2_TILE_VALID);
                    }
                }
        }
    }
    if (lane == 0 && (u.flags & 1)) {
        *reinterpret_cast<volatile uint32_t*>(&w.tiles[u.tileC].version) = cver + (uint32_t)L;
        st_relaxed_gpu(&w.tiles[u.tileC].state, PB2_TILE_VALID);
    }
    __threadfence();
    __syncwarp();
    // release: parsec_update_deps_with_counter on the successor units; a ready unit contributes nparts ring entries
    for (int e0 = 0; e0 < u.succ_count; e0 += 32) {
        const int e = e0 + lane;
        int nparts = 0, sid = -1;
        if (e < u.succ_count) {
            sid = g.usucc[u.succ_begin + e];
            if (atomicSub(&g.udep[sid], 1) == 1) nparts = g.units[sid].nparts;
        }
        // exclusive scan of nparts over the warp
        int incl = nparts;
        for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
        const int total = __shfl_sync(0xffffffffu, incl, 31);
        if (total) {
            unsigned long long base = 0;
            if (lane == 0) base = atomicAdd(&w.ctl->tail.v, (unsigned long long)total);
            base = __shfl_sync(0xffffffffu, base, 0);
            for (int p = 0; p < nparts; ++p)
                st_release_gpu(&w.ring[((uint32_t)base + (uint32_t)(incl - nparts + p)) & w.cap_mask], (int32_t)PB2_SUCC_MAKE(sid, p));
        }
    }
    // out-edges into other GPUs' windows, member by member (a member with remote successors is always the last of
    // its unit: build_gemm2_units does not fuse across it)
    if (w.rs_begin) for (int i = 0; i < L; ++i) release_remote_warp(w, g.segs[u.seg_begin + i].task);
    if (lane == 0 && (int32_t)(rbase + L) == w.ntasks) {
        __threadfence();
        st_release_gpu(reinterpret_cast<int32_t*>(&w.ctl->done.v), kDoneOK);
    }
    (void)unit_id;
}

}  // namespace gemm2

__global__ void __launch_bounds__(gemm::kThreads, 1)
pb2_engine_gemm2_kernel(Win2Dev g) {
    using namespace gemm2;
    const WinDev& w = g.w;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    __shared__ Shared2 sh;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg = threadIdx.x >> 7;

    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) { mbar_init(&sh.full[s], 1); mbar_init(&sh.empty[s], kConsumers); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    uint32_t p_stage = 0, p_phase = 0, c_stage = 0, c_phase = 0;

    for (;;) {
        // ---------------- pop the next (part, unit), stage its tiles in
        if (threadIdx.x == 0) {
            Job j; memset(&j, 0, sizeof j);
            const int32_t e = pop_entry(w);
            if (e == kEmpty) { j.stop = 1; }
            else {
                __threadfence();
                j.unit = PB2_SUCC_TASK((uint32_t)e); j.part = PB2_SUCC_FLOW((uint32_t)e);
                const GUnit u = g.units[j.unit];
                j.is_gemm = u.flags & 1; j.pushout = (u.flags >> 1) & 1;
                j.seg_begin = u.seg_begin; j.seg_count = u.seg_count; j.tileC = u.tileC;
                const int mparts = (u.M + kPartRows - 1) / kPartRows;
                j.m0 = (j.part % mparts) * kPartRows; j.M = u.M; j.N = u.N; j.K = u.K;
                j.n0 = (j.part / mparts) * kPartCols; j.Nj = min(kPartCols, u.N - j.n0);
            }
            sh.job = j;
        }
        __syncthreads();
        if (sh.job.stop) break;
        {
            // stage in every INVALID tile the job reads (same protocol as the other kernels)
            const int nseg = sh.job.is_gemm ? sh.job.seg_count : 0;
            for (int i = -1; i < 2 * nseg; ++i) {
                int tile_id; uint8_t acc;
                if (i < 0) { if (!sh.job.is_gemm) break; tile_id = sh.job.tileC; acc = PB2_FLOW_ACCESS_RW; }
                else { const GSeg s = g.segs[sh.job.seg_begin + (i >> 1)]; tile_id = (i & 1) ? s.tileB : s.tileA; acc = PB2_FLOW_ACCESS_READ; }
                pb2_tile_t* tile = &w.tiles[tile_id];
                if (threadIdx.x == 0) sh.need = ld_acquire_gpu(&tile->state) != PB2_TILE_VALID;
                __syncthreads();
                if (sh.need) {
                    const int ns = tile_slices(w, tile->bytes);
                    if (ns == 1) stage_in_flow(stage_ctx(w), tile, acc, &sh.decide);
                    else stage_in_slices(stage_ctx(w), tile_id, ns, 0, ns, &sh.decide);     // take what nobody has claimed, wait for the rest
                    fence_proxy_async();
                }
                __syncthreads();
            }
            if (!sh.job.is_gemm) {
                const GSeg s = g.segs[sh.job.seg_begin];
                if (threadIdx.x < 4) reinterpret_cast<uint4*>(&sh.task)[threadIdx.x] =
                    __ldg(reinterpret_cast<const uint4*>(&w.tasks[s.task]) + threadIdx.x);
                __syncthreads();
                const pb2_task_t& t = sh.task;
                for (int f = 0; f < t.nb_flows; ++f) {
                    if (t.tile[f] < 0 || !(t.access[f] & PB2_FLOW_ACCESS_READ)) continue;
                    pb2_tile_t* tile = &w.tiles[t.tile[f]];
                    if (threadIdx.x == 0) sh.need = ld_acquire_gpu(&tile->state) != PB2_TILE_VALID;
                    __syncthreads();
                    if (sh.need) { stage_in_flow(stage_ctx(w), tile, t.access[f], &sh.decide); fence_proxy_async(); }
                    __syncthreads();
                }
            }
        }
        const Job job = sh.job;

        if (job.is_gemm) {
            const int kblocks = (job.K + BK - 1) / BK;
            if (warp == 1) {
                // ===== TMA producer: 128 rows of A, 256 rows of B per k-block, every member of the chain
                if (lane == 0) {
                    fence_proxy_async();
                    for (int s = 0; s < job.seg_count; ++s) {
                        const GSeg sg = g.segs[job.seg_begin + s];
                        const CUtensorMap* mapA = &g.tmaps[sg.tileA];
                        const CUtensorMap* mapB = &g.tmaps[sg.tileB];
                        if (s + 1 < job.seg_count) {        // the next member's descriptors: fetch them now, not on first use
                            const GSeg nx = g.segs[job.seg_begin + s + 1];
                            asm volatile("prefetch.tensormap [%0];" :: "l"(&g.tmaps[nx.tileA]) : "memory");
                            asm volatile("prefetch.tensormap [%0];" :: "l"(&g.tmaps[nx.tileB]) : "memory");
                        }
                        for (int kb = 0; kb < kblocks; ++kb) {
                            mbar_wait(&sh.empty[p_stage], p_phase ^ 1);
                            uint8_t* sa = smem + p_stage * kStageBytes;
                            if (g.debug & 1) {
                                mbar_arrive(&sh.full[p_stage]);
                            } else {
                                mbar_expect_tx(&sh.full[p_stage], kStageBytes);
                                tma_load_2d(sa, mapA, &sh.full[p_stage], kb * BK, job.m0);
                                tma_load_2d(sa + kAStageBytes, mapB, &sh.full[p_stage], kb * BK, job.n0);
                                tma_load_2d(sa + kAStageBytes + kBStageBytes / 2, mapB, &sh.full[p_stage], kb * BK, job.n0 + 128);
                            }
                            if (++p_stage == kStages) { p_stage = 0; p_phase ^= 1; }
                        }
                    }
                }
            } else if (wg >= 1) {
                // ===== consumers: rows m0 + 64 * cw .. of the part, the whole chain into one accumulator
                const int cw = wg - 1;
                uint8_t* Cbase = reinterpret_cast<uint8_t*>(w.tiles[job.tileC].dev_ptr);
                {   // pull the part's C rows into L2 now, so that the read-modify-write after the chain does not pay DRAM latency
                    const int t = threadIdx.x - 128, row = job.m0 + (t >> 1);
                    if (row < job.M)
                        for (int b = (t & 1) * 128; b < job.Nj * 2; b += 256)
                            asm volatile("prefetch.global.L2 [%0];" :: "l"(Cbase + ((size_t)row * job.N + job.n0) * 2 + b));
                }
                float acc[128];
#pragma unroll
                for (int i = 0; i < 128; ++i) acc[i] = 0.f;
                const int n = job.seg_count * kblocks;
                if (g.debug & 2) {
                    for (int i = 0; i < n; ++i) {
                        mbar_wait(&sh.full[c_stage], c_phase);
                        if ((threadIdx.x & 127) == 0) mbar_arrive(&sh.empty[c_stage]);
                        if (++c_stage == kStages) { c_stage = 0; c_phase ^= 1; }
                    }
                } else {
                    mma_kblocks(acc, smem, sh.full, sh.empty, c_stage, c_phase, n, true, cw);
                }
                if (!(g.debug & 4)) epilogue_add(acc, Cbase, job.N, job.m0 + cw * 64, job.n0, job.M, job.n0 + job.Nj);
                fence_proxy_async();
            }
        } else {
            // ---------------- a non-GEMM member of the DAG (e.g. a panel stand-in): the whole CTA runs it in place
            const pb2_task_t& t = sh.task;
            BodyArgs a;
            for (int f = 0; f < PB2_MAX_FLOWS; ++f) {
                const bool has = f < t.nb_flows && t.tile[f] >= 0;
                a.flow[f] = has ? w.tiles[t.tile[f]].dev_ptr : nullptr;
                a.bytes[f] = has ? w.tiles[t.tile[f]].bytes : 0;
            }
            a.elem0 = 0; a.part = 0;
            a.iparam[0] = t.iparam[0]; a.iparam[1] = t.iparam[1]; a.iparam[2] = t.iparam[2]; a.fparam = t.fparam;
            const unsigned long long r = run_hbm_body(t.body, a, sh.red);
            if (threadIdx.x == 0) {
                w.result[g.segs[job.seg_begin].task] = r;
                if ((t.body == PB2_BODY_CHECK_I32 || t.body == PB2_BODY_CHECK_F32) && (r >> 32)) atomicAdd(&w.ctl->body_errors.v, r >> 32);
            }
            fence_proxy_async();
            for (int f = 0; f < t.nb_flows; ++f)
                if (t.tile[f] >= 0 && (t.access[f] & PB2_FLOW_PUSHOUT) && (t.access[f] & PB2_FLOW_ACCESS_WRITE)) {
                    pb2_tile_t* tile = &w.tiles[t.tile[f]];
                    cta_copy<false>(tile->src_ptr, tile->dev_ptr, tile->bytes);
                    if (threadIdx.x == 0) atomicAdd(&w.ctl->bytes_d2h.v, (unsigned long long)tile->bytes);
                }
        }
        __threadfence();
        __syncthreads();             // every store of the part is done and visible

        // ---------------- part complete: pushout of this part's C rows, then unit retirement by the last part
        if (job.is_gemm && job.pushout) {
            pb2_tile_t* tile = &w.tiles[job.tileC];
            const size_t row_bytes = (size_t)job.N * 2;
            const int rows = min(kPartRows, job.M - job.m0);
            if (rows > 0 && job.Nj == job.N) {
                cta_copy<false>(reinterpret_cast<uint8_t*>(tile->src_ptr) + (size_t)job.m0 * row_bytes,
                                reinterpret_cast<const uint8_t*>(tile->dev_ptr) + (size_t)job.m0 * row_bytes, (size_t)rows * row_bytes);
                if (threadIdx.x == 0) atomicAdd(&w.ctl->bytes_d2h.v, (unsigned long long)rows * row_bytes);
            } else if (rows > 0) {
                // a column block of a tile wider than one part: row segments
                for (int r = 0; r < rows; ++r) {
                    const size_t o = (size_t)(job.m0 + r) * row_bytes + (size_t)job.n0 * 2;
                    cta_copy<false>(reinterpret_cast<uint8_t*>(tile->src_ptr) + o, reinterpret_cast<const uint8_t*>(tile->dev_ptr) + o, (size_t)job.Nj * 2);
                }
                if (threadIdx.x == 0) atomicAdd(&w.ctl->bytes_d2h.v, (unsigned long long)rows * (unsigned long long)job.Nj * 2ull);
            }
            __syncthreads();
        }
        if (warp == 0) {
            int last = 0;
            if (lane == 0) { __threadfence(); last = atomicSub(&g.parts_left[job.unit], 1) == 1; }
            last = __shfl_sync(0xffffffffu, last, 0);
            if (last) { __threadfence(); retire_unit_warp(g, g.units[job.unit], job.unit); }
        }
        __syncthreads();             // sh.job is rewritten by the next pop
    }
}

static inline int pb2_gemm2_launch(const Win2Dev& g, int nworkers, cudaStream_t stream) {
    static bool attr_set = false;
    if (!attr_set) {
        if (cudaFuncSetAttribute(pb2_engine_gemm2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, gemm::kSmemBytes) != cudaSuccess) return PB2_ERR_DEVICE;
        attr_set = true;
    }
    if (nworkers < 1) return PB2_ERR_BAD_PARAM;
    pb2_engine_gemm2_kernel<<<nworkers, gemm::kThreads, gemm::kSmemBytes, stream>>>(g);
    return cudaGetLastError() == cudaSuccess ? PB2_SUCCESS : PB2_ERR_DEVICE;
}

}  // namespace pb2
