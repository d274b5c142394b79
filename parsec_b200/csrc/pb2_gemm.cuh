// pb2_gemm.cuh -- the tensor-core (wgmma / TMA / mbarrier) engine kernel of PB2_BODY_GEMM_BF16 windows.
//
// The task body restates what the reference reaches through `dyld=cublasDgemm` / cublasDgemm_v2
// (tests/dsl/dtd/dtd_test_simple_gemm.c:450,527; tests/runtime/cuda/nvlink.jdf:136-152): one tile
// GEMM per task, C(M x N) += A(M x K) * B(K x N).  Here in bf16 with fp32 accumulation in registers
// (BASELINE config 3); tiles are K-contiguous for both operands: A row-major [M][K], B stored
// [N][K] (== column-major K x N, what a "TN" cuBLAS call consumes), C row-major [M][N].
//
// The host groups GEMM tasks into UNITS (build_gemm2_units, pb2_window_plan.cpp): a maximal chain of tasks that accumulate into the same C
// tile and whose only missing dependency is the previous link (the C(i,j) k-chain of dtd_test_simple_gemm.c:675-696,
// the k-chains of a tile Cholesky); with gemm_mode 1 or 2 every task is a unit of its own.  A unit's C is cut into
// sub-tiles of 128 rows x 256 columns, run by nparts = min(sub-tiles, kMaxParts) independent parts: part p runs
// sub-tiles p, p + nparts, p + 2 nparts, ...  For each sub-tile the worker keeps the 128 x 256 fp32 accumulator in the
// registers of its two consumer warpgroups across ALL the members of the chain and touches C once:
// C_out = bf16(C_in + sum_k A_k B_k^T).  This is the reference's "keep the released successor for the same execution
// stream" (es->next_task, scheduling.c:517-530) taken to its conclusion: 32 dependent tasks become one accumulation.
// Members still retire one by one, in chain order, with their own sequence numbers, versions and out-edges (the
// dependency trace is unchanged); only the intermediate bf16 roundings of C disappear.  Scheduling entities on the
// device are units (counter-mode dependency words), ring entries are (part, unit).
// The other tasks of the DAG (HBM bodies: FILL, SCALE, COPY, AXPY, CHECK, ... between the chains) are units of one
// task, or of one read group with the producer that runs with it (as in HBM windows); one wider than part_bytes is cut into byte-slice parts like a wide task of an HBM window.  A whole CTA runs each
// part with the HBM workers' run_task_part (pb2_worker.cuh), and the last part to finish retires the unit.
//
// One CTA per SM is one worker.  Three warpgroups (384 threads):
//   warpgroup 0 : warp 0 retires a unit and releases its out-edges; one lane of warp 1 is the TMA producer
//   warpgroups 1, 2 : consumers; each issues `wgmma.mma_async` m64n256k16 for its 64 rows of the sub-tile and keeps
//                 the 64 x 256 fp32 accumulator in registers, then adds it into C (bf16) itself
// Operands stream through a 4-stage smem ring of {A 128x64, B 256x64} bf16 128B-swizzled boxes filled by TMA
// (`cp.async.bulk.tensor.2d`) from per-tile tensor maps; the producer fills the next sub-tile's stages while the
// consumers run the epilogue of the current one.
#pragma once
#include <cuda.h>
#include "pb2_sched.cuh"
#include "pb2_worker.cuh"

namespace pb2 {

namespace gemm {

constexpr int BK = 64, UK = 16;     // BM, BN: pb2_window_layout.h
constexpr int kStages = 4;
constexpr int kAStageBytes = BM * BK * 2;          // 16 KiB
constexpr int kBStageBytes = BN * BK * 2;          // 32 KiB
constexpr int kStageBytes = kAStageBytes + kBStageBytes;
constexpr int kThreads = 384;
constexpr int kConsumers = 2;                      // warpgroups 1 and 2, 64 rows of A each
constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align*/;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) { }
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        :: "r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async;" ::: "memory"); }
// Acquire a tensor map the host wrote into global memory (system scope: the writer is the host), so that the TMA unit
// does not use a descriptor it cached when an earlier, since destroyed window had its maps at that address.
__device__ __forceinline__ void tmap_acquire(const CUtensorMap* m) {
    asm volatile("fence.proxy.tensormap::generic.acquire.sys [%0], 128;" :: "l"(m) : "memory");
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N) : "memory"); }

// D(64 x 256, fp32 registers) (+)= A[smem, 64 x 16] * B[smem, 256 x 16]^T, both K-major bf16.  Register d[4c + i] of
// thread (warp w, lane l) of the warpgroup holds row 16w + l/4 + 8*(i/2), column 8c + 2*(l%4) + i%2.
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %130, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
        "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
        "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
        "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,"
        "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,"
        "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,"
        "%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, "
        "%128, %129, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}

// K-major, 128B-swizzled wgmma operand descriptor: start>>4 [0,14) | LBO=1 [16,30) (unused with this swizzle) |
// SBO = 1024>>4 [32,46) (eight 128-byte rows) | layout SWIZZLE_128B = 1 [62,64).  Stepping K by 16 elements inside
// the 128-byte swizzle atom adds 32 bytes to the start address.
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3ffffu) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}

// Consumer warpgroup `cw` (0 or 1): run `n` k-blocks of the smem ring into acc (zeroed by the first one when `zero`).
// A k-block's stage goes back to the producer once the wgmma group of the NEXT k-block has been issued and the
// group reading it has retired, so one group is always in flight.
__device__ __forceinline__ void mma_kblocks(float (&acc)[128], uint8_t* smem, uint64_t* full, uint64_t* empty,
                                            uint32_t& stage, uint32_t& phase, int n, bool zero, int cw) {
    int prev = -1;
    for (int i = 0; i < n; ++i) {
        mbar_wait(&full[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * kStageBytes);
        const uint64_t da = make_desc(sa + cw * 64 * 128), db = make_desc(sa + kAStageBytes);
        wg_fence();
#pragma unroll
        for (int k = 0; k < BK / UK; ++k)
            wgmma_m64n256k16(acc, da + (uint64_t)(k * UK * 2 >> 4), db + (uint64_t)(k * UK * 2 >> 4),
                             (zero && i == 0 && k == 0) ? 0u : 1u);
        wg_commit();
        wg_wait<1>();
        if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
        prev = (int)stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    wg_wait<0>();
    if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
}

// C(row0.., col0..) += acc for this warpgroup's 64 x 256 block, rows < row_end and columns < col_end (bf16, ldc
// elements per row).  C is read and written at L2: it may have been written by another SM earlier in the window.
__device__ __forceinline__ void epilogue_add(const float (&acc)[128], uint8_t* Cbase, int ldc, int row0, int col0,
                                             int row_end, int col_end) {
    const int t = threadIdx.x & 127, l = t & 31;
    const int r0 = row0 + 16 * (t >> 5) + (l >> 2), r1 = r0 + 8;
    const int c0 = col0 + 2 * (l & 3);
#pragma unroll
    for (int g = 0; g < 32; g += 4) {           // four column blocks at a time: loads in flight before the stores
        uint32_t v0[4], v1[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int col = c0 + 8 * (g + c);
            v0[c] = (r0 < row_end && col < col_end) ? __ldcg(reinterpret_cast<const unsigned int*>(Cbase + ((size_t)r0 * ldc + col) * 2)) : 0u;
            v1[c] = (r1 < row_end && col < col_end) ? __ldcg(reinterpret_cast<const unsigned int*>(Cbase + ((size_t)r1 * ldc + col) * 2)) : 0u;
        }
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int col = c0 + 8 * (g + c), j = 4 * (g + c);
            if (col < col_end) {
                if (r0 < row_end)
                    __stcg(reinterpret_cast<unsigned int*>(Cbase + ((size_t)r0 * ldc + col) * 2),
                           pack_bf16(bf16_lo(v0[c]) + acc[j], bf16_hi(v0[c]) + acc[j + 1]));
                if (r1 < row_end)
                    __stcg(reinterpret_cast<unsigned int*>(Cbase + ((size_t)r1 * ldc + col) * 2),
                           pack_bf16(bf16_lo(v1[c]) + acc[j + 2], bf16_hi(v1[c]) + acc[j + 3]));
            }
        }
    }
}

}  // namespace gemm

struct Win2Dev {
    WinDev w;                       // task-level arrays (descriptors, tiles, outputs, ctl, ring)
    const GUnit* units;
    const GSeg*  segs;
    const int32_t* usucc;
    int32_t* udep;
    int32_t* parts_left;
    const CUtensorMap* tmaps;       // one per tile (w.ntiles)
    int32_t nunits;
    int32_t fresh_tmaps;            // first launch since tmaps were written: every producer acquires all of them first
    TraceDev trace;                 // part records of a traced window (null otherwise); the HBM kernel takes them beside w
};

namespace gemm {

struct Job {
    int32_t unit, part, stop, is_gemm;
    int32_t seg_begin, seg_count, tileC, nparts;
    int32_t M, N, K, pushout;
    int32_t mblocks, nsub;          // GEMM units: sub-tiles of C, ceil(M / BM) per column block; nsub = 0 otherwise
};

struct Shared {
    alignas(16) Job job;
    TaskSmem ts;                    // non-GEMM units: run_task_part's state; GEMM units stage in with its need / decide
    GroupSmem gs;                   // non-GEMM units: the read group the unit's first task leads or runs with
    uint64_t full[kStages];
    uint64_t empty[kStages];
};

// whole warp: the unit is complete (all parts): retire its members in chain order, release its out-edges.  The members
// of a read group retire in member order, right after the producer that runs with them (flag bit 2), which is the
// unit's first member: they saw the version it wrote (seen_version of a group led by its first member was stored with
// each part, group_part_results).
template <bool PRIO>
__device__ __forceinline__ void retire_unit_warp(const Win2Dev& g, const GUnit& u) {
    const WinDev& w = g.w;
    const int lane = threadIdx.x & 31;
    const int L = u.seg_count;
    unsigned long long ebase = 0, rbase = 0;
    uint32_t vx = 0;
    if (lane == 0) {
        ebase = atomicAdd(&w.ctl->evt.v, (unsigned long long)(2 * L));
        rbase = atomicAdd(&w.ctl->retired.v, (unsigned long long)L);
        *reinterpret_cast<volatile unsigned long long*>(&w.ctl->progress_ns.v) = globaltimer_ns();
        if (u.flags & 4) vx = epilog_written_flows(w, w.tasks[g.segs[u.seg_begin].task], w.tasks[g.segs[u.seg_begin + 1].task].tile[0]);
    }
    ebase = __shfl_sync(0xffffffffu, ebase, 0);
    rbase = __shfl_sync(0xffffffffu, rbase, 0);
    vx = __shfl_sync(0xffffffffu, vx, 0);
    const uint32_t cver = (u.flags & 1) ? *reinterpret_cast<volatile uint32_t*>(&w.tiles[u.tileC].version) : 0u;
    for (int i = lane; i < L; i += 32) {
        const GSeg s = g.segs[u.seg_begin + i];
        w.start_seq[s.task] = (uint32_t)(ebase + 2 * i);
        w.end_seq[s.task] = (uint32_t)(ebase + 2 * i + 1);
        w.retire_log[rbase + i] = s.task;
        w.worker[s.task] = (int32_t)blockIdx.x;
        if (u.flags & 1) {
            w.seen_version[s.task * PB2_MAX_FLOWS + 0] = *reinterpret_cast<volatile uint32_t*>(&w.tiles[s.tileA].version);
            w.seen_version[s.task * PB2_MAX_FLOWS + 1] = *reinterpret_cast<volatile uint32_t*>(&w.tiles[s.tileB].version);
            w.seen_version[s.task * PB2_MAX_FLOWS + 2] = cver + (uint32_t)i;
            w.result[s.task] = 0;
        } else if (u.flags & 4) {
            if (i > 0) w.seen_version[s.task * PB2_MAX_FLOWS] = vx;     // the producer's epilog ran above
        } else {
            epilog_written_flows(w, w.tasks[s.task]);      // part 0 stored seen_version (run_task_part)
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
        if (total && PRIO) {
            const uint32_t first = reserve_lane_slots(w.lanes, nparts ? (int)w.lane[sid] : 0, nparts);
            for (int p = 0; p < nparts; ++p) st_release_gpu(&w.ring[first + (uint32_t)p], (int32_t)PB2_SUCC_MAKE(sid, p));
        } else if (total) {
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
}

// Consumer warpgroup `cw` (0 or 1) of a GEMM unit's part: sub-tiles job.part, job.part + nparts, ..., rows m0 + 64 * cw
// .. of each, the whole chain into one accumulator, added into C at Cbase.  stage / phase: the consumers' place in the
// smem ring, carried from one part to the next.
__device__ __forceinline__ void consume_part(const Job& job, uint8_t* smem, uint64_t* full, uint64_t* empty, uint8_t* Cbase,
                                             uint32_t& stage, uint32_t& phase, int cw) {
    const int kblocks = (job.K + BK - 1) / BK;
    float acc[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    for (int sub = job.part; sub < job.nsub; sub += job.nparts) {
        const int m0 = (sub % job.mblocks) * BM, n0 = (sub / job.mblocks) * BN, Nj = min(BN, job.N - n0);
        {   // pull the sub-tile's C rows into L2 now, so that the read-modify-write after the chain does not pay DRAM latency
            const int t = threadIdx.x - 128, row = m0 + (t >> 1);
            if (row < job.M)
                for (int b = (t & 1) * 128; b < Nj * 2; b += 256)
                    asm volatile("prefetch.global.L2 [%0];" :: "l"(Cbase + ((size_t)row * job.N + n0) * 2 + b));
        }
        mma_kblocks(acc, smem, full, empty, stage, phase, job.seg_count * kblocks, true, cw);
        epilogue_add(acc, Cbase, job.N, m0 + cw * 64, n0, job.M, n0 + Nj);
    }
}

// consume_part out of line, for the LINKED kernels.  In relocatable code ptxas serializes every wgmma of a function that
// reaches a call it cannot see into (C7509 for the extern pb2_linked_body; silently for an indirect or weak callee),
// and the kernel reaches the application's body; this function makes no call, so its wgmma groups stay pipelined.
// Under the standard call ABI it saves the callee-saved registers its 128 contiguous accumulator registers cover (ptxas
// counts them as spill stores) once per call, outside the k-block loop.  The ring position goes in and comes back by
// value (stage in the low word, phase in the high word), so nothing of the caller's lives in local memory across the call.
static __device__ __noinline__ uint64_t consume_part_outlined(Shared* sp, uint8_t* smem, uint8_t* Cbase, uint64_t ring, int cw) {
    uint32_t stage = (uint32_t)ring, phase = (uint32_t)(ring >> 32);
    consume_part(sp->job, smem, sp->full, sp->empty, Cbase, stage, phase, cw);
    return stage | ((uint64_t)phase << 32);
}

// All threads (LINKED instantiations), in place of the body of a task marked PB2_TASK_GEMM_BODY: the application's
// GEMM-worker body gets its task's whole tiles in the 80-byte block *lp, with check 0, as run_linked_part hands them,
// and the operand ring as scratch (include/pb2_device_body.h).  The ring is idle: the consumers of every GEMM unit that
// ran on this worker before waited on full[] for each TMA load of the unit and on each of its wgmma groups, before the
// barrier that ended the unit.  The fences order the body's generic accesses to the ring after those async-proxy
// accesses, and before the TMA writes of the units after it (the caller's barrier follows the second one).
// Built with PB2_LINKED_GEMM_BODY_ENTRY (the kernels linked with PB2_LINK_GEMM_BODY_ENTRY), the call goes to the
// application's pb2_linked_gemm_body instead, which only these kernels reach, so it has their register budget.
static_assert(PB2_GEMM_BODY_SMEM_BYTES == kStages * kStageBytes, "a GEMM-worker body gets the whole operand ring");
static_assert(kSmemBytes - kStages * kStageBytes == PB2_GEMM_BODY_SMEM_ALIGN, "the ring is aligned up to 1024 bytes");
// A task of a body declared in parts (pb2_engine_set_gemm_body_parts) calls it once per part, each over whole tiles
// (run_task_part<..., GEMM_BODY_PARTS>) with its part index in args.part and the count in lp->nparts.
static __device__ __forceinline__ unsigned long long run_gemm_worker_body(TaskSmem* sp, pb2_gemm_body_args_t* lp, uint8_t* ring,
                                                                          int nparts) {
    static_assert(sizeof(BodyArgs) % 4 == 0 && sizeof(BodyArgs) / 4 <= kThreads, "one word of BodyArgs per thread");
    if (threadIdx.x < sizeof(BodyArgs) / 4)
        reinterpret_cast<uint32_t*>(&lp->args)[threadIdx.x] = reinterpret_cast<const uint32_t*>(&sp->args)[threadIdx.x];
    if (threadIdx.x == 0) { lp->check = 0; lp->k0 = 0; lp->nparts = (unsigned)nparts; lp->reserved = 0; }
    __syncthreads();
    fence_proxy_async();
#ifdef PB2_LINKED_GEMM_BODY_ENTRY
    const unsigned long long r = pb2_linked_gemm_body(sp->task.body, &lp->args, reinterpret_cast<unsigned int*>(ring));
#else
    const unsigned long long r = pb2_linked_body(sp->task.body, &lp->args, reinterpret_cast<unsigned int*>(ring));
#endif
    fence_proxy_async();
    return r;
}

// All threads, on the worker whose part of a GEMM-worker task in parts retires it: every written flow marked PUSHOUT,
// copied home whole.  Its parts wrote it on other SMs; their stores are visible (each part's __threadfence before it
// counted parts_left down) and the copy reads through L2.
template <bool TRACE>
__device__ __forceinline__ void push_out_whole_flows(const WinDev& w, const pb2_task_t& t, PartSmem* rec) {
#pragma unroll 1
    for (int f = 0; f < (int)t.nb_flows; ++f) {
        if (t.tile[f] < 0 || !(t.access[f] & PB2_FLOW_PUSHOUT) || !(t.access[f] & PB2_FLOW_ACCESS_WRITE)) continue;
        const pb2_tile_t* tile = &w.tiles[t.tile[f]];
        cta_copy<false>(tile->src_ptr, tile->dev_ptr, tile->bytes);
        if (threadIdx.x == 0) atomicAdd(&w.ctl->bytes_d2h.v, (unsigned long long)tile->bytes);
        if (TRACE && threadIdx.x == 0) rec->out_bytes += tile->bytes;
    }
}

}  // namespace gemm

// PRIO: queue_policy 1 (priority lanes of units, pop_prio).  TRACE: write a record of every part into g.trace (PartSmem,
// then trace_part); the untraced instantiations never touch it.  The built-in instantiations are in
// pb2_window_kernels.cu, one per object, beside the HBM kernel of the same PRIO and TRACE; the engine launches every
// instantiation with gemm::kThreads threads and the operand ring, gemm::kSmemBytes, as dynamic shared memory.
// LINKED: body ids PB2_BODY_LINKED_0 .. _7 call the application's pb2_linked_body, a task marked PB2_TASK_GEMM_BODY with
// the operand ring as its scratch (run_gemm_worker_body); built only in
// pb2_engine_linked_gemm.cu, as relocatable device code that pb2_engine_link_bodies_ex links with the application's
// image when PB2_LINK_GEMM_WINDOWS is set.  The other instantiations compile as if the flag did not exist.
template <bool PRIO, bool TRACE, bool LINKED = false>
__global__ void __launch_bounds__(gemm::kThreads, 1)
pb2_engine_gemm2_kernel(Win2Dev g) {
    using namespace gemm;
    const WinDev& w = g.w;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    __shared__ Shared sh;
    PartSmem* rec = nullptr;
    if constexpr (TRACE) { __shared__ PartSmem part_rec; rec = &part_rec; }
    pb2_body_check_t* lk = nullptr;          // LINKED: what a linked body is handed (run_linked_part)
    pb2_gemm_body_args_t* lg = nullptr;      // ... the same block, as a GEMM-worker body reads it (run_gemm_worker_body)
    if constexpr (LINKED) {
        __shared__ pb2_gemm_body_args_t linked_args;
        lg = &linked_args; lk = reinterpret_cast<pb2_body_check_t*>(&linked_args);
    }

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg = threadIdx.x >> 7;

    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) { mbar_init(&sh.full[s], 1); mbar_init(&sh.empty[s], kConsumers); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // The maps of a live window stay at their addresses and never change, so what a launch caches stays valid for the
    // next launches of the window; only the first one has to drop what an earlier window left at those addresses.
    if (g.fresh_tmaps && warp == 1 && lane == 0)
        for (int i = 0; i < w.ntiles; ++i) tmap_acquire(&g.tmaps[i]);
    __syncthreads();

    uint32_t p_stage = 0, p_phase = 0, c_stage = 0, c_phase = 0;

    for (;;) {
        // ---------------- pop the next (part, unit), stage its tiles in
        if (threadIdx.x == 0) {
            Job j; memset(&j, 0, sizeof j);
            const int32_t e = pop_entry<PRIO>(w);
            if (e == kEmpty) { j.stop = 1; }
            else {
                __threadfence();
                if (TRACE) *rec = PartSmem{globaltimer_ns(), 0, 0, 0, 0, 0, 0};
                j.unit = PB2_SUCC_TASK((uint32_t)e); j.part = PB2_SUCC_FLOW((uint32_t)e);
                const GUnit u = g.units[j.unit];
                j.is_gemm = u.flags & 1; j.pushout = (u.flags >> 1) & 1;
                j.seg_begin = u.seg_begin; j.seg_count = u.seg_count; j.tileC = u.tileC; j.nparts = u.nparts;
                j.M = u.M; j.N = u.N; j.K = u.K;
                if (j.is_gemm) { j.mblocks = (u.M + BM - 1) / BM; j.nsub = j.mblocks * ((u.N + BN - 1) / BN); }
            }
            sh.job = j;
        }
        __syncthreads();
        if (sh.job.stop) break;
        {
            // GEMM units: stage in every INVALID tile the job reads (same protocol as the other kernels)
            const int nseg = sh.job.is_gemm ? sh.job.seg_count : 0;
            for (int i = -1; i < 2 * nseg; ++i) {
                int tile_id; uint8_t acc;
                if (i < 0) { if (!sh.job.is_gemm) break; tile_id = sh.job.tileC; acc = PB2_FLOW_ACCESS_RW; }
                else { const GSeg s = g.segs[sh.job.seg_begin + (i >> 1)]; tile_id = (i & 1) ? s.tileB : s.tileA; acc = PB2_FLOW_ACCESS_READ; }
                pb2_tile_t* tile = &w.tiles[tile_id];
                if (threadIdx.x == 0) sh.ts.need = ld_acquire_gpu(&tile->state) != PB2_TILE_VALID;
                __syncthreads();
                if (sh.ts.need) {
                    const int ns = tile_slices(w, tile->bytes);
                    if (TRACE && threadIdx.x == 0) rec->flags |= PB2_PART_WAITED_INPUT;
                    unsigned long long* moved = TRACE ? &rec->in_bytes : nullptr;
                    if (ns == 1) stage_in_flow<TRACE>(stage_ctx(w), tile, acc, &sh.ts.decide, nullptr, moved);
                    else stage_in_slices<TRACE>(stage_ctx(w), tile_id, ns, 0, ns, &sh.ts.decide, nullptr, moved);     // take what nobody has claimed, wait for the rest
                    fence_proxy_async();
                }
                __syncthreads();
            }
            if (TRACE && sh.job.is_gemm && threadIdx.x == 0) rec->t_in = globaltimer_ns();
        }
        const Job& job = sh.job;       // read from shared memory, not held in registers across the wgmma loop

        // The part's sub-tiles are job.part, job.part + nparts, ...: sub-tile `sub` is rows m0 .. m0 + 127 and columns
        // n0 .. n0 + Nj - 1 of C.  The producer and the consumers walk the same sequence, so the ring's stage and phase
        // carry over from one sub-tile to the next.
        if (job.is_gemm) {
            const int kblocks = (job.K + BK - 1) / BK;
            if (warp == 1) {
                // ===== TMA producer: 128 rows of A, 256 rows of B per k-block, every member of the chain
                if (lane == 0) {
                    fence_proxy_async();
                    for (int sub = job.part; sub < job.nsub; sub += job.nparts) {
                        const int m0 = (sub % job.mblocks) * BM, n0 = (sub / job.mblocks) * BN;
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
                                mbar_expect_tx(&sh.full[p_stage], kStageBytes);
                                tma_load_2d(sa, mapA, &sh.full[p_stage], kb * BK, m0);
                                tma_load_2d(sa + kAStageBytes, mapB, &sh.full[p_stage], kb * BK, n0);
                                tma_load_2d(sa + kAStageBytes + kBStageBytes / 2, mapB, &sh.full[p_stage], kb * BK, n0 + 128);
                                if (++p_stage == kStages) { p_stage = 0; p_phase ^= 1; }
                            }
                        }
                    }
                }
            } else if (wg >= 1) {
                // ===== consumers: rows m0 + 64 * cw .. of each sub-tile, the whole chain into one accumulator
                uint8_t* Cbase = reinterpret_cast<uint8_t*>(w.tiles[job.tileC].dev_ptr);
                if constexpr (LINKED) {
                    const uint64_t ring = consume_part_outlined(&sh, smem, Cbase, c_stage | ((uint64_t)c_phase << 32), wg - 1);
                    c_stage = (uint32_t)ring; c_phase = (uint32_t)(ring >> 32);
                } else {
                    consume_part(job, smem, sh.full, sh.empty, Cbase, c_stage, c_phase, wg - 1);
                }
                fence_proxy_async();
            }
        } else {
            // ---------------- an HBM body in the DAG (element-wise task, panel stand-in): the whole CTA runs this
            // part's byte slice of its flows in place, as a worker of an HBM window does, with the read group its
            // task leads or runs with (a producer fused with its group: run_fused_part, or run_linked_part in check
            // mode).  Later units read the tiles through TMA: the generic stores of a stage-in and of the body are
            // followed by fence.proxy.async.
            const int32_t id = g.segs[job.seg_begin].task;
            if (threadIdx.x < 4) reinterpret_cast<uint4*>(&sh.ts.task)[threadIdx.x] =
                __ldg(reinterpret_cast<const uint4*>(&w.tasks[id]) + threadIdx.x);
            const uint32_t gd = load_group_members(w, id, sh.gs);
            if (threadIdx.x == 0) { sh.gs.n = (int)(gd & 15u); sh.gs.fused = (gd & PB2_GROUP_FUSED) != 0; }
            __syncthreads();
            const unsigned long long r = run_task_part<false, TRACE, LINKED>(w, sh.ts, nullptr, id, job.part, job.nparts, [&] {
                if (sh.ts.need) fence_proxy_async();
                unsigned long long body_r;
                if constexpr (LINKED) body_r = (sh.ts.task.flags & PB2_TASK_GEMM_BODY) ? run_gemm_worker_body(&sh.ts, lg, smem, job.nparts)
                                             : linked_reader_group(w, sh.gs) ? run_linked_group_part<kThreads>(&sh.ts, &sh.gs, lk, w.tasks, w.seen_version)
                                             : is_linked_body(sh.ts.task.body) ? run_linked_part<kThreads>(&sh.ts, &sh.gs, lk)
                                             : sh.gs.fused ? run_fused_part<kThreads>(&sh.ts, &sh.gs)
                                                           : run_hbm_body(sh.ts.task.body, sh.ts.args, sh.ts.red);
                else body_r = sh.gs.fused ? run_fused_part<kThreads>(&sh.ts, &sh.gs) : run_hbm_body(sh.ts.task.body, sh.ts.args, sh.ts.red);
                fence_proxy_async();
                return body_r;
            }, rec);
            // the leader of a group of linked readers is a reader; run_linked_group_part gave its members their results
            if (sh.gs.n && !sh.gs.fused && !(LINKED && (sh.ts.task.flags & PB2_TASK_READER)))
                group_part_results<kThreads, TRACE>(w, sh.ts, sh.gs, id, job.part, r, rec);
            // CHECK parts add their mismatch counts, linked readers their sums; the first element comes from part 0
            if (threadIdx.x == 0) store_part_results<LINKED>(w, sh.ts.task, id, job.part, job.nparts, r, sh.gs);
        }
        __threadfence();
        __syncthreads();             // every store of the part is done and visible
        // a GEMM unit's exec ends here: its TMA operand stream cannot be told apart from its MMAs
        if (TRACE && job.is_gemm && threadIdx.x == 0) rec->t_exec = globaltimer_ns();

        // ---------------- part complete: pushout of its sub-tiles' C rows, then unit retirement by the last part
        if (job.is_gemm && job.pushout) {
            pb2_tile_t* tile = &w.tiles[job.tileC];
            const size_t row_bytes = (size_t)job.N * 2;
            for (int sub = job.part; sub < job.nsub; sub += job.nparts) {
                const int m0 = (sub % job.mblocks) * BM, n0 = (sub / job.mblocks) * BN, Nj = min(BN, job.N - n0);
                const int rows = min(BM, job.M - m0);
                if (Nj == job.N) {
                    cta_copy<false>(reinterpret_cast<uint8_t*>(tile->src_ptr) + (size_t)m0 * row_bytes,
                                    reinterpret_cast<const uint8_t*>(tile->dev_ptr) + (size_t)m0 * row_bytes, (size_t)rows * row_bytes);
                    if (threadIdx.x == 0) atomicAdd(&w.ctl->bytes_d2h.v, (unsigned long long)rows * row_bytes);
                    if (TRACE && threadIdx.x == 0) rec->out_bytes += (unsigned long long)rows * row_bytes;
                } else {
                    // a column block of a tile wider than one sub-tile: row segments
                    for (int r = 0; r < rows; ++r) {
                        const size_t o = (size_t)(m0 + r) * row_bytes + (size_t)n0 * 2;
                        cta_copy<false>(reinterpret_cast<uint8_t*>(tile->src_ptr) + o, reinterpret_cast<const uint8_t*>(tile->dev_ptr) + o, (size_t)Nj * 2);
                    }
                    if (threadIdx.x == 0) atomicAdd(&w.ctl->bytes_d2h.v, (unsigned long long)rows * (unsigned long long)Nj * 2ull);
                    if (TRACE && threadIdx.x == 0) rec->out_bytes += (unsigned long long)rows * (unsigned long long)Nj * 2ull;
                }
            }
            // a pushout writes the whole tile back, as every other body's does: the part that runs the last sub-tile also
            // copies the bytes of the tile past C
            const size_t c_bytes = (size_t)job.M * row_bytes;
            if (job.part == (job.nsub - 1) % job.nparts && tile->bytes > c_bytes) {
                cta_copy<false>(reinterpret_cast<uint8_t*>(tile->src_ptr) + c_bytes,
                                reinterpret_cast<const uint8_t*>(tile->dev_ptr) + c_bytes, tile->bytes - c_bytes);
                if (threadIdx.x == 0) atomicAdd(&w.ctl->bytes_d2h.v, (unsigned long long)(tile->bytes - c_bytes));
                if (TRACE && threadIdx.x == 0) rec->out_bytes += (unsigned long long)(tile->bytes - c_bytes);
            }
            __syncthreads();
        }
        if constexpr (LINKED) {
            // ---------------- a part of a GEMM-worker task in parts: the worker that counts the last part pushes the
            // task's flows out whole, after every part's stores, then records its part and retires the unit
            if (!job.is_gemm && job.nparts > 1 && (sh.ts.task.flags & PB2_TASK_GEMM_BODY)) {
                if (threadIdx.x == 0) { __threadfence(); sh.ts.last = atomicSub(&g.parts_left[job.unit], 1) == 1; }
                __syncthreads();
                const bool last = sh.ts.last != 0;
                if (last) {
                    __threadfence();
                    push_out_whole_flows<TRACE>(w, sh.ts.task, rec);
                    __threadfence();
                    __syncthreads();
                }
                if (warp == 0) {
                    if (TRACE && lane == 0) {
                        if (last) rec->t_out = globaltimer_ns();
                        trace_part(g.trace, job.unit, job.part, *rec, last);
                    }
                    if (last) retire_unit_warp<PRIO>(g, g.units[job.unit]);
                }
                __syncthreads();     // sh.job is rewritten by the next pop
                continue;
            }
        }
        if (warp == 0) {
            int last = 0;
            if (TRACE && lane == 0 && job.is_gemm) rec->t_out = globaltimer_ns();
            if (lane == 0) { __threadfence(); last = atomicSub(&g.parts_left[job.unit], 1) == 1; }
            if (TRACE && lane == 0) trace_part(g.trace, job.unit, job.part, *rec, last);
            last = __shfl_sync(0xffffffffu, last, 0);
            if (last) { __threadfence(); retire_unit_warp<PRIO>(g, g.units[job.unit]); }
        }
        __syncthreads();             // sh.job is rewritten by the next pop
    }
}

}  // namespace pb2
