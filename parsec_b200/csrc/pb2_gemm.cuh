// pb2_gemm.cuh -- tensor-core (wgmma / TMA / mbarrier) engine kernel for PB2_BODY_GEMM_BF16 windows.
//
// The task body restates what the reference reaches through `dyld=cublasDgemm` / cublasDgemm_v2
// (tests/dsl/dtd/dtd_test_simple_gemm.c:450,527; tests/runtime/cuda/nvlink.jdf:136-152): one tile
// GEMM per task, C(M x N) += A(M x K) * B(K x N).  Here in bf16 with fp32 accumulation in registers
// (BASELINE config 3); tiles are K-contiguous for both operands: A row-major [M][K], B stored
// [N][K] (== column-major K x N, what a "TN" cuBLAS call consumes), C row-major [M][N].
//
// One CTA per SM is one worker.  Three warpgroups (384 threads):
//   warpgroup 0 : warp 0 is the scheduler (ring pop / dependency release / retire) and, one lane, the TMA producer
//   warpgroups 1, 2 : consumers; each issues `wgmma.mma_async` m64n256k16 for its 64 rows of the sub-tile and keeps
//                 the 64 x 256 fp32 accumulator in registers, then adds it into C (bf16) itself
// A task is executed as ceil(M/128) x ceil(N/256) accumulator sub-tiles of 128 x 256 fp32.  Operands stream
// through a 4-stage smem ring of {A 128x64, B 256x64} bf16 128B-swizzled boxes filled by TMA
// (`cp.async.bulk.tensor.2d`) from per-tile tensor maps; the producer fills the next sub-tile's stages while the
// consumers run the epilogue of the current one.
#pragma once
#include <cuda.h>
#include "pb2_sched.cuh"

namespace pb2 {

namespace gemm {

constexpr int BM = 128, BN = 256, BK = 64, UK = 16;
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

struct Shared {
    alignas(16) pb2_task_t task;    // filled with four 16-byte loads
    uint64_t full[kStages];
    uint64_t empty[kStages];
    int32_t  id;
    int32_t  need;
    int32_t  decide;
    int32_t  last;
    uint32_t red[32];
};

}  // namespace gemm

__global__ void __launch_bounds__(gemm::kThreads, 1)
pb2_engine_gemm_kernel(WinDev w, const CUtensorMap* __restrict__ tmaps) {
    using namespace gemm;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    __shared__ Shared sh;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg = threadIdx.x >> 7;

    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) { mbar_init(&sh.full[s], 1); mbar_init(&sh.empty[s], kConsumers); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    // pipeline state persists across tasks
    uint32_t p_stage = 0, p_phase = 0;     // producer
    uint32_t c_stage = 0, c_phase = 0;     // consumers

    for (;;) {
        if (threadIdx.x == 0) {
            const int32_t id = pop_task(w);
            if (id != kEmpty) {
                __threadfence();
                w.start_seq[id] = (uint32_t)atomicAdd(&w.ctl->evt.v, 1ull);
                w.worker[id] = (int32_t)blockIdx.x;
            }
            sh.id = id;
        }
        __syncthreads();
        const int32_t id = sh.id;
        if (id == kEmpty) break;
        if (threadIdx.x < 4) reinterpret_cast<uint4*>(&sh.task)[threadIdx.x] =
            __ldg(reinterpret_cast<const uint4*>(&w.tasks[id]) + threadIdx.x);
        __syncthreads();
        const pb2_task_t& t = sh.task;

        // ---- stage in (same protocol as the HBM kernel) ----
        if (threadIdx.x == 0) {
            int need = 0;
            for (int f = 0; f < t.nb_flows; ++f)
                if (t.tile[f] >= 0 && (t.access[f] & PB2_FLOW_ACCESS_READ) &&
                    ld_acquire_gpu(&w.tiles[t.tile[f]].state) != PB2_TILE_VALID) need |= 1 << f;
            sh.need = need;
        }
        __syncthreads();
        {
            const int need = sh.need;
            for (int f = 0; f < t.nb_flows; ++f) {
                if (t.tile[f] < 0) continue;
                pb2_tile_t* tile = &w.tiles[t.tile[f]];
                if ((need >> f) & 1) stage_in_flow(stage_ctx(w), tile, t.access[f], &sh.decide);
                if (threadIdx.x == 0)
                    w.seen_version[id * PB2_MAX_FLOWS + f] = *reinterpret_cast<volatile uint32_t*>(&tile->version);
            }
            if (need) { fence_proxy_async(); __syncthreads(); }
        }

        const bool is_gemm = (t.body == PB2_BODY_GEMM_BF16);
        unsigned long long hbm_result = 0;
        if (!is_gemm && t.body != PB2_BODY_NOP) {
            // GEMM windows may carry a few HBM-bound tasks of the same DAG (e.g. a panel task): run them in place
            BodyArgs a;
            for (int f = 0; f < PB2_MAX_FLOWS; ++f) {
                const bool has = f < t.nb_flows && t.tile[f] >= 0;
                a.flow[f] = has ? w.tiles[t.tile[f]].dev_ptr : nullptr;
                a.bytes[f] = has ? w.tiles[t.tile[f]].bytes : 0;
            }
            a.elem0 = 0; a.part = 0;
            a.iparam[0] = t.iparam[0]; a.iparam[1] = t.iparam[1]; a.iparam[2] = t.iparam[2]; a.fparam = t.fparam;
            hbm_result = run_hbm_body(t.body, a, sh.red);
            fence_proxy_async();
            __syncthreads();
        }
        const int M = t.iparam[0], N = t.iparam[1], K = t.iparam[2];
        const int mblocks = is_gemm ? (M + BM - 1) / BM : 0;
        const int nblocks = is_gemm ? (N + BN - 1) / BN : 0;
        const int kblocks = (K + BK - 1) / BK;
        const int nsub = mblocks * nblocks;

        if (warp == 0) {
            // ===== TMA producer =====
            if (lane == 0 && nsub > 0) {
                fence_proxy_async();    // operand tiles may have been written by generic-proxy stores
                const CUtensorMap* mapA = &tmaps[t.tile[0]];
                const CUtensorMap* mapB = &tmaps[t.tile[1]];
                for (int sub = 0; sub < nsub; ++sub) {
                    const int mb = sub / nblocks, nb = sub % nblocks;
                    for (int kb = 0; kb < kblocks; ++kb) {
                        mbar_wait(&sh.empty[p_stage], p_phase ^ 1);
                        uint8_t* sa = smem + p_stage * kStageBytes;
                        uint8_t* sb = sa + kAStageBytes;
                        mbar_expect_tx(&sh.full[p_stage], kStageBytes);
                        tma_load_2d(sa, mapA, &sh.full[p_stage], kb * BK, mb * BM);
                        tma_load_2d(sb, mapB, &sh.full[p_stage], kb * BK, nb * BN);
                        tma_load_2d(sb + kBStageBytes / 2, mapB, &sh.full[p_stage], kb * BK, nb * BN + 128);
                        if (++p_stage == kStages) { p_stage = 0; p_phase ^= 1; }
                    }
                }
            }
        } else if (wg >= 1) {
            // ===== consumer warpgroups: wgmma into registers, then C += acc -> bf16 =====
            if (nsub > 0) {
                const int cw = wg - 1;
                uint8_t* Cbase = reinterpret_cast<uint8_t*>(w.tiles[t.tile[2]].dev_ptr);
                float acc[128];
#pragma unroll
                for (int i = 0; i < 128; ++i) acc[i] = 0.f;
                for (int sub = 0; sub < nsub; ++sub) {
                    const int mb = sub / nblocks, nb = sub % nblocks;
                    mma_kblocks(acc, smem, sh.full, sh.empty, c_stage, c_phase, kblocks, true, cw);
                    epilogue_add(acc, Cbase, N, mb * BM + cw * 64, nb * BN, M, N);
                }
                fence_proxy_async();   // C may be consumed through TMA by a later task on another SM
            }
        }
        __syncthreads();

        // ---- pushout (PARSEC_PUSHOUT on the last k, dtd_test_simple_gemm.c:687) ----
        for (int f = 0; f < t.nb_flows; ++f) {
            if (t.tile[f] >= 0 && (t.access[f] & PB2_FLOW_PUSHOUT) && (t.access[f] & PB2_FLOW_ACCESS_WRITE)) {
                pb2_tile_t* tile = &w.tiles[t.tile[f]];
                cta_copy<false>(tile->src_ptr, tile->dev_ptr, tile->bytes);
                if (threadIdx.x == 0) atomicAdd(&w.ctl->bytes_d2h.v, (unsigned long long)tile->bytes);
            }
        }
        __syncthreads();

        if (threadIdx.x < 32) {
            __threadfence();
            if (threadIdx.x == 0) {
                w.result[id] = hbm_result;
                if ((t.body == PB2_BODY_CHECK_I32 || t.body == PB2_BODY_CHECK_F32) && (hbm_result >> 32))
                    atomicAdd(&w.ctl->body_errors.v, hbm_result >> 32);
                for (int f = 0; f < t.nb_flows; ++f) {
                    if (t.tile[f] < 0 || !(t.access[f] & PB2_FLOW_ACCESS_WRITE)) continue;
                    pb2_tile_t* tile = &w.tiles[t.tile[f]];
                    *reinterpret_cast<volatile uint32_t*>(&tile->version) =
                        *reinterpret_cast<volatile uint32_t*>(&tile->version) + 1;
                    if (!(t.access[f] & PB2_FLOW_ACCESS_READ)) st_relaxed_gpu(&tile->state, PB2_TILE_VALID);
                }
                w.end_seq[id] = (uint32_t)atomicAdd(&w.ctl->evt.v, 1ull);
                sh.last = retire_task(w, id) ? 1 : 0;
                __threadfence();
            }
            __syncwarp();
            release_successors_warp(w, t);
            release_remote_warp(w, id);
            if (threadIdx.x == 0 && sh.last) {
                __threadfence();
                st_release_gpu(reinterpret_cast<int32_t*>(&w.ctl->done.v), kDoneOK);
            }
        }
        __syncthreads();
    }
}

static inline int pb2_gemm_nworkers(int sm_count) { return sm_count; }

static inline int pb2_gemm_launch(const WinDev& w, const CUtensorMap* tmaps, int nworkers, cudaStream_t stream) {
    static bool attr_set = false;
    if (!attr_set) {
        if (cudaFuncSetAttribute(pb2_engine_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 gemm::kSmemBytes) != cudaSuccess) return PB2_ERR_DEVICE;
        attr_set = true;
    }
    pb2_engine_gemm_kernel<<<nworkers, gemm::kThreads, gemm::kSmemBytes, stream>>>(w, tmaps);
    return cudaGetLastError() == cudaSuccess ? PB2_SUCCESS : PB2_ERR_DEVICE;
}

}  // namespace pb2
