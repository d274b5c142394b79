// GEMM-worker bodies whose tasks run in parts (pb2_engine_set_gemm_body_parts), that the GPU tests
// (tests/test_gemm_body_parts_gpu.py) and tools/ab_gemm_body_parts.py link into GEMM engine windows.  Application code,
// not part of the library.  Every part of a task gets the task's whole tiles, its part index in args.part and the part
// count in pb2_gemm_body_args_t::nparts, and splits the work by them itself.  Built by the Makefile with
// -maxrregcount=168 (the GEMM window kernels' budget) into gemm_part_bodies.cubin, and with -DGEMM_PART_READER_GROUP,
// which adds the group form of SUM, into gemm_part_group_bodies.cubin.
//   PB2_BODY_LINKED_0  DGEMM  C (M x N, row-major fp64) += A (M x K, row-major) * B (N x K, row-major)^T on the FP64
//                             tensor cores; flows A, B, C; iparam = M, N, K.  The DGEMM of gemm_entry_bodies.cu (same
//                             blocking, same k order), where part p runs the C blocks p, p + nparts, ...: every C element
//                             gets the same DMMA sequence for any part count.  Through pb2_linked_gemm_body only.
//   PB2_BODY_LINKED_1  PART   the part probe, through either entry point: writes (nparts << 16) | (part + 1) into word
//                             `part` of flow 0 and returns what it saw (probe_result below).
//   PB2_BODY_LINKED_2  ADD    flow 0 (int32) += iparam[0], element-wise; sliceable; result 0.
//   PB2_BODY_LINKED_3  SUM    reader: the sum of flow 0's int32 elements, as a 64-bit integer modulo 2^64.
#include <stdint.h>
#include "pb2_device_body.h"

enum { DGEMM = 20, PART = 21, ADD = 22, SUM = 23 };

namespace {

// The blocking of gemm_entry_bodies.cu: C blocks of BM x BN, 12 warps as 4 x 3 of 32 x 32 each, K through NST ring
// stages of BK, rows padded to LD doubles.
constexpr int BM = 128, BN = 96, BK = 16, LD = BK + 4, NST = 5, WM = 32, WN = 32;
constexpr int kStageDoubles = (BM + BN) * LD;
static_assert(NST * kStageDoubles * 8 <= PB2_GEMM_BODY_SMEM_BYTES, "the stages fit in the operand ring");
static_assert((BM / WM) * (BN / WN) == 12, "one 32 x 32 block of C per warp of the 384-thread worker");

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ double lds(uint32_t a) {
    double v;
    asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(a));
    return v;
}

__device__ __forceinline__ void mma_m16n8k8(double (&d)[4], const double (&a)[4], const double (&b)[2]) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
}

// The part's index and count: a GEMM-worker body's `a` points into a pb2_gemm_body_args_t.
__device__ __forceinline__ uint32_t nparts_of(const pb2_body_args_t* a) {
    return reinterpret_cast<const pb2_gemm_body_args_t*>(a)->nparts;
}

template <bool VEC>
__device__ __forceinline__ void load_stage(uint32_t st, const double* A, const double* B, int M, int N, int K, int m0, int n0,
                                           int k0) {
    constexpr int W = VEC ? 2 : 1, PER_ROW = BK / W;
#pragma unroll 1
    for (int i = threadIdx.x; i < (BM + BN) * PER_ROW; i += blockDim.x) {
        const int r = i / PER_ROW, c = (i % PER_ROW) * W;
        const bool isa = r < BM;
        const int row = isa ? m0 + r : n0 + (r - BM), k = k0 + c;
        const bool ok = row < (isa ? M : N) && k < K;
        const double* src = (isa ? A : B) + (ok ? (size_t)row * K + k : 0);
        const uint32_t dst = st + (uint32_t)(r * LD + c) * 8u;
        if constexpr (VEC)
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" :: "r"(dst), "l"(src), "r"(ok ? 16 : 0) : "memory");
        else
            asm volatile("st.shared.f64 [%0], %1;" :: "r"(dst), "d"(ok ? __ldcg(src) : 0.0) : "memory");
    }
}

// C blocks part, part + nparts, ... of the task's C; each as gemm_entry_bodies.cu computes it.
template <bool VEC>
__device__ void dgemm_tile(const pb2_body_args_t* a, uint32_t ring, int M, int N, int K, int part, int nparts) {
    const double* A = static_cast<const double*>(a->flow[0]);
    const double* B = static_cast<const double*>(a->flow[1]);
    double* C = static_cast<double*>(a->flow[2]);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int wm = (warp / (BN / WN)) * WM, wn = (warp % (BN / WN)) * WN;
    const int mblocks = (M + BM - 1) / BM, nblocks = (N + BN - 1) / BN, nk = (K + BK - 1) / BK;
#pragma unroll 1
    for (int blk = part; blk < mblocks * nblocks; blk += nparts) {
        const int m0 = (blk % mblocks) * BM, n0 = (blk / mblocks) * BN;
        const bool live = m0 + wm < M && n0 + wn < N;
        double acc[2][4][4];
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int v = 0; v < 4; ++v) acc[i][j][v] = 0.0;
#pragma unroll 1
        for (int s = 0; s < NST - 1; ++s) {
            if (s < nk) load_stage<VEC>(ring + s * kStageDoubles * 8, A, B, M, N, K, m0, n0, s * BK);
            asm volatile("cp.async.commit_group;" ::: "memory");
        }
#pragma unroll 1
        for (int kb = 0; kb < nk; ++kb) {
            asm volatile("cp.async.wait_group %0;" :: "n"(NST - 2) : "memory");
            __syncthreads();
            const int nxt = kb + NST - 1;
            if (nxt < nk) load_stage<VEC>(ring + (nxt % NST) * kStageDoubles * 8, A, B, M, N, K, m0, n0, nxt * BK);
            asm volatile("cp.async.commit_group;" ::: "memory");
            if (!live) continue;
            const uint32_t As = ring + (uint32_t)((kb % NST) * kStageDoubles + (wm + g) * LD + t) * 8u;
            const uint32_t Bs = ring + (uint32_t)((kb % NST) * kStageDoubles + (BM + wn + g) * LD + t) * 8u;
#pragma unroll
            for (int kk = 0; kk < BK; kk += 8) {
                double fa[2][4], fb[4][2];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const uint32_t p = Bs + (uint32_t)(8 * j * LD + kk) * 8u;
                    fb[j][0] = lds(p); fb[j][1] = lds(p + 32);
                }
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const uint32_t p = As + (uint32_t)(16 * i * LD + kk) * 8u;
                    fa[i][0] = lds(p); fa[i][1] = lds(p + 8 * LD * 8); fa[i][2] = lds(p + 32); fa[i][3] = lds(p + 8 * LD * 8 + 32);
                }
#pragma unroll
                for (int i = 0; i < 2; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) mma_m16n8k8(acc[i][j], fa[i], fb[j]);
            }
        }
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();
        if (!live) continue;
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = m0 + wm + 16 * i + g + 8 * h;
                if (row >= M) continue;
#pragma unroll
                for (int j = 0; j < 4; ++j)
#pragma unroll
                    for (int v = 0; v < 2; ++v) {
                        const int col = n0 + wn + 8 * j + 2 * t + v;
                        if (col < N) {
                            double* c = C + (size_t)row * N + col;
                            __stcg(c, __ldcg(c) + acc[i][j][2 * h + v]);
                        }
                    }
            }
    }
}

__device__ unsigned long long dgemm(const pb2_body_args_t* a, unsigned int* scratch) {
    const int M = a->iparam[0], N = a->iparam[1], K = a->iparam[2];
    const int part = (int)a->part, nparts = (int)nparts_of(a);
    if (M <= 0 || N <= 0 || K <= 0 || !a->flow[0] || !a->flow[1] || !a->flow[2] ||
        (uint64_t)M * K * 8 > a->bytes[0] || (uint64_t)N * K * 8 > a->bytes[1] || (uint64_t)M * N * 8 > a->bytes[2] ||
        nparts < 1 || part >= nparts)
        return ~0ull;
    const uint32_t ring = smem_u32(scratch);
    if (K % 2 == 0) dgemm_tile<true>(a, ring, M, N, K, part, nparts);
    else dgemm_tile<false>(a, ring, M, N, K, part, nparts);
    return 0;
}

// The part probe.  Thread 0 stores (nparts << 16) | (part + 1) into word `part` of flow 0.  The result is
// (part << 48) | (nparts << 40), with bit 32 set when scratch is not 1024-byte aligned shared memory, bit 33 when
// blockDim.x is not 384, bit 34 when the part did not get the whole tile (bytes[0] != iparam[0] or elem0 != 0), bit 35
// when it was reached through pb2_linked_body, and bit 36 when part >= nparts or the ring does not read back what the
// CTA wrote over it.
__device__ unsigned long long part_probe(const pb2_body_args_t* a, unsigned int* ring, bool entry) {
    const uint32_t part = a->part, nparts = nparts_of(a);
    const uint32_t n = PB2_GEMM_BODY_SMEM_BYTES / 4;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) ring[i] = (i * 0x9E3779B1u) ^ part;
    __syncthreads();
    uint32_t bad = 0;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) bad |= ring[n - 1 - i] != (((n - 1 - i) * 0x9E3779B1u) ^ part);
    bad = __syncthreads_or(bad);
    unsigned long long r = ((unsigned long long)part << 48) | ((unsigned long long)(nparts & 0xFFu) << 40);
    if (!__isShared(ring) || smem_u32(ring) % PB2_GEMM_BODY_SMEM_ALIGN) r |= 1ull << 32;
    if (blockDim.x != 384) r |= 1ull << 33;
    if (a->bytes[0] != (uint32_t)a->iparam[0] || a->elem0 != 0) r |= 1ull << 34;
    if (!entry) r |= 1ull << 35;
    if (part >= nparts || bad) r |= 1ull << 36;
    if (threadIdx.x == 0 && a->flow[0] && (part + 1) * 4 <= a->bytes[0])
        static_cast<uint32_t*>(a->flow[0])[part] = (nparts << 16) | (part + 1);
    return r;
}

__device__ unsigned long long add(const pb2_body_args_t* a) {
    int* x = static_cast<int*>(a->flow[0]);
    const uint32_t n = a->bytes[0] / 4;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) x[i] += a->iparam[0];
    return 0;
}

__device__ __forceinline__ long long partial_sum(const void* flow, uint32_t bytes) {
    const int* x = static_cast<const int*>(flow);
    long long s = 0;
    for (uint32_t i = threadIdx.x; i < bytes / 4; i += blockDim.x) s += x[i];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    return s;
}

__device__ unsigned long long sum(const pb2_body_args_t* a) {
    __shared__ unsigned long long total;
    if (threadIdx.x == 0) total = 0;
    __syncthreads();
    const long long s = partial_sum(a->flow[0], a->bytes[0]);
    if ((threadIdx.x & 31) == 0 && s) atomicAdd(&total, (unsigned long long)s);
    __syncthreads();
    const unsigned long long r = total;
    __syncthreads();
    return r;
}

}  // namespace

extern "C" __device__ unsigned long long pb2_linked_gemm_body(int body, const pb2_body_args_t* a, unsigned int* scratch) {
    switch (body) {
    case DGEMM: return dgemm(a, scratch);
    case PART: return part_probe(a, scratch, true);
    default: return ~0ull;
    }
}

extern "C" __device__ unsigned long long pb2_linked_body(int body, const pb2_body_args_t* a, unsigned int* scratch) {
    switch (body) {
    case PART: return part_probe(a, scratch, false);
    case ADD: return add(a);
    case SUM: return sum(a);
    default: return ~0ull;          // DGEMM included: it needs more than the HBM kernels' 80 registers
    }
}

#ifdef GEMM_PART_READER_GROUP
extern "C" __device__ unsigned long long pb2_linked_reader_group(const pb2_reader_group_t* g, unsigned long long* results,
                                                                 unsigned int* scratch) {
    (void)scratch;
    const long long s = partial_sum(g->flow, g->bytes);
    if ((threadIdx.x & 31) == 0 && s)
        for (uint32_t m = 0; m < g->n; ++m) atomicAdd(&results[m], (unsigned long long)s);
    return 0;
}
#endif
