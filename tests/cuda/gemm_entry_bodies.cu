// GEMM-worker bodies behind their own entry point, pb2_linked_gemm_body (PB2_LINK_GEMM_BODY_ENTRY), that the GPU tests
// (tests/test_gemm_body_entry_gpu.py) and tools/ab_gemm_body_entry.py link into GEMM engine windows.  Application code,
// not part of the library.  Only the GEMM window kernels call pb2_linked_gemm_body, so it has their budget of 168
// registers per thread (PB2_GEMM_BODY_MAX_REGS); pb2_linked_body is linked into the HBM window kernels as well and has
// to fit their 80.  Built by the Makefile with -maxrregcount=168 into gemm_entry_bodies.cubin (relocatable sm_90a) and
// .ptx, and with -DGEMM_ENTRY_READER_GROUP, which adds the group form of SUM (pb2_linked_reader_group), into
// gemm_entry_group_bodies.cubin.
//   PB2_BODY_LINKED_0  DGEMM  C (M x N, row-major fp64) += A (M x K, row-major) * B (N x K, row-major)^T on the FP64
//                             tensor cores; flows A, B, C; iparam = M, N, K.  The DGEMM of gemm_worker_bodies.cu with
//                             32 x 32 of C per warp instead of 32 x 16, and the same k order (see below).  Through
//                             pb2_linked_gemm_body only: pb2_linked_body returns ~0 for it.
//   PB2_BODY_LINKED_1  PROBE  the ring probe of gemm_worker_bodies.cu through either entry point; its result has bit 35
//                             set when it was reached through pb2_linked_body.
//   PB2_BODY_LINKED_2  ADD    flow 0 (int32) += iparam[0], element-wise; sliceable; result 0.
//   PB2_BODY_LINKED_3  SUM    reader: the sum of flow 0's int32 elements, as a 64-bit integer modulo 2^64.
#include <stdint.h>
#include "pb2_device_body.h"

enum { DGEMM = 20, PROBE = 21, ADD = 22, SUM = 23 };

namespace {

// DGEMM blocking: C blocks of BM x BN, one per pass of the CTA, 12 warps as 4 x 3 of 32 x 32 each (2 x 4 tiles of
// mma.m16n8k8 fp64: 64 accumulator registers, with room for one k-step's fragments, 16 more, within 168).  K advances BK
// at a time through NST ring stages; each stage holds A[BM][LD] and B[BN][LD] with rows padded to LD doubles, so the
// fragment loads of a half-warp (rows g = 0..3, columns t = 0..3) hit 16 different 8-byte bank pairs.  BK is that of
// gemm_worker_bodies.cu: every C element then gets the same DMMA sequence, from zero, in the same k steps of 8 (the
// zero padding past K included), and the same final C += acc, so both fixtures give the same bits.
constexpr int BM = 128, BN = 96, BK = 16, LD = BK + 4, NST = 5, WM = 32, WN = 32;
constexpr int kStageDoubles = (BM + BN) * LD;
static_assert(NST * kStageDoubles * 8 <= PB2_GEMM_BODY_SMEM_BYTES, "the stages fit in the operand ring");
static_assert((BM / WM) * (BN / WN) == 12, "one 32 x 32 block of C per warp of the 384-thread worker");

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// scratch reaches the body as a generic pointer: shared-window addresses make the loads and stores LDS / STS
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

// Stage `st` <- k-columns k0 .. k0 + BK - 1 of rows m0.. of A and n0.. of B, zeros outside the matrices.  VEC (K even:
// every row starts 16-byte aligned) copies 16-byte pairs with cp.async, bypassing L1, and leaves them in flight;
// otherwise the doubles are loaded from L2 and stored one by one.
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

template <bool VEC>
__device__ void dgemm_tile(const pb2_body_args_t* a, uint32_t ring, int M, int N, int K) {
    const double* A = static_cast<const double*>(a->flow[0]);
    const double* B = static_cast<const double*>(a->flow[1]);
    double* C = static_cast<double*>(a->flow[2]);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int wm = (warp / (BN / WN)) * WM, wn = (warp % (BN / WN)) * WN;
    const int mblocks = (M + BM - 1) / BM, nblocks = (N + BN - 1) / BN, nk = (K + BK - 1) / BK;
#pragma unroll 1
    for (int blk = 0; blk < mblocks * nblocks; ++blk) {
        const int m0 = (blk % mblocks) * BM, n0 = (blk / mblocks) * BN;
        // a warp whose 32 x 32 lies wholly past M or N (the last block of a ragged edge) stages and waits, but leaves
        // the tensor cores to the others
        const bool live = m0 + wm < M && n0 + wn < N;
        double acc[2][4][4];
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int v = 0; v < 4; ++v) acc[i][j][v] = 0.0;
        // prologue: NST - 1 stages in flight (one commit group each, empty past the last k-block)
#pragma unroll 1
        for (int s = 0; s < NST - 1; ++s) {
            if (s < nk) load_stage<VEC>(ring + s * kStageDoubles * 8, A, B, M, N, K, m0, n0, s * BK);
            asm volatile("cp.async.commit_group;" ::: "memory");
        }
#pragma unroll 1
        for (int kb = 0; kb < nk; ++kb) {
            asm volatile("cp.async.wait_group %0;" :: "n"(NST - 2) : "memory");
            __syncthreads();        // stage kb % NST is complete for every thread; stage (kb - 1) % NST is free again
            const int nxt = kb + NST - 1;
            if (nxt < nk) load_stage<VEC>(ring + (nxt % NST) * kStageDoubles * 8, A, B, M, N, K, m0, n0, nxt * BK);
            asm volatile("cp.async.commit_group;" ::: "memory");
            if (!live) continue;
            const uint32_t As = ring + (uint32_t)((kb % NST) * kStageDoubles + (wm + g) * LD + t) * 8u;
            const uint32_t Bs = ring + (uint32_t)((kb % NST) * kStageDoubles + (BM + wn + g) * LD + t) * 8u;
#pragma unroll
            for (int kk = 0; kk < BK; kk += 8) {
                // all fragments of the k-step (16 doubles), then the 8 DMMAs: each A fragment feeds four, each B two
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
        __syncthreads();            // the ring is reused by the next block
        if (!live) continue;
        // C += acc: c0, c1 at (row g, columns 2t, 2t + 1) of each 16 x 8 tile, c2, c3 eight rows below.  C goes through
        // L2: an earlier task of the chain may have written it on another SM.
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
    if (M <= 0 || N <= 0 || K <= 0 || !a->flow[0] || !a->flow[1] || !a->flow[2] ||
        (uint64_t)M * K * 8 > a->bytes[0] || (uint64_t)N * K * 8 > a->bytes[1] || (uint64_t)M * N * 8 > a->bytes[2])
        return ~0ull;
    const uint32_t ring = smem_u32(scratch);
    if (K % 2 == 0) dgemm_tile<true>(a, ring, M, N, K);
    else dgemm_tile<false>(a, ring, M, N, K);
    return 0;
}

__device__ __forceinline__ uint32_t pattern(uint32_t i, uint32_t key) {
    uint32_t x = (i + 1u) * 0x9E3779B1u ^ key;
    x ^= x >> 15; x *= 0x85EBCA77u; x ^= x >> 13;
    return x;
}

// The ring probe of gemm_worker_bodies.cu: the mismatch count of a pattern written over the whole ring and read back
// by other warps, with bit 32 set when scratch is not 1024-byte aligned, bit 33 when blockDim.x is not 384, bit 34
// when scratch is not shared memory, and bit 35 when it was not reached through pb2_linked_gemm_body.
__device__ unsigned long long probe(const pb2_body_args_t* a, unsigned int* ring, bool entry) {
    const uint32_t n = PB2_GEMM_BODY_SMEM_BYTES / 4;
    const uint32_t key = (uint32_t)a->iparam[0] * 0x2545F491u + (uint32_t)a->iparam[1] * 0x61C88647u + (uint32_t)a->iparam[2];
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) ring[i] = pattern(i, key);
    __syncthreads();
    uint32_t bad = 0;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) bad += ring[n - 1 - i] != pattern(n - 1 - i, key);   // another warp's words
    for (int o = 16; o > 0; o >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, o);
    __syncthreads();
    if (threadIdx.x == 0) ring[0] = 0;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) atomicAdd(&ring[0], bad);
    __syncthreads();
    unsigned long long r = ring[0];
    if (!__isShared(ring)) r |= 1ull << 34;
    else if (smem_u32(ring) % PB2_GEMM_BODY_SMEM_ALIGN) r |= 1ull << 32;
    if (blockDim.x != 384) r |= 1ull << 33;
    if (!entry) r |= 1ull << 35;
    return r;
}

__device__ unsigned long long add(const pb2_body_args_t* a) {
    int* x = static_cast<int*>(a->flow[0]);
    const uint32_t n = a->bytes[0] / 4;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) x[i] += a->iparam[0];
    return 0;
}

// The int32 elements of flow .. flow + bytes, summed per thread as 64-bit integers.
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
    __syncthreads();                // total is free again for the next call
    return r;
}

}  // namespace

extern "C" __device__ unsigned long long pb2_linked_gemm_body(int body, const pb2_body_args_t* a, unsigned int* scratch) {
    switch (body) {
    case DGEMM: return dgemm(a, scratch);
    case PROBE: return probe(a, scratch, true);
    default: return ~0ull;
    }
}

extern "C" __device__ unsigned long long pb2_linked_body(int body, const pb2_body_args_t* a, unsigned int* scratch) {
    switch (body) {
    case PROBE: return probe(a, scratch, false);
    case ADD: return add(a);
    case SUM: return sum(a);
    default: return ~0ull;          // DGEMM included: it needs more than the HBM kernels' 80 registers
    }
}

#ifdef GEMM_ENTRY_READER_GROUP
// Every member of a call is a SUM (the only reader declared with the group form): one pass, one sum for all.
extern "C" __device__ unsigned long long pb2_linked_reader_group(const pb2_reader_group_t* g, unsigned long long* results,
                                                                 unsigned int* scratch) {
    (void)scratch;
    const long long s = partial_sum(g->flow, g->bytes);
    if ((threadIdx.x & 31) == 0 && s)
        for (uint32_t m = 0; m < g->n; ++m) atomicAdd(&results[m], (unsigned long long)s);
    return 0;
}
#endif
