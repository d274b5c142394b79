// pb2_dev_utils.cuh -- small sm_90a device helpers shared by the engine kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pb2 {

__device__ __forceinline__ int32_t ld_acquire_gpu(const int32_t* p) {
    int32_t v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ int32_t ld_acquire_sys(const int32_t* p) {
    int32_t v;
    asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ int32_t ld_relaxed_sys(const int32_t* p) {
    int32_t v;
    asm volatile("ld.relaxed.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void fence_acq_rel_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }
__device__ __forceinline__ void st_release_sys(int32_t* p, int32_t v) {
    asm volatile("st.release.sys.global.s32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ int32_t ld_relaxed_gpu(const int32_t* p) {
    int32_t v;
    asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_gpu(int32_t* p, int32_t v) {
    asm volatile("st.release.gpu.global.s32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_gpu(int32_t* p, int32_t v) {
    asm volatile("st.relaxed.gpu.global.s32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
    uint64_t t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ uint32_t smid() {
    uint32_t r;
    asm volatile("mov.u32 %0, %smid;" : "=r"(r));
    return r;
}

// 16-byte streaming accesses that bypass L1: tile payloads are produced by other SMs inside the
// same kernel, so they must be read at L2 (the coherence point), and they are touched once.
__device__ __forceinline__ uint4 ld_stream(const uint4* p) { return __ldcg(p); }
__device__ __forceinline__ void  st_stream(uint4* p, const uint4& v) { __stcg(p, v); }

// Source may be cudaHostRegister'ed system memory or a peer GPU: plain coherent load, no L1 allocate.
__device__ __forceinline__ uint4 ld_remote(const uint4* p) {
    uint4 r;
    asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
    return r;
}

// Stores of bytes nobody is expected to read back soon (a fused unit's tile, checked on the SM before it is stored):
// with the policy of l2_evict_first() the lines they write are the first L2 evicts.
__device__ __forceinline__ uint64_t l2_evict_first() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void st_v4_policy(uint4* p, const uint4& v, uint64_t pol) {
    asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.u32 [%0], {%1,%2,%3,%4}, %5;"
                 :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_u32_policy(uint32_t* p, uint32_t v, uint64_t pol) {
    asm volatile("st.global.L1::no_allocate.L2::cache_hint.u32 [%0], %1, %2;" :: "l"(p), "r"(v), "l"(pol) : "memory");
}

__device__ __forceinline__ uint32_t lanemask_lt() {
    uint32_t m;
    asm volatile("mov.u32 %0, %lanemask_lt;" : "=r"(m));
    return m;
}

// ---------------------------------------------------------------------------------------------
// TMA bulk mover (cp.async.bulk, 1-D): global -> shared -> global through a kBulkDepth-deep shared-memory ring with
// mbarrier completion.  One elected thread drives the whole pipeline, so a copy costs no payload registers and
// keeps up to kBulkDepth x kBulkChunk bytes of LOADS in flight per CTA whatever the latency of the source (pinned host
// memory over PCIe, a peer GPU over NVLink, local HBM): what a link delivers is bytes in flight / round trip, and a
// 64-thread worker that pulls a tile is one of a few hundred CTAs doing so at any moment.  The store of chunk i and
// the reload of the slot of chunk i-1 overlap (wait_group.read 1), so depth-1 loads stay in flight all the time.
// Depth 3 x 4 KiB is the measured choice (r02, tools/r02_probe24.sh): the resident Ex05 window is unchanged against depth 2
// (0.617 / 0.620 ms), a window that pulls 0.22 GiB per rank from its neighbour goes from 0.958 to 0.879 ms (4 x 2 KiB:
// 0.918); a 4-deep ring of 4 KiB chunks (16 KiB per worker, 203 KiB per SM) leaves the SM 28 KiB of L1 and the resident
// window drops from 60 to 46 M tasks/s.
// Requires 16-byte aligned addresses and a byte count that is a multiple of 16; callers fall back to the SIMT loops
// of pb2_bodies.cuh otherwise.
// This is the device-side replacement of the cudaMemcpyAsync per flow in parsec_default_gpu_stage_in / _stage_out
// (parsec/mca/device/device_gpu.c:1623-1662, :1673-1724).
// ---------------------------------------------------------------------------------------------
#ifndef PB2_BULK_CHUNK
#define PB2_BULK_CHUNK 4096
#endif
#ifndef PB2_BULK_DEPTH
#define PB2_BULK_DEPTH 3
#endif
constexpr uint32_t kBulkChunk = PB2_BULK_CHUNK;
constexpr int kBulkDepth = PB2_BULK_DEPTH;
static_assert(kBulkDepth >= 2 && kBulkDepth <= 8, "bulk ring depth");

struct alignas(128) BulkSmem {
    uint8_t  buf[kBulkDepth][kBulkChunk];
    uint64_t bar[kBulkDepth];
    uint32_t parity;        // bit s: the phase barrier s will complete next (persists across copies; owned by thread 0)
};

__device__ __forceinline__ uint32_t smem_addr_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void bulk_init(BulkSmem& b) {     // thread 0, once per kernel, followed by a barrier
    for (int s = 0; s < kBulkDepth; ++s)
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_addr_u32(&b.bar[s])) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    b.parity = 0;
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_addr_u32(bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(smem_addr_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_addr_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                 :: "l"(gdst), "r"(smem_addr_u32(smem_src)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
// at most N bulk groups may still be reading their shared-memory source
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" :: "n"(N) : "memory"); }
__device__ __forceinline__ void bulk_wait_all0()  { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_bar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok = 0;
    while (!ok) {
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n"
                     : "=r"(ok) : "r"(smem_addr_u32(bar)), "r"(parity) : "memory");
    }
}

// Whole CTA calls (uniform arguments); thread 0 moves `bytes` (multiple of 16, both pointers 16-byte aligned).
// On return the bytes are written and ordered before a following __threadfence()/release by any thread of the CTA.
__device__ __forceinline__ void cta_bulk_copy(void* dst, const void* src, size_t bytes, BulkSmem& b) {
    if (threadIdx.x == 0 && bytes) {
        const uint8_t* s = reinterpret_cast<const uint8_t*>(src);
        uint8_t* d = reinterpret_cast<uint8_t*>(dst);
        const size_t n = (bytes + kBulkChunk - 1) / kBulkChunk;
        uint32_t par = b.parity;
        // the source may have been written by generic-proxy stores a barrier ago (a body's output that is pushed out)
        asm volatile("fence.proxy.async;" ::: "memory");
        size_t issued = 0;                               // chunks whose load has been issued; chunk c uses slot c % depth
        for (; issued < n && issued < (size_t)kBulkDepth; ++issued) {
            const size_t off = issued * kBulkChunk;
            bulk_g2s(b.buf[issued], s + off, (uint32_t)(bytes - off < kBulkChunk ? bytes - off : kBulkChunk), &b.bar[issued]);
        }
        for (size_t i = 0; i < n; ++i) {
            const int slot = (int)(i % kBulkDepth);
            bulk_bar_wait(&b.bar[slot], (par >> slot) & 1u); par ^= (1u << slot);
            const size_t off = i * kBulkChunk;
            bulk_s2g(d + off, b.buf[slot], (uint32_t)(bytes - off < kBulkChunk ? bytes - off : kBulkChunk));
            if (i >= 1 && issued < n) {
                // the slot of chunk i-1: its store is the second most recent group, and it has finished READING the
                // buffer once at most one group (the store just issued) still has reads pending
                bulk_wait_read<1>();
                const int fs = (int)((i - 1) % kBulkDepth);           // == issued % depth
                const size_t noff = issued * kBulkChunk;
                bulk_g2s(b.buf[fs], s + noff, (uint32_t)(bytes - noff < kBulkChunk ? bytes - noff : kBulkChunk), &b.bar[fs]);
                ++issued;
            }
        }
        bulk_wait_all0();
        asm volatile("fence.proxy.async;" ::: "memory");
        b.parity = par;
    }
    __syncthreads();
}

}  // namespace pb2
