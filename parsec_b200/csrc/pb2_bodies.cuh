// pb2_bodies.cuh -- HBM-bound task bodies run in place by the persistent engine kernel.
//
// Each body is executed by one whole CTA (the "worker") over one tile.  All payload
// accesses are 16-byte, fully coalesced, L1-bypassing (ld.global.cg / st.global.cg) with
// UNROLL independent requests in flight per thread (the checked form of a producer, run_hbm_body<true>, also compares
// every value it stores with a constant, and stores with an L2 evict-first policy); ragged tails (bytes % 16, bytes % 4)
// are handled by scalar epilogues so empty and odd-sized tiles are legal.
//
// Reference bodies these restate (the reference ships them as toy <<<1,1>>> kernels or CPU code):
//   examples/Ex05_Broadcast.jdf:33-39,53-57, examples/Ex02_Chain.jdf:44-50,
//   tests/runtime/cuda/ping_kernel.cu:13-21,
//   tests/dsl/dtd/dtd_test_new_tile_cuda_kernels.cu:14-56,
//   contrib/build_with_parsec/write_check.cu:7-35,
//   tests/runtime/cuda/get_best_device_check.jdf:82.
#pragma once
#include <stddef.h>
#include "pb2_dev_utils.cuh"
#include "../../include/pb2_device_body.h"

namespace pb2 {

#ifndef PB2_UNROLL
#define PB2_UNROLL 4
#endif
constexpr int kUnroll = PB2_UNROLL;

// What the checked form of a producer body (run_fused_part) does besides storing: every element it stores is compared
// with the group leader's constant k, and the stores carry the L2 evict-first policy `pol` (the group never reads the
// tile back).
struct Checked {
    uint32_t k;
    uint32_t diff;      // OR of (element ^ k) over the elements this thread stored: 0 iff all of them equal k
    uint64_t pol;
};

// f(uint4& v, uint32_t first_elem_index) ; elements are 4-byte lanes x,y,z,w, read from src (READ) and written to dst
// (WRITE) at the same offsets.  CHECKED: the stores go through ck (WRITE implied).  Tiles are below 4 GiB
// (pb2_tile_t::bytes is 32-bit), so all indices are 32-bit: half the address registers of a size_t loop.
template <bool READ, bool WRITE, bool CHECKED = false, class F>
__device__ __forceinline__ void cta_vec_loop(const void* src, void* dst, uint32_t bytes, F f, Checked* ck = nullptr) {
    const uint4* p = reinterpret_cast<const uint4*>(src);
    uint4* q = reinterpret_cast<uint4*>(dst);
    auto store = [&](uint32_t i, const uint4& v) {
        if (CHECKED) {
            ck->diff |= ((v.x ^ ck->k) | (v.y ^ ck->k)) | ((v.z ^ ck->k) | (v.w ^ ck->k));
            st_v4_policy(q + i, v, ck->pol);
        } else if (WRITE) st_stream(q + i, v);
    };
    const uint32_t nvec = bytes >> 4;
    const uint32_t tid = threadIdx.x, nt = blockDim.x;
    const uint32_t per_iter = nt * kUnroll;
    uint32_t base = 0;
    for (; base + per_iter <= nvec; base += per_iter) {
        uint4 v[kUnroll];
#pragma unroll
        for (int j = 0; j < kUnroll; ++j) {
            if (READ) v[j] = ld_stream(p + (base + j * nt + tid));
            else      v[j] = make_uint4(0, 0, 0, 0);
        }
#pragma unroll
        for (int j = 0; j < kUnroll; ++j) {
            f(v[j], (base + j * nt + tid) * 4u);
            store(base + j * nt + tid, v[j]);
        }
    }
    for (uint32_t i = base + tid; i < nvec; i += nt) {
        uint4 v = READ ? ld_stream(p + i) : make_uint4(0, 0, 0, 0);
        f(v, i * 4u);
        store(i, v);
    }
    // scalar 4-byte tail (bytes not a multiple of 16)
    const uint32_t nelem = bytes >> 2;
    const uint32_t* e = reinterpret_cast<const uint32_t*>(src);
    uint32_t* o = reinterpret_cast<uint32_t*>(dst);
    for (uint32_t i = (nvec << 2) + tid; i < nelem; i += nt) {
        uint4 v = make_uint4(READ ? __ldcg(e + i) : 0u, 0, 0, 0);
        // present the single element in lane x only; f must treat y,z,w as don't-care here (and the check ignores them)
        uint4 w = v;
        f(w, i);
        if (CHECKED) { ck->diff |= w.x ^ ck->k; st_u32_policy(o + i, w.x, ck->pol); }
        else if (WRITE) __stcg(o + i, w.x);
    }
}

// dst[:] = src[:] for arbitrary byte counts and alignments.  Tile slots are 16-byte aligned; a
// ragged collection in host memory (tile size not a multiple of 16) gives sources that are only
// 4-byte (or 1-byte) aligned, handled by the narrower paths.
// 'remote' source = host-pinned or peer memory (stage-in), else local HBM.
template <bool REMOTE_SRC>
__device__ __forceinline__ void cta_copy_simt(void* dst, const void* src, size_t bytes64) {
    // callers cut copies into pieces below 4 GiB (tiles are); 32-bit indices keep the register count down
    const uint32_t bytes = (uint32_t)bytes64;
    const uint32_t tid = threadIdx.x, nt = blockDim.x;
    const uintptr_t al = reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(src);
    uint32_t done = 0;
    if ((al & 15) == 0) {
        uint4* d = reinterpret_cast<uint4*>(dst);
        const uint4* s = reinterpret_cast<const uint4*>(src);
        const uint32_t nvec = bytes >> 4;
        constexpr int U = kUnroll;
        const uint32_t per_iter = nt * U;
        uint32_t base = 0;
        for (; base + per_iter <= nvec; base += per_iter) {
            uint4 v[U];
#pragma unroll
            for (int j = 0; j < U; ++j)
                v[j] = REMOTE_SRC ? ld_remote(s + base + j * nt + tid) : ld_stream(s + base + j * nt + tid);
#pragma unroll
            for (int j = 0; j < U; ++j) st_stream(d + base + j * nt + tid, v[j]);
        }
        for (uint32_t i = base + tid; i < nvec; i += nt)
            st_stream(d + i, REMOTE_SRC ? ld_remote(s + i) : ld_stream(s + i));
        done = nvec << 4;
    } else if ((al & 3) == 0) {
        uint32_t* d = reinterpret_cast<uint32_t*>(dst);
        const uint32_t* s = reinterpret_cast<const uint32_t*>(src);
        const uint32_t n = bytes >> 2;
        constexpr int U = 8;
        const uint32_t per_iter = nt * U;
        uint32_t base = 0;
        for (; base + per_iter <= n; base += per_iter) {
            uint32_t v[U];
#pragma unroll
            for (int j = 0; j < U; ++j) v[j] = __ldcg(s + base + j * nt + tid);
#pragma unroll
            for (int j = 0; j < U; ++j) __stcg(d + base + j * nt + tid, v[j]);
        }
        for (uint32_t i = base + tid; i < n; i += nt) __stcg(d + i, __ldcg(s + i));
        done = n << 2;
    }
    const unsigned char* sb = reinterpret_cast<const unsigned char*>(src);
    unsigned char* db = reinterpret_cast<unsigned char*>(dst);
    for (uint32_t i = done + tid; i < bytes; i += nt) db[i] = sb[i];
}

// The tile mover.  With a bulk ring (HBM-body kernels) the 16-byte aligned bulk of the copy goes through TMA
// (cp.async.bulk global -> shared -> global, see pb2_dev_utils.cuh) and only a ragged tail (< 16 bytes) or an
// unaligned pair of addresses takes the SIMT loops; without one (the GEMM kernels keep their shared memory for
// operand stages) everything is SIMT.  Ends with a CTA barrier in the bulk case.
template <bool REMOTE_SRC>
__device__ __forceinline__ void cta_copy(void* dst, const void* src, size_t bytes, BulkSmem* bulk = nullptr) {
    const uintptr_t al = reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(src);
    if (bulk != nullptr && (al & 15) == 0 && bytes >= 16) {
        const size_t body = bytes & ~(size_t)15;
        cta_bulk_copy(dst, src, body, *bulk);
        if (bytes != body)
            cta_copy_simt<REMOTE_SRC>(reinterpret_cast<uint8_t*>(dst) + body, reinterpret_cast<const uint8_t*>(src) + body, bytes - body);
        return;
    }
    cta_copy_simt<REMOTE_SRC>(dst, src, bytes);
}

#ifndef PB2_CHECK_UNROLL
#define PB2_CHECK_UNROLL 16
#endif
// OR over the slice of (element ^ k): zero iff every 4-byte element equals k.  Read-only, 16-byte loads,
// PB2_CHECK_UNROLL independent requests per thread in flight.
__device__ __forceinline__ uint32_t cta_xor_scan(const void* ptr, uint32_t bytes, uint32_t k) {
    const uint4* p = reinterpret_cast<const uint4*>(ptr);
    const uint32_t nvec = bytes >> 4, tid = threadIdx.x, nt = blockDim.x;
    constexpr uint32_t U = PB2_CHECK_UNROLL;
    uint32_t diff = 0, i = tid;
    for (; i + (U - 1) * nt < nvec; i += U * nt) {
        uint4 v[U];
#pragma unroll
        for (uint32_t j = 0; j < U; ++j) v[j] = ld_stream(p + i + j * nt);
#pragma unroll
        for (uint32_t j = 0; j < U; ++j) diff |= ((v[j].x ^ k) | (v[j].y ^ k)) | ((v[j].z ^ k) | (v[j].w ^ k));
    }
    for (; i < nvec; i += nt) {
        const uint4 v = ld_stream(p + i);
        diff |= ((v.x ^ k) | (v.y ^ k)) | ((v.z ^ k) | (v.w ^ k));
    }
    const uint32_t* e = reinterpret_cast<const uint32_t*>(ptr);
    for (uint32_t j = (nvec << 2) + tid; j < (bytes >> 2); j += nt) diff |= __ldcg(e + j) ^ k;
    return diff;
}

// Block-wide sum of a 32-bit count; result valid in thread 0.  smem: >= 32 uint32.
__device__ __forceinline__ uint32_t cta_reduce_sum(uint32_t v, uint32_t* smem) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) smem[warp] = v;
    __syncthreads();
    uint32_t r = 0;
    if (warp == 0) {
        r = (lane < (int)((blockDim.x + 31) >> 5)) ? smem[lane] : 0u;
        for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
    }
    __syncthreads();
    return r;
}

// The number of 4-byte elements of the slice that differ from k, counted exactly; result valid in thread 0.
__device__ __forceinline__ uint32_t cta_count_ne(const void* ptr, uint32_t bytes, uint32_t k, uint32_t* red_smem) {
    uint32_t bad = 0;
    const uint32_t nvec_elems = (bytes >> 4) << 2;
    cta_vec_loop<true, false>(ptr, nullptr, bytes, [&](uint4& v, uint32_t i) {
        if (i < nvec_elems) bad += (v.x != k) + (v.y != k) + (v.z != k) + (v.w != k);
        else                bad += (v.x != k);
    });
    return cta_reduce_sum(bad, red_smem);
}

struct BodyArgs {
    void*    flow[4];     // device pointers of this part's slice of the flows' tiles
    uint32_t bytes[4];    // bytes of the slice
    uint32_t elem0;       // index of the slice's first 4-byte element inside the tile (IOTA-style bodies)
    uint32_t part;        // part index (CHECK reports the tile's first element from part 0 only)
    int32_t  iparam[3];
    float    fparam;
};
// linked bodies (include/pb2_device_body.h) are handed TaskSmem::args as a pb2_body_args_t
static_assert(sizeof(BodyArgs) == sizeof(pb2_body_args_t) && alignof(BodyArgs) == alignof(pb2_body_args_t) &&
              offsetof(BodyArgs, bytes) == offsetof(pb2_body_args_t, bytes) &&
              offsetof(BodyArgs, elem0) == offsetof(pb2_body_args_t, elem0) &&
              offsetof(BodyArgs, part) == offsetof(pb2_body_args_t, part) &&
              offsetof(BodyArgs, iparam) == offsetof(pb2_body_args_t, iparam) &&
              offsetof(BodyArgs, fparam) == offsetof(pb2_body_args_t, fparam), "BodyArgs and pb2_body_args_t differ");

// Returns the body result (only meaningful in thread 0): CHECK -> (mismatches << 32) | first element bits.
// CHECKED: the checked form of a producer that runs with its read group as one unit (run_fused_part, pb2_hbm.cuh).  The
// body writes its output flow (flow 1 for COPY and AXPY, else flow 0) as the unchecked form does, through ck: each
// thread ORs (element ^ ck->k) of every whole 4-byte element it stores into ck->diff (a byte tail, MEMSET's or COPY's,
// is stored but not checked, as cta_xor_scan does not check it).  Bodies without a checked form (NOP, CHECK, ADD_AT)
// return ~0 there; form_read_groups (pb2_window_plan.cpp) fuses none of them.
template <bool CHECKED = false>
__device__ __forceinline__ uint64_t run_hbm_body(int body, const BodyArgs& a, uint32_t* red_smem, Checked* ck = nullptr) {
    switch (body) {
    case PB2_BODY_NOP:
        return CHECKED ? ~0ull : 0;
    case PB2_BODY_FILL_I32: {
        const uint32_t k = (uint32_t)a.iparam[0];
        cta_vec_loop<false, true, CHECKED>(a.flow[0], a.flow[0], a.bytes[0], [k](uint4& v, uint32_t) { v = make_uint4(k, k, k, k); }, ck);
        return 0;
    }
    case PB2_BODY_FILL_F32: {
        const uint32_t k = __float_as_uint(a.fparam);
        cta_vec_loop<false, true, CHECKED>(a.flow[0], a.flow[0], a.bytes[0], [k](uint4& v, uint32_t) { v = make_uint4(k, k, k, k); }, ck);
        return 0;
    }
    case PB2_BODY_MEMSET_U8: {
        const uint32_t b = (uint32_t)a.iparam[0] & 0xffu;
        const uint32_t k = b | (b << 8) | (b << 16) | (b << 24);
        cta_vec_loop<false, true, CHECKED>(a.flow[0], a.flow[0], a.bytes[0] & ~3u, [k](uint4& v, uint32_t) { v = make_uint4(k, k, k, k); }, ck);
        unsigned char* db = reinterpret_cast<unsigned char*>(a.flow[0]);
        for (size_t i = (a.bytes[0] & ~3u) + threadIdx.x; i < a.bytes[0]; i += blockDim.x) db[i] = (unsigned char)b;
        return 0;
    }
    case PB2_BODY_CHECK_I32:
    case PB2_BODY_CHECK_F32: {
        if (CHECKED) return ~0ull;
        const uint32_t k = (body == PB2_BODY_CHECK_I32) ? (uint32_t)a.iparam[0] : __float_as_uint(a.fparam);
        // Fast path: OR of (element ^ k) over the slice -- three LOP3 per 16 bytes, no predicates, no per-thread count.
        // A slice with a mismatch (the exception) is counted exactly by a second, slower pass.
        uint32_t total = 0;
        if (__syncthreads_or(cta_xor_scan(a.flow[0], a.bytes[0], k) != 0u)) total = cta_count_ne(a.flow[0], a.bytes[0], k, red_smem);
        uint32_t first = 0;
        if (threadIdx.x == 0 && a.part == 0 && a.bytes[0] >= 4) first = __ldcg(reinterpret_cast<const uint32_t*>(a.flow[0]));
        return ((uint64_t)total << 32) | first;
    }
    case PB2_BODY_INCR_I32: {
        const uint32_t k = (uint32_t)a.iparam[0];
        cta_vec_loop<true, true, CHECKED>(a.flow[0], a.flow[0], a.bytes[0], [k](uint4& v, uint32_t) { v.x += k; v.y += k; v.z += k; v.w += k; }, ck);
        return 0;
    }
    case PB2_BODY_SCALE_I32: {
        const int32_t k = a.iparam[0];
        cta_vec_loop<true, true, CHECKED>(a.flow[0], a.flow[0], a.bytes[0], [k](uint4& v, uint32_t) {
            v.x = (uint32_t)((int32_t)v.x * k); v.y = (uint32_t)((int32_t)v.y * k);
            v.z = (uint32_t)((int32_t)v.z * k); v.w = (uint32_t)((int32_t)v.w * k);
        }, ck);
        return 0;
    }
    case PB2_BODY_ADD_IOTA_I32: {
        const uint32_t e0 = a.elem0;
        cta_vec_loop<true, true, CHECKED>(a.flow[0], a.flow[0], a.bytes[0], [e0](uint4& v, uint32_t i) {
            const uint32_t j = e0 + i;
            v.x += j; v.y += j + 1; v.z += j + 2; v.w += j + 3;
        }, ck);
        return 0;
    }
    case PB2_BODY_IOTA_I32: {
        const uint32_t e0 = a.elem0;
        cta_vec_loop<false, true, CHECKED>(a.flow[0], a.flow[0], a.bytes[0], [e0](uint4& v, uint32_t i) {
            const uint32_t j = e0 + i;
            v = make_uint4(j, j + 1, j + 2, j + 3);
        }, ck);
        return 0;
    }
    case PB2_BODY_INCR_F32: {
        const float k = a.fparam;
        cta_vec_loop<true, true, CHECKED>(a.flow[0], a.flow[0], a.bytes[0], [k](uint4& v, uint32_t) {
            v.x = __float_as_uint(__uint_as_float(v.x) + k); v.y = __float_as_uint(__uint_as_float(v.y) + k);
            v.z = __float_as_uint(__uint_as_float(v.z) + k); v.w = __float_as_uint(__uint_as_float(v.w) + k);
        }, ck);
        return 0;
    }
    case PB2_BODY_ADD_AT_I32: {
        if (CHECKED) return ~0ull;
        const long long rel = (long long)a.iparam[0] - (long long)a.elem0;     // the element may live in another part
        if (threadIdx.x == 0 && rel >= 0 && (size_t)rel * 4 + 4 <= a.bytes[0]) {
            uint32_t* e = reinterpret_cast<uint32_t*>(a.flow[0]) + rel;
            __stcg(e, __ldcg(e) + (uint32_t)a.iparam[1]);
        }
        return 0;
    }
    case PB2_BODY_COPY: {
        const uint32_t n = a.bytes[0] < a.bytes[1] ? a.bytes[0] : a.bytes[1];
        if (!CHECKED) { cta_copy<false>(a.flow[1], a.flow[0], n); return 0; }
        // through registers, where the check sees the bytes (cta_copy's bulk path never has them there)
        cta_vec_loop<true, true, true>(a.flow[0], a.flow[1], n, [](uint4&, uint32_t) {}, ck);
        const unsigned char* sb = reinterpret_cast<const unsigned char*>(a.flow[0]);
        unsigned char* db = reinterpret_cast<unsigned char*>(a.flow[1]);
        for (uint32_t i = (n & ~3u) + threadIdx.x; i < n; i += blockDim.x) __stcg(db + i, __ldcg(sb + i));
        return 0;
    }
    case PB2_BODY_AXPY_F32: {
        const float k = a.fparam;
        const uint4* x = reinterpret_cast<const uint4*>(a.flow[0]);
        const uint32_t* xe = reinterpret_cast<const uint32_t*>(a.flow[0]);
        const uint32_t n = a.bytes[0] < a.bytes[1] ? a.bytes[0] : a.bytes[1];
        const uint32_t nvec_elems = (n >> 4) << 2;
        cta_vec_loop<true, true, CHECKED>(a.flow[1], a.flow[1], n, [&](uint4& v, uint32_t i) {
            if (i < nvec_elems) {
                const uint4 xv = ld_stream(x + (i >> 2));
                v.x = __float_as_uint(fmaf(k, __uint_as_float(xv.x), __uint_as_float(v.x)));
                v.y = __float_as_uint(fmaf(k, __uint_as_float(xv.y), __uint_as_float(v.y)));
                v.z = __float_as_uint(fmaf(k, __uint_as_float(xv.z), __uint_as_float(v.z)));
                v.w = __float_as_uint(fmaf(k, __uint_as_float(xv.w), __uint_as_float(v.w)));
            } else {
                v.x = __float_as_uint(fmaf(k, __uint_as_float(__ldcg(xe + i)), __uint_as_float(v.x)));
            }
        }, ck);
        return 0;
    }
    default:
        return ~0ull;
    }
}

}  // namespace pb2
