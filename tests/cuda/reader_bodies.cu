// Device bodies for linked readers (include/pb2_device_body.h, PB2_LINK_READERS) that the tests
// (tests/test_linked_readers.py, tests/test_linked_readers_gpu.py) and tools/ab_linked_readers.py link into engine
// windows.  Built by the Makefile into reader_bodies.cubin (relocatable sm_90a) and reader_bodies.ptx.  Integer
// arithmetic only (wrapping int32, sums modulo 2^64), so numpy reproduces every result bit for bit.  All are sliceable.
//   PB2_BODY_LINKED_0  COUNT_NE  reader: the elements of flow0 that differ from iparam[0] (the built-in CHECK's count)
//   PB2_BODY_LINKED_1  SUM_I64   reader: the sum of the int32 elements of flow0, as a 64-bit value
//   PB2_BODY_LINKED_2  COUNT_GT  reader: the elements of flow0 greater than iparam[0]
//   PB2_BODY_LINKED_3  AXPB      producer: flow1[i] = iparam[0] * flow0[i] + iparam[1], result 0
//   PB2_BODY_LINKED_4  FILL      producer: flow0[i] = iparam[0], result 0
//   PB2_BODY_LINKED_5  SUM_CTL   SUM_I64 for a body that is not declared a reader: a task keeps part 0's result
//   PB2_BODY_LINKED_6  FAIL      reader that returns ~0 (a bad body)
// Only the whole 4-byte elements of a slice count; the loads are plain loads, which L1 may serve.
#include <stdint.h>
#include "pb2_device_body.h"

enum { COUNT_NE = 20, SUM_I64, COUNT_GT, AXPB, FILL, SUM_CTL, FAIL };

// The sum over the CTA of op(element) over flow0's whole elements; thread 0 has it.  scratch: two words per warp.
template <class Op>
static __device__ unsigned long long reduce_i32(const pb2_body_args_t* a, unsigned int* scratch, Op op) {
    const uint4* q = static_cast<const uint4*>(a->flow[0]);
    const int32_t* e = static_cast<const int32_t*>(a->flow[0]);
    const uint32_t n = a->bytes[0] >> 2, nvec = n >> 2, nt = blockDim.x;
    unsigned long long acc = 0;
    uint32_t i = threadIdx.x;
    for (; i + 3 * nt < nvec; i += 4 * nt) {
        const uint4 v0 = q[i], v1 = q[i + nt], v2 = q[i + 2 * nt], v3 = q[i + 3 * nt];
        acc += op(v0.x) + op(v0.y) + op(v0.z) + op(v0.w) + op(v1.x) + op(v1.y) + op(v1.z) + op(v1.w);
        acc += op(v2.x) + op(v2.y) + op(v2.z) + op(v2.w) + op(v3.x) + op(v3.y) + op(v3.z) + op(v3.w);
    }
    for (; i < nvec; i += nt) { const uint4 v = q[i]; acc += op(v.x) + op(v.y) + op(v.z) + op(v.w); }
    for (uint32_t j = (nvec << 2) + threadIdx.x; j < n; j += nt) acc += op((uint32_t)e[j]);
    for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    const uint32_t warp = threadIdx.x >> 5, nw = (nt + 31) >> 5;
    if ((threadIdx.x & 31) == 0) { scratch[2 * warp] = (uint32_t)acc; scratch[2 * warp + 1] = (uint32_t)(acc >> 32); }
    __syncthreads();
    unsigned long long r = 0;
    if (threadIdx.x == 0)
        for (uint32_t w = 0; w < nw; ++w) r += scratch[2 * w] | ((unsigned long long)scratch[2 * w + 1] << 32);
    __syncthreads();
    return r;
}

static __device__ void fill(const pb2_body_args_t* a) {
    const uint32_t k = (uint32_t)a->iparam[0];
    uint32_t* y = static_cast<uint32_t*>(a->flow[0]);
    for (uint32_t i = threadIdx.x; i < (a->bytes[0] >> 2); i += blockDim.x) y[i] = k;
}

static __device__ void axpb(const pb2_body_args_t* a) {
    const int32_t* x = static_cast<const int32_t*>(a->flow[0]);
    int32_t* y = static_cast<int32_t*>(a->flow[1]);
    const uint32_t n = (a->bytes[0] < a->bytes[1] ? a->bytes[0] : a->bytes[1]) >> 2;
    const uint32_t m = (uint32_t)a->iparam[0], b = (uint32_t)a->iparam[1];
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) y[i] = (int32_t)(m * (uint32_t)x[i] + b);
}

extern "C" __device__ unsigned long long pb2_linked_body(int body, const pb2_body_args_t* a, unsigned int* scratch) {
    const uint32_t k = (uint32_t)a->iparam[0];
    switch (body) {
    case COUNT_NE: return reduce_i32(a, scratch, [k](uint32_t v) { return (unsigned long long)(v != k); });
    case COUNT_GT: return reduce_i32(a, scratch, [k](uint32_t v) { return (unsigned long long)((int32_t)v > (int32_t)k); });
    case SUM_I64:
    case SUM_CTL: return reduce_i32(a, scratch, [](uint32_t v) { return (unsigned long long)(long long)(int32_t)v; });
    case AXPB: axpb(a); return 0;
    case FILL: fill(a); return 0;
    case FAIL: return ~0ull;
    default: return 0;
    }
}
