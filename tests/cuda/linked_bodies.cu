// Device bodies the GPU tests (tests/test_linked_bodies_gpu.py) and tools/ab_linked.py link into HBM engine windows
// (pb2_engine_link_bodies).  Built by the Makefile into linked_bodies.cubin (relocatable sm_90a) and linked_bodies.ptx.
// Integer arithmetic only (wrapping int32), so numpy reproduces every output bit for bit.
//   PB2_BODY_LINKED_0  AXPB     flow1[i] = iparam[0] * flow0[i] + iparam[1]                    (sliceable)
//   PB2_BODY_LINKED_1  STENCIL  flow3[i] = iparam[0] * c[i-1] + iparam[1] * c[i] + iparam[2] * c[i+1] over the
//                               centre tile c = flow1, c[-1] = last element of flow0, c[n] = first element of flow2
//                               (0 where that flow has no tile)                                (whole tiles)
//   PB2_BODY_LINKED_2  SUM      result = sum of the int32 elements of flow0 modulo 2^32        (sliceable)
//   PB2_BODY_LINKED_3  FILL     flow0[:] = iparam[0], the built-in FILL_I32 restated            (sliceable)
#include <stdint.h>
#include "pb2_device_body.h"

enum { AXPB = 20, STENCIL = 21, SUM = 22, FILL = 23 };

static __device__ void axpb(const pb2_body_args_t* a) {
    const int32_t* x = static_cast<const int32_t*>(a->flow[0]);
    int32_t* y = static_cast<int32_t*>(a->flow[1]);
    const uint32_t n = (a->bytes[0] < a->bytes[1] ? a->bytes[0] : a->bytes[1]) >> 2;
    const uint32_t m = (uint32_t)a->iparam[0], b = (uint32_t)a->iparam[1];
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) y[i] = (int32_t)(m * (uint32_t)__ldcg(x + i) + b);
}

static __device__ void stencil(const pb2_body_args_t* a) {
    const int32_t* l = static_cast<const int32_t*>(a->flow[0]);
    const int32_t* c = static_cast<const int32_t*>(a->flow[1]);
    const int32_t* r = static_cast<const int32_t*>(a->flow[2]);
    int32_t* o = static_cast<int32_t*>(a->flow[3]);
    const uint32_t n = a->bytes[1] >> 2;
    const uint32_t wl = (uint32_t)a->iparam[0], wc = (uint32_t)a->iparam[1], wr = (uint32_t)a->iparam[2];
    const uint32_t left = (l && a->bytes[0] >= 4) ? (uint32_t)__ldcg(l + (a->bytes[0] >> 2) - 1) : 0u;
    const uint32_t right = (r && a->bytes[2] >= 4) ? (uint32_t)__ldcg(r) : 0u;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        const uint32_t p = i == 0 ? left : (uint32_t)__ldcg(c + i - 1);
        const uint32_t q = i == n - 1 ? right : (uint32_t)__ldcg(c + i + 1);
        o[i] = (int32_t)(wl * p + wc * (uint32_t)__ldcg(c + i) + wr * q);
    }
}

// the CTA's sum through scratch: one word per warp, then warp 0 adds them
static __device__ unsigned long long sum(const pb2_body_args_t* a, unsigned int* scratch) {
    const uint32_t* x = static_cast<const uint32_t*>(a->flow[0]);
    const uint32_t n = a->bytes[0] >> 2;
    uint32_t v = 0;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) v += __ldcg(x + i);
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
    __syncthreads();
    uint32_t t = 0;
    if (threadIdx.x == 0)
        for (uint32_t w = 0; w < (blockDim.x + 31) / 32; ++w) t += scratch[w];
    __syncthreads();
    return t;
}

static __device__ void fill(const pb2_body_args_t* a) {
    const uint32_t k = (uint32_t)a->iparam[0];
    const uint4 kv = make_uint4(k, k, k, k);
    uint4* q = static_cast<uint4*>(a->flow[0]);
    const uint32_t nvec = a->bytes[0] >> 4, nt = blockDim.x;
    uint32_t i = threadIdx.x;
    for (; i + 3 * nt < nvec; i += 4 * nt) {
        __stcg(q + i, kv); __stcg(q + i + nt, kv); __stcg(q + i + 2 * nt, kv); __stcg(q + i + 3 * nt, kv);
    }
    for (; i < nvec; i += nt) __stcg(q + i, kv);
    uint32_t* e = static_cast<uint32_t*>(a->flow[0]);
    for (uint32_t j = (nvec << 2) + threadIdx.x; j < (a->bytes[0] >> 2); j += nt) e[j] = k;
}

extern "C" __device__ unsigned long long pb2_linked_body(int body, const pb2_body_args_t* a, unsigned int* scratch) {
    switch (body) {
    case AXPB: axpb(a); return 0;
    case STENCIL: stencil(a); return 0;
    case SUM: return sum(a, scratch);
    case FILL: fill(a); return 0;
    default: return 0;
    }
}
