// Device bodies with a checked form (include/pb2_device_body.h, pb2_engine_link_bodies_checked) that the GPU tests
// (tests/test_checked_linked_gpu.py) and tools/ab_linked.py link into HBM engine windows.  Built by the Makefile into
// checked_bodies.cubin (relocatable sm_90a) and checked_bodies.ptx.  Integer arithmetic only (wrapping int32), so numpy
// reproduces every output bit for bit.  Both are sliceable and checked; each writes one flow.
//   PB2_BODY_LINKED_0  FILL  flow0[i] = iparam[0], the built-in FILL_I32 restated
//   PB2_BODY_LINKED_1  AXPB  flow1[i] = iparam[0] * flow0[i] + iparam[1]: an output that varies with its input
// In check mode every thread returns the OR of (element ^ k0) over the elements it stored: nonzero iff one differed.
#include <stdint.h>
#include "pb2_device_body.h"

enum { FILL = 20, AXPB = 21 };

static __device__ uint32_t fill(const pb2_body_check_t* c) {
    const pb2_body_args_t* a = &c->args;
    const uint32_t k = (uint32_t)a->iparam[0];
    const uint4 kv = make_uint4(k, k, k, k);
    uint4* q = static_cast<uint4*>(a->flow[0]);
    const uint32_t nvec = a->bytes[0] >> 4, nt = blockDim.x;
    uint32_t i = threadIdx.x;
    bool stored = i < nvec;
    for (; i + 3 * nt < nvec; i += 4 * nt) {
        __stcg(q + i, kv); __stcg(q + i + nt, kv); __stcg(q + i + 2 * nt, kv); __stcg(q + i + 3 * nt, kv);
    }
    for (; i < nvec; i += nt) __stcg(q + i, kv);
    uint32_t* e = static_cast<uint32_t*>(a->flow[0]);
    for (uint32_t j = (nvec << 2) + threadIdx.x; j < (a->bytes[0] >> 2); j += nt) { e[j] = k; stored = true; }
    return c->check && stored ? k ^ c->k0 : 0u;
}

static __device__ uint32_t axpb(const pb2_body_check_t* c) {
    const pb2_body_args_t* a = &c->args;
    const int32_t* x = static_cast<const int32_t*>(a->flow[0]);
    int32_t* y = static_cast<int32_t*>(a->flow[1]);
    const uint32_t n = (a->bytes[0] < a->bytes[1] ? a->bytes[0] : a->bytes[1]) >> 2;
    const uint32_t m = (uint32_t)a->iparam[0], b = (uint32_t)a->iparam[1], k0 = c->k0;
    uint32_t diff = 0;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        const uint32_t v = m * (uint32_t)__ldcg(x + i) + b;
        y[i] = (int32_t)v;
        diff |= v ^ k0;
    }
    return c->check ? diff : 0u;
}

extern "C" __device__ unsigned long long pb2_linked_body(int body, const pb2_body_args_t* a, unsigned int* scratch) {
    const pb2_body_check_t* c = (const pb2_body_check_t*)a;
    switch (body) {
    case FILL: return fill(c);
    case AXPB: return axpb(c);
    default: return 0;
    }
}
