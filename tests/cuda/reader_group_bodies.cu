// The bodies of tests/cuda/reader_bodies.cu, with the group form of its readers (pb2_linked_reader_group,
// include/pb2_device_body.h), that tests/test_reader_groups_linked.py, tests/test_reader_groups_linked_gpu.py and
// tools/ab_linked_readers.py link with PB2_LINK_READER_GROUPS.  Built by the Makefile into reader_group_bodies.cubin
// (relocatable sm_90a) and reader_group_bodies.ptx.  The group form covers the readers COUNT_NE, SUM_I64, COUNT_GT and
// FAIL (which sets its member's result to ~0 and returns ~0); the producers FILL and AXPB are no readers, so they are
// declared in neither mask and run fused with a group through pb2_linked_body alone.  Integer arithmetic only, so a
// member's result of a chunk is the integer pb2_linked_body returns for it, and numpy reproduces every result.
#include "reader_bodies.cu"

namespace {

// COUNT_NE and COUNT_GT as one test: with u = v ^ 2^31 (the order of int32 as unsigned), member m counts an element
// when u - lo[m] > span[m] (unsigned): lo = k ^ 2^31, span 0 for COUNT_NE (u != lo); lo 0, span k ^ 2^31 for COUNT_GT
// (u > span); lo 0, span ~0 (never) for the others.  Every summing member (SUM_I64, and SUM_CTL as in pb2_linked_body)
// has the same result, so one 64-bit sum serves them all; the counts take 32 bits per thread.
struct Members { uint32_t lo[PB2_GROUP_MAX], span[PB2_GROUP_MAX]; uint32_t sum, fail; };

__device__ __forceinline__ void members_of(const pb2_reader_group_t* g, Members& c) {
    c.sum = c.fail = 0;
#pragma unroll
    for (int m = 0; m < PB2_GROUP_MAX; ++m) {
        const int b = m < (int)g->n ? g->body[m] : 0;
        const uint32_t k = (uint32_t)g->iparam[m][0] ^ 0x80000000u;
        c.lo[m] = b == COUNT_NE ? k : 0u;
        c.span[m] = b == COUNT_NE ? 0u : b == COUNT_GT ? k : ~0u;
        if (b == SUM_I64 || b == SUM_CTL) c.sum |= 1u << m;
        if (b == FAIL) c.fail |= 1u << m;
    }
}

// What every member counts or adds over the elements v[0 .. N), on the same loaded values.
template <int N>
__device__ __forceinline__ void add_elems(const Members& c, uint32_t (&cnt)[PB2_GROUP_MAX], long long& sum, const uint32_t* v) {
#pragma unroll
    for (int j = 0; j < N; ++j) {
        sum += (int32_t)v[j];
        const uint32_t u = v[j] ^ 0x80000000u;
#pragma unroll
        for (int m = 0; m < PB2_GROUP_MAX; ++m) cnt[m] += u - c.lo[m] > c.span[m] ? 1u : 0u;
    }
}

}  // namespace

extern "C" __device__ unsigned long long pb2_linked_reader_group(const pb2_reader_group_t* g, unsigned long long* results,
                                                                 unsigned int* scratch) {
    (void)scratch;
    Members c;
    members_of(g, c);
    uint32_t cnt[PB2_GROUP_MAX];
#pragma unroll
    for (int m = 0; m < PB2_GROUP_MAX; ++m) cnt[m] = 0;
    long long sum = 0;
    // one pass of 16-byte loads, two in flight per thread, then the whole elements past the last 16 bytes
    const uint4* q = static_cast<const uint4*>(g->flow);
    const uint32_t* e = static_cast<const uint32_t*>(g->flow);
    const uint32_t ne = g->bytes >> 2, nvec = ne >> 2, nt = blockDim.x;
    uint32_t i = threadIdx.x;
#pragma unroll 1
    for (; i + nt < nvec; i += 2 * nt) {
        const uint4 v0 = q[i], v1 = q[i + nt];
        const uint32_t v[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
        add_elems<8>(c, cnt, sum, v);
    }
    if (i < nvec) {
        const uint4 v0 = q[i];
        const uint32_t v[4] = {v0.x, v0.y, v0.z, v0.w};
        add_elems<4>(c, cnt, sum, v);
    }
#pragma unroll 1
    for (uint32_t j = (nvec << 2) + threadIdx.x; j < ne; j += nt) add_elems<1>(c, cnt, sum, &e[j]);
    // one warp reduction per counting member and one for the sum, one shared atomicAdd per member per warp
    const bool lead = (threadIdx.x & 31) == 0;
#pragma unroll
    for (int m = 0; m < PB2_GROUP_MAX; ++m) {
        if (c.span[m] == ~0u) continue;
        uint32_t n = cnt[m];
        for (int s = 16; s; s >>= 1) n += __shfl_xor_sync(0xffffffffu, n, s);
        if (lead && n) atomicAdd(&results[m], (unsigned long long)n);
    }
    if (c.sum) {
        for (int s = 16; s; s >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, s);
        if (lead && sum)
            for (int m = 0; m < PB2_GROUP_MAX; ++m)
                if ((c.sum >> m) & 1u) atomicAdd(&results[m], (unsigned long long)sum);
    }
    if (c.fail && threadIdx.x == 0)
        for (int m = 0; m < PB2_GROUP_MAX; ++m)
            if ((c.fail >> m) & 1u) results[m] = ~0ull;
    return c.fail ? ~0ull : 0ull;
}
