// l2_probe.cu -- measures, on the box it runs on, the two ceilings the Ex05 window kernel can hit:
//   (1) L2 (LTS) throughput: every SM streams a buffer that fits in L2 (ld.global.cg 16 B, 4 in flight per thread);
//   (2) the Ex05 mix: one tile write followed by F reads of the same tile, tiles > L2 in total.
// Prints one JSON line.  Development aid behind MEASURED numbers quoted in DESIGN.md; not part of the product path.
// With --compressible, a second line: 1 GiB written with a constant and with random words, on cudaMalloc memory and on
// compressible memory (cuMemCreate with CU_MEM_ALLOCATION_COMP_GENERIC, fetched through the runtime: no -lcuda).
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdint.h>
#include <string.h>

__global__ void __launch_bounds__(256) read_kernel(const uint4* __restrict__ p, size_t nvec, int reps, unsigned long long* sink) {
    uint4 acc = make_uint4(0, 0, 0, 0);
    const size_t gsz = (size_t)gridDim.x * blockDim.x;
    for (int r = 0; r < reps; ++r)
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i + 3 * gsz < nvec; i += 4 * gsz) {
            uint4 a = __ldcg(p + i), b = __ldcg(p + i + gsz), c = __ldcg(p + i + 2 * gsz), d = __ldcg(p + i + 3 * gsz);
            acc.x ^= a.x ^ b.x ^ c.x ^ d.x; acc.y ^= a.y ^ b.y ^ c.y ^ d.y;
        }
    if (acc.x == 0x12345678u && acc.y == 0x9abcdef0u) *sink = acc.x;
}
__global__ void __launch_bounds__(256) write_kernel(uint4* __restrict__ p, size_t nvec, uint32_t v) {
    const size_t gsz = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += gsz) __stcg(p + i, make_uint4(v, v, v, v));
}
__global__ void __launch_bounds__(256) write_random_kernel(uint4* __restrict__ p, size_t nvec, uint32_t seed) {
    const size_t gsz = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += gsz) {
        uint32_t h = (uint32_t)i * 2654435761u ^ seed;          // a few multiply-xorshift rounds per word: no run repeats
        uint32_t w[4];
        for (int k = 0; k < 4; ++k) { h ^= h >> 15; h *= 0x2c1b3c6du; h ^= h >> 12; h *= 0x297a2d39u; h ^= h >> 15; w[k] = h; }
        __stcg(p + i, make_uint4(w[0], w[1], w[2], w[3]));
    }
}

// bytes of compressible memory on device 0, or nullptr (*granted tells whether the driver granted compression).
static void* compressible_malloc(size_t bytes, int* granted) {
    void* fn[7] = {};
    const char* names[7] = {"cuMemCreate", "cuMemGetAllocationPropertiesFromHandle", "cuMemAddressReserve", "cuMemMap",
                            "cuMemSetAccess", "cuDeviceGetAttribute", "cuMemGetAllocationGranularity"};
    cudaDriverEntryPointQueryResult q;
    for (int i = 0; i < 7; ++i)
        if (cudaGetDriverEntryPoint(names[i], &fn[i], cudaEnableDefault, &q) != cudaSuccess || !fn[i]) return nullptr;
    CUmemAllocationProp prop;
    memset(&prop, 0, sizeof prop);
    prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    prop.location.id = 0;
    prop.allocFlags.compressionType = CU_MEM_ALLOCATION_COMP_GENERIC;
    size_t g = 0;
    if (((decltype(&cuMemGetAllocationGranularity))fn[6])(&g, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM) != CUDA_SUCCESS) return nullptr;
    bytes = (bytes + g - 1) / g * g;
    CUmemGenericAllocationHandle h;
    if (((decltype(&cuMemCreate))fn[0])(&h, bytes, &prop, 0) != CUDA_SUCCESS) return nullptr;
    CUmemAllocationProp got;
    memset(&got, 0, sizeof got);
    ((decltype(&cuMemGetAllocationPropertiesFromHandle))fn[1])(&got, h);
    *granted = got.allocFlags.compressionType == CU_MEM_ALLOCATION_COMP_GENERIC;
    CUdeviceptr ptr = 0;
    if (((decltype(&cuMemAddressReserve))fn[2])(&ptr, bytes, g, 0, 0) != CUDA_SUCCESS) return nullptr;
    if (((decltype(&cuMemMap))fn[3])(ptr, bytes, 0, h, 0) != CUDA_SUCCESS) return nullptr;
    CUmemAccessDesc a;
    memset(&a, 0, sizeof a);
    a.location = prop.location;
    a.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    if (((decltype(&cuMemSetAccess))fn[4])(ptr, bytes, &a, 1) != CUDA_SUCCESS) return nullptr;
    return (void*)ptr;                 // the probe's process ends here: it is never unmapped
}

// Best of 5 writes of 1 GiB at grid: a constant (random = 0) or random words, in GB/s of bytes written.
static double write_gbs(uint4* p, size_t big, int grid, int random) {
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    float best = 1e30f;
    for (int it = 0; it < 6; ++it) {               // the first round only warms up
        cudaEventRecord(e0);
        if (random) write_random_kernel<<<grid, 256>>>(p, big / 16, 0x9e3779b9u * (it + 1));
        else write_kernel<<<grid, 256>>>(p, big / 16, it);
        cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        if (it && ms < best) best = ms;
    }
    return (double)big / best / 1e6;
}

static int compressible_probe(int grid) {
    const size_t big = 1ull << 30;
    int attr = 0, granted = 0;
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuDeviceGetAttribute", &fn, cudaEnableDefault, &q) == cudaSuccess && fn)
        ((decltype(&cuDeviceGetAttribute))fn)(&attr, CU_DEVICE_ATTRIBUTE_GENERIC_COMPRESSION_SUPPORTED, 0);
    uint4* plain = nullptr;
    cudaMalloc(&plain, big);
    uint4* comp = attr ? (uint4*)compressible_malloc(big, &granted) : nullptr;
    printf("{\"probe\": \"compressible\", \"generic_compression_supported\": %d, \"granted\": %d, "
           "\"plain_const_write_gbs\": %.1f, \"plain_random_write_gbs\": %.1f",
           attr, granted, write_gbs(plain, big, grid, 0), write_gbs(plain, big, grid, 1));
    if (comp) printf(", \"compressible_const_write_gbs\": %.1f, \"compressible_random_write_gbs\": %.1f",
                     write_gbs(comp, big, grid, 0), write_gbs(comp, big, grid, 1));
    printf(", \"bytes\": %zu, \"error\": \"%s\"}\n", big, cudaGetErrorString(cudaGetLastError()));
    return 0;
}

int main(int argc, char** argv) {
    cudaDeviceProp prop; cudaGetDeviceProperties(&prop, 0);
    int clk_khz = 0; cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
    const size_t small = 48ull << 20, big = 1ull << 30;
    uint4 *a, *b; unsigned long long* sink;
    cudaMalloc(&a, small); cudaMalloc(&b, big); cudaMalloc(&sink, 8);
    cudaMemset(a, 1, small); cudaMemset(b, 1, big);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    const int grid = prop.multiProcessorCount * 8;
    float best_l2 = 1e30f, best_dram = 1e30f, best_copy = 1e30f;
    const int reps = 20;
    for (int it = 0; it < 5; ++it) {
        read_kernel<<<grid, 256>>>(a, small / 16, 2, sink);            // warm L2
        cudaEventRecord(e0); read_kernel<<<grid, 256>>>(a, small / 16, reps, sink); cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1); if (ms < best_l2) best_l2 = ms;
        cudaEventRecord(e0); read_kernel<<<grid, 256>>>(b, big / 16, 1, sink); cudaEventRecord(e1); cudaEventSynchronize(e1);
        cudaEventElapsedTime(&ms, e0, e1); if (ms < best_dram) best_dram = ms;
        cudaEventRecord(e0); write_kernel<<<grid, 256>>>(b, big / 16, it); cudaEventRecord(e1); cudaEventSynchronize(e1);
        cudaEventElapsedTime(&ms, e0, e1); if (ms < best_copy) best_copy = ms;
    }
    const double l2_gbs = (double)small * reps / best_l2 / 1e6, dram_gbs = (double)big / best_dram / 1e6, wr_gbs = (double)big / best_copy / 1e6;
    printf("{\"probe\": \"l2\", \"sms\": %d, \"sm_clock_mhz_attr\": %d, \"l2_read_gbs\": %.1f, \"l2_bytes_per_clk_at_attr_clock\": %.0f, "
           "\"dram_read_gbs\": %.1f, \"dram_write_gbs\": %.1f, \"l2_size_mb\": %d}\n",
           prop.multiProcessorCount, clk_khz / 1000, l2_gbs, l2_gbs * 1e9 / (clk_khz * 1e3), dram_gbs, wr_gbs, prop.l2CacheSize >> 20);
    if (argc > 1 && !strcmp(argv[1], "--compressible")) return compressible_probe(grid);
    return 0;
}
