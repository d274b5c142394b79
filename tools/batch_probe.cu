// batch_probe.cu -- what moves 4096 tiles of 256 KiB from registered host memory to the device fastest:
// one cudaMemcpyAsync per tile, cudaMemcpyBatchAsync of 128 tiles, or one copy of everything.
// nvcc -arch=sm_90a tools/batch_probe.cu -o tools/batch_probe && tools/batch_probe
#include <cuda_runtime.h>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <vector>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); return 1; } } while (0)
static double now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
int main() {
    const size_t tile = 256 << 10, n = 4096, bytes = tile * n;
    char* h = (char*)aligned_alloc(4096, bytes);
    for (size_t i = 0; i < bytes; i += 4096) h[i] = 1;
    CK(cudaHostRegister(h, bytes, cudaHostRegisterPortable | cudaHostRegisterMapped));
    char* d; CK(cudaMalloc(&d, bytes));
    cudaStream_t s; CK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    for (int rep = 0; rep < 2; ++rep) {
        double t0 = now();
        CK(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, s));
        double t1 = now(); CK(cudaStreamSynchronize(s)); double t2 = now();
        printf("one copy:            issue %.2f ms, total %.2f ms = %.1f GB/s\n", (t1 - t0) * 1e3, (t2 - t0) * 1e3, bytes / (t2 - t0) / 1e9);
        t0 = now();
        for (size_t i = 0; i < n; ++i) CK(cudaMemcpyAsync(d + i * tile, h + i * tile, tile, cudaMemcpyHostToDevice, s));
        t1 = now(); CK(cudaStreamSynchronize(s)); t2 = now();
        printf("per tile:            issue %.2f ms, total %.2f ms = %.1f GB/s\n", (t1 - t0) * 1e3, (t2 - t0) * 1e3, bytes / (t2 - t0) / 1e9);
        for (size_t batch : {32, 128, 512}) {
            std::vector<void*> dsts(batch), srcs(batch); std::vector<size_t> sizes(batch, tile);
            cudaMemcpyAttributes at{}; at.srcAccessOrder = cudaMemcpySrcAccessOrderStream; at.flags = 0;
            size_t idx0 = 0, fail = 0;
            t0 = now();
            for (size_t b = 0; b < n; b += batch) {
                // scattered destinations, like slots handed out by a heap: reverse order inside the batch
                for (size_t i = 0; i < batch; ++i) { srcs[i] = h + (b + i) * tile; dsts[i] = d + (b + batch - 1 - i) * tile; }
                CK(cudaMemcpyBatchAsync(dsts.data(), srcs.data(), sizes.data(), batch, &at, &idx0, 1, &fail, s));
            }
            t1 = now(); CK(cudaStreamSynchronize(s)); t2 = now();
            printf("batches of %3zu:      issue %.2f ms, total %.2f ms = %.1f GB/s\n", batch, (t1 - t0) * 1e3, (t2 - t0) * 1e3, bytes / (t2 - t0) / 1e9);
        }
    }
    return 0;
}
