// pb2_engine_priv.hpp -- host-side engine object shared by the translation units of libparsec_b200.so
// (pb2_engine.cu: windows; pb2_stream.cu: the streaming ring + persistent kernel).
#pragma once
#include <cuda_runtime.h>
#include <stdio.h>
#include <map>
#include <mutex>
#include <string>
#include <utility>
#include "../../include/pb2_engine.h"

struct pb2_engine_s {
    int cuda_device = 0;
    cudaDeviceProp prop{};
    pb2_engine_params_t params{};
    cudaStream_t stream = nullptr;       // where engine work is enqueued
    cudaStream_t own_stream = nullptr;   // created by the engine
    cudaStream_t up_stream = nullptr;    // descriptor uploads of the NEXT window: not ordered behind the running one
    cudaStream_t dma_stream = nullptr;   // pb2_engine_prefetch_h2d
    cudaEvent_t dma_ev = nullptr;
    bool dma_pending = false;
    int nworkers = 0;
    int32_t stage_slice_bytes = 64 * 1024;   // stage-in granularity: every CTA that needs a tile pulls the slices nobody has claimed
    int nworkers_gemm = 0;
    std::string last_error;
    std::mutex mu;
    bool shared_windows = false;
    const int32_t* next_rs_begin = nullptr;   // remote out-degree CSR of the next shared window (not owned)
    std::map<void*, std::pair<size_t, void*>> registered;   // host ptr -> (bytes, device alias)
};

#define PB2_CUDA(e, call)                                                                        \
    do {                                                                                         \
        cudaError_t err__ = (call);                                                              \
        if (err__ != cudaSuccess) {                                                              \
            char buf__[512];                                                                     \
            snprintf(buf__, sizeof buf__, "%s:%d %s -> %s", __FILE__, __LINE__, #call,           \
                     cudaGetErrorString(err__));                                                 \
            if (e) (e)->last_error = buf__;                                                      \
            fprintf(stderr, "pb2: CUDA error %s\n", buf__);                                      \
            return PB2_ERR_DEVICE;                                                               \
        }                                                                                        \
    } while (0)

