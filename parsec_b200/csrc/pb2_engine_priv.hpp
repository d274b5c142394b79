// pb2_engine_priv.hpp -- host-side engine object shared by the translation units of libparsec_b200.so
// (pb2_engine.cu: windows; pb2_stream.cu: the streaming ring + persistent kernel).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdio.h>
#include <map>
#include <mutex>
#include <string>
#include <utility>
#include "../../include/pb2_engine.h"
#include "pb2_window_layout.h"

struct pb2_engine_s {
    int cuda_device = 0;
    cudaDeviceProp prop{};
    pb2_engine_params_t params{};
    cudaStream_t stream = nullptr;       // where engine work is enqueued
    cudaStream_t own_stream = nullptr;   // created by the engine
    cudaStream_t up_stream = nullptr;    // descriptor uploads of the NEXT window: not ordered behind the running one
    cudaStream_t dma_stream = nullptr;   // pb2_engine_prefetch_h2d
    cudaStream_t arm_stream = nullptr;   // re-arms the other copy of an HBM window's per-run state beside its run
    cudaEvent_t dma_ev = nullptr;
    bool dma_pending = false;
    int nworkers = 0;
    int32_t stage_slice_bytes = 64 * 1024;   // stage-in granularity: every CTA that needs a tile pulls the slices nobody has claimed
    int nworkers_gemm = 0;
    std::string last_error;
    std::mutex mu;
    bool shared_windows = false;
    bool window_trace = false;           // windows created from now on record per-task device time stamps
    const int32_t* next_rs_begin = nullptr;   // remote out-degree CSR of the next shared window (not owned)
    std::map<void*, std::pair<size_t, void*>> registered;   // host ptr -> (bytes, device alias)
    // pb2_engine_link_bodies: the module of the linked HBM window kernels, each kernel and its worker count by
    // (queue_policy 1) + 2 * (trace), what the linker made of the untraced one of this engine's policy, and which
    // linked body ids may be cut into parts (bit i: PB2_BODY_LINKED_0 + i) and which have a checked form
    CUmodule linked_module = nullptr;
    CUfunction linked_fn[4] = {};
    int linked_nworkers[4] = {};
    int32_t linked_regs = 0, linked_local = 0, linked_smem = 0;
    uint32_t linked_sliceable = 0, linked_checked = 0;
    // linked with PB2_LINK_GEMM_WINDOWS: the same module's linked GEMM window kernels, their worker counts and what the
    // linker made of the untraced one of this engine's policy (else linked_gemm is false and the rest stays zero)
    bool linked_gemm = false;
    CUfunction linked_gemm_fn[4] = {};
    int linked_gemm_nworkers[4] = {};
    int32_t linked_gemm_regs = 0, linked_gemm_local = 0, linked_gemm_smem = 0;
};

// The argument check of pb2_engine_link_bodies(_checked, _ex) and pb2_device_link_bodies(_checked, _ex): nullptr, or why
// the arguments are refused.
static inline const char* link_args_error(const void* image, size_t bytes, int format, uint32_t sliceable, uint32_t checked,
                                          uint32_t flags = 0) {
    if (flags & ~(uint32_t)PB2_LINK_GEMM_WINDOWS) return "link flags have an unknown bit (PB2_LINK_GEMM_WINDOWS is the only flag)";
    if (!image || !bytes) return "linked body image is NULL or empty";
    if (format != PB2_IMAGE_PTX && format != PB2_IMAGE_CUBIN) return "linked body image format must be PB2_IMAGE_PTX or PB2_IMAGE_CUBIN";
    if (sliceable >> 8) return "sliceable mask has bits above bit 7 (there are 8 linked body ids)";
    if (checked >> 8) return "checked mask has bits above bit 7 (there are 8 linked body ids)";
    // a fused producer's parts cut its tile as its readers' parts do
    if (checked & ~sliceable) return "checked mask has a bit that is clear in the sliceable mask (a checked body must be sliceable)";
    return nullptr;
}

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

