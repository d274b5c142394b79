// pb2_engine_priv.hpp -- host-side engine object shared by the translation units of libparsec_b200.so
// (pb2_engine.cu: windows; pb2_window_kernels.cu: the built-in window kernels; pb2_stream.cu: the streaming ring +
// persistent kernel).
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

// One window kernel as the engine launches it: the function, its launch shape, and what the compiler or the linker made
// of it (registers, local bytes per thread, static shared memory).
struct WindowKernel {
    CUfunction fn = nullptr;
    unsigned grid = 0, block = 0, dyn_smem = 0;
    int32_t regs = 0, local = 0, static_smem = 0;
};

// The host symbols of the built-in HBM and GEMM window kernels of variant v = (queue_policy 1) + 2 * (trace):
// window_kernels_<v> is defined by the object the Makefile compiles from pb2_window_kernels.cu with PB2_WINDOW_VARIANT=v.
struct WindowKernelSymbols { const void* hbm; const void* gemm; };
WindowKernelSymbols window_kernels_0();
WindowKernelSymbols window_kernels_1();
WindowKernelSymbols window_kernels_2();
WindowKernelSymbols window_kernels_3();

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
    // Compressible tile memory (pb2_engine_malloc_ex): the granule of such an allocation, 0 where the device or the
    // driver offers none; every allocation the L2 compresses, base -> (handle, mapped bytes), freed by pb2_engine_free
    // or with the engine; whether the last allocation of a granule or more was granted compression.
    size_t comp_granule = 0;
    std::map<void*, std::pair<CUmemGenericAllocationHandle, size_t>> compressible;
    bool slab_compressible = false;
    // Every window kernel by [built-in, linked][kind: HBM, GEMM][(queue_policy 1) + 2 * (trace)].  A built-in entry
    // is resolved when a window first needs it, under mu; pb2_engine_link_bodies_ex resolves the linked HBM entries,
    // and with PB2_LINK_GEMM_WINDOWS the linked GEMM entries (an entry that is not resolved has a null fn).
    WindowKernel kernels[2][2][4];
    // pb2_engine_link_bodies: the module of the linked window kernels, and which linked body ids may be cut into parts
    // (bit i: PB2_BODY_LINKED_0 + i), which have a checked form, which are readers (PB2_LINK_READERS) and which readers
    // have the group form (PB2_LINK_READER_GROUPS) and which get the GEMM worker's operand ring (PB2_LINK_GEMM_BODIES),
    // and whether the GEMM kernels call those through pb2_linked_gemm_body (PB2_LINK_GEMM_BODY_ENTRY)
    CUmodule linked_module = nullptr;
    uint32_t linked_sliceable = 0, linked_checked = 0, linked_readers = 0, linked_reader_groups = 0, linked_gemm_bodies = 0;
    bool linked_gemm_body_entry = false;
    // pb2_engine_set_gemm_body_parts: parts per task of GEMM-worker body PB2_BODY_LINKED_0 + i
    int32_t gemm_body_parts[8] = {1, 1, 1, 1, 1, 1, 1, 1};
};

// The readers mask of link flags (PB2_LINK_READERS): bit i, PB2_BODY_LINKED_0 + i is a reader.
static inline uint32_t link_readers(uint32_t flags) { return (flags >> 8) & 0xFFu; }
// The reader groups mask of link flags (PB2_LINK_READER_GROUPS): bit i, reader PB2_BODY_LINKED_0 + i has the group form.
static inline uint32_t link_reader_groups(uint32_t flags) { return (flags >> 16) & 0xFFu; }

// The GEMM-worker bodies mask of link flags (PB2_LINK_GEMM_BODIES): bit i, PB2_BODY_LINKED_0 + i gets the operand ring.
static inline uint32_t link_gemm_bodies(uint32_t flags) { return (flags >> 24) & 0xFFu; }

// The argument check of pb2_engine_link_bodies(_checked, _ex) and pb2_device_link_bodies(_checked, _ex): nullptr, or why
// the arguments are refused.
static inline const char* link_args_error(const void* image, size_t bytes, int format, uint32_t sliceable, uint32_t checked,
                                          uint32_t flags = 0) {
    if (flags & ~(uint32_t)(PB2_LINK_GEMM_WINDOWS | PB2_LINK_GEMM_BODY_ENTRY | PB2_LINK_READERS(0xFFu) |
                            PB2_LINK_READER_GROUPS(0xFFu) | PB2_LINK_GEMM_BODIES(0xFFu)))
        return "link flags have an unknown bit (PB2_LINK_GEMM_WINDOWS, PB2_LINK_GEMM_BODY_ENTRY, PB2_LINK_READERS(mask), "
               "bits 8..15, PB2_LINK_READER_GROUPS(mask), bits 16..23, and PB2_LINK_GEMM_BODIES(mask), bits 24..31, are "
               "the only flags)";
    if (!image || !bytes) return "linked body image is NULL or empty";
    if (format != PB2_IMAGE_PTX && format != PB2_IMAGE_CUBIN) return "linked body image format must be PB2_IMAGE_PTX or PB2_IMAGE_CUBIN";
    if (sliceable >> 8) return "sliceable mask has bits above bit 7 (there are 8 linked body ids)";
    if (checked >> 8) return "checked mask has bits above bit 7 (there are 8 linked body ids)";
    // a fused producer's parts cut its tile as its readers' parts do
    if (checked & ~sliceable) return "checked mask has a bit that is clear in the sliceable mask (a checked body must be sliceable)";
    // a read group's parts and chunks cut the tile as every member's parts do
    if (link_readers(flags) & ~sliceable) return "readers mask has a bit that is clear in the sliceable mask (a reader must be sliceable)";
    if (link_reader_groups(flags) & ~link_readers(flags))
        return "link flags have an unknown bit: the reader groups mask has a bit that is clear in the readers mask (only a "
               "reader has the group form)";
    if (link_gemm_bodies(flags) && !(flags & PB2_LINK_GEMM_WINDOWS))
        return "GEMM-worker bodies mask without PB2_LINK_GEMM_WINDOWS (a GEMM-worker body runs in GEMM windows only)";
    // the ring is the worker's own: such a body runs whole, never in parts, in a read group or fused with one
    if (link_gemm_bodies(flags) & sliceable)
        return "GEMM-worker bodies mask has a bit that is set in the sliceable mask (a GEMM-worker body runs as one part; "
               "it can be neither checked nor a reader)";
    if ((flags & PB2_LINK_GEMM_BODY_ENTRY) && !link_gemm_bodies(flags))
        return "PB2_LINK_GEMM_BODY_ENTRY without a PB2_LINK_GEMM_BODIES mask (the entry point is called for GEMM-worker "
               "bodies only)";
    return nullptr;
}

// The argument check of pb2_engine_set_gemm_body_parts and pb2_device_set_gemm_body_parts: nullptr, or why the call is
// refused with the code in *rc.  linked: an image is linked; gemm_bodies: the link's GEMM-worker mask.
static inline const char* gemm_body_parts_error(bool linked, uint32_t gemm_bodies, int body, int32_t nparts, int* rc) {
    *rc = PB2_ERR_NOT_FOUND;
    if (!linked) return "no image is linked yet: part counts are declared for the GEMM-worker bodies of a link";
    *rc = PB2_ERR_BAD_PARAM;
    if (body < PB2_BODY_LINKED_0 || body > PB2_BODY_LINKED_7) return "body is not a linked body id (PB2_BODY_LINKED_0 .. _7)";
    if (!((gemm_bodies >> (body - PB2_BODY_LINKED_0)) & 1u))
        return "body is not a GEMM-worker body of the link (its bit is clear in the PB2_LINK_GEMM_BODIES mask)";
    *rc = PB2_ERR_VALUE_OUT_OF_BOUNDS;
    if (nparts < 1 || nparts > PB2_GEMM_BODY_MAX_PARTS) return "nparts must be 1 .. PB2_GEMM_BODY_MAX_PARTS (32)";
    *rc = PB2_SUCCESS;
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

