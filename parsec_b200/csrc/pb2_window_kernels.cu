// pb2_window_kernels.cu -- the built-in window kernels of one variant v = (queue_policy 1) + 2 * (window trace): the
// Makefile compiles this file once per v with -DPB2_WINDOW_VARIANT=v.  Each object holds one HBM and one GEMM kernel,
// because a second HBM kernel calling the same __noinline__ helpers in one translation unit makes ptxas give them the
// standard call ABI, which costs the kernel a stack frame and spills at its 80-register budget (pb2_hbm.cuh).  The
// engine launches them through its kernel table (pb2_engine.cu), by the host symbols window_kernels_<v> returns.
#include <cuda_runtime.h>

#include "pb2_hbm.cuh"
#include "pb2_gemm.cuh"
#include "pb2_engine_priv.hpp"

#if !defined(PB2_WINDOW_VARIANT) || PB2_WINDOW_VARIANT < 0 || PB2_WINDOW_VARIANT > 3
#error "compile with -DPB2_WINDOW_VARIANT=v, v = (queue_policy 1) + 2 * (trace) in 0..3"
#endif

namespace pb2 {

constexpr bool kPrio = (PB2_WINDOW_VARIANT & 1) != 0, kTrace = (PB2_WINDOW_VARIANT & 2) != 0;

template __global__ void pb2_engine_hbm_kernel<kPrio, kTrace>(WinDev, TraceDev);
template __global__ void pb2_engine_gemm2_kernel<kPrio, kTrace>(Win2Dev);

}  // namespace pb2

#define PB2_WINDOW_KERNELS_FN_(v) window_kernels_##v
#define PB2_WINDOW_KERNELS_FN(v) PB2_WINDOW_KERNELS_FN_(v)

WindowKernelSymbols PB2_WINDOW_KERNELS_FN(PB2_WINDOW_VARIANT)() {
    return {reinterpret_cast<const void*>(pb2::pb2_engine_hbm_kernel<pb2::kPrio, pb2::kTrace>),
            reinterpret_cast<const void*>(pb2::pb2_engine_gemm2_kernel<pb2::kPrio, pb2::kTrace>)};
}
