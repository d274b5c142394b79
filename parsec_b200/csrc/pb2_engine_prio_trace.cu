// pb2_engine_prio_trace.cu -- the traced queue_policy 1 instantiations of the window kernels, in a translation unit of
// their own for the same reason as pb2_engine_prio.cu.
#include <cuda_runtime.h>

#include "pb2_hbm.cuh"
#include "pb2_gemm.cuh"

namespace pb2 {

cudaError_t pb2_hbm_prio_trace_launch(const WinDev& w, const TraceDev& tr, int nworkers, int threads, cudaStream_t stream) {
    pb2_engine_hbm_kernel<true, true><<<nworkers, threads, 0, stream>>>(w, tr);
    return cudaGetLastError();
}

int pb2_gemm2_prio_trace_launch(const Win2Dev& g, int nworkers, cudaStream_t stream) {
    return pb2_gemm2_launch<true, true>(g, nworkers, stream);
}

}  // namespace pb2
