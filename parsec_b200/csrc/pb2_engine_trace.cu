// pb2_engine_trace.cu -- the traced FIFO instantiations of the window kernels (pb2_engine_set_window_trace), in a
// translation unit of their own so that the untraced kernels compile exactly as they do without them (see pb2_hbm.cuh).
#include <cuda_runtime.h>

#include "pb2_hbm.cuh"
#include "pb2_gemm.cuh"

namespace pb2 {

cudaError_t pb2_hbm_trace_launch(const WinDev& w, const TraceDev& tr, int nworkers, int threads, cudaStream_t stream) {
    pb2_engine_hbm_kernel<false, true><<<nworkers, threads, 0, stream>>>(w, tr);
    return cudaGetLastError();
}

int pb2_gemm2_trace_launch(const Win2Dev& g, int nworkers, cudaStream_t stream) {
    return pb2_gemm2_launch<false, true>(g, nworkers, stream);
}

}  // namespace pb2
