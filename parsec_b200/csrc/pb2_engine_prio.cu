// pb2_engine_prio.cu -- the queue_policy 1 (priority lanes) instantiations of the window kernels, in a translation
// unit of their own so that the FIFO kernels of pb2_engine.cu compile exactly as they do without them (see pb2_hbm.cuh).
#include <cuda_runtime.h>

#include "pb2_hbm.cuh"
#include "pb2_gemm.cuh"

namespace pb2 {

cudaError_t pb2_hbm_prio_launch(const WinDev& w, int nworkers, int threads, cudaStream_t stream) {
    pb2_engine_hbm_kernel<true, false><<<nworkers, threads, 0, stream>>>(w, TraceDev{});
    return cudaGetLastError();
}

int pb2_gemm2_prio_launch(const Win2Dev& g, int nworkers, cudaStream_t stream) {
    return pb2_gemm2_launch<true, false>(g, nworkers, stream);
}

}  // namespace pb2
