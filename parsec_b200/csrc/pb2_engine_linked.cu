// pb2_engine_linked.cu -- the HBM window kernel with application bodies (pb2_hbm.cuh, LINKED = true), all four queue
// policy x trace instantiations.  Not part of the library's own device code: the Makefile compiles this file with
// -rdc=true to a relocatable sm_90a cubin, which is embedded in libparsec_b200.so (pb2_linked_image.S) and linked with
// the application's image by pb2_engine_link_bodies.  pb2_linked_body is resolved there.  The kernels are looked up by
// the names of kLinkedKernels[0] (pb2_engine.cu), in the engine's kernel table's order.
#include <cuda_runtime.h>

#include "pb2_hbm.cuh"

namespace pb2 {

template __global__ void pb2_engine_hbm_kernel<false, false, true>(WinDev, TraceDev);
template __global__ void pb2_engine_hbm_kernel<true, false, true>(WinDev, TraceDev);
template __global__ void pb2_engine_hbm_kernel<false, true, true>(WinDev, TraceDev);
template __global__ void pb2_engine_hbm_kernel<true, true, true>(WinDev, TraceDev);

}  // namespace pb2
