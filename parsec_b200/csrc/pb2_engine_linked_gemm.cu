// pb2_engine_linked_gemm.cu -- the GEMM window kernel with application bodies (pb2_gemm.cuh, LINKED = true), all four
// queue policy x trace instantiations.  Like pb2_engine_linked.cu, not part of the library's own device code: the
// Makefile compiles this file with -rdc=true to a second relocatable sm_90a cubin, embedded in libparsec_b200.so
// (pb2_linked_image.S), which pb2_engine_link_bodies_ex adds to the link only with PB2_LINK_GEMM_WINDOWS.  A translation
// unit of its own: the HBM kernels' __noinline__ stage-in helpers are instantiated once per caller kernel per unit, and
// a GEMM kernel beside them would change the linked HBM kernels' code (pb2_hbm.cuh).  The kernels are looked up by the
// names of kLinkedKernels[1] (pb2_engine.cu), in the engine's kernel table's order.  The Makefile builds it four times:
// plain, with PB2_LINKED_READER_GROUPS, with PB2_LINKED_GEMM_BODY_ENTRY, and with both.
#include <cuda_runtime.h>

#include "pb2_gemm.cuh"

namespace pb2 {

template __global__ void pb2_engine_gemm2_kernel<false, false, true>(Win2Dev);
template __global__ void pb2_engine_gemm2_kernel<true, false, true>(Win2Dev);
template __global__ void pb2_engine_gemm2_kernel<false, true, true>(Win2Dev);
template __global__ void pb2_engine_gemm2_kernel<true, true, true>(Win2Dev);

}  // namespace pb2
