// conv_gemm instantiations (conv_gemm.cuh), one file per group of epilogue variants so that they compile in parallel.
#include "conv_gemm.cuh"

namespace uc {
template int conv_launch<kEpiRelu, false>(const ConvKernelParams&, int, bool, cudaStream_t);
template int conv_launch<kEpiGelu, false>(const ConvKernelParams&, int, bool, cudaStream_t);
template int conv_launch<kEpiGeluLn, false>(const ConvKernelParams&, int, bool, cudaStream_t);
}  // namespace uc
