// The convolution kernels of the bf16x3 precision mode (split bf16 hi + lo operands) in Ric, RicHalo and Halo modes;
// its tap launches run the bf16 kernels (conv_bf16.cu).
#include "conv_wgmma.cuh"

namespace dsu {

template cudaError_t launch_mode<ConvMode::Ric, true, __nv_bfloat16>(const ConvParams&, cudaStream_t);
template cudaError_t launch_mode<ConvMode::RicHalo, true, __nv_bfloat16>(const ConvParams&, cudaStream_t);
template cudaError_t launch_mode<ConvMode::Halo, true, __nv_bfloat16>(const ConvParams&, cudaStream_t);

}  // namespace dsu
