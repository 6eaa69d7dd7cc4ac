// The convolution kernels of the fp16x3 precision mode (split fp16 hi + lo operands) in Ric, RicHalo and Halo modes;
// its tap launches run the fp16 kernels (conv_fp16.cu).
#include "conv_wgmma.cuh"

namespace dsu {

template cudaError_t launch_mode<ConvMode::Ric, true, __half>(const ConvParams&, cudaStream_t);
template cudaError_t launch_mode<ConvMode::RicHalo, true, __half>(const ConvParams&, cudaStream_t);
template cudaError_t launch_mode<ConvMode::Halo, true, __half>(const ConvParams&, cudaStream_t);

}  // namespace dsu
