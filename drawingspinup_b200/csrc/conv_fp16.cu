// The convolution kernels of the fp16 precision mode (single-pass fp16 operands), every mode.  Split-fp16 tap launches
// run these too: tap mode takes the split from its K masks.
#include "conv_wgmma.cuh"

namespace dsu {

template cudaError_t launch_mode<ConvMode::Tap, false, __half>(const ConvParams&, cudaStream_t);
template cudaError_t launch_mode<ConvMode::Ric, false, __half>(const ConvParams&, cudaStream_t);
template cudaError_t launch_mode<ConvMode::RicHalo, false, __half>(const ConvParams&, cudaStream_t);
template cudaError_t launch_mode<ConvMode::Halo, false, __half>(const ConvParams&, cudaStream_t);

}  // namespace dsu
