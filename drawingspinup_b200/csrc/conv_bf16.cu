// The convolution kernels of the bf16 precision mode (single-pass bf16 operands), every mode.  Split-bf16 tap launches
// run these too: tap mode takes the split from its K masks.
#include "conv_wgmma.cuh"

namespace dsu {

template cudaError_t launch_mode<ConvMode::Tap, false, __nv_bfloat16>(const ConvParams&, cudaStream_t);
template cudaError_t launch_mode<ConvMode::Ric, false, __nv_bfloat16>(const ConvParams&, cudaStream_t);
template cudaError_t launch_mode<ConvMode::RicHalo, false, __nv_bfloat16>(const ConvParams&, cudaStream_t);
template cudaError_t launch_mode<ConvMode::Halo, false, __nv_bfloat16>(const ConvParams&, cudaStream_t);

}  // namespace dsu
