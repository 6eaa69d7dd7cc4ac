// launch_conv: one convolution launch, dispatched on its mode and precision to the launch_mode instantiations of the
// precision's translation unit (conv_fp16.cu, conv_fp16x3.cu, conv_bf16.cu, conv_bf16x3.cu).  The kernels are in
// conv_wgmma.cuh.
#include "conv_wgmma.cuh"

namespace dsu {

// instantiated elsewhere: no kernel is compiled in this translation unit
extern template cudaError_t launch_mode<ConvMode::Tap, false, __half>(const ConvParams&, cudaStream_t);
extern template cudaError_t launch_mode<ConvMode::Ric, false, __half>(const ConvParams&, cudaStream_t);
extern template cudaError_t launch_mode<ConvMode::RicHalo, false, __half>(const ConvParams&, cudaStream_t);
extern template cudaError_t launch_mode<ConvMode::Halo, false, __half>(const ConvParams&, cudaStream_t);
extern template cudaError_t launch_mode<ConvMode::Ric, true, __half>(const ConvParams&, cudaStream_t);
extern template cudaError_t launch_mode<ConvMode::RicHalo, true, __half>(const ConvParams&, cudaStream_t);
extern template cudaError_t launch_mode<ConvMode::Halo, true, __half>(const ConvParams&, cudaStream_t);
extern template cudaError_t launch_mode<ConvMode::Tap, false, __nv_bfloat16>(const ConvParams&, cudaStream_t);
extern template cudaError_t launch_mode<ConvMode::Ric, false, __nv_bfloat16>(const ConvParams&, cudaStream_t);
extern template cudaError_t launch_mode<ConvMode::RicHalo, false, __nv_bfloat16>(const ConvParams&, cudaStream_t);
extern template cudaError_t launch_mode<ConvMode::Halo, false, __nv_bfloat16>(const ConvParams&, cudaStream_t);
extern template cudaError_t launch_mode<ConvMode::Ric, true, __nv_bfloat16>(const ConvParams&, cudaStream_t);
extern template cudaError_t launch_mode<ConvMode::RicHalo, true, __nv_bfloat16>(const ConvParams&, cudaStream_t);
extern template cudaError_t launch_mode<ConvMode::Halo, true, __nv_bfloat16>(const ConvParams&, cudaStream_t);

namespace {

// the launch's precision: split fp16 or split bf16 (Tap mode reads the split from the K masks), fp16 or bf16
template <ConvMode kMode>
cudaError_t launch_prec(const ConvParams& p, cudaStream_t stream) {
    if constexpr (kMode != ConvMode::Tap)
        if (p.exact) return p.bf16 ? launch_mode<kMode, true, __nv_bfloat16>(p, stream) : launch_mode<kMode, true, __half>(p, stream);
    return p.bf16 ? launch_mode<kMode, false, __nv_bfloat16>(p, stream) : launch_mode<kMode, false, __half>(p, stream);
}

}  // namespace

cudaError_t launch_conv(const ConvParams& p, cudaStream_t stream) {
    if (conv_smem_bytes(p.mode, p.Cout, p.ksize, p.up) > kSmemMax || p.b_bytes != p.Cout * 128)
        return cudaErrorInvalidConfiguration;
    switch (p.mode) {
        case ConvMode::Tap: return launch_prec<ConvMode::Tap>(p, stream);
        case ConvMode::Ric: return launch_prec<ConvMode::Ric>(p, stream);
        case ConvMode::RicHalo: return launch_prec<ConvMode::RicHalo>(p, stream);
        case ConvMode::Halo: return launch_prec<ConvMode::Halo>(p, stream);
    }
    return cudaErrorInvalidConfiguration;
}

}  // namespace dsu
