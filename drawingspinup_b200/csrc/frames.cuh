// Launch wrappers of the per-pixel frame kernels (frames.cu).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "act.cuh"

namespace dsu {

cudaError_t ingest_f32(const float* x, int B, int cin, int cpad, int H, int W, const ActOut& out, cudaStream_t st);
// x channels RGB | mask (has_mask) | posXY (has_pos), the rest of the 8-channel group zero.  edge == nullptr && derive_edge:
// burn the edges pos2edge would find in `pos` (run_render.py:31-57 fused into the ingest).  `pos` may be null when neither
// has_pos nor derive_edge reads it.
cudaError_t ingest_u8(const uint8_t* color, const uint8_t* pos, const uint8_t* edge, int derive_edge, bool has_mask, bool has_pos,
                      int B, int H, int W, const ActOut& out, cudaStream_t st);
// 2x2 / stride 2 max-pool of C channels from `in` to `out`, both fp16, both bf16 or both fp32; a lo plane is an error (the
// split modes pool only in stage 1, whose activations are fp32)
cudaError_t maxpool2(const ActOut& in, const ActOut& out, int B, int Hin, int Win, int C, cudaStream_t st);
cudaError_t frames_to_tensor(const uint8_t* color, const uint8_t* pos, const uint8_t* edge, int B, int H, int W,
                             float* pre, float* mask, cudaStream_t st);
cudaError_t to_image_space(const float* x, uint8_t* out, size_t n, cudaStream_t st);
cudaError_t overlap_edge(const uint8_t* edge, uint8_t* rgba, size_t npix, cudaStream_t st);
cudaError_t compose_rgba(const float* y, const float* mask, int B, int H, int W, uint8_t* out, cudaStream_t st);
cudaError_t pos2edge(const uint8_t* pos, int B, int H, int W, uint8_t* edge, cudaStream_t st);
// conv_12 of a final layer split into output-channel pieces: part[piece][3][B*H*W] partial dot products -> sum in piece
// order + b12 (+ tanh) -> y [B,3,H,W] fp32 and / or rgba [B,H,W,4] (to_u8, alpha byte of pixel p at alpha_src[p *
// alpha_stride], 255 without alpha_src); either output may be null
cudaError_t conv12_tail(const float* part, int npieces, const float* b12, int tanh_flag, int B, int H, int W, float* y,
                        uint8_t* rgba, const uint8_t* alpha_src, int alpha_stride, cudaStream_t st);

// nn.InstanceNorm2d between a convolution (raw fp32 output x[B][HW][C] left by its epilogue) and its activation, followed by
// the stores the fused epilogue would have done.  Three small launches: statistics (fp64 accumulation), finish, apply.
struct InstNormApply {
    const float* x;          // raw convolution output, fp32 NHWC, pitch C
    float2* stats;           // [B][C] (mean, 1/sqrt(var + eps)) - written by the call
    int B, HW, C;
    int act;                 // 0 none, 1 ReLU, 2 LeakyReLU(0.2), applied after the normalisation
    float* resid;            // fp32 residual stream [pix][C] to write, or null
    ActOut out;              // main output, ReLU first when out_relu
    ActOut out2;             // second copy taken before out_relu
    int out_relu;
};
// Each plane's statistics are taken in min(64, ceil(HW / 4096)) slices of ceil(HW / slices) pixels, one block per (slice,
// 32 channels, frame); `acc` holds one (sum, sum of squares) slot per slice, summed in slice order by the finish step.
constexpr int kInormMaxSlices = 64;
cudaError_t instance_norm(const InstNormApply& a, double* acc /* [B][C][kInormMaxSlices][2] scratch */, cudaStream_t st);

}  // namespace dsu
