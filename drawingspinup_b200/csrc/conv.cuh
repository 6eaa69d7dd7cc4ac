// Parameter blocks shared by the fused convolution kernel and the engine that plans a network.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "act.cuh"

namespace dsu {

constexpr int kTileH = 8;       // output patch rows per CTA
constexpr int kTileW = 16;      // output patch cols per CTA
constexpr int kTileM = 128;     // output pixels per CTA = two warpgroups x wgmma M = 64
constexpr int kChunkK = 64;     // 16-bit (fp16 / bf16) K elements per smem row (128 B, SWIZZLE_128B)
constexpr int kABytes = kTileM * 128;   // bytes of one A stage
constexpr int kThreads = 256;   // two warpgroups: producers, MMA issuers and epilogue alike
constexpr int kStages = 4;      // A + B ring depth; chunk q + 2 is loaded while the MMAs of chunk q run
constexpr int kMaxSeg = 6;      // concat segments (second half = lo planes in exact mode)
constexpr int kChannelAlign = 32;   // stored activation widths are multiples of this (the epilogue's 32-column batches)
// widest output-channel piece of one launch (the widest Cout launch_mode instantiates in that precision; fp16 and bf16
// share the single-pass value, split fp16 and split bf16 the split one)
constexpr int kMaxPiece(bool exact) { return exact ? 128 : 256; }

// Which mainloop and A producer a convolution launch runs.  This is the one statement of the rule (engine.cu compile_layer
// records the plan-time mode, conv_mode applies the run-time knobs):
//   * stage-1 (RIC) layers run RicHalo; knob `ric_halo` = 0 keeps them on Ric.
//   * a stage-2 layer runs Halo when it is stride 1 without fused upsampling and either conv0-shaped or Cout <= 64 (wider layers
//     measured slower on 8 x 16 halo tiles, DESIGN section 7); plan-time knob `halo` (DSU_HALO) = 0 keeps all but conv0 on
//     Tap, and run-time knob `first` = 0 sends conv0 to Tap.  Every other layer runs Tap.
// The run-time alternatives use the same chunks and weight packing as the plan-time mode.
//
// Output-channel pieces.  Every activation is stored with its width rounded up to a multiple of 32 (kChannelAlign; the
// padding channels hold exact zeros).  A layer whose padded width exceeds kMaxPiece (128 in split fp16 / bf16, 256 in fp16 / bf16) runs as
// several launches over contiguous channel ranges, widest first (split-fp16 160 -> 128 + 32, fp16 384 -> 256 + 128), each
// with its own weight tiles, affine and output channel offset; the residual stream and the instance-norm scratch keep the
// layer's full pitch (EpiParams::resid_pitch).  The mode above is decided once per layer on its padded width, so every piece
// runs the same mode.
enum class ConvMode : int {
    Tap,        // conv_wgmma_kernel: each A slot gathered from global memory per (chunk, slot) with cp.async
    Ric,        // conv_wgmma_kernel: stage-1 deformable, the bilinear corners gathered from global memory
    RicHalo,    // conv_halo_kernel at every width: stage-1 deformable, stencil and corners staged in shared memory, the A
                // fragments blended straight into registers
    Halo,       // conv_halo_kernel: stride 1, A fragments read with ldmatrix from a shared-memory input halo
};

// One 16-byte (8-channel) K slot: which tap of which source segment fills it.
// plain conv: one entry per (chunk, slot).  RIC conv: one entry per (64-channel block, slot) - the
// tap is the chunk's position inside the block.  Halo mode: per chunk as for a plain conv, plus one entry per
// (channel block, 16-byte slot of a halo pixel) saying what the halo holds (ConvParams::hslots).
struct Slot {
    int8_t dy, dx;      // plain: tap offset (kh - pad, kw - pad)
    uint8_t seg;        // source segment index (lo plane = seg + kMaxSeg/2)
    uint8_t valid;      // 0 -> zero fill (K padding)
    uint16_t choff;     // first channel inside the segment buffer
    uint8_t hslot;      // halo mode: the 16-byte slot of the halo pixel that holds these 8 channels
    uint8_t pad_;
};
static_assert(sizeof(Slot) == 8, "Slot must be 8 bytes");

struct Seg {
    const __half* ptr;
    int pitch;          // channels per pixel in the buffer
    int pad_;
};

struct EpiParams {
    const float* scale;     // [Cout] pre-activation affine (folded BN / bias); never null
    const float* shift;
    const float* scale2;    // [Cout] post-activation affine (conv_11_a.2) or null
    const float* shift2;
    int act;                // 0 none, 1 ReLU, 2 LeakyReLU(0.2)
    int resid_in, resid_out;
    float* resid;           // fp32 residual stream [pix][resid_pitch], from this launch's first channel
    int resid_pitch;        // channels per pixel of `resid`: the layer's padded width (> Cout for an output-channel piece)
    ActOut out;             // main output (after residual), ReLU first when out_relu
    ActOut out2;            // second, un-ReLU'd copy (skip connection)
    int out_relu;
    // fused conv_12 (1x1, +bias, optional tanh) tail
    const float* w12;       // [3][Cout] or null
    const float* b12;       // [3]
    int tanh_flag;
    float* y_nchw;          // [B,3,H,W] fp32 or null
    uint8_t* y_rgba;        // [B,H,W,4] uint8 or null (to_image_space + alpha)
    const uint8_t* alpha_src;   // alpha byte of pixel p at alpha_src[p * alpha_stride]
    int alpha_stride;
    // one piece of a final layer split into output-channel pieces: the three conv_12 partial dot products of its channels
    // go to y_part[o][pix] (B*H*W pixels) instead of y_nchw / y_rgba; conv12_tail (frames.cuh) sums the pieces
    float* y_part;
};

struct ConvParams {
    int B, Hout, Wout;      // output geometry
    int Hin, Win;           // source buffer geometry (before the fused nearest x2)
    int Hv, Wv;             // virtual conv-input geometry = (Hin << up, Win << up)
    ConvMode mode;
    int stride, up, exact;
    int bf16;               // bf16 operands, single pass or split (exact): the kernels' element type is __nv_bfloat16, not __half
    int nchunks, nblocks, Cout;
    int b_bytes;            // bytes per B stage = Cout x 128 (one chunk's weight tile in wpack)
    // K-step masks as launch constants so the issuing warpgroups stay uniform (kmask: which of the 4 K=16 steps are
    // issued against B tile 0; kmask2, split fp16: which of A steps 0-1 are issued against B steps 2-3): every chunk uses
    // *_full except the ragged tail (tap mode: the last chunk; RIC: all chunks of the last channel block), which uses *_last
    uint32_t kmask_full, kmask_last, kmask2_full, kmask2_last;
    const Slot* slots;      // plain: [nchunks][8]; RIC: [nblocks][8]
    const uint8_t* wpack;   // pre-swizzled B tiles
    Seg seg[kMaxSeg];
    // RIC stencil of the output level, per pixel: octant (tap rotation) and, in rotated tap
    // order m = (octant + k) & 7, the bilinear fractions (ly, lx) relative to the static quadrant of m
    const float2* ric_lyx;  // [Hout*Wout][8]
    const uint8_t* ric_oct; // [Hout*Wout]
    const uint2* ric_wh;    // [Hout*Wout][8] the 4 bilinear weights of each rotated tap as fp16 {w00,w01 | w10,w11} (packed-half2 blend,
                            // fp16 mode; split fp16, bf16 and split bf16 blend in fp32 from ric_lyx)
    EpiParams epi;
    // sub-pixel class of a fused nearest-x2 + 3x3 convolution: the launch is a 2x2 convolution over the LOW-resolution
    // source whose output pixel (oy, ox) of the Hout x Wout grid lands at (2*oy + sub_py, 2*ox + sub_px) of the
    // (2*Hout) x (2*Wout) output buffer
    int sub, sub_py, sub_px;
    // halo mode: the channels are walked in blocks of 128 bytes per pixel; the (tile rows + ksize - 1) x (kTileW + ksize - 1)
    // input halo of each block, origin (ty0 - pad_y, tx0 - pad_x), is staged in shared memory once and the A fragments of
    // every tap are read from it straight into registers
    int ksize, pad_y, pad_x;
    const Slot* hslots;     // [nblocks][8]: the channels of each 16-byte slot of a halo pixel
    int n128;               // Cout a multiple of 128: issue N = 128 wgmma instructions (else N = 64 / 32)
};

cudaError_t launch_conv(const ConvParams& p, cudaStream_t stream);

}  // namespace dsu
