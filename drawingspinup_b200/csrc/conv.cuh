// Parameter blocks shared by the fused convolution kernel and the engine that plans a network.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace dsu {

constexpr int kTileH = 8;       // output patch rows per CTA
constexpr int kTileW = 16;      // output patch cols per CTA
constexpr int kTileM = 128;     // output pixels per CTA = two warpgroups x wgmma M = 64
constexpr int kChunkK = 64;     // fp16 K elements per smem row (128 B, SWIZZLE_128B)
constexpr int kABytes = kTileM * 128;   // bytes of one A stage
constexpr int kThreads = 256;   // two warpgroups: producers, MMA issuers and epilogue alike
constexpr int kStages = 4;      // A + B ring depth; chunk q + 2 is loaded while the MMAs of chunk q run
constexpr int kMaxSeg = 6;      // concat segments (second half = lo planes in exact mode)

// One 16-byte (8-channel) K slot: which tap of which source segment fills it.
// plain conv: one entry per (chunk, slot).  RIC conv: one entry per (64-channel block, slot) - the
// tap is the chunk's position inside the block.
struct Slot {
    int8_t dy, dx;      // plain: tap offset (kh - pad, kw - pad)
    uint8_t seg;        // source segment index (lo plane = seg + kMaxSeg/2)
    uint8_t valid;      // 0 -> zero fill (K padding)
    uint16_t choff;     // first channel inside the segment buffer
    uint16_t pad_;
};
static_assert(sizeof(Slot) == 8, "Slot must be 8 bytes");

// Host-side description of one K chunk (8 slots = 64 K elements) of the implicit GEMM; the kernel gets the masks as
// launch constants (kmask_full / kmask_last).
struct ChunkHdr {
    uint8_t kmask;      // which of the 4 K=16 steps are issued against B tile 0
    uint8_t kmask2;     // exact mode: which of A steps 0-1 (the hi half) are issued against B steps 2-3 (W_lo)
};

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
    float* resid;           // fp32 residual stream [pix][Cout]
    __half* out_hi;         // main fp16 output (after residual), optional ReLU
    __half* out_lo;         // lo plane (exact mode) or null
    int out_pitch, out_choff, out_relu;
    __half* out2_hi;        // second, un-ReLU'd copy (skip connection) or null
    __half* out2_lo;
    int out2_pitch, out2_choff;
    // stage 1 in split-fp16 mode keeps its activations in fp32 (same bytes as hi + lo planes; the RIC producers blend in fp32
    // anyway and split after the blend): when non-null these replace out_hi/out_lo and out2_hi/out2_lo (same pitch / choff)
    float* out_f32;
    float* out2_f32;
    // fused conv_12 (1x1, +bias, optional tanh) tail
    const float* w12;       // [3][Cout] or null
    const float* b12;       // [3]
    int tanh_flag;
    float* y_nchw;          // [B,3,H,W] fp32 or null
    uint8_t* y_rgba;        // [B,H,W,4] uint8 or null (to_image_space + alpha)
    const uint8_t* alpha_src;   // alpha byte of pixel p at alpha_src[p * alpha_stride]
    int alpha_stride;
};

struct ConvParams {
    int B, Hout, Wout;      // output geometry
    int Hin, Win;           // source buffer geometry (before the fused nearest x2)
    int Hv, Wv;             // virtual conv-input geometry = (Hin << up, Win << up)
    int stride, up, ric, exact;
    int nchunks, nblocks, Cout;
    int b_bytes;            // bytes per B stage = Cout x 128 (one chunk's weight tile in wpack)
    // K-step masks (ChunkHdr semantics) as launch constants so the issuing warpgroups stay uniform:
    // every chunk uses *_full except the ragged tail (tap mode: the last chunk; RIC: all chunks of the last
    // channel block), which uses *_last
    uint32_t kmask_full, kmask_last, kmask2_full, kmask2_last;
    const Slot* slots;      // plain: [nchunks][8]; RIC: [nblocks][8]
    const uint8_t* wpack;   // pre-swizzled B tiles
    Seg seg[kMaxSeg];
    // RIC stencil of the output level, per pixel: octant (tap rotation) and, in rotated tap
    // order m = (octant + k) & 7, the bilinear fractions (ly, lx) relative to the static quadrant of m
    const float2* ric_lyx;  // [Hout*Wout][8]
    const uint8_t* ric_oct; // [Hout*Wout]
    const uint2* ric_wh;    // [Hout*Wout][8] the 4 bilinear weights of each rotated tap as fp16 {w00,w01 | w10,w11} (packed-half2 blend)
    EpiParams epi;
    // sub-pixel class of a fused nearest-x2 + 3x3 convolution: the launch is a 2x2 convolution over the LOW-resolution
    // source whose output pixel (oy, ox) of the Hout x Wout grid lands at (2*oy + sub_py, 2*ox + sub_px) of the
    // (2*Hout) x (2*Wout) output buffer
    int sub, sub_py, sub_px;
    // first layer (one 8-channel segment, stride 1): stage the (kTileH + ksize - 1) x (kTileW + ksize - 1) input halo of the
    // tile once in shared memory and build every A chunk from it instead of from global memory
    int halo, ksize, pad;
    int n128;               // Cout a multiple of 128: issue N = 128 wgmma instructions (else N = 64 / 32)
};

cudaError_t launch_conv(const ConvParams& p, cudaStream_t stream);
size_t conv_smem_bytes(const ConvParams& p);

}  // namespace dsu
