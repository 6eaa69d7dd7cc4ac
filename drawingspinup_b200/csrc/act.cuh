// Activation storage: how a value that crosses a kernel boundary sits in HBM (NHWC, DESIGN section 3), and the device
// helpers that convert and store it.  A buffer holds one of five forms, chosen per handle by engine.cu act_out:
//   * fp16, one plane (fp16 mode);
//   * bf16, one plane (bf16 mode): the same 2-byte elements, pitch and padding as the fp16 plane;
//   * fp16 hi = fp16(v) and lo = fp16(v - hi), two planes (split-fp16 stage 2);
//   * bf16 hi = bf16(v) and lo = bf16(v - hi), two planes (split-bf16 stage 2), laid out like the split-fp16 planes;
//   * fp32 (stage 1 of both split modes: the RIC producers blend in fp32 and split after the blend).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

namespace dsu {

// Where a kernel stores channel c of pixel p: element p * pitch + choff + c of `f32` when it is non-null, else of `hi`
// (and of `lo` when non-null).  All null: no store.  `bf16`: the `hi` (and `lo`) plane holds bf16 bits, not fp16.
struct ActOut {
    __half* hi;
    __half* lo;
    float* f32;
    int pitch, choff;
    int bf16;
};

// Two fp32 <-> one 32-bit word of two 16-bit storage elements of type T (__half or __nv_bfloat16), round to nearest even
template <typename T>
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    if constexpr (std::is_same<T, __nv_bfloat16>::value) {
        __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
        return *reinterpret_cast<uint32_t*>(&h);
    } else {
        __half2 h = __floats2half2_rn(a, b);
        return *reinterpret_cast<uint32_t*>(&h);
    }
}
template <typename T>
__device__ __forceinline__ float2 unpack_h2(uint32_t v) {
    if constexpr (std::is_same<T, __nv_bfloat16>::value) return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v));
    else return __half22float2(*reinterpret_cast<const __half2*>(&v));
}
template <typename T>
__device__ __forceinline__ void unpack8(const uint4& raw, float* f) {
    float2 a = unpack_h2<T>(raw.x), b = unpack_h2<T>(raw.y), c = unpack_h2<T>(raw.z), d = unpack_h2<T>(raw.w);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
// 8 fp32 -> packed T (one plane)
template <typename T>
__device__ __forceinline__ uint4 pack8(const float* f) {
    return make_uint4(pack_h2<T>(f[0], f[1]), pack_h2<T>(f[2], f[3]), pack_h2<T>(f[4], f[5]), pack_h2<T>(f[6], f[7]));
}
// 2 fp32 -> packed T hi and residual lo = T(v - hi), T = __half (split fp16) or __nv_bfloat16 (split bf16)
template <typename T>
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
    hi = pack_h2<T>(a, b);
    const float2 r = unpack_h2<T>(hi);
    lo = pack_h2<T>(a - r.x, b - r.y);
}
// 8 fp32 -> packed T hi and residual lo, two channels at a time
template <typename T>
__device__ __forceinline__ void split8(const float* f, uint4& hi, uint4& lo) {
    split2<T>(f[0], f[1], hi.x, lo.x); split2<T>(f[2], f[3], hi.y, lo.y);
    split2<T>(f[4], f[5], hi.z, lo.z); split2<T>(f[6], f[7], hi.w, lo.w);
}

// exact fp32 -> uint8 of custom_transforms.py:7-8: ((clip(x,-1,1)+1)/2*255) truncated, fp32 ops in order
__device__ __forceinline__ uint8_t to_u8(float x) {
    x = fminf(fmaxf(x, -1.0f), 1.0f);
    float t = __fmul_rn(__fmul_rn(__fadd_rn(x, 1.0f), 0.5f), 255.0f);
    return static_cast<uint8_t>(static_cast<int>(t));
}

// N (a multiple of 4) fp32 values -> fp32 at dst
template <int N>
__device__ __forceinline__ void store_f32(float* dst, const float* f) {
#pragma unroll
    for (int c = 0; c < N / 4; ++c) reinterpret_cast<float4*>(dst)[c] = make_float4(f[4 * c], f[4 * c + 1], f[4 * c + 2], f[4 * c + 3]);
}

// N (a multiple of 8) channels of pixel `pix`, starting at channel c of the view, in the view's form.  kLo = false: the
// caller knows there is no lo plane, and the store does not test for one.
template <int N, bool kLo = true>
__device__ __forceinline__ void store_act(const ActOut& o, size_t pix, int c, const float* f) {
    const size_t i = pix * o.pitch + o.choff + c;
    if (o.f32) {
        store_f32<N>(o.f32 + i, f);
    } else if (o.hi) {
        if (kLo && o.lo) {
            uint4 h[N / 8], l[N / 8];
            if (o.bf16) {
#pragma unroll
                for (int q = 0; q < N / 8; ++q) split8<__nv_bfloat16>(f + 8 * q, h[q], l[q]);
            } else {
#pragma unroll
                for (int q = 0; q < N / 8; ++q) split8<__half>(f + 8 * q, h[q], l[q]);
            }
#pragma unroll
            for (int q = 0; q < N / 8; ++q) { reinterpret_cast<uint4*>(o.hi + i)[q] = h[q]; reinterpret_cast<uint4*>(o.lo + i)[q] = l[q]; }
        } else if (o.bf16) {
#pragma unroll
            for (int q = 0; q < N / 8; ++q) reinterpret_cast<uint4*>(o.hi + i)[q] = pack8<__nv_bfloat16>(f + 8 * q);
        } else {
#pragma unroll
            for (int q = 0; q < N / 8; ++q) reinterpret_cast<uint4*>(o.hi + i)[q] = pack8<__half>(f + 8 * q);
        }
    }
}

}  // namespace dsu
