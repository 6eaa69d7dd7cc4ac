// Device helpers shared by the convolution kernels: fp16 pack/split, the exact uint8 conversion and
// the fused epilogue (accumulator row -> BN/activation/residual -> fp16 NHWC / fp32 / uint8).
#pragma once
#include "conv.cuh"
#include "ptx.cuh"

namespace dsu {

__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float2 unpack_h2(uint32_t v) {
    return __half22float2(*reinterpret_cast<const __half2*>(&v));
}
__device__ __forceinline__ void unpack8(const uint4& raw, float* f) {
    float2 a = unpack_h2(raw.x), b = unpack_h2(raw.y), c = unpack_h2(raw.z), d = unpack_h2(raw.w);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
// 8 fp32 -> packed fp16 hi and residual lo = fp16(v - hi)
__device__ __forceinline__ void split8(const float* f, uint4& hi, uint4& lo) {
    hi.x = pack_h2(f[0], f[1]); hi.y = pack_h2(f[2], f[3]); hi.z = pack_h2(f[4], f[5]); hi.w = pack_h2(f[6], f[7]);
    float r[8];
    unpack8(hi, r);
    lo.x = pack_h2(f[0] - r[0], f[1] - r[1]); lo.y = pack_h2(f[2] - r[2], f[3] - r[3]);
    lo.z = pack_h2(f[4] - r[4], f[5] - r[5]); lo.w = pack_h2(f[6] - r[6], f[7] - r[7]);
}

// exact fp32 -> uint8 of custom_transforms.py:7-8: ((clip(x,-1,1)+1)/2*255) truncated, fp32 ops in order
__device__ __forceinline__ uint8_t to_u8(float x) {
    x = fminf(fmaxf(x, -1.0f), 1.0f);
    float t = __fmul_rn(__fmul_rn(__fadd_rn(x, 1.0f), 0.5f), 255.0f);
    return static_cast<uint8_t>(static_cast<int>(t));
}

// epilogue parameters in shared memory: [scale C][shift C][scale2 C][shift2 C][w12 3C][b12 4]
__device__ __forceinline__ void load_epilogue_params(const ConvParams& p, float* s_par, int tid, int nthreads) {
    const int C = p.Cout;
    for (int i = tid; i < C; i += nthreads) {
        s_par[i] = p.epi.scale[i];
        s_par[C + i] = p.epi.shift[i];
        s_par[2 * C + i] = p.epi.scale2 ? p.epi.scale2[i] : 1.0f;
        s_par[3 * C + i] = p.epi.shift2 ? p.epi.shift2[i] : 0.0f;
        if (p.epi.w12) {
            s_par[4 * C + i] = p.epi.w12[i];
            s_par[5 * C + i] = p.epi.w12[C + i];
            s_par[6 * C + i] = p.epi.w12[2 * C + i];
        }
    }
    if (p.epi.w12 && tid < 3) s_par[7 * C + tid] = p.epi.b12[tid];
}

// 8 fp32 -> packed fp16 (hi plane only)
__device__ __forceinline__ uint4 pack8(const float* f) {
    return make_uint4(pack_h2(f[0], f[1]), pack_h2(f[2], f[3]), pack_h2(f[4], f[5]), pack_h2(f[6], f[7]));
}

// 32 channels of one pixel -> fp16 NHWC (hi plane, plus the split-fp16 lo plane when kLo and `lo` is non-null)
template <bool kLo>
__device__ __forceinline__ void store32(__half* hi, __half* lo, const float* f) {
    if (kLo && lo) {
        uint4 h[4], l[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) split8(f + 8 * c, h[c], l[c]);
#pragma unroll
        for (int c = 0; c < 4; ++c) { reinterpret_cast<uint4*>(hi)[c] = h[c]; reinterpret_cast<uint4*>(lo)[c] = l[c]; }
    } else {
#pragma unroll
        for (int c = 0; c < 4; ++c) reinterpret_cast<uint4*>(hi)[c] = pack8(f + 8 * c);
    }
}

// 32 channels of one pixel -> fp32 NHWC (stage-1 activations of the split-fp16 mode)
__device__ __forceinline__ void store32_f32(float* dst, const float* f) {
#pragma unroll
    for (int c = 0; c < 8; ++c) reinterpret_cast<float4*>(dst)[c] = make_float4(f[4 * c], f[4 * c + 1], f[4 * c + 2], f[4 * c + 3]);
}

// One 32-column batch of one accumulator row after the K-split partial sums were added: folded BN / bias, activation,
// optional post-activation affine, residual stream, fp16 stores, conv_12 partial dot products.  The activation, the
// second affine and the lo plane are compile-time (dispatched once per row in epilogue_row), which keeps run-time tests
// out of the 32-element loops.
template <int kAct, int kScale2, bool kLo>   // kAct / kScale2 = -1: decided at run time (cold generic variant)
__device__ __forceinline__ void epilogue_batch(const ConvParams& p, const float* s_par, const float* v, size_t opix, int cb,
                                               bool tail, float* y3) {
    const EpiParams& e = p.epi;
    const int C = p.Cout;
    float f[32];
    {
        const float4* sc = reinterpret_cast<const float4*>(s_par + cb);
        const float4* sh = reinterpret_cast<const float4*>(s_par + C + cb);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const float4 a = sc[q], b = sh[q];
            f[4 * q] = fmaf(v[4 * q], a.x, b.x);
            f[4 * q + 1] = fmaf(v[4 * q + 1], a.y, b.y);
            f[4 * q + 2] = fmaf(v[4 * q + 2], a.z, b.z);
            f[4 * q + 3] = fmaf(v[4 * q + 3], a.w, b.w);
        }
    }
    const int act = kAct >= 0 ? kAct : e.act;
    if (act == 1) {
#pragma unroll
        for (int c = 0; c < 32; ++c) f[c] = fmaxf(f[c], 0.0f);
    } else if (act == 2) {           // LeakyReLU(0.2): max(x, 0.2 x) == (x > 0 ? x : 0.2 x) for every input
#pragma unroll
        for (int c = 0; c < 32; ++c) f[c] = fmaxf(f[c], 0.2f * f[c]);
    }
    if (kScale2 > 0 || (kScale2 < 0 && e.scale2)) {
        const float4* sc = reinterpret_cast<const float4*>(s_par + 2 * C + cb);
        const float4* sh = reinterpret_cast<const float4*>(s_par + 3 * C + cb);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const float4 a = sc[q], b = sh[q];
            f[4 * q] = fmaf(f[4 * q], a.x, b.x);
            f[4 * q + 1] = fmaf(f[4 * q + 1], a.y, b.y);
            f[4 * q + 2] = fmaf(f[4 * q + 2], a.z, b.z);
            f[4 * q + 3] = fmaf(f[4 * q + 3], a.w, b.w);
        }
    }
    if (e.resid_in) {
        const float4* rp = reinterpret_cast<const float4*>(e.resid + opix * C + cb);
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const float4 rv = rp[c];
            f[4 * c] += rv.x; f[4 * c + 1] += rv.y; f[4 * c + 2] += rv.z; f[4 * c + 3] += rv.w;
        }
    }
    if (e.resid_out) {
        float4* rp = reinterpret_cast<float4*>(e.resid + opix * C + cb);
#pragma unroll
        for (int c = 0; c < 8; ++c) rp[c] = make_float4(f[4 * c], f[4 * c + 1], f[4 * c + 2], f[4 * c + 3]);
    }
    if (e.out2_f32) store32_f32(e.out2_f32 + opix * e.out2_pitch + e.out2_choff + cb, f);
    else if (e.out2_hi)
        store32<kLo>(e.out2_hi + opix * e.out2_pitch + e.out2_choff + cb,
                     e.out2_lo ? e.out2_lo + opix * e.out2_pitch + e.out2_choff + cb : nullptr, f);
    if (e.out_relu) {
#pragma unroll
        for (int c = 0; c < 32; ++c) f[c] = fmaxf(f[c], 0.0f);
    }
    if (e.out_f32) store32_f32(e.out_f32 + opix * e.out_pitch + e.out_choff + cb, f);
    else if (e.out_hi)
        store32<kLo>(e.out_hi + opix * e.out_pitch + e.out_choff + cb,
                     e.out_lo ? e.out_lo + opix * e.out_pitch + e.out_choff + cb : nullptr, f);
    if (tail) {
#pragma unroll
        for (int c = 0; c < 32; ++c) {
            y3[0] = fmaf(f[c], s_par[4 * C + cb + c], y3[0]);
            y3[1] = fmaf(f[c], s_par[5 * C + cb + c], y3[1]);
            y3[2] = fmaf(f[c], s_par[6 * C + cb + c], y3[2]);
        }
    }
}

// One accumulator row (= one output pixel, all Cout columns) per thread, read from the fp32 row `acc` the MMA
// warpgroups staged in shared memory.  The `csplit` threads that share a row (chalf 0 .. csplit-1) split the 32-column
// batches; the conv_12 tail needs a whole row in one thread, so only chalf 0 runs it.
constexpr uint32_t kEpiAll = 0xFFFFu;   // variant mask (bit = variant index)
template <uint32_t kMask = kEpiAll, bool kSub = false>
__device__ __forceinline__ void epilogue_row(const ConvParams& p, const float* s_par, const float* acc,
                                             int n, int oy, int ox, int chalf, int csplit = 2) {
    const EpiParams& e = p.epi;
    const int C = p.Cout;
    const bool pix_ok = oy < p.Hout && ox < p.Wout;
    // kSub: (oy, ox) index the low-resolution grid of one sub-pixel class; the output buffer is twice as large in y and x
    const size_t opix = kSub ? (static_cast<size_t>(n) * (2 * p.Hout) + (2 * oy + p.sub_py)) * (2 * p.Wout) + (2 * ox + p.sub_px)
                             : (static_cast<size_t>(n) * p.Hout + oy) * p.Wout + ox;
    const int ncb = C / 32;
    const bool tail = e.w12 != nullptr;
    const int cb_first = tail ? 0 : chalf, cb_step = tail ? 1 : csplit;
    const bool active = tail ? (chalf == 0) : (chalf < ncb);
    if (!active || !pix_ok) return;
    // uniform variant index: activation | second affine | lo plane
    const int variant = e.act | (e.scale2 ? 4 : 0) | ((e.out_lo || e.out2_lo) ? 8 : 0);
    float y3[3] = {0.0f, 0.0f, 0.0f};
    for (int cbi = cb_first; cbi < ncb; cbi += cb_step) {
        const int cb = cbi * 32;
        float v[32];
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const float4 a = reinterpret_cast<const float4*>(acc + cb)[c];
            v[4 * c] = a.x; v[4 * c + 1] = a.y; v[4 * c + 2] = a.z; v[4 * c + 3] = a.w;
        }
        // variants the planner emits (engine.cu build_plan): act 0/1/2, second affine only with ReLU (conv_11_a.2), +8 = lo plane;
        // kMask limits what a kernel instantiates (code size), anything else runs the cold run-time variant
#define DSU_EPI_CASE(N, A, S2, LO)                                                                                        \
    case N:                                                                                                               \
        if constexpr ((kMask >> N) & 1u) { epilogue_batch<A, S2, LO>(p, s_par, v, opix, cb, tail, y3); handled = true; } \
        break;
        bool handled = false;
        switch (variant) {
            DSU_EPI_CASE(0, 0, 0, false)
            DSU_EPI_CASE(1, 1, 0, false)
            DSU_EPI_CASE(2, 2, 0, false)
            DSU_EPI_CASE(5, 1, 1, false)
            DSU_EPI_CASE(8, 0, 0, true)
            DSU_EPI_CASE(9, 1, 0, true)
            DSU_EPI_CASE(10, 2, 0, true)
            DSU_EPI_CASE(13, 1, 1, true)
            default: break;
        }
        if (!handled) epilogue_batch<-1, -1, true>(p, s_par, v, opix, cb, tail, y3);
#undef DSU_EPI_CASE
    }
    if (tail) {
        const size_t plane = static_cast<size_t>(p.Hout) * p.Wout;
        const size_t pin = static_cast<size_t>(oy) * p.Wout + ox;
        uint8_t rgb[3];
#pragma unroll
        for (int o = 0; o < 3; ++o) {
            float yv = y3[o] + s_par[7 * C + o];
            if (e.tanh_flag) yv = tanhf(yv);
            if (e.y_nchw) e.y_nchw[(static_cast<size_t>(n) * 3 + o) * plane + pin] = yv;
            rgb[o] = to_u8(yv);
        }
        if (e.y_rgba) {
            const uint8_t a = e.alpha_src ? e.alpha_src[opix * e.alpha_stride] : 255;
            reinterpret_cast<uchar4*>(e.y_rgba)[opix] = make_uchar4(rgb[0], rgb[1], rgb[2], a);
        }
    }
}

}  // namespace dsu
