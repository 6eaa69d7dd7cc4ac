// The fused epilogue of the convolution kernels: accumulator row -> BN/activation/residual -> activation stores
// (act.cuh) / fp32 / uint8.
#pragma once
#include "conv.cuh"
#include "ptx.cuh"

namespace dsu {

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

// One 32-column batch of one accumulator row after the K-split partial sums were added: folded BN / bias, activation,
// optional post-activation affine, residual stream, activation stores, conv_12 partial dot products.  The activation, the
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
        const float4* rp = reinterpret_cast<const float4*>(e.resid + opix * e.resid_pitch + cb);
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const float4 rv = rp[c];
            f[4 * c] += rv.x; f[4 * c + 1] += rv.y; f[4 * c + 2] += rv.z; f[4 * c + 3] += rv.w;
        }
    }
    if (e.resid_out) {
        float4* rp = reinterpret_cast<float4*>(e.resid + opix * e.resid_pitch + cb);
#pragma unroll
        for (int c = 0; c < 8; ++c) rp[c] = make_float4(f[4 * c], f[4 * c + 1], f[4 * c + 2], f[4 * c + 3]);
    }
    store_act<32, kLo>(e.out2, opix, cb, f);
    if (e.out_relu) {
#pragma unroll
        for (int c = 0; c < 32; ++c) f[c] = fmaxf(f[c], 0.0f);
    }
    store_act<32, kLo>(e.out, opix, cb, f);
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
// warpgroups staged in shared memory.  The two threads that share a row (chalf 0 / 1) split the 32-column batches; the
// conv_12 tail needs a whole row in one thread, so only chalf 0 runs it.
template <bool kSub>
__device__ __forceinline__ void epilogue_row(const ConvParams& p, const float* s_par, const float* acc,
                                             int n, int oy, int ox, int chalf) {
    const EpiParams& e = p.epi;
    const int C = p.Cout;
    const bool pix_ok = oy < p.Hout && ox < p.Wout;
    // kSub: (oy, ox) index the low-resolution grid of one sub-pixel class; the output buffer is twice as large in y and x
    const size_t opix = kSub ? (static_cast<size_t>(n) * (2 * p.Hout) + (2 * oy + p.sub_py)) * (2 * p.Wout) + (2 * ox + p.sub_px)
                             : (static_cast<size_t>(n) * p.Hout + oy) * p.Wout + ox;
    const int ncb = C / 32;
    const bool tail = e.w12 != nullptr;
    const int cb_first = tail ? 0 : chalf, cb_step = tail ? 1 : 2;
    const bool active = tail ? (chalf == 0) : (chalf < ncb);
    if (!active || !pix_ok) return;
    // uniform variant index: activation | second affine | lo plane
    const int variant = e.act | (e.scale2 ? 4 : 0) | ((e.out.lo || e.out2.lo) ? 8 : 0);
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
        // anything else runs the cold run-time variant
#define DSU_EPI_CASE(N, A, S2, LO) \
    case N: epilogue_batch<A, S2, LO>(p, s_par, v, opix, cb, tail, y3); break;
        switch (variant) {
            DSU_EPI_CASE(0, 0, 0, false)
            DSU_EPI_CASE(1, 1, 0, false)
            DSU_EPI_CASE(2, 2, 0, false)
            DSU_EPI_CASE(5, 1, 1, false)
            DSU_EPI_CASE(8, 0, 0, true)
            DSU_EPI_CASE(9, 1, 0, true)
            DSU_EPI_CASE(10, 2, 0, true)
            DSU_EPI_CASE(13, 1, 1, true)
            default: epilogue_batch<-1, -1, true>(p, s_par, v, opix, cb, tail, y3); break;
        }
#undef DSU_EPI_CASE
    }
    if (tail && e.y_part) {            // one piece of a split conv_12: partial sums only (the final layer is never a sub-pixel class)
        const size_t npix = static_cast<size_t>(p.B) * p.Hout * p.Wout;
#pragma unroll
        for (int o = 0; o < 3; ++o) e.y_part[o * npix + opix] = y3[o];
    } else if (tail) {
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
