// Fused convolution as an implicit GEMM on the Hopper tensor cores (wgmma, fp32 accumulators in registers).
//
// One CTA computes a kTileH x kTileW patch (128 output pixels = GEMM M) of one frame for all Cout channels (GEMM N).
// K = taps x input channels, walked in 64-element chunks through a kStages-deep ring of shared-memory stages; each
// stage holds the A operand (one 128-byte SWIZZLE_128B row per output pixel) and the chunk's pre-swizzled weight tile
// (B operand, one 128-byte row per output channel).  Both warpgroups (256 threads) do everything in turn:
//   * PRODUCE chunk q + 2 while the MMAs of chunk q run.  Each 16-byte slot of an A row is 8 channels of one tap of one
//     concat segment (slot table), so plain 3x3 / 7x7 taps, stride 2, fused nearest-x2 upsampling, sub-pixel classes
//     and channel concatenation are pure address arithmetic (cp.async with zero fill at the border).  The first layer
//     (one 8-channel segment, stride 1) stages the tile's input halo in shared memory once and builds its A chunks from
//     there (49 taps of the 7x7 conv0 read each input pixel 49 times).  RIC (stage-1
//     deformable) layers blend the four bilinear corners of the rotated tap in registers and store the result.
//     The weight tile is streamed with cp.async.
//   * ISSUE wgmma: warpgroup w multiplies A rows 64w .. 64w+63 by the whole weight tile into its register accumulators.
//   * after the last chunk, STAGE the accumulators to shared memory as fp32 rows and run the fused epilogue: folded BN /
//     activation / residual, fp16 NHWC (hi [+lo] planes), fp32 activations, the fp32 residual stream, or the conv_12
//     1x1 + tanh + uint8 composite tail (one pixel row per thread, two threads per row).
// "Exact" mode (split fp16): a K chunk holds 32 channels as [a_hi | a_lo], its weight tile [W_hi | W_lo] in one
// 128-byte row; A steps 0-3 are issued against B steps 0,1,0,1 and A steps 0,1 again against B steps 2,3 into the
// same accumulator: a_hi*W_hi + a_lo*W_hi + a_hi*W_lo, fp32-grade products at 3x the tensor work.
#include "conv_device.cuh"

namespace dsu {

namespace {

constexpr int kModeTap = 0, kModeRic = 1, kModeRicExact = 2, kModeHalo = 3;

struct SmemLayout {
    uint32_t stage_bytes;   // A tile + B tile
    uint32_t par;           // epilogue parameters, after the ring (the staged accumulators reuse the ring)
    uint32_t halo;          // first-layer input halo (hi plane, then the lo plane in exact mode)
    uint32_t total;         // from the 1024-aligned base
};

// pixels of the first-layer halo of one tile
__host__ __device__ inline int halo_pixels(int ksize) { return (kTileH + ksize - 1) * (kTileW + ksize - 1); }

__host__ __device__ inline uint32_t acc_pitch(int cout) { return static_cast<uint32_t>(cout) + 4; }   // floats per staged row

__host__ __device__ inline SmemLayout smem_layout(int cout, int b_bytes, uint32_t halo_bytes) {
    SmemLayout L;
    L.stage_bytes = kABytes + b_bytes;
    const uint32_t ring = kStages * L.stage_bytes, staged = kTileM * acc_pitch(cout) * 4;
    L.par = ((ring > staged ? ring : staged) + 15u) & ~15u;
    L.halo = (L.par + (7 * cout + 4) * 4 + 15u) & ~15u;
    L.total = L.halo + halo_bytes;
    return L;
}

__host__ __device__ inline uint32_t halo_bytes(const ConvParams& p) {
    return p.halo ? static_cast<uint32_t>(halo_pixels(p.ksize)) * 16u * (p.exact ? 2u : 1u) : 0u;
}

// ---- first layer: the tile's (kTileH + k - 1) x (kTileW + k - 1) input pixels (8 channels, hi [+ lo] plane) with cp.async,
// zeros outside the image.  Every slot of the single segment reads the same 8 channels (choff of slot 0).
__device__ __forceinline__ void load_halo(const ConvParams& p, uint32_t halo, int tid, int n, int ty0, int tx0) {
    const int hw = kTileW + p.ksize - 1, npix = halo_pixels(p.ksize);
    const size_t frame_in = static_cast<size_t>(n) * p.Hin * p.Win;
    const int choff = p.slots[0].choff;
    for (int i = tid; i < npix * (p.exact ? 2 : 1); i += kThreads) {
        const int plane = i >= npix, pix = i - plane * npix;
        const int y = ty0 - p.pad + pix / hw, x = tx0 - p.pad + pix % hw;
        const bool ok = static_cast<unsigned>(y) < static_cast<unsigned>(p.Hin) && static_cast<unsigned>(x) < static_cast<unsigned>(p.Win);
        const Seg sg = p.seg[plane ? kMaxSeg / 2 : 0];
        const __half* src = sg.ptr + choff + (ok ? (frame_in + static_cast<size_t>(y) * p.Win + x) * sg.pitch : 0);
        cp_async16(halo + 16u * i, src, ok ? 16u : 0u);
    }
}

// ---- first layer: chunk q's A rows copied out of the halo (same slot table and row mapping as tap mode)
__device__ __forceinline__ void produce_halo(const ConvParams& p, int q, uint32_t a, uint32_t halo, int tid) {
    const int j = tid & 7, prow = tid >> 3;
    const Slot sl = p.slots[q * 8 + j];
    const int hw = kTileW + p.ksize - 1;
    const uint32_t plane = sl.seg >= kMaxSeg / 2 ? static_cast<uint32_t>(halo_pixels(p.ksize)) * 16u : 0u;
    const uint32_t dst0 = a + static_cast<uint32_t>(prow) * 128u + (static_cast<uint32_t>(j ^ (prow & 7)) << 4);
    const int hx = (prow & 15) + sl.dx + p.pad;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int hy = (prow >> 4) + 2 * i + sl.dy + p.pad;
        const uint4 v = sl.valid ? ld_shared_v4(halo + plane + 16u * static_cast<uint32_t>(hy * hw + hx)) : make_uint4(0u, 0u, 0u, 0u);
        st_shared_v4(dst0 + i * 4096u, v);
    }
}

__device__ __forceinline__ constexpr int ric_r0(int m) { return (m >= 2 && m <= 5) ? 0 : 1; }   // first corner row - 1 + 1
__device__ __forceinline__ constexpr int ric_c0(int m) { return (m >= 4) ? 0 : 1; }

// ---- tap mode: chunk q's A rows with cp.async (zero fill outside the image / for K padding)
__device__ __forceinline__ void produce_tap(const ConvParams& p, int q, uint32_t a, int tid, int n, int ty0, int tx0) {
    const int j = tid & 7;          // slot (16 B column) of the row
    const int prow = tid >> 3;      // 0..31; item i covers row prow + 32*i
    const Slot sl = p.slots[q * 8 + j];
    const Seg sg = p.seg[sl.seg];
    const __half* sbase = sg.ptr + sl.choff;
    const uint32_t dst0 = a + static_cast<uint32_t>(prow) * 128u + (static_cast<uint32_t>(j ^ (prow & 7)) << 4);
    const size_t frame_in = static_cast<size_t>(n) * p.Hin * p.Win;
    const int ox = tx0 + (prow & 15), oy0 = ty0 + (prow >> 4);
    const int vx = ox * p.stride + sl.dx;
    const bool okx = sl.valid && static_cast<unsigned>(vx) < static_cast<unsigned>(p.Wv);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int vy = (oy0 + 2 * i) * p.stride + sl.dy;
        const bool ok = okx && static_cast<unsigned>(vy) < static_cast<unsigned>(p.Hv);
        const size_t pix = frame_in + static_cast<size_t>(vy >> p.up) * p.Win + (vx >> p.up);
        cp_async16(dst0 + i * 4096u, ok ? sbase + pix * sg.pitch : sbase, ok ? 16u : 0u);
    }
}

// ---- RIC: chunk q = (channel block q / 9, tap q % 9).  torchvision's deform_conv2d bilinear rule with the engine's
// stencil tables: tap t != 4 samples the 2x2 corner set of its rotated sector m at fractions (ly, lx); corners outside
// the (virtual, nearest-x2) image read as zero.  Same operation order as the reference port of the weights:
// w00*n00, then fma w01*n01, w10*n10, w11*n11.
template <bool kExact>
__device__ __forceinline__ void produce_ric(const ConvParams& p, int q, uint32_t a, int tid, int n, int ty0, int tx0) {
    const int blk = q / 9, t = q - 9 * blk;
    const int kq = t < 4 ? t : t - 1;                     // circle index of a rotated tap
    const size_t frame_in = static_cast<size_t>(n) * p.Hin * p.Win;
    // fp16: one item = (row, slot j), 4 rows per thread; split-fp16: one item = (row, data slot d) -> hi slot d, lo slot d + 4
    constexpr int kSlots = kExact ? 4 : 8, kRowsPer = kExact ? 2 : 4, kRowStep = kTileM / kRowsPer;
    const int d = tid % kSlots, prow = tid / kSlots;
    const Slot sl = p.slots[blk * 8 + d];
    const Seg sg = p.seg[sl.seg];
#pragma unroll
    for (int i = 0; i < kRowsPer; ++i) {
        const int r = prow + kRowStep * i;
        const int oy = ty0 + (r >> 4), ox = tx0 + (r & 15);
        const bool live = sl.valid && oy < p.Hout && ox < p.Wout;
        const size_t e = live ? static_cast<size_t>(oy) * p.Wout + ox : 0;
        int dy0 = 0, dx0 = 0, m = 0;
        if (t != 4) {
            m = (kq + __ldg(p.ric_oct + e)) & 7;
            dy0 = ric_r0(m) - 1; dx0 = ric_c0(m) - 1;
        }
        // corner (cy, cx) of the sample -> pointer into the source (null when outside the image)
        auto corner = [&](int cy, int cx, bool& ok) {
            const int vy = oy + dy0 + cy, vx = ox + dx0 + cx;
            ok = live && static_cast<unsigned>(vy) < static_cast<unsigned>(p.Hv) && static_cast<unsigned>(vx) < static_cast<unsigned>(p.Wv);
            return ok ? frame_in + static_cast<size_t>(vy >> p.up) * p.Win + (vx >> p.up) : 0;
        };
        const uint32_t row = a + static_cast<uint32_t>(r) * 128u;
        const uint32_t swz = static_cast<uint32_t>(r & 7);
        if constexpr (!kExact) {
            const __half* src = sg.ptr + sl.choff;
            uint4 out;
            if (t == 4) {
                bool ok;
                const size_t pix = corner(0, 0, ok);
                out = ldg128_if(src + pix * sg.pitch, ok);
            } else {
                const uint2 wv = live ? __ldg(p.ric_wh + e * 8 + m) : make_uint2(0u, 0u);
                const __half2 wa = *reinterpret_cast<const __half2*>(&wv.x), wb = *reinterpret_cast<const __half2*>(&wv.y);
                const __half2 w00 = __low2half2(wa), w01 = __high2half2(wa), w10 = __low2half2(wb), w11 = __high2half2(wb);
                bool k00, k01, k10, k11;
                const size_t p00 = corner(0, 0, k00), p01 = corner(0, 1, k01), p10 = corner(1, 0, k10), p11 = corner(1, 1, k11);
                const uint4 n00 = ldg128_if(src + p00 * sg.pitch, k00), n01 = ldg128_if(src + p01 * sg.pitch, k01);
                const uint4 n10 = ldg128_if(src + p10 * sg.pitch, k10), n11 = ldg128_if(src + p11 * sg.pitch, k11);
                const __half2* h00 = reinterpret_cast<const __half2*>(&n00);
                const __half2* h01 = reinterpret_cast<const __half2*>(&n01);
                const __half2* h10 = reinterpret_cast<const __half2*>(&n10);
                const __half2* h11 = reinterpret_cast<const __half2*>(&n11);
                __half2* o = reinterpret_cast<__half2*>(&out);
#pragma unroll
                for (int c = 0; c < 4; ++c) o[c] = __hfma2(w11, h11[c], __hfma2(w10, h10[c], __hfma2(w01, h01[c], __hmul2(w00, h00[c]))));
            }
            st_shared_v4(row + ((static_cast<uint32_t>(d) ^ swz) << 4), out);
        } else {
            // split-fp16 stage 1 keeps fp32 activations: 8 channels = two 16-byte loads per corner
            const float* src = reinterpret_cast<const float*>(sg.ptr) + sl.choff;
            float f[8];
            auto load8 = [&](size_t pix, bool ok, float* v) {
                const uint4 lo = ldg128_if(src + pix * sg.pitch, ok), hi = ldg128_if(src + pix * sg.pitch + 4, ok);
                v[0] = __uint_as_float(lo.x); v[1] = __uint_as_float(lo.y); v[2] = __uint_as_float(lo.z); v[3] = __uint_as_float(lo.w);
                v[4] = __uint_as_float(hi.x); v[5] = __uint_as_float(hi.y); v[6] = __uint_as_float(hi.z); v[7] = __uint_as_float(hi.w);
            };
            if (t == 4) {
                bool ok;
                const size_t pix = corner(0, 0, ok);
                load8(pix, ok, f);
            } else {
                const float2 l = live ? __ldg(p.ric_lyx + e * 8 + m) : make_float2(0.0f, 0.0f);
                const float hy = 1.0f - l.x, hx = 1.0f - l.y;
                const float w0 = __fmul_rn(hy, hx), w1 = __fmul_rn(hy, l.y), w2 = __fmul_rn(l.x, hx), w3 = __fmul_rn(l.x, l.y);
                bool k00, k01, k10, k11;
                const size_t p00 = corner(0, 0, k00), p01 = corner(0, 1, k01), p10 = corner(1, 0, k10), p11 = corner(1, 1, k11);
                float v00[8], v01[8], v10[8], v11[8];
                load8(p00, k00, v00); load8(p01, k01, v01); load8(p10, k10, v10); load8(p11, k11, v11);
#pragma unroll
                for (int c = 0; c < 8; ++c) f[c] = __fmaf_rn(w3, v11[c], __fmaf_rn(w2, v10[c], __fmaf_rn(w1, v01[c], __fmul_rn(w0, v00[c]))));
            }
            uint4 hi, lo;
            split8(f, hi, lo);
            st_shared_v4(row + ((static_cast<uint32_t>(d) ^ swz) << 4), hi);
            st_shared_v4(row + ((static_cast<uint32_t>(d + 4) ^ swz) << 4), lo);
        }
    }
}

template <int kMode>
__device__ __forceinline__ void produce(const ConvParams& p, int q, uint32_t stage, uint32_t halo, int tid, int n, int ty0, int tx0) {
    if constexpr (kMode == kModeTap) produce_tap(p, q, stage, tid, n, ty0, tx0);
    else if constexpr (kMode == kModeHalo) produce_halo(p, q, stage, halo, tid);
    else produce_ric<kMode == kModeRicExact>(p, q, stage, tid, n, ty0, tx0);
    // weight tile of chunk q
    const uint8_t* src = p.wpack + static_cast<size_t>(q) * p.b_bytes;
    for (int i = tid; i < p.b_bytes / 16; i += kThreads) cp_async16(stage + kABytes + 16u * i, src + 16 * i, 16u);
}

// the K steps of one chunk: every PN-column piece of the accumulator against the matching PN rows of the weight tile
template <int NC, int PN>
__device__ __forceinline__ void mma_chunk(float* acc, uint64_t da, uint64_t db, uint32_t km, uint32_t km2) {
    constexpr uint64_t kPieceStep = PN * 128 / 16;        // descriptor units between PN-row weight pieces
    auto step = [&](int ka, int kb) {
#pragma unroll
        for (int j = 0; j < NC / PN; ++j) Wgmma<PN>::mma(acc + j * (PN / 2), da + 2 * ka, db + 2 * kb + j * kPieceStep);
    };
    if (km2) {
        // split-fp16: A = [a_hi | a_lo] (steps 0-1 | 2-3), B = [W_hi | W_lo]; a_hi*W_hi + a_lo*W_hi + a_hi*W_lo
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if ((km >> k) & 1) step(k, k & 1);
#pragma unroll
        for (int k = 0; k < 2; ++k)
            if ((km2 >> k) & 1) step(k, 2 + k);
    } else {
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if ((km >> k) & 1) step(k, k);
    }
}

}  // namespace

// NC = Cout, PN = wgmma N per instruction (a divisor of NC: 32, 64 or 128)
template <int NC, int PN, int kMode>
__global__ void __launch_bounds__(kThreads, 1)
conv_wgmma_kernel(const __grid_constant__ ConvParams p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw_u32 = smem_u32(smem_raw);
    const uint32_t base = (raw_u32 + 1023u) & ~1023u;     // SWIZZLE_128B atoms are 1024-byte aligned
    uint8_t* smem = smem_raw + (base - raw_u32);
    const SmemLayout L = smem_layout(NC, p.b_bytes, halo_bytes(p));
    const uint32_t halo = base + L.halo;
    float* s_par = reinterpret_cast<float*>(smem + L.par);

    const int tid = threadIdx.x;
    const int wg = tid >> 7;
    const int n = blockIdx.z;
    const int ty0 = blockIdx.y * kTileH;
    const int tx0 = blockIdx.x * kTileW;
    const int nq = p.nchunks;
    // chunks with the ragged K tail: the last one (tap / halo mode) or the 9 taps of the last channel block (RIC)
    const int tail_from = (kMode == kModeRic || kMode == kModeRicExact) ? (p.nblocks - 1) * 9 : nq - 1;

    load_epilogue_params(p, s_par, tid, kThreads);

    float acc[NC / 2];
#pragma unroll
    for (int i = 0; i < NC / 2; ++i) acc[i] = 0.0f;

    if constexpr (kMode == kModeHalo) {                   // the halo must be complete before any chunk is built from it
        load_halo(p, halo, tid, n, ty0, tx0);
        cp_async_commit();
        cp_async_wait<0>();
        __syncthreads();
    }
    // prologue: chunks 0 and 1; every iteration commits one cp.async group so that "chunk q has landed" is wait_group 1
#pragma unroll
    for (int s = 0; s < kStages - 2; ++s) {
        if (s < nq) produce<kMode>(p, s, base + s * L.stage_bytes, halo, tid, n, ty0, tx0);
        cp_async_commit();
    }
    for (int q = 0; q < nq; ++q) {
        cp_async_wait<kStages - 3>();
        fence_proxy_async_smem();
        __syncthreads();                                  // chunk q is in shared memory; the MMAs of chunk q - 2 have retired
        const uint32_t stage = base + (q % kStages) * L.stage_bytes;
        const uint64_t da = wgmma_desc_sw128(stage + wg * (kABytes / 2), 1024), db = wgmma_desc_sw128(stage + kABytes, 1024);
        const bool tail = q >= tail_from;
        wgmma_fence();
        mma_chunk<NC, PN>(acc, da, db, tail ? p.kmask_last : p.kmask_full, tail ? p.kmask2_last : p.kmask2_full);
        wgmma_commit();
        wgmma_wait<1>();                                  // this warpgroup's MMAs of chunk q - 1 have retired
        if (q + kStages - 2 < nq) produce<kMode>(p, q + kStages - 2, base + ((q + kStages - 2) % kStages) * L.stage_bytes, halo, tid, n, ty0, tx0);
        cp_async_commit();
    }
    wgmma_wait<0>();
    cp_async_wait<0>();
    __syncthreads();                                      // the ring is free: stage the accumulators over it

    {
        float* staged = reinterpret_cast<float*>(smem);
        const int w = (tid >> 5) & 3, l = tid & 31;
        const int r0 = wg * 64 + 16 * w + (l >> 2), c0 = 2 * (l & 3);
#pragma unroll
        for (int i = 0; i < NC / 2; i += 2) {
            const int r = r0 + 8 * ((i >> 1) & 1), c = c0 + 8 * (i >> 2);
            *reinterpret_cast<float2*>(staged + r * acc_pitch(NC) + c) = make_float2(acc[i], acc[i + 1]);
        }
    }
    __syncthreads();
    {
        const int r = tid & (kTileM - 1);                 // patch pixel; two threads per row split the 32-column batches
        const float* row = reinterpret_cast<const float*>(smem) + r * acc_pitch(NC);
        if (p.sub) epilogue_row<kEpiAll, true>(p, s_par, row, n, ty0 + (r >> 4), tx0 + (r & 15), tid >> 7);
        else epilogue_row<kEpiAll, false>(p, s_par, row, n, ty0 + (r >> 4), tx0 + (r & 15), tid >> 7);
    }
}

size_t conv_smem_bytes(const ConvParams& p) {
    return smem_layout(p.Cout, p.b_bytes, halo_bytes(p)).total + 1024;
}

namespace {

template <int NC, int PN, int kMode>
cudaError_t launch_nc(const ConvParams& p, cudaStream_t stream) {
    // one flag per device: the attribute is per function and context
    static bool attr_set[64] = {};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    const size_t smem = conv_smem_bytes(p);
    if (dev >= 64 || !attr_set[dev]) {
        e = cudaFuncSetAttribute(conv_wgmma_kernel<NC, PN, kMode>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
        if (e != cudaSuccess) return e;
        if (dev < 64) attr_set[dev] = true;
    }
    dim3 grid((p.Wout + kTileW - 1) / kTileW, (p.Hout + kTileH - 1) / kTileH, p.B);
    conv_wgmma_kernel<NC, PN, kMode><<<grid, kThreads, smem, stream>>>(p);
    return cudaGetLastError();
}

template <int kMode>
cudaError_t launch_mode(const ConvParams& p, cudaStream_t stream) {
    switch (p.Cout) {
        case 32: return launch_nc<32, 32, kMode>(p, stream);
        case 64: return launch_nc<64, 64, kMode>(p, stream);
        case 96: return launch_nc<96, 32, kMode>(p, stream);
        case 128: return p.n128 ? launch_nc<128, 128, kMode>(p, stream) : launch_nc<128, 64, kMode>(p, stream);
        default: break;
    }
    if constexpr (kMode != kModeRicExact) {              // split-fp16 configurations stop at 128 channels (engine.cu dsu_create)
        switch (p.Cout) {
            case 160: return launch_nc<160, 32, kMode>(p, stream);
            case 192: return launch_nc<192, 64, kMode>(p, stream);
            case 224: return launch_nc<224, 32, kMode>(p, stream);
            case 256: return p.n128 ? launch_nc<256, 128, kMode>(p, stream) : launch_nc<256, 64, kMode>(p, stream);
            default: break;
        }
    }
    return cudaErrorInvalidConfiguration;
}

}  // namespace

cudaError_t launch_conv(const ConvParams& p, cudaStream_t stream) {
    if (conv_smem_bytes(p) > 227 * 1024 || p.b_bytes != p.Cout * 128) return cudaErrorInvalidConfiguration;
    if (p.halo) return launch_mode<kModeHalo>(p, stream);
    if (!p.ric) return launch_mode<kModeTap>(p, stream);
    return p.exact ? launch_mode<kModeRicExact>(p, stream) : launch_mode<kModeRic>(p, stream);
}

}  // namespace dsu
