// Fused convolution as an implicit GEMM on the Hopper tensor cores (wgmma, fp32 accumulators in registers).
//
// One CTA computes a tile of output pixels (GEMM M) of one frame for all Cout channels (GEMM N), K = taps x input
// channels walked in 64-element chunks.  Two warpgroups (256 threads) do everything in turn.  Two mainloops, one per
// source of the A operand:
//
// conv_wgmma_kernel (Tap and Ric modes: A from global memory): a kTileH x kTileW patch (128 pixels).  Each chunk goes
// through a kStages-deep ring of shared-memory stages holding the A operand (one 128-byte SWIZZLE_128B row per output
// pixel) and the chunk's pre-swizzled weight tile (B operand, one 128-byte row per output channel).
//   * PRODUCE chunk q + 2 while the MMAs of chunk q run.  Tap mode: each 16-byte slot of an A row is 8 channels of one
//     tap of one concat segment (slot table), so stride 2 and fused nearest-x2 upsampling are pure address arithmetic
//     (cp.async with zero fill at the border).  Ric mode (stage-1 deformable layers, the gather producer) loads the four
//     bilinear corners of the rotated tap straight from global memory, blends them in registers and stores the result.
//     The weight tile is streamed with cp.async.
//   * ISSUE wgmma: warpgroup w multiplies A rows 64w .. 64w+63 by the whole weight tile into its register accumulators.
//
// conv_halo_kernel (Halo and RicHalo modes: A from a shared-memory input halo): the concat is walked in channel blocks of
// 128 bytes per pixel (8 groups of 8 channels, or 4 groups as hi + lo in exact mode).  The tile's input halo of a block is
// loaded once with cp.async (double-buffered: block b + 1 lands while the taps of block b run) and every chunk's A
// fragments are built from it straight into registers (wgmma RS form, double-buffered across chunks), so an input pixel
// crosses L2 once per block instead of once per tap, and no A tile passes through shared memory.  Halo mode
// (halo_rows(Cout) x kTileW patch) reads the fragments with ldmatrix; RicHalo mode (8 x 16 patch: the tile +- 1 source
// pixel per block, with the tile's stencil staged once per CTA) blends them from the rotated tap's corners in the halo
// with the same helpers as the gather producer.  Weight tiles stream through a ring of bulk copies on mbarriers (one
// thread issues each tile), and the halos complete on mbarriers too, so the mainloop has no block barrier.
//
// After the last chunk both kernels STAGE the accumulators to shared memory as fp32 rows and run the fused epilogue:
// folded BN / activation / residual, fp16 NHWC (hi [+lo] planes), fp32 activations, the fp32 residual stream, or the
// conv_12 1x1 + tanh + uint8 composite tail (one pixel row per thread, two threads per row).
// "Exact" mode (split fp16): a K chunk holds 32 channels as [a_hi | a_lo], its weight tile [W_hi | W_lo] in one
// 128-byte row; A steps 0-3 are issued against B steps 0,1,0,1 and A steps 0,1 again against B steps 2,3 into the
// same accumulator: a_hi*W_hi + a_lo*W_hi + a_hi*W_lo, fp32-grade products at 3x the tensor work.
// Every kernel takes the element type T of its operands: __half (fp16, split fp16) or __nv_bfloat16 (bf16, single pass
// like fp16, with the same chunks, tiles and launch shapes; only the wgmma type and the RIC blend differ; split bf16, the
// split-fp16 chunks, tiles and shapes with bf16 hi / lo parts: a 16-bit significand with fp32's exponent range).
#pragma once
#include <type_traits>

#include "conv_device.cuh"

namespace dsu {

namespace {

__host__ __device__ constexpr uint32_t acc_pitch(int cout) { return static_cast<uint32_t>(cout) + 4; }   // floats per staged row

__host__ __device__ constexpr uint32_t par_bytes(int cout) { return (7 * cout + 4) * 4; }

// RicHalo mode: every corner of the 3 x 3 neighbourhoods of a tile lies in source rows (ty0 >> up) - 1 .. ((ty0 + kTileH) >> up)
// and columns (tx0 >> up) - 1 .. ((tx0 + kTileW) >> up): 10 x 18 pixels at up = 0, 6 x 10 with the fused nearest x2
__host__ __device__ constexpr int ric_halo_rows(int up) { return (kTileH >> up) + 2; }
__host__ __device__ constexpr int ric_halo_cols(int up) { return (kTileW >> up) + 2; }
constexpr uint32_t kStenBytes = kTileM * 8 * 8;

// Halo mode: output rows per tile.  16 x 16 tiles halve the weight traffic per pixel; above 64 channels the two m64 blocks
// per warpgroup would not fit the register file next to the accumulators, so those layers keep 8 x 16.
__host__ __device__ constexpr int halo_rows(int cout) { return cout <= 64 ? 16 : 8; }

// whether a launch of this mode runs conv_halo_kernel (A fragments built in registers from a shared-memory input halo)
// rather than conv_wgmma_kernel (A tiles gathered from global memory into a shared-memory ring)
__host__ __device__ constexpr bool uses_halo_kernel(ConvMode mode) { return mode == ConvMode::Halo || mode == ConvMode::RicHalo; }

// CTAs per SM a conv_halo_kernel instantiation is built for.  A RicHalo CTA spends most of each chunk building the next
// chunk's fragments and at its barrier, with only two warps per SM sub-partition to hide the shared-memory latency, so the
// tensor cores idle.  Up to 64 channels a second CTA fits: <= 128 registers per thread (launch bounds; ptxas keeps two
// 8-byte values in a 16-byte stack slot) and <= 90 KB of shared memory each (ring 4 x 8 KB, two 22.5 KB halos, 8 KB
// stencil, parameters).
__host__ __device__ constexpr int ric_ctas_per_sm(ConvMode mode, int cout) {
    return mode == ConvMode::RicHalo && cout <= 64 ? 2 : 1;
}

// conv_halo_kernel: deepest weight ring (stages) a launch is given when shared memory allows.  Halo mode streams a weight
// tile per chunk against a few ldmatrix per warp, so it takes up to kMaxRing stages.  RicHalo chunks are bound by building
// the fragments, and a deeper ring measured slower there (DESIGN section 7), so they keep kStages.
constexpr int kMaxRing = 8;
__host__ __device__ constexpr int ring_cap(ConvMode mode) { return mode == ConvMode::Halo ? kMaxRing : kStages; }

constexpr uint32_t kSmemMax = 227u * 1024u;      // dynamic shared memory per CTA (sm_90)

// Shared memory from the 1024-aligned base: a ring of `stages` stages, then (RicHalo / Halo) two input-halo buffers and the
// RicHalo stencil entries ([rotated tap m][tile pixel] x 8 B) or the Halo zero row (16 B, the A rows of K-padding slots), then
// the epilogue parameters and (conv_halo_kernel) the mbarriers.  The staged fp32 accumulators reuse everything before `par`.
struct SmemLayout {
    uint32_t stages;        // ring depth: kStages in conv_wgmma_kernel; conv_halo_kernel: as deep as 227 KB allows, <= ring_cap
    uint32_t stage_bytes;   // A tile + B tile (conv_halo_kernel: B tile only)
    uint32_t halo;          // two input halos of halo_bytes each (halo_bytes = 0 in Tap / Ric mode)
    uint32_t halo_bytes;
    uint32_t aux;           // stencil (RicHalo) or zero row (Halo)
    uint32_t par;
    uint32_t bars;          // conv_halo_kernel: full[stages], empty[stages], halo full[2], halo empty[2] (8 B each)
    uint32_t total;
};

__host__ __device__ constexpr SmemLayout smem_layout_at(ConvMode mode, int cout, int ksize, int up, int stages) {
    const bool halo = mode == ConvMode::Halo, ric_halo = mode == ConvMode::RicHalo;
    const int rows = halo ? halo_rows(cout) : kTileH;
    SmemLayout L{};
    L.stages = static_cast<uint32_t>(stages);
    L.stage_bytes = (uses_halo_kernel(mode) ? 0u : static_cast<uint32_t>(kABytes)) + static_cast<uint32_t>(cout) * 128u;
    L.halo = L.stages * L.stage_bytes;
    L.halo_bytes = halo       ? static_cast<uint32_t>((rows + ksize - 1) * (kTileW + ksize - 1)) * 128u
                   : ric_halo ? static_cast<uint32_t>(ric_halo_rows(up) * ric_halo_cols(up)) * 128u : 0u;
    L.aux = L.halo + 2 * L.halo_bytes;
    const uint32_t main_end = L.aux + (halo ? 16u : ric_halo ? kStenBytes : 0u);
    const uint32_t staged = static_cast<uint32_t>(rows * kTileW) * acc_pitch(cout) * 4u;
    L.par = ((main_end > staged ? main_end : staged) + 15u) & ~15u;
    L.bars = L.par + par_bytes(cout);                    // a multiple of 8
    L.total = L.bars + (uses_halo_kernel(mode) ? (2 * L.stages + 4) * 8u : 0u);
    return L;
}

__host__ __device__ constexpr SmemLayout smem_layout(ConvMode mode, int cout, int ksize, int up) {
    if (!uses_halo_kernel(mode)) return smem_layout_at(mode, cout, ksize, up, kStages);
    SmemLayout L = smem_layout_at(mode, cout, ksize, up, ring_cap(mode));
    for (int s = ring_cap(mode) - 1; s >= kStages && L.total + 1024u > kSmemMax; --s)     // conv_smem_bytes <= 227 KB
        L = smem_layout_at(mode, cout, ksize, up, s);
    return L;
}

// dynamic shared memory of a launch: the layout plus the slack for aligning the base to 1024 bytes
constexpr size_t conv_smem_bytes(ConvMode mode, int cout, int ksize, int up) { return smem_layout(mode, cout, ksize, up).total + 1024; }

// Every RicHalo launch fits: the widest piece of either precision at both source scales (up = 1: the fused nearest x2).
// With no A ring, fp16 Cout 256 at up = 0 takes 189 KB (ring 4 x 32 KB, two 22.5 KB halos, stencil, parameters).
static_assert(conv_smem_bytes(ConvMode::RicHalo, kMaxPiece(false), 3, 0) <= kSmemMax &&
              conv_smem_bytes(ConvMode::RicHalo, kMaxPiece(false), 3, 1) <= kSmemMax &&
              conv_smem_bytes(ConvMode::RicHalo, kMaxPiece(true), 3, 0) <= kSmemMax &&
              conv_smem_bytes(ConvMode::RicHalo, kMaxPiece(true), 3, 1) <= kSmemMax,
              "a RicHalo launch exceeds 227 KB of shared memory");

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

// ---- RIC: chunk q = (channel block q / 9, tap q % 9).  One A-row item = (output pixel r, data slot d).  fp16: slot d of
// the row, 4 rows per thread; split fp16 / bf16: 8 fp32 channels -> hi slot d, lo slot d + 4, 2 rows per thread.
template <bool kExact>
struct RicItems {
    static constexpr int kSlots = kExact ? 4 : 8, kRowsPer = kExact ? 2 : 4, kRowStep = kTileM / kRowsPer;
};

// torchvision's deform_conv2d bilinear rule with the engine's stencil tables, per element: a rotated tap blends the 2x2
// corner set of its sector in the operation order of the reference port of the weights: w00*n00, then fma w01*n01, w10*n10,
// w11*n11.  fp16: the stencil entry holds the four fp16 weights {w00,w01 | w10,w11} and one call blends a packed-half2 word
// (two channels).  Split fp16: the entry holds the fractions (ly, lx), the weights and the blend are fp32 with explicit
// rounding, one channel per call (split bf16 likewise).  bf16: the split-fp16 entry and fp32 blend, one call per bf16 word (two channels), rounded
// once to bf16 (a bf16 blend would round four partial sums at 2^-8 each).  The weight type selects the rule (RicWeightsH:
// packed-half2; RicWeightsF: fp32), and every RIC A producer goes through these functions, so they all agree bit for bit.
struct RicWeightsH { __half2 w00, w01, w10, w11; };
struct RicWeightsF { float w0, w1, w2, w3; };

// whether the RIC producers of a launch read the fp32 fractions (ric_lyx) and blend in fp32, not the fp16 weights (ric_wh)
template <bool kExact, typename T>
constexpr bool kBlendF32 = kExact || std::is_same<T, __nv_bfloat16>::value;

__device__ __forceinline__ __half2 h2_of(uint32_t v) { return *reinterpret_cast<const __half2*>(&v); }

__device__ __forceinline__ RicWeightsH ric_weights(uint2 wv) {
    const __half2 wa = h2_of(wv.x), wb = h2_of(wv.y);
    return {__low2half2(wa), __high2half2(wa), __low2half2(wb), __high2half2(wb)};
}
__device__ __forceinline__ RicWeightsF ric_weights(float2 l) {
    const float hy = 1.0f - l.x, hx = 1.0f - l.y;
    return {__fmul_rn(hy, hx), __fmul_rn(hy, l.y), __fmul_rn(l.x, hx), __fmul_rn(l.x, l.y)};
}
__device__ __forceinline__ uint32_t ric_blend(const RicWeightsH& w, uint32_t n00, uint32_t n01, uint32_t n10, uint32_t n11) {
    const __half2 o = __hfma2(w.w11, h2_of(n11), __hfma2(w.w10, h2_of(n10), __hfma2(w.w01, h2_of(n01), __hmul2(w.w00, h2_of(n00)))));
    return *reinterpret_cast<const uint32_t*>(&o);
}
__device__ __forceinline__ float ric_blend(const RicWeightsF& w, float v00, float v01, float v10, float v11) {
    return __fmaf_rn(w.w3, v11, __fmaf_rn(w.w2, v10, __fmaf_rn(w.w1, v01, __fmul_rn(w.w0, v00))));
}
__device__ __forceinline__ uint32_t ric_blend(const RicWeightsF& w, uint32_t n00, uint32_t n01, uint32_t n10, uint32_t n11) {
    const float2 a = unpack_h2<__nv_bfloat16>(n00), b = unpack_h2<__nv_bfloat16>(n01);
    const float2 c = unpack_h2<__nv_bfloat16>(n10), d = unpack_h2<__nv_bfloat16>(n11);
    return pack_h2<__nv_bfloat16>(ric_blend(w, a.x, b.x, c.x, d.x), ric_blend(w, a.y, b.y, c.y, d.y));
}

// One A-row item of the gather producer: the centre tap copies corner (0, 0); a rotated tap blends its corners
// with the stencil entry `entry()` (fp16 weights or fp32 fractions: the blend rule above).  `fetch(cy, cx, h)` returns 16
// source bytes of corner (cy, cx), zeros outside the (virtual, nearest-x2) image: the 8 fp16 / bf16 channels (h = 0), or
// fp32 channels 4h .. 4h + 3.
template <bool kExact, typename T, typename Entry, typename Fetch>
__device__ __forceinline__ void ric_item(bool centre, const Entry& entry, const Fetch& fetch, uint32_t row, int d, uint32_t swz) {
    if constexpr (!kExact) {
        uint4 out;
        if (centre) {
            out = fetch(0, 0, 0);
        } else {
            const auto w = ric_weights(entry());
            const uint4 n00 = fetch(0, 0, 0), n01 = fetch(0, 1, 0), n10 = fetch(1, 0, 0), n11 = fetch(1, 1, 0);
            out = make_uint4(ric_blend(w, n00.x, n01.x, n10.x, n11.x), ric_blend(w, n00.y, n01.y, n10.y, n11.y),
                             ric_blend(w, n00.z, n01.z, n10.z, n11.z), ric_blend(w, n00.w, n01.w, n10.w, n11.w));
        }
        st_shared_v4(row + ((static_cast<uint32_t>(d) ^ swz) << 4), out);
    } else {
        // stage 1 of both split modes keeps fp32 activations: 8 channels = two 16-byte fetches per corner
        auto load8 = [&](int cy, int cx, float* v) {
            const uint4 lo = fetch(cy, cx, 0), hi = fetch(cy, cx, 1);
            v[0] = __uint_as_float(lo.x); v[1] = __uint_as_float(lo.y); v[2] = __uint_as_float(lo.z); v[3] = __uint_as_float(lo.w);
            v[4] = __uint_as_float(hi.x); v[5] = __uint_as_float(hi.y); v[6] = __uint_as_float(hi.z); v[7] = __uint_as_float(hi.w);
        };
        float f[8];
        if (centre) {
            load8(0, 0, f);
        } else {
            const RicWeightsF w = ric_weights(entry());
            float v00[8], v01[8], v10[8], v11[8];
            load8(0, 0, v00); load8(0, 1, v01); load8(1, 0, v10); load8(1, 1, v11);
#pragma unroll
            for (int c = 0; c < 8; ++c) f[c] = ric_blend(w, v00[c], v01[c], v10[c], v11[c]);
        }
        uint4 hi, lo;
        split8<T>(f, hi, lo);
        st_shared_v4(row + ((static_cast<uint32_t>(d) ^ swz) << 4), hi);
        st_shared_v4(row + ((static_cast<uint32_t>(d + 4) ^ swz) << 4), lo);
    }
}

// ---- RIC gather producer: octant, stencil entry and the four corners of every item straight from L2 / global memory
template <bool kExact, typename T>
__device__ __forceinline__ void produce_ric(const ConvParams& p, int q, uint32_t a, int tid, int n, int ty0, int tx0) {
    using It = RicItems<kExact>;
    const int blk = q / 9, t = q - 9 * blk;
    const int kq = t < 4 ? t : t - 1;                     // circle index of a rotated tap
    const size_t frame_in = static_cast<size_t>(n) * p.Hin * p.Win;
    const int d = tid % It::kSlots, prow = tid / It::kSlots;
    const Slot sl = p.slots[blk * 8 + d];
    const Seg sg = p.seg[sl.seg];
    constexpr size_t kEsz = kExact ? sizeof(float) : sizeof(__half);
    const uint8_t* src = reinterpret_cast<const uint8_t*>(sg.ptr) + sl.choff * kEsz;
    const size_t pitch = static_cast<size_t>(sg.pitch) * kEsz;
#pragma unroll
    for (int i = 0; i < It::kRowsPer; ++i) {
        const int r = prow + It::kRowStep * i;
        const int oy = ty0 + (r >> 4), ox = tx0 + (r & 15);
        const bool live = sl.valid && oy < p.Hout && ox < p.Wout;
        const size_t e = live ? static_cast<size_t>(oy) * p.Wout + ox : 0;
        int dy0 = 0, dx0 = 0, m = 0;
        if (t != 4) {
            m = (kq + __ldg(p.ric_oct + e)) & 7;
            dy0 = ric_r0(m) - 1; dx0 = ric_c0(m) - 1;
        }
        auto fetch = [&](int cy, int cx, int h) {
            const int vy = oy + dy0 + cy, vx = ox + dx0 + cx;
            const bool ok = live && static_cast<unsigned>(vy) < static_cast<unsigned>(p.Hv) && static_cast<unsigned>(vx) < static_cast<unsigned>(p.Wv);
            const size_t pix = ok ? frame_in + static_cast<size_t>(vy >> p.up) * p.Win + (vx >> p.up) : 0;
            return ldg128_if(src + pix * pitch + 16 * h, ok);
        };
        auto entry = [&]() {
            if constexpr (kBlendF32<kExact, T>) return live ? __ldg(p.ric_lyx + e * 8 + m) : make_float2(0.0f, 0.0f);
            else return live ? __ldg(p.ric_wh + e * 8 + m) : make_uint2(0u, 0u);
        };
        ric_item<kExact, T>(t == 4, entry, fetch, a + static_cast<uint32_t>(r) * 128u, d, static_cast<uint32_t>(r & 7));
    }
}

// The stencil entries of the tile's 128 pixels (fp16 weights or, kF32, fp32 fractions: 8 B per rotated tap), stored
// [m][pixel] so that the items of one load phase (neighbouring pixels, any sectors) hit distinct banks; zeros outside
// Hout x Wout.  The octants go to registers (ric_lane): a lane's output pixels never change across chunks.  (They are read
// with plain loads: a tile row of octant bytes is not 4-byte aligned when Wout is not a multiple of 4.)
template <bool kF32>
__device__ __forceinline__ void stage_ric_stencil(const ConvParams& p, uint32_t sten, int tid, int ty0, int tx0) {
    const uint8_t* table = kF32 ? reinterpret_cast<const uint8_t*>(p.ric_lyx) : reinterpret_cast<const uint8_t*>(p.ric_wh);
    for (int i = tid; i < kTileM * 8; i += kThreads) {
        const int r = i >> 3, m = i & 7;
        const int oy = ty0 + (r >> 4), ox = tx0 + (r & 15);
        const bool ok = oy < p.Hout && ox < p.Wout;
        const size_t e = ok ? static_cast<size_t>(oy) * p.Wout + ox : 0;
        cp_async8(sten + static_cast<uint32_t>(m * kTileM + r) * 8u, table + (e * 8 + m) * 8, ok ? 8u : 0u);
    }
}

// the octant of tile pixel r (0 outside Hout x Wout)
__device__ __forceinline__ uint32_t ric_oct(const ConvParams& p, int r, int ty0, int tx0) {
    const int oy = ty0 + (r >> 4), ox = tx0 + (r & 15);
    return (oy < p.Hout && ox < p.Wout) ? static_cast<uint32_t>(__ldg(p.ric_oct + static_cast<size_t>(oy) * p.Wout + ox)) : 0u;
}

// The input of channel block `blk` for the whole tile: source rows (ty0 >> up) - 1 + [0, ric_halo_rows), columns
// (tx0 >> up) - 1 + [0, ric_halo_cols), 128 B per pixel, pixel-major, 16-byte slot s at ((s ^ (pixel & 7)) << 4).  Slot s
// holds group s (fp16) or half s & 1 of group s / 2 (fp32: channels 4 (s & 1) .. + 3) of the block's RIC slot table.
// Zeros outside [0, Hin) x [0, Win) (torchvision's border rule: corners outside the virtual image read zero) and for
// K-padding slots.
template <bool kExact>
__device__ __forceinline__ void load_ric_halo(const ConvParams& p, int blk, uint32_t halo, int tid, int n, int ty0, int tx0) {
    const int hw = ric_halo_cols(p.up), npix = ric_halo_rows(p.up) * hw;
    const int y0 = (ty0 >> p.up) - 1, x0 = (tx0 >> p.up) - 1;
    const int s = tid & 7;                                // the 8 threads of a pixel copy its 128 bytes
    const Slot sl = p.slots[blk * 8 + (kExact ? s >> 1 : s)];
    const Seg sg = p.seg[sl.seg];
    constexpr size_t kEsz = kExact ? sizeof(float) : sizeof(__half);
    const uint8_t* sbase = reinterpret_cast<const uint8_t*>(sg.ptr) + (sl.choff + (kExact ? 4 * (s & 1) : 0)) * kEsz;
    const size_t pitch = static_cast<size_t>(sg.pitch) * kEsz;
    const size_t frame_in = static_cast<size_t>(n) * p.Hin * p.Win;
    for (int pix = tid >> 3; pix < npix; pix += kThreads / 8) {
        const int hy = pix / hw, hx = pix - hy * hw;
        const int y = y0 + hy, x = x0 + hx;
        const bool ok = sl.valid && static_cast<unsigned>(y) < static_cast<unsigned>(p.Hin) && static_cast<unsigned>(x) < static_cast<unsigned>(p.Win);
        const uint8_t* src = ok ? sbase + (frame_in + static_cast<size_t>(y) * p.Win + x) * pitch : sbase;
        cp_async16(halo + static_cast<uint32_t>(pix) * 128u + (static_cast<uint32_t>(s ^ (pix & 7)) << 4), src, ok ? 16u : 0u);
    }
}

// ---- RicHalo mode, A in registers.  Lane l of warp w in warpgroup wg holds the A fragments of tile pixels
// r = 64 wg + 16 w + l / 4 and r + 8 (fragment rows l / 4 and l / 4 + 8: tile row 4 wg + w, columns l / 4 and l / 4 + 8),
// columns 2 (l % 4), +1 of the 16-byte slots 2k and 2k + 1 of K step k: the layout ldsm_x4 returns and mma_rs takes,
// a[k][0 | 1] = slot 2k of pixel r | r + 8, a[k][2 | 3] = slot 2k + 1.  What a lane needs in every chunk:
struct RicLane {
    int r;              // tile pixel of fragment row l / 4 (the other row is r + 8)
    int oy, ox;         // its output pixel (the other one is (oy, ox + 8))
    uint32_t live;      // bit j: pixel r + 8j lies inside Hout x Wout
    uint32_t oct;       // byte j: octant of pixel r + 8j; byte 2 (fp16): octant of the ldmatrix row pixel
    int ax;             // fp16: output column of the pixel whose row address this lane gives ldmatrix (row oy, slot 2k + aslot)
    int aslot;
};

__device__ __forceinline__ RicLane ric_lane(const ConvParams& p, int tid, int ty0, int tx0) {
    const int wg = tid >> 7, w = (tid >> 5) & 3, l = tid & 31;
    RicLane ln;
    ln.r = 64 * wg + 16 * w + (l >> 2);
    ln.oy = ty0 + (ln.r >> 4);
    ln.ox = tx0 + (ln.r & 15);
    ln.live = (ln.oy < p.Hout && ln.ox < p.Wout ? 1u : 0u) | (ln.oy < p.Hout && ln.ox + 8 < p.Wout ? 2u : 0u);
    // ldmatrix: lanes 0-7 / 8-15 give the rows of matrices 0 / 1 (pixels 0-7 / 8-15 of the warp's tile row, slot 2k),
    // lanes 16-31 the same pixels for slot 2k + 1
    const int ra = (ln.r & ~15) + (l & 7) + 8 * ((l >> 3) & 1);
    ln.ax = tx0 + (ra & 15);
    ln.aslot = l >> 4;
    ln.oct = ric_oct(p, ln.r, ty0, tx0) | ric_oct(p, ln.r + 8, ty0, tx0) << 8 | ric_oct(p, ra, ty0, tx0) << 16;
    return ln;
}

// Chunk q's A fragments from the block's halo and the tile's stencil: the same corners, entries, blend helpers, centre
// tap and zero rule as the gather producer (produce_ric), so the fragments hold exactly the values it stores.  A corner
// (vy, vx) of the virtual image is halo pixel ((vy >> up) - y0, (vx >> up) - x0); pixels past Hout / Wout in ragged tiles
// stay inside the halo and produce zeros (`live`).  K-padding slots are zeros in the halo and blend to zeros.
//   fp16 / bf16: per corner and K step one ldsm_x4 gathers the corner of each fragment row (every lane gives the row address
//   of its ldmatrix pixel's corner), then each register is one blend of two channels with its row's weights (packed-half2
//   in fp16, fp32 and one rounding in bf16).
//   Split fp16 / bf16: K steps 0-1 are the hi and 2-3 the lo parts of the chunk's 32 fp32 channels.  Channels 2t, 2t + 1 (t = l % 4)
//   of group g sit in halo slot 2g + (t >> 1) at byte 8 (t & 1): one ld.shared.v2 per corner, group and pixel; the blend is
//   split once, hi into K step g / 2 and lo into g / 2 + 2.
template <bool kExact, typename T>
__device__ __forceinline__ void build_ric_a(const ConvParams& p, int q, uint32_t halo, uint32_t sten, const RicLane& ln,
                                            int lane, int ty0, int tx0, uint32_t (*a)[4]) {
    const int t = q % 9, kq = t < 4 ? t : t - 1;
    const int hw = ric_halo_cols(p.up), y0 = (ty0 >> p.up) - 1, x0 = (tx0 >> p.up) - 1;
    auto hpix = [&](int vy, int vx) { return ((vy >> p.up) - y0) * hw + (vx >> p.up) - x0; };
    auto sector = [&](int j, int& dy0, int& dx0) {     // rotated tap m of pixel j: stencil entry and first corner offset
        const int m = (kq + (ln.oct >> (8 * j))) & 7;
        dy0 = ric_r0(m) - 1; dx0 = ric_c0(m) - 1;
        return m;
    };
    if constexpr (!kExact) {
        auto slot = [&](int hp, int k) { return halo + static_cast<uint32_t>(hp) * 128u + ((static_cast<uint32_t>(2 * k + ln.aslot) ^ static_cast<uint32_t>(hp & 7)) << 4); };
        if (t == 4) {
            const int hp = hpix(ln.oy, ln.ax);
#pragma unroll
            for (int k = 0; k < 4; ++k) ldsm_x4(a[k], slot(hp, k));
        } else {
            int dy0, dx0;
            sector(2, dy0, dx0);
            const int vy = ln.oy + dy0, vx = ln.ax + dx0;
            const int h00 = hpix(vy, vx), h01 = hpix(vy, vx + 1), h10 = hpix(vy + 1, vx), h11 = hpix(vy + 1, vx + 1);
            auto weights = [](uint2 raw) {        // the staged entry: fp32 fractions (bf16) or fp16 weights
                if constexpr (kBlendF32<kExact, T>) return ric_weights(make_float2(__uint_as_float(raw.x), __uint_as_float(raw.y)));
                else return ric_weights(raw);
            };
            decltype(weights(uint2{})) w[2];
#pragma unroll
            for (int j = 0; j < 2; ++j) w[j] = weights(ld_shared_v2(sten + static_cast<uint32_t>(sector(j, dy0, dx0) * kTileM + ln.r + 8 * j) * 8u));
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                uint32_t n00[4], n01[4], n10[4], n11[4];
                ldsm_x4(n00, slot(h00, k)); ldsm_x4(n01, slot(h01, k)); ldsm_x4(n10, slot(h10, k)); ldsm_x4(n11, slot(h11, k));
#pragma unroll
                for (int i = 0; i < 4; ++i) a[k][i] = ric_blend(w[i & 1], n00[i], n01[i], n10[i], n11[i]);
            }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int i = 0; i < 4; ++i)
                if (!((ln.live >> (i & 1)) & 1)) a[k][i] = 0u;
    } else {
        // The centre tap and the rotated taps are separate straight-line paths, each issuing all its shared-memory loads
        // of a pixel before the first blend, so the loads overlap instead of each group waiting for its own.
        const uint32_t th = static_cast<uint32_t>((lane & 3) >> 1), tb = static_cast<uint32_t>(lane & 1) * 8u;
        auto ld = [&](int hp, int g) {
            const uint32_t s = 2u * g + th;
            const uint2 v = ld_shared_v2(halo + static_cast<uint32_t>(hp) * 128u + ((s ^ static_cast<uint32_t>(hp & 7)) << 4) + tb);
            return make_float2(__uint_as_float(v.x), __uint_as_float(v.y));
        };
        auto put = [&](int j, int g, float2 f) {
            if (!((ln.live >> j) & 1)) f = make_float2(0.0f, 0.0f);
            uint32_t hi, lo;
            split2<T>(f.x, f.y, hi, lo);
            a[g >> 1][j + 2 * (g & 1)] = hi;
            a[2 + (g >> 1)][j + 2 * (g & 1)] = lo;
        };
        if (t == 4) {
            float2 v[2][4];
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int hp = hpix(ln.oy, ln.ox + 8 * j);
#pragma unroll
                for (int g = 0; g < 4; ++g) v[j][g] = ld(hp, g);
            }
#pragma unroll
            for (int j = 0; j < 2; ++j)
#pragma unroll
                for (int g = 0; g < 4; ++g) put(j, g, v[j][g]);
        } else {
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                int dy0, dx0;
                const uint2 raw = ld_shared_v2(sten + static_cast<uint32_t>(sector(j, dy0, dx0) * kTileM + ln.r + 8 * j) * 8u);
                const int vy = ln.oy + dy0, vx = ln.ox + 8 * j + dx0;
                const int h00 = hpix(vy, vx), h01 = hpix(vy, vx + 1), h10 = hpix(vy + 1, vx), h11 = hpix(vy + 1, vx + 1);
                float2 v00[4], v01[4], v10[4], v11[4];
#pragma unroll
                for (int g = 0; g < 4; ++g) { v00[g] = ld(h00, g); v01[g] = ld(h01, g); v10[g] = ld(h10, g); v11[g] = ld(h11, g); }
                const RicWeightsF w = ric_weights(make_float2(__uint_as_float(raw.x), __uint_as_float(raw.y)));
#pragma unroll
                for (int g = 0; g < 4; ++g)
                    put(j, g, make_float2(ric_blend(w, v00[g].x, v01[g].x, v10[g].x, v11[g].x),
                                          ric_blend(w, v00[g].y, v01[g].y, v10[g].y, v11[g].y)));
            }
        }
    }
}

// weight tile of chunk q (cp.async)
__device__ __forceinline__ void produce_b(const ConvParams& p, int q, uint32_t dst, int tid) {
    const uint8_t* src = p.wpack + static_cast<size_t>(q) * p.b_bytes;
    for (int i = tid; i < p.b_bytes / 16; i += kThreads) cp_async16(dst + 16u * i, src + 16 * i, 16u);
}

// chunk q: A rows and weight tile
template <ConvMode kMode, bool kExact, typename T>
__device__ __forceinline__ void produce(const ConvParams& p, int q, uint32_t stage, int tid, int n, int ty0, int tx0) {
    if constexpr (kMode == ConvMode::Tap) produce_tap(p, q, stage, tid, n, ty0, tx0);
    else produce_ric<kExact, T>(p, q, stage, tid, n, ty0, tx0);
    produce_b(p, q, stage + kABytes, tid);
}

// the K steps of one chunk: every PN-column piece of the accumulator against the matching PN rows of the weight tile
template <int NC, int PN, typename T>
__device__ __forceinline__ void mma_chunk(float* acc, uint64_t da, uint64_t db, uint32_t km, uint32_t km2) {
    constexpr uint64_t kPieceStep = PN * 128 / 16;        // descriptor units between PN-row weight pieces
    auto step = [&](int ka, int kb) {
#pragma unroll
        for (int j = 0; j < NC / PN; ++j) Wgmma<PN, T>::mma(acc + j * (PN / 2), da + 2 * ka, db + 2 * kb + j * kPieceStep);
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

// the same K steps with A from registers: a[mb][k] = K step k of m64 block mb; in split-fp16 the hi fragments (steps 0-1)
// are used for both a_hi*W_hi and a_hi*W_lo.  Every step is issued, also in the ragged last chunk: its K-padding slots
// read zeros against zero weights and add exact zeros, and a branch-free sequence keeps the wgmmas back to back.
template <int NC, int PN, int MB, bool kExact, typename T>
__device__ __forceinline__ void mma_chunk_rs(float (*acc)[NC / 2], const uint32_t (*a)[4][4], uint64_t db) {
    constexpr uint64_t kPieceStep = PN * 128 / 16;
    auto step = [&](int ka, int kb) {
#pragma unroll
        for (int mb = 0; mb < MB; ++mb)
#pragma unroll
            for (int j = 0; j < NC / PN; ++j) Wgmma<PN, T>::mma_rs(acc[mb] + j * (PN / 2), a[mb][ka], db + 2 * kb + j * kPieceStep);
    };
#pragma unroll
    for (int k = 0; k < 4; ++k) step(k, kExact ? (k & 1) : k);
    if constexpr (kExact) {
#pragma unroll
        for (int k = 0; k < 2; ++k) step(k, 2 + k);
    }
}

// ---- halo mode: the input halo of channel block `blk` with cp.async, zeros outside the image.  Pixel-major, 128 B per
// pixel, 16-byte slot s at ((s ^ (pixel & 7)) << 4): any 8 consecutive halo pixels are bank-conflict free for ldmatrix.
template <int kRows>
__device__ __forceinline__ void load_halo(const ConvParams& p, int blk, uint32_t halo, int tid, int n, int ty0, int tx0) {
    const int hw = kTileW + p.ksize - 1, npix = (kRows + p.ksize - 1) * hw;
    const int s = tid & 7;                                // the 8 threads of a pixel copy its 128 contiguous bytes
    const Slot sl = p.hslots[blk * 8 + s];
    const Seg sg = p.seg[sl.seg];
    const __half* sbase = sg.ptr + sl.choff;
    const size_t frame_in = static_cast<size_t>(n) * p.Hin * p.Win;
    for (int pix = tid >> 3; pix < npix; pix += kThreads / 8) {
        const int hy = pix / hw, hx = pix - hy * hw;
        const int y = ty0 - p.pad_y + hy, x = tx0 - p.pad_x + hx;
        const bool ok = sl.valid && static_cast<unsigned>(y) < static_cast<unsigned>(p.Hin) && static_cast<unsigned>(x) < static_cast<unsigned>(p.Win);
        const __half* src = ok ? sbase + (frame_in + static_cast<size_t>(y) * p.Win + x) * sg.pitch : sbase;
        cp_async16(halo + static_cast<uint32_t>(pix) * 128u + (static_cast<uint32_t>(s ^ (pix & 7)) << 4), src, ok ? 16u : 0u);
    }
}

// ---- halo mode: chunk q's A fragments of this warp (rows pb[mb] of each m64 block) from the halo into registers.  Lanes
// 0-15 address the 16 rows of slot 2k, lanes 16-31 those of slot 2k + 1; each slot reads its halo pixel shifted by its own
// tap, so taps of several channel groups may share a chunk.  K-padding slots read 16 zero bytes.
template <int MB>
__device__ __forceinline__ void load_a(const ConvParams& p, int q, uint32_t halo, uint32_t zero, const int* pb, int lane,
                                       uint32_t (*a)[4][4]) {
    const int hw = kTileW + p.ksize - 1;
    const uint2* slots = reinterpret_cast<const uint2*>(p.slots) + q * 8 + (lane >> 4);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint2 raw = __ldg(slots + 2 * k);
        Slot sl;
        memcpy(&sl, &raw, sizeof(sl));
        const int shift = (sl.dy + p.pad_y) * hw + sl.dx + p.pad_x;
#pragma unroll
        for (int mb = 0; mb < MB; ++mb) {
            const int pix = pb[mb] + shift;
            const uint32_t addr = sl.valid ? halo + static_cast<uint32_t>(pix) * 128u + (static_cast<uint32_t>(sl.hslot ^ (pix & 7)) << 4) : zero;
            ldsm_x4(a[mb][k], addr);
        }
    }
}

// accumulators (MB m64 blocks per warpgroup) -> fp32 rows in shared memory -> fused epilogue, one pixel row per thread pair
template <int NC, int MB>
__device__ __forceinline__ void store_tile(const ConvParams& p, uint8_t* smem, const float* s_par, float (*acc)[NC / 2],
                                           int tid, int n, int ty0, int tx0) {
    constexpr int kM = 128 * MB;
    float* staged = reinterpret_cast<float*>(smem);
    {
        const int wg = tid >> 7, w = (tid >> 5) & 3, l = tid & 31;
#pragma unroll
        for (int mb = 0; mb < MB; ++mb) {
            const int r0 = wg * (kM / 2) + mb * 64 + 16 * w + (l >> 2), c0 = 2 * (l & 3);
#pragma unroll
            for (int i = 0; i < NC / 2; i += 2) {
                const int r = r0 + 8 * ((i >> 1) & 1), c = c0 + 8 * (i >> 2);
                *reinterpret_cast<float2*>(staged + r * acc_pitch(NC) + c) = make_float2(acc[mb][i], acc[mb][i + 1]);
            }
        }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < MB; ++i) {
        const int r = (tid & 127) + 128 * i;              // patch pixel; two threads per row split the 32-column batches
        const float* row = staged + r * acc_pitch(NC);
        if (p.sub) epilogue_row<true>(p, s_par, row, n, ty0 + (r >> 4), tx0 + (r & 15), tid >> 7);
        else epilogue_row<false>(p, s_par, row, n, ty0 + (r >> 4), tx0 + (r & 15), tid >> 7);
    }
}

}  // namespace

// NC = Cout, PN = wgmma N per instruction (a divisor of NC: 32, 64 or 128), T the operand type.  Tap mode reads the
// split K steps from the K masks, so it is instantiated with kExact = false for the single-pass and split forms of each T.
template <int NC, int PN, ConvMode kMode, bool kExact, typename T>
__global__ void __launch_bounds__(kThreads, 1)
conv_wgmma_kernel(const __grid_constant__ ConvParams p) {
    static_assert(!uses_halo_kernel(kMode), "conv_wgmma_kernel: Tap and Ric modes only");
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw_u32 = smem_u32(smem_raw);
    const uint32_t base = (raw_u32 + 1023u) & ~1023u;     // SWIZZLE_128B atoms are 1024-byte aligned
    uint8_t* smem = smem_raw + (base - raw_u32);
    const SmemLayout L = smem_layout(kMode, NC, p.ksize, p.up);
    float* s_par = reinterpret_cast<float*>(smem + L.par);

    const int tid = threadIdx.x;
    const int wg = tid >> 7;
    const int n = blockIdx.z;
    const int ty0 = blockIdx.y * kTileH;
    const int tx0 = blockIdx.x * kTileW;
    const int nq = p.nchunks;
    // chunks with the ragged K tail: the last one (tap mode) or the 9 taps of the last channel block (RIC)
    const int tail_from = kMode != ConvMode::Tap ? (p.nblocks - 1) * 9 : nq - 1;

    load_epilogue_params(p, s_par, tid, kThreads);

    float acc[1][NC / 2];
#pragma unroll
    for (int i = 0; i < NC / 2; ++i) acc[0][i] = 0.0f;

    // prologue: chunks 0 and 1; every iteration commits one cp.async group so that "chunk q has landed" is wait_group 1
#pragma unroll
    for (int s = 0; s < kStages - 2; ++s) {
        if (s < nq) produce<kMode, kExact, T>(p, s, base + s * L.stage_bytes, tid, n, ty0, tx0);
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
        mma_chunk<NC, PN, T>(acc[0], da, db, tail ? p.kmask_last : p.kmask_full, tail ? p.kmask2_last : p.kmask2_full);
        wgmma_commit();
        wgmma_wait<1>();                                  // this warpgroup's MMAs of chunk q - 1 have retired
        if (q + kStages - 2 < nq) produce<kMode, kExact, T>(p, q + kStages - 2, base + ((q + kStages - 2) % kStages) * L.stage_bytes, tid, n, ty0, tx0);
        cp_async_commit();
    }
    wgmma_wait<0>();
    cp_async_wait<0>();
    __syncthreads();                                      // the ring is free: stage the accumulators over it
    store_tile<NC, 1>(p, smem, s_par, acc, tid, n, ty0, tx0);
}

// Halo and RicHalo modes.  Chunk q belongs to channel block q / k^2 (every block but the last has
// exactly k^2 chunks, one per tap; in Halo mode the last one may pack several taps of its few channel groups into a chunk).
// The mainloop is an mbarrier pipeline (below, and DESIGN section 4a): weight tiles in a ring of SmemLayout::stages
// bulk-copied stages, halos with full / empty barriers per buffer, the halo of block b + 1 issued in the first iteration of
// block b (it lands k^2 - 1 iterations before it is read; the buffer it overwrites was last read in iteration b k^2 - 2).
// The chunk loop is unrolled by two so that the fragment buffers have fixed registers.  The two modes differ only in the
// fragment source: Halo mode ldmatrix'es each slot's
// tap-shifted halo pixel (load_a); RicHalo mode blends the rotated tap's corners from the halo with the stencil staged in
// the prologue (build_ric_a), with 8 x 16 tiles and k^2 = 9 taps per block.  RicHalo layers up to 64 channels run two
// CTAs per SM (ric_ctas_per_sm) with one fragment buffer, so one CTA's fragment building and barriers overlap the other's
// MMAs.
template <int NC, int PN, ConvMode kMode, bool kExact, typename T>
__global__ void __launch_bounds__(kThreads, ric_ctas_per_sm(kMode, NC))
conv_halo_kernel(const __grid_constant__ ConvParams p) {
    constexpr bool kRic = kMode == ConvMode::RicHalo;
    static_assert(uses_halo_kernel(kMode), "conv_halo_kernel: Halo and RicHalo modes only");
    constexpr int kRows = kRic ? kTileH : halo_rows(NC), kM = kRows * kTileW, MB = kM / 128;     // MB: m64 blocks per warpgroup
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw_u32 = smem_u32(smem_raw);
    const uint32_t base = (raw_u32 + 1023u) & ~1023u;
    uint8_t* smem = smem_raw + (base - raw_u32);
    const SmemLayout L = smem_layout(kMode, NC, p.ksize, p.up);
    float* s_par = reinterpret_cast<float*>(smem + L.par);
    const uint32_t aux = base + L.aux;                    // zero row (Halo) or stencil (RicHalo)

    const int tid = threadIdx.x;
    const int wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
    const int n = blockIdx.z;
    const int ty0 = blockIdx.y * kRows;
    const int tx0 = blockIdx.x * kTileW;
    const int nq = p.nchunks, kk = kRic ? 9 : p.ksize * p.ksize;
    const int hw = kTileW + p.ksize - 1;

    load_epilogue_params(p, s_par, tid, kThreads);
    if (!kRic && tid < 4) reinterpret_cast<uint32_t*>(smem + L.aux)[tid] = 0u;

    // Halo: halo pixel of this lane's A row in each m64 block, for the tap (0, 0) of the halo origin
    int pb[MB];
#pragma unroll
    for (int mb = 0; mb < MB; ++mb) {
        const int r = wg * (kM / 2) + mb * 64 + warp * 16 + (lane & 15);
        pb[mb] = (r >> 4) * hw + (r & 15);
    }
    RicLane ln{};
    if constexpr (kRic) ln = ric_lane(p, tid, ty0, tx0);
    float acc[MB][NC / 2];
#pragma unroll
    for (int mb = 0; mb < MB; ++mb)
#pragma unroll
        for (int i = 0; i < NC / 2; ++i) acc[mb][i] = pinned_zero();   // not 0.0f: see pinned_zero
    // [buffer][m64 block][K step][register].  Two-CTA instantiations keep one buffer (128 registers per thread): each
    // CTA waits for its MMAs before it builds the next chunk, and the other CTA's MMAs fill the gap.
    constexpr bool kOneBuf = ric_ctas_per_sm(kMode, NC) > 1;
    uint32_t a[2][MB][4][4];

    // mbarriers: full[s] completes when the weight tile in stage s has landed (one arrive with its byte count by the
    // issuing thread), empty[s] when both warpgroups' MMAs have stopped reading it (one arrive per warpgroup); halo full[i]
    // when every thread's cp.async of the block in buffer i have landed, halo empty[i] when every warp has built its last
    // fragments from it (one arrive per warp)
    const int S = static_cast<int>(L.stages);
    const uint32_t bars = base + L.bars;
    auto full_bar = [&](int s) { return bars + 8u * static_cast<uint32_t>(s); };
    auto empty_bar = [&](int s) { return bars + 8u * static_cast<uint32_t>(S + s); };
    auto hfull_bar = [&](int blk) { return bars + 8u * static_cast<uint32_t>(2 * S + (blk & 1)); };
    auto hempty_bar = [&](int blk) { return bars + 8u * static_cast<uint32_t>(2 * S + 2 + (blk & 1)); };
    if (tid == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), 2);
        }
        for (int i = 0; i < 2; ++i) {
            mbar_init(hfull_bar(i), kThreads);
            mbar_init(hempty_bar(i), kThreads / 32);
        }
        fence_mbar_init();
    }
    __syncthreads();                                      // barriers initialised, the zero row written

    auto halo_buf = [&](int blk) { return base + L.halo + static_cast<uint32_t>(blk & 1) * L.halo_bytes; };
    // every thread: its share of block blk's halo, then one arrive on the buffer's full barrier when it has landed
    auto load_block = [&](int blk) {
        if constexpr (kRic) load_ric_halo<kExact>(p, blk, halo_buf(blk), tid, n, ty0, tx0);
        else load_halo<kRows>(p, blk, halo_buf(blk), tid, n, ty0, tx0);
        cp_async_mbar_arrive(hfull_bar(blk));
    };
    auto load_frags = [&](int q, int b, uint32_t (*dst)[4][4]) {      // chunk q of channel block b
        if constexpr (kRic) build_ric_a<kExact, T>(p, q, halo_buf(b), aux, ln, lane, ty0, tx0, dst[0]);
        else load_a<MB>(p, q, halo_buf(b), aux, pb, lane, dst);
    };
    // thread 0: weight tile of chunk c (one bulk copy) into stage s
    auto produce_w = [&](int c, int s) {
        mbar_arrive_expect_tx(full_bar(s), static_cast<uint32_t>(p.b_bytes));
        bulk_copy_g2s(base + static_cast<uint32_t>(s) * L.stage_bytes, p.wpack + static_cast<size_t>(c) * p.b_bytes,
                      static_cast<uint32_t>(p.b_bytes), full_bar(s));
    };

    // prologue: (RicHalo: the tile's stencil with) the halo of block 0, and the weight tiles of chunks 0 .. S - 3
    if constexpr (kRic) stage_ric_stencil<kBlendF32<kExact, T>>(p, aux, tid, ty0, tx0);
    load_block(0);
    if (tid == 0)
        for (int c = 0; c < S - 2 && c < nq; ++c) produce_w(c, c);
    mbar_wait(hfull_bar(0), 0);
    load_frags(0, 0, a[0]);

    // Iteration q: wait for the weights of chunk q, issue its MMAs, wait for the MMAs of chunk q - 1 (two buffers) or q (one)
    // and release that chunk's stage, issue the weights of chunk q + S - 2 into the stage of chunk q - 2 once both
    // warpgroups released it, build the fragments of chunk q + 1 (waiting for its block's halo if it is the block's first
    // chunk, releasing the halo after the block's last), and in the first chunk of block b issue the halo of block b + 1
    // into the buffer block b - 1 used.  No block barrier: the warpgroups meet only at the mbarriers, so one may run a chunk
    // ahead of the other.  qs / qph: stage and phase parity of chunk q.  Halo mode carries chunk q's channel block and tap
    // position (k^2 is a run-time value there); RicHalo divides by the constant 9, which keeps two registers free for the
    // two-CTA instantiations.
    int qs = 0, cblk = 0, cqt = 0;
    uint32_t qph = 0;
    auto step = [&](int q, const uint32_t (*cur)[4][4], uint32_t (*nxt)[4][4]) {
        mbar_wait(full_bar(qs), qph);
        const uint64_t db = wgmma_desc_sw128(base + static_cast<uint32_t>(qs) * L.stage_bytes, 1024);
        wgmma_fence();
        mma_chunk_rs<NC, PN, MB, kExact, T>(acc, cur, db);
        wgmma_commit();
        if constexpr (kOneBuf) {
            wgmma_wait<0>();                              // the MMAs of chunk q have retired: the one buffer is free
            if ((tid & 127) == 0) mbar_arrive(empty_bar(qs));
        } else {
            wgmma_wait<1>();                              // the MMAs of chunk q - 1 have retired: `nxt` is free
            if (q > 0 && (tid & 127) == 0) mbar_arrive(empty_bar(qs > 0 ? qs - 1 : S - 1));
        }
        if (tid == 0 && q + S - 2 < nq) {
            // chunk q + S - 2 goes to stage (qs - 2) mod S, one round after chunk q - 2 there
            const int ps = qs >= 2 ? qs - 2 : qs + S - 2;
            if (q >= 2) mbar_wait(empty_bar(ps), qs >= 2 ? qph : qph ^ 1u);
            produce_w(q + S - 2, ps);
        }
        // chunk q: block blk, tap position qt in it; chunk q + 1: block nb, position nt
        const int blk = kRic ? q / 9 : cblk, qt = kRic ? q - 9 * blk : cqt;
        const bool next_blk = qt + 1 == kk;
        const int nb = next_blk ? blk + 1 : blk, nt = next_blk ? 0 : qt + 1;
        if (q + 1 < nq) {
            if (next_blk) mbar_wait(hfull_bar(nb), static_cast<uint32_t>(nb >> 1) & 1u);
            load_frags(q + 1, nb, nxt);
            if (nt + 1 == kk || q + 2 == nq) {
                __syncwarp();
                if (lane == 0) mbar_arrive(hempty_bar(nb));
            }
        }
        if (qt == 0 && blk + 1 < p.nblocks) {
            if (blk >= 1) mbar_wait(hempty_bar(blk + 1), (static_cast<uint32_t>((blk + 1) >> 1) & 1u) ^ 1u);
            load_block(blk + 1);
        }
        cblk = nb;
        cqt = nt;
        if (++qs == S) {
            qs = 0;
            qph ^= 1u;
        }
    };
    for (int q = 0; q < nq; q += 2) {
        step(q, a[0], a[kOneBuf ? 0 : 1]);
        if (q + 1 < nq) step(q + 1, a[kOneBuf ? 0 : 1], a[0]);
    }
    wgmma_wait<0>();
    __syncthreads();                                      // ring and halos are free: stage the accumulators over them
    store_tile<NC, MB>(p, smem, s_par, acc, tid, n, ty0, tx0);
}

// launch_mode<kMode, kExact, T> launches the instantiation for p.Cout (and p.n128) of one mode and precision.  It is
// explicitly instantiated once per precision, in conv_fp16.cu, conv_fp16x3.cu, conv_bf16.cu and conv_bf16x3.cu; conv_wgmma.cu
// dispatches to those instantiations without instantiating any kernel itself.  The four precisions are thereby separate
// translation units, which the build compiles in parallel.
template <ConvMode kMode, bool kExact, typename T, int NC, int PN>
cudaError_t launch_one(const ConvParams& p, cudaStream_t stream) {
    constexpr int kRows = kMode == ConvMode::Halo ? halo_rows(NC) : kTileH;
    void (*kernel)(ConvParams);
    if constexpr (uses_halo_kernel(kMode)) kernel = conv_halo_kernel<NC, PN, kMode, kExact, T>;
    else kernel = conv_wgmma_kernel<NC, PN, kMode, kExact, T>;
    static bool attr_set[64] = {};                        // the attribute is per function and context: one flag per device
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess && !(dev < 64 && attr_set[dev])) {
        e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax);
        // two CTAs per SM need the largest shared-memory carveout of the unified L1 / shared-memory array
        if (e == cudaSuccess && ric_ctas_per_sm(kMode, NC) > 1)
            e = cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        if (e == cudaSuccess && dev < 64) attr_set[dev] = true;
    }
    if (e != cudaSuccess) return e;
    dim3 grid((p.Wout + kTileW - 1) / kTileW, (p.Hout + kRows - 1) / kRows, p.B);
    kernel<<<grid, kThreads, conv_smem_bytes(kMode, NC, p.ksize, p.up), stream>>>(p);
    return cudaGetLastError();
}

template <ConvMode kMode, bool kExact, typename T>
cudaError_t launch_mode(const ConvParams& p, cudaStream_t stream) {
    switch (p.Cout) {
        case 32: return launch_one<kMode, kExact, T, 32, 32>(p, stream);
        case 64: return launch_one<kMode, kExact, T, 64, 64>(p, stream);
        case 96: return launch_one<kMode, kExact, T, 96, 32>(p, stream);
        case 128: return p.n128 ? launch_one<kMode, kExact, T, 128, 128>(p, stream) : launch_one<kMode, kExact, T, 128, 64>(p, stream);
        default: break;
    }
    if constexpr (!kExact) {              // split launches stop at 128 channels (wider layers run in pieces, conv.cuh kMaxPiece)
        switch (p.Cout) {
            case 160: return launch_one<kMode, kExact, T, 160, 32>(p, stream);
            case 192: return launch_one<kMode, kExact, T, 192, 64>(p, stream);
            case 224: return launch_one<kMode, kExact, T, 224, 32>(p, stream);
            case 256: return p.n128 ? launch_one<kMode, kExact, T, 256, 128>(p, stream) : launch_one<kMode, kExact, T, 256, 64>(p, stream);
            default: break;
        }
    }
    return cudaErrorInvalidConfiguration;
}

}  // namespace dsu
