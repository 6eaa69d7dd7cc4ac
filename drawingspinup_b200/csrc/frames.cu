// HBM-bound per-pixel kernels around the convolution stack: frame ingest (uint8 / fp32 -> activation
// storage, act.cuh), 2x2 max-pool, and the stand-alone uint8 steps of the reference's frame loop
// (custom_transforms.py:7-35, data.py:23-47, test_stage1.py:68-70, run_render.py:31-57).
// One thread per pixel (or per 8-channel group), 128-bit accesses where the layout allows.
#include "frames.cuh"

namespace dsu {

namespace {

// ToTensor + Normalize(0.5, 0.5) of custom_transforms.py:18-22: (u8/255 - 0.5)/0.5, fp32 ops in order
__device__ __forceinline__ float norm_u8(uint8_t v) {
    return __fdiv_rn(__fsub_rn(__fdiv_rn(static_cast<float>(v), 255.0f), 0.5f), 0.5f);
}

__global__ void ingest_f32_kernel(const float* __restrict__ x, int cin, int cpad, size_t npix_frame, size_t npix, ActOut out) {
    const size_t p = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
    if (p >= npix) return;
    const size_t n = p / npix_frame, q = p % npix_frame;
    const float* xp = x + n * cin * npix_frame + q;
    for (int g = 0; g < cpad; g += 8) {
        float v[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) v[c] = (g + c < cin) ? xp[static_cast<size_t>(g + c) * npix_frame] : 0.0f;
        store_act<8>(out, p, g, v);
    }
}

__global__ void frames_to_tensor_kernel(const uchar4* __restrict__ color, const uchar4* __restrict__ pos,
                                        const uint8_t* __restrict__ edge, size_t npix_frame, size_t npix,
                                        float* __restrict__ pre, float* __restrict__ mask_out) {
    const size_t p = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
    if (p >= npix) return;
    const size_t n = p / npix_frame, r = p % npix_frame;
    uchar4 c = color[p];
    const uchar4 q = pos[p];
    const float mask = __fdiv_rn(static_cast<float>(c.w), 255.0f);
    if (edge && edge[p] < 255) { c.x = 0; c.y = 0; c.z = 0; }
    float* o = pre + n * 6 * npix_frame + r;
    o[0] = norm_u8(c.x); o[npix_frame] = norm_u8(c.y); o[2 * npix_frame] = norm_u8(c.z);
    o[3 * npix_frame] = mask; o[4 * npix_frame] = norm_u8(q.x); o[5 * npix_frame] = norm_u8(q.y);
    if (mask_out) mask_out[p] = mask;
}

// 2x2 / stride 2 max-pool over NHWC fp16 (8 channels per thread)
__global__ void maxpool2_kernel(const __half* __restrict__ in, int in_pitch, int B, int Hin, int Win, int C, __half* out, int out_pitch) {
    const int Ho = Hin / 2, Wo = Win / 2, G = C / 8;
    const size_t total = static_cast<size_t>(B) * Ho * Wo * G;
    const size_t t = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
    if (t >= total) return;
    const int g = static_cast<int>(t % G);
    const size_t op = t / G;
    const int ox = static_cast<int>(op % Wo);
    const int oy = static_cast<int>((op / Wo) % Ho);
    const int n = static_cast<int>(op / (static_cast<size_t>(Wo) * Ho));
    float best[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const size_t ip = (static_cast<size_t>(n) * Hin + 2 * oy + (k >> 1)) * Win + 2 * ox + (k & 1);
        float v[8];
        unpack8(*reinterpret_cast<const uint4*>(in + ip * in_pitch + g * 8), v);
#pragma unroll
        for (int c = 0; c < 8; ++c)      // strict > keeps the first maximum, like F.max_pool2d's value
            if (k == 0 || v[c] > best[c]) best[c] = v[c];
    }
    *reinterpret_cast<uint4*>(out + op * out_pitch + g * 8) = pack8(best);
}

// the same pool over fp32 NHWC (4 channels per thread)
__global__ void maxpool2_f32_kernel(const float* __restrict__ in, int in_pitch, int B, int Hin, int Win, int C, float* out,
                                    int out_pitch) {
    const int Ho = Hin / 2, Wo = Win / 2, G = C / 4;
    const size_t total = static_cast<size_t>(B) * Ho * Wo * G;
    const size_t t = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
    if (t >= total) return;
    const int g = static_cast<int>(t % G);
    const size_t op = t / G;
    const int ox = static_cast<int>(op % Wo);
    const int oy = static_cast<int>((op / Wo) % Ho);
    const int n = static_cast<int>(op / (static_cast<size_t>(Wo) * Ho));
    float4 best = make_float4(0, 0, 0, 0);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const size_t ip = (static_cast<size_t>(n) * Hin + 2 * oy + (k >> 1)) * Win + 2 * ox + (k & 1);
        const float4 v = *reinterpret_cast<const float4*>(in + ip * in_pitch + g * 4);
        if (k == 0) best = v;
        else {      // strict > keeps the first maximum, like the fp16 kernel above and F.max_pool2d's value
            if (v.x > best.x) best.x = v.x;
            if (v.y > best.y) best.y = v.y;
            if (v.z > best.z) best.z = v.z;
            if (v.w > best.w) best.w = v.w;
        }
    }
    *reinterpret_cast<float4*>(out + op * out_pitch + g * 4) = best;
}

__global__ void to_image_space_kernel(const float* __restrict__ x, uint8_t* __restrict__ out, size_t n) {
    const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
    if (i < n) out[i] = to_u8(x[i]);
}

__global__ void overlap_edge_kernel(const uint8_t* __restrict__ edge, uchar4* rgba, size_t npix) {
    const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
    if (i < npix && edge[i] < 255) rgba[i] = make_uchar4(0, 0, 0, 255);
}

__global__ void compose_rgba_kernel(const float* __restrict__ y, const float* __restrict__ mask,
                                    size_t npix_frame, size_t npix, uchar4* __restrict__ out) {
    const size_t p = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
    if (p >= npix) return;
    const size_t n = p / npix_frame, r = p % npix_frame;
    const float* yp = y + n * 3 * npix_frame + r;
    const uint8_t a = static_cast<uint8_t>(static_cast<int>(__fmul_rn(mask[p], 255.0f)));   // (mask*255).astype(uint8)
    out[p] = make_uchar4(to_u8(yp[0]), to_u8(yp[npix_frame]), to_u8(yp[2 * npix_frame]), a);
}

// pos2edge (run_render.py:31-57): per channel Sobel-3 (BORDER_REFLECT_101) in float64 on u8/255 with
// the background (alpha < 255) forced to 2, max magnitude over the 3 channels > 0.3.
__device__ __forceinline__ bool pos_is_edge(const uchar4* __restrict__ f, int x, int y, int H, int W) {
    double v[3][3][3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        int yy = y + i - 1;
        yy = yy < 0 ? -yy : (yy >= H ? 2 * H - 2 - yy : yy);
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            int xx = x + j - 1;
            xx = xx < 0 ? -xx : (xx >= W ? 2 * W - 2 - xx : xx);
            const uchar4 q = f[static_cast<size_t>(yy) * W + xx];
            const bool bg = q.w < 255;
            v[0][i][j] = bg ? 2.0 : static_cast<double>(__fdiv_rn(static_cast<float>(q.x), 255.0f));
            v[1][i][j] = bg ? 2.0 : static_cast<double>(__fdiv_rn(static_cast<float>(q.y), 255.0f));
            v[2][i][j] = bg ? 2.0 : static_cast<double>(__fdiv_rn(static_cast<float>(q.z), 255.0f));
        }
    }
    double best = 0.0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const double gx = (v[c][0][2] - v[c][0][0]) + 2.0 * (v[c][1][2] - v[c][1][0]) + (v[c][2][2] - v[c][2][0]);
        const double gy = (v[c][2][0] - v[c][0][0]) + 2.0 * (v[c][2][1] - v[c][0][1]) + (v[c][2][2] - v[c][0][2]);
        best = fmax(best, sqrt(gx * gx + gy * gy));
    }
    return best > 0.3;
}
__global__ void pos2edge_kernel(const uchar4* __restrict__ pos, int B, int H, int W, uint8_t* __restrict__ edge) {
    const size_t p = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
    const size_t npf = static_cast<size_t>(H) * W;
    if (p >= npf * B) return;
    edge[p] = pos_is_edge(pos + (p / npf) * npf, static_cast<int>(p % W), static_cast<int>((p / W) % H), H, W) ? 255 : 0;
}


__global__ void ingest_u8_kernel(const uchar4* __restrict__ color, const uchar4* __restrict__ pos,
                                 const uint8_t* __restrict__ edge, int derive_edge, int H, int W, size_t npix, ActOut out) {
    const size_t p = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
    if (p >= npix) return;
    uchar4 c = color[p];
    const uchar4 q = pos[p];
    const float mask = __fdiv_rn(static_cast<float>(c.w), 255.0f);      // alpha BEFORE the edge burn-in (data.py:28)
    // overlap_edge_on_img: burn where the stored edge map (255 - pos2edge, run_render.py:117-120) is < 255.  derive_edge: no edge
    // map given - the same predicate straight from the pos frame (pos2edge fused into the ingest, nothing crosses PCIe)
    bool burn = false;
    if (edge) burn = edge[p] < 255;
    else if (derive_edge) {
        const size_t npf = static_cast<size_t>(H) * W;
        burn = pos_is_edge(pos + (p / npf) * npf, static_cast<int>(p % W), static_cast<int>((p / W) % H), H, W);
    }
    if (burn) { c.x = 0; c.y = 0; c.z = 0; }
    float v[8] = {norm_u8(c.x), norm_u8(c.y), norm_u8(c.z), mask, norm_u8(q.x), norm_u8(q.y), 0.0f, 0.0f};
    store_act<8>(out, p, 0, v);
}


// ---- nn.InstanceNorm2d (norm_layer='instance_norm', models.py:34-35; defaults: affine=False, no running stats, eps 1e-5,
// biased variance) between a convolution and its activation.  The convolution's epilogue leaves its raw fp32 output
// x[B][HW][C] in a scratch buffer; (1) per-(frame, channel, slice) sum and sum of squares in fp64, each block storing its
// partials to its own slot; (2) the slots summed in slice order, mean / 1/sqrt(var + eps); (3) normalise, activation, and
// the stores the fused epilogue would have done (residual stream, un-ReLU'd second copy, output).  Every sum runs in one
// fixed order, so the statistics are bit-reproducible run to run and independent of the batch a frame is in.
__global__ void instnorm_stats_kernel(const float* __restrict__ x, int HW, int C, int rows_per_slice, double* acc) {
    __shared__ double s_sum[8][33], s_sq[8][33];
    const int lane = threadIdx.x & 31, row = threadIdx.x >> 5;              // 8 pixel rows x 32 channels per block step
    const int c = blockIdx.x * 32 + lane, n = blockIdx.z;
    const int p0 = blockIdx.y * rows_per_slice, p1 = min(HW, p0 + rows_per_slice);
    double s = 0.0, q = 0.0;
    if (c < C) {
        const float* base = x + static_cast<size_t>(n) * HW * C + c;
        for (int p = p0 + row; p < p1; p += 8) {
            const double v = static_cast<double>(base[static_cast<size_t>(p) * C]);
            s += v; q += v * v;
        }
    }
    s_sum[row][lane] = s; s_sq[row][lane] = q;
    __syncthreads();
    if (row == 0 && c < C) {
#pragma unroll
        for (int r = 1; r < 8; ++r) { s += s_sum[r][lane]; q += s_sq[r][lane]; }
        double* slot = acc + ((static_cast<size_t>(n) * C + c) * kInormMaxSlices + blockIdx.y) * 2;
        slot[0] = s;
        slot[1] = q;
    }
}

__global__ void instnorm_finish_kernel(const double* __restrict__ acc, int total, int HW, int slices, float2* stats) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const double* slot = acc + static_cast<size_t>(i) * kInormMaxSlices * 2;
    double s = 0.0, q = 0.0;
    for (int k = 0; k < slices; ++k) { s += slot[2 * k]; q += slot[2 * k + 1]; }
    const double mean = s / HW;
    double var = q / HW - mean * mean;
    var = var < 0.0 ? 0.0 : var;
    stats[i] = make_float2(static_cast<float>(mean), static_cast<float>(1.0 / sqrt(var + 1e-5)));
}

__global__ void instnorm_apply_kernel(InstNormApply a) {
    const int G = a.C / 8;
    const size_t total = static_cast<size_t>(a.B) * a.HW * G;
    const size_t t = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
    if (t >= total) return;
    const int g = static_cast<int>(t % G);
    const size_t pix = t / G;
    const int n = static_cast<int>(pix / a.HW);
    const float* src = a.x + pix * a.C + g * 8;
    const float4 x0 = reinterpret_cast<const float4*>(src)[0], x1 = reinterpret_cast<const float4*>(src)[1];
    float v[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
    const float2* st = a.stats + static_cast<size_t>(n) * a.C + g * 8;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const float2 ms = st[c];
        v[c] = (v[c] - ms.x) * ms.y;
        if (a.act == 1) v[c] = fmaxf(v[c], 0.0f);
        else if (a.act == 2) v[c] = fmaxf(v[c], 0.2f * v[c]);
    }
    if (a.resid) store_f32<8>(a.resid + pix * a.C + g * 8, v);
    store_act<8>(a.out2, pix, g * 8, v);
    if (a.out_relu) {
#pragma unroll
        for (int c = 0; c < 8; ++c) v[c] = fmaxf(v[c], 0.0f);
    }
    store_act<8>(a.out, pix, g * 8, v);
}

inline unsigned blocks_for(size_t n, int threads) { return static_cast<unsigned>((n + threads - 1) / threads); }

}  // namespace

cudaError_t ingest_f32(const float* x, int B, int cin, int cpad, int H, int W, const ActOut& out, cudaStream_t st) {
    const size_t npf = static_cast<size_t>(H) * W, np = npf * B;
    ingest_f32_kernel<<<blocks_for(np, 256), 256, 0, st>>>(x, cin, cpad, npf, np, out);
    return cudaGetLastError();
}
cudaError_t ingest_u8(const uint8_t* color, const uint8_t* pos, const uint8_t* edge, int derive_edge, int B, int H, int W,
                      const ActOut& out, cudaStream_t st) {
    const size_t np = static_cast<size_t>(H) * W * B;
    ingest_u8_kernel<<<blocks_for(np, 256), 256, 0, st>>>(reinterpret_cast<const uchar4*>(color), reinterpret_cast<const uchar4*>(pos), edge,
                                                          derive_edge, H, W, np, out);
    return cudaGetLastError();
}
cudaError_t frames_to_tensor(const uint8_t* color, const uint8_t* pos, const uint8_t* edge, int B, int H, int W,
                             float* pre, float* mask, cudaStream_t st) {
    const size_t npf = static_cast<size_t>(H) * W, np = npf * B;
    frames_to_tensor_kernel<<<blocks_for(np, 256), 256, 0, st>>>(reinterpret_cast<const uchar4*>(color),
                                                                 reinterpret_cast<const uchar4*>(pos), edge, npf, np, pre, mask);
    return cudaGetLastError();
}
cudaError_t maxpool2(const ActOut& in, const ActOut& out, int B, int Hin, int Win, int C, cudaStream_t st) {
    if (in.lo || out.lo || !in.f32 != !out.f32) return cudaErrorInvalidValue;
    const size_t opix = static_cast<size_t>(B) * (Hin / 2) * (Win / 2);
    if (in.f32)
        maxpool2_f32_kernel<<<blocks_for(opix * (C / 4), 256), 256, 0, st>>>(in.f32 + in.choff, in.pitch, B, Hin, Win, C,
                                                                             out.f32 + out.choff, out.pitch);
    else
        maxpool2_kernel<<<blocks_for(opix * (C / 8), 256), 256, 0, st>>>(in.hi + in.choff, in.pitch, B, Hin, Win, C,
                                                                         out.hi + out.choff, out.pitch);
    return cudaGetLastError();
}
cudaError_t to_image_space(const float* x, uint8_t* out, size_t n, cudaStream_t st) {
    to_image_space_kernel<<<blocks_for(n, 256), 256, 0, st>>>(x, out, n);
    return cudaGetLastError();
}
cudaError_t overlap_edge(const uint8_t* edge, uint8_t* rgba, size_t npix, cudaStream_t st) {
    overlap_edge_kernel<<<blocks_for(npix, 256), 256, 0, st>>>(edge, reinterpret_cast<uchar4*>(rgba), npix);
    return cudaGetLastError();
}
cudaError_t compose_rgba(const float* y, const float* mask, int B, int H, int W, uint8_t* out, cudaStream_t st) {
    const size_t npf = static_cast<size_t>(H) * W, np = npf * B;
    compose_rgba_kernel<<<blocks_for(np, 256), 256, 0, st>>>(y, mask, npf, np, reinterpret_cast<uchar4*>(out));
    return cudaGetLastError();
}
cudaError_t pos2edge(const uint8_t* pos, int B, int H, int W, uint8_t* edge, cudaStream_t st) {
    const size_t np = static_cast<size_t>(H) * W * B;
    pos2edge_kernel<<<blocks_for(np, 256), 256, 0, st>>>(reinterpret_cast<const uchar4*>(pos), B, H, W, edge);
    return cudaGetLastError();
}

cudaError_t instance_norm(const InstNormApply& a, double* acc, cudaStream_t st) {
    if (a.C % 8 || a.B < 1 || a.HW < 1 || !a.x || !a.stats || !acc) return cudaErrorInvalidValue;
    int slices = (a.HW + 4095) / 4096;                       // >= 4096 pixels per block and channel group, at most 64 slices
    slices = slices > kInormMaxSlices ? kInormMaxSlices : slices;
    const int rows = (a.HW + slices - 1) / slices;
    instnorm_stats_kernel<<<dim3((a.C + 31) / 32, slices, a.B), 256, 0, st>>>(a.x, a.HW, a.C, rows, acc);
    instnorm_finish_kernel<<<blocks_for(static_cast<size_t>(a.B) * a.C, 128), 128, 0, st>>>(acc, a.B * a.C, a.HW, slices,
                                                                                          a.stats);
    const size_t total = static_cast<size_t>(a.B) * a.HW * (a.C / 8);
    instnorm_apply_kernel<<<blocks_for(total, 256), 256, 0, st>>>(a);
    return cudaGetLastError();
}

}  // namespace dsu
