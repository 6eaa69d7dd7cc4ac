// Network planner + C ABI (include/dsu_b200.h) of the stylization engine.
//
// Turns the constructor arguments of GeneratorJ / GeneratorJ_RIC (training/models.py:24-111,
// 200-291) and a loaded state dict into a list of fused convolution launches (conv_wgmma.cuh):
// BatchNorm (eval) is folded into per-channel scale/shift, conv weights are rounded to fp16
// (hi [+lo]) or bf16 (hi [+lo]) and pre-swizzled into tensor-core tiles, skip connections / nearest-x2 upsampling /
// stride / concat become slot tables, and the dead stage-1 smoother conv (models.py:348-350) is
// dropped.  Activations live in NHWC workspace buffers owned by the handle, in one of the forms of act.cuh.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cctype>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <set>
#include <string>
#include <vector>

#include "../../include/dsu_b200.h"
#include "conv.cuh"
#include "frames.cuh"

using namespace dsu;

namespace {

thread_local std::string g_err;

int fail(int code, const std::string& msg) {
    g_err = msg;
    return code;
}
#define CUDA_TRY(expr)                                                                         \
    do {                                                                                       \
        cudaError_t e__ = (expr);                                                              \
        if (e__ != cudaSuccess)                                                                \
            return fail(DSU_E_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e__));      \
    } while (0)

enum BufId { SK0 = 0, P0, O1, P1, O2, TT, UU, V2, V1, C11, S0, NBUF };

struct SegDef {
    int buf, choff, nch;   // buffer, first channel, channels consumed (multiple of 8: the stored, padded width)
    int wch0, wn;          // first weight input channel, real weight channels (<= nch)
};

// stored width of an activation of c channels (conv.cuh: output-channel pieces)
int padded(int c) { return (c + kChannelAlign - 1) / kChannelAlign * kChannelAlign; }

struct LayerDef {
    std::string name, wkey, bkey, bn, bn2;
    int k = 3, pad = 1, stride = 1, up = 0, ric = 0, cout = 0, level_out = 0;
    int n0 = 0, nw = 0;    // output-channel piece (conv.cuh): first channel and width of this launch, of the padded(cout) channels
    std::vector<SegDef> segs;
    int act = 0;
    int out_buf = -1, out_choff = 0, out_relu = 0, out2_buf = -1;
    int resid_in = 0, resid_out = 0, final = 0;
    int inorm = 0;         // norm_layer='instance_norm': the epilogue leaves the raw fp32 output in a scratch buffer; a type-2 step normalises
    // sub-pixel class py*2+px of a nearest-x2 + 3x3 convolution (models.py:180-192, SURVEY 8a row a7):
    // out(2y+py, 2x+px) = sum over a,b in {0,1} of Wc[a][b] * in(y+a-1+py, x+b-1+px), Wc = sums of the 3x3 taps that hit the
    // same source pixel - exact including the zero border, 4 taps instead of 9 per output pixel.  k = 2 for such a layer and
    // wk = 3 is the kernel size of the stored weights; -1 = ordinary layer
    int sub = -1, wk = 0;
    int pad_y = 0, pad_x = 0;  // padding above / left of the window (compiled at finalize; a sub-pixel class pads (1 - py, 1 - px))
    // compiled at finalize
    int first = 0;         // conv0-shaped: one <= 8-channel segment, stride 1, k > 3
    ConvMode mode = ConvMode::Tap;  // plan-time mode (Tap, Halo or Ric); conv_mode applies the run-time knobs
    int nchunks = 0, nblocks = 0;
    uint32_t kmask_full = 0xF, kmask_last = 0xF, kmask2_full = 0, kmask2_last = 0;
    Slot* d_slots = nullptr;
    Slot* d_hslots = nullptr;  // halo mode: [nblocks][8] channels of each 16-byte slot of a halo pixel
    uint8_t* d_wpack = nullptr;
    float *d_scale = nullptr, *d_shift = nullptr, *d_scale2 = nullptr, *d_shift2 = nullptr;   // [nw]: this piece's channels
    float* d_w12 = nullptr;   // final layer: [3][nw] conv_12 weights of this piece's channels
    double macs_per_px = 0;   // live MACs per output pixel
    int live() const { return std::min(nw, cout - n0); }   // real (not padding) output channels of the piece
};

struct Step {
    int type;    // 0 conv, 1 maxpool, 2 instance norm + activation + stores of layer `layer` (after its last launch),
                 // 3 conv_12 of a final layer that ran in pieces (after its last piece)
    int layer;
    int src, src_choff, C, dst;
};

// Development knobs: read ONCE from the environment (DSU_<NAME>) by dsu_create, adjustable per handle through
// dsu_set_knob (tests / tools).
struct Knobs {
    int first = 1;            // the first layer builds its A chunks from a shared-memory input halo; 0 = tap mode (global loads)
    int halo = 1;             // plan-time: the other stride-1 layers without fused upsampling and Cout <= 64 in halo mode; 0 = tap mode
    int n128 = 1;             // Cout a multiple of 128: N = 128 wgmma instructions; 0 = N = 64 (two instructions per K step)
    int subpixel = 1;         // plan-time: stage-2 nearest-x2 + 3x3 as four 2x2 sub-pixel convolutions
    int derive_edge = 0;      // stage 2, no edge map passed: burn the edges pos2edge finds in the pos frames (fused into the ingest)
    int ric_halo = 1;         // RIC layers read stencil and corners from shared memory (conv_halo_kernel); 0 = gather from global memory
};
struct KnobName { const char* name; int Knobs::*field; };
const KnobName kKnobNames[] = {
    {"first", &Knobs::first}, {"n128", &Knobs::n128}, {"subpixel", &Knobs::subpixel}, {"derive_edge", &Knobs::derive_edge},
    {"halo", &Knobs::halo}, {"ric_halo", &Knobs::ric_halo},
};
Knobs knobs_from_env() {
    Knobs k;
    for (const KnobName& kn : kKnobNames) {
        std::string env = "DSU_";
        for (const char* c = kn.name; *c; ++c) env += static_cast<char>(std::toupper(static_cast<unsigned char>(*c)));
        if (const char* v = std::getenv(env.c_str())) k.*(kn.field) = std::atoi(v);
    }
    return k;
}

// Every C-ABI entry point runs on the handle's device and leaves the caller's current device as it found it.
struct DeviceGuard {
    int prev = -1;
    cudaError_t err = cudaSuccess;
    explicit DeviceGuard(int dev) {
        err = cudaGetDevice(&prev);
        if (err == cudaSuccess && prev != dev) err = cudaSetDevice(dev);
        else if (err == cudaSuccess) prev = -1;          // nothing to restore
    }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};
#define DEVICE_GUARD(h)                                                                        \
    DeviceGuard guard__((h)->cfg.device);                                                      \
    if (guard__.err != cudaSuccess) return fail(DSU_E_CUDA, std::string("cudaSetDevice: ") + cudaGetErrorString(guard__.err))

struct Level {
    int h = 0, w = 0;
    float2* lyx = nullptr;    // [h*w][8] bilinear fractions in rotated tap order
    uint8_t* oct = nullptr;   // [h*w] octant (tap rotation) of the pixel
    uint2* wh = nullptr;      // [h*w][8] fp16 bilinear weights {w00,w01,w10,w11} per rotated tap
    float max_clamp = 0;      // largest adjustment needed to express a tap in its static quadrant
};

}  // namespace

struct dsu_engine {
    dsu_config cfg{};
    Knobs knobs;
    int cin_pad = 8;
    bool exact = false, finalized = false;
    bool bf16 = false;        // DSU_PREC_BF16 / BF16X3: bf16 weights and activation planes (the fp16 / split-fp16 plan)
    std::map<std::string, std::vector<int64_t>> expected;
    std::vector<std::string> expected_order;
    std::map<std::string, std::vector<float>> w;
    std::set<std::string> loaded;
    std::vector<LayerDef> layers;
    std::vector<Step> steps;
    bool f32_acts = false;    // stage 1 in a split mode: activation buffers hold fp32 instead of hi + lo planes
    int buf_level[NBUF]{}, buf_C[NBUF]{};
    bool buf_used[NBUF]{};
    float* d_b12 = nullptr;
    int tail_pieces = 1;      // pieces of the final layer; > 1: its epilogues leave conv_12 partials in tail_part
    // shape-dependent state
    int B = 0, H = 0, W = 0;
    __half* buf_hi[NBUF]{};
    __half* buf_lo[NBUF]{};
    size_t buf_cap[NBUF]{};
    float* resid = nullptr;
    size_t resid_cap = 0;
    float* inorm_x = nullptr;      // norm_layer='instance_norm': raw fp32 output of the convolution being normalised
    float2* inorm_stats = nullptr; // [B][Cmax] (mean, 1/sqrt(var + eps))
    double* inorm_acc = nullptr;   // [B][Cmax][kInormMaxSlices][2] partial sum, sum of squares of each statistics slice
    size_t inorm_cap = 0, inorm_stats_cap = 0;   // bytes of inorm_x, inorm_stats
    float* tail_part = nullptr;    // [tail_pieces][3][B*H*W] conv_12 partial dot products of the final layer's pieces
    size_t tail_cap = 0;
    Level lv[3];
    std::map<std::pair<int, int>, std::vector<float>> user_offsets;
    uint8_t *io_color = nullptr, *io_pos = nullptr, *io_edge = nullptr, *io_out = nullptr;
    size_t io_cap = 0;
};

namespace {

// ------------------------------------------------------------------ configuration -> plan
std::string conv12_prefix(const dsu_config& c) { return c.tanh ? "conv_12.0" : "conv_12"; }

void expect(dsu_engine* E, const std::string& key, std::vector<int64_t> shape) {
    E->expected[key] = shape;
    E->expected_order.push_back(key);
}

void expect_bn(dsu_engine* E, const std::string& p, int c) {
    expect(E, p + ".weight", {c});
    expect(E, p + ".bias", {c});
    expect(E, p + ".running_mean", {c});
    expect(E, p + ".running_var", {c});
    expect(E, p + ".num_batches_tracked", {});
}

int build_plan(dsu_engine* E) {
    const dsu_config& c = E->cfg;
    const int* f = c.filters;
    const bool ric = c.kind == DSU_KIND_GENERATORJ_RIC;
    const bool bn = c.norm == DSU_NORM_BATCH;
    const bool inorm = c.norm == DSU_NORM_INSTANCE;     // the twelve norm_layer modules are nn.InstanceNorm2d (no state)
    const int cin = c.input_channels, cp = E->cin_pad;
    const int k0 = ric ? 3 : 7;
    auto conv_keys = [&](const std::string& p, int co, int ci, int k, bool may_bias) {
        expect(E, p + ".weight", {co, ci, k, k});
        if (may_bias && c.use_bias) expect(E, p + ".bias", {co});
    };
    // state-dict layout (SURVEY.md 8a row a8; models.py:41-111 / 220-284)
    conv_keys("conv0.conv", f[0], cin, k0, true);
    if (bn) expect_bn(E, "conv0.normalization", f[0]);
    conv_keys("conv1.conv", f[1], f[0], 3, true);
    if (bn) expect_bn(E, "conv1.normalization", f[1]);
    conv_keys("conv2.conv", f[2], f[1], 3, true);
    if (bn) expect_bn(E, "conv2.normalization", f[2]);
    for (int i = 0; i < c.resnet_blocks; ++i) {
        const std::string p = "resnets." + std::to_string(i) + ".";
        conv_keys(p + "conv_0", f[2], f[2], 3, true);
        if (bn) expect_bn(E, p + "normalization", f[2]);
        conv_keys(p + "conv_1", f[2], f[2], 3, true);
    }
    conv_keys("upconv2.1", f[4], f[3] + f[2], 3, false);
    if (bn) expect_bn(E, "upconv2.2", f[4]);
    conv_keys("upconv1.1", f[4], f[4] + f[1], 3, false);
    if (bn) expect_bn(E, "upconv1.2", f[4]);
    conv_keys("conv_11.0", f[5], f[0] + f[4] + cin, k0, true);
    if (c.append_smoothers) {
        conv_keys("conv_11_a.0", f[5], f[5], 3, true);
        expect_bn(E, "conv_11_a.2", f[5]);
        conv_keys("conv_11_a.3", f[5], f[5], 3, true);
    }
    expect(E, conv12_prefix(c) + ".weight", {3, f[5], 1, 1});
    expect(E, conv12_prefix(c) + ".bias", {3});

    // activation buffers, every width stored padded to a multiple of 32 (x to 8 behind conv0's channels in SK0)
    int F[6];
    for (int i = 0; i < 6; ++i) F[i] = padded(f[i]);
    auto setbuf = [&](int b, int level, int C) { E->buf_level[b] = level; E->buf_C[b] = C; E->buf_used[b] = true; };
    setbuf(SK0, 0, F[0] + cp);
    setbuf(O1, 1, F[1]);
    setbuf(O2, 2, F[2]);
    if (ric) { setbuf(P0, 1, F[0]); setbuf(P1, 2, F[1]); }
    if (c.resnet_blocks > 0) { setbuf(TT, 2, F[2]); setbuf(UU, 2, F[2]); }
    setbuf(V2, 1, F[4]);
    setbuf(V1, 0, F[4]);
    setbuf(C11, 0, F[5]);
    if (c.append_smoothers && !ric) setbuf(S0, 0, F[5]);

    // in stage 1 the deformable calls pass only .weight, so conv biases are never applied (models.py:302-351)
    auto bias_of = [&](const std::string& p) { return (c.use_bias && !ric) ? p + ".bias" : std::string(); };
    // one launch per output-channel piece, widest first (conv.cuh); a one-piece layer keeps its name, pieces get ".n<i>"
    const int cap = kMaxPiece(E->exact);
    auto add = [&](LayerDef L) {
        const int cpad = padded(L.cout), np = (cpad + cap - 1) / cap;
        const std::string base = L.name;
        for (int i = 0; i < np; ++i) {
            LayerDef P = L;
            P.n0 = i * cap; P.nw = std::min(cap, cpad - P.n0);
            if (np > 1) P.name = base + ".n" + std::to_string(i);
            E->layers.push_back(P);
            E->steps.push_back(Step{0, (int)E->layers.size() - 1, 0, 0, 0, 0});
        }
        if (L.final && np > 1) { E->tail_pieces = np; E->steps.push_back(Step{3, (int)E->layers.size() - 1, 0, 0, 0, 0}); }
    };
    auto add_norm = [&]() { if (inorm) E->steps.push_back(Step{2, (int)E->layers.size() - 1, 0, 0, 0, 0}); };
    {
        LayerDef L; L.name = "conv0"; L.wkey = "conv0.conv.weight"; L.bkey = bias_of("conv0.conv");
        L.bn = bn ? "conv0.normalization" : ""; L.k = k0; L.pad = k0 / 2; L.ric = ric; L.cout = f[0]; L.level_out = 0;
        L.segs = {{SK0, F[0], cp, 0, cin}}; L.act = 2; L.out_buf = SK0; L.out_choff = 0; L.inorm = inorm;
        add(L); add_norm();
    }
    if (ric) E->steps.push_back(Step{1, -1, SK0, 0, F[0], P0});
    {
        LayerDef L; L.name = "conv1"; L.wkey = "conv1.conv.weight"; L.bkey = bias_of("conv1.conv");
        L.bn = bn ? "conv1.normalization" : ""; L.stride = ric ? 1 : 2; L.ric = ric; L.cout = f[1]; L.level_out = 1;
        L.segs = {{ric ? P0 : SK0, 0, F[0], 0, f[0]}}; L.act = 2; L.out_buf = O1; L.inorm = inorm;
        add(L); add_norm();
    }
    if (ric) E->steps.push_back(Step{1, -1, O1, 0, F[1], P1});
    const bool has_res = c.resnet_blocks > 0;
    {
        LayerDef L; L.name = "conv2"; L.wkey = "conv2.conv.weight"; L.bkey = bias_of("conv2.conv");
        L.bn = bn ? "conv2.normalization" : ""; L.stride = ric ? 1 : 2; L.ric = ric; L.cout = f[2]; L.level_out = 2;
        L.segs = {{ric ? P1 : O1, 0, F[1], 0, f[1]}}; L.act = 2;
        if (has_res) { L.out_buf = TT; L.out_relu = 1; L.out2_buf = O2; L.resid_out = 1; }
        else L.out_buf = O2;
        L.inorm = inorm;
        add(L); add_norm();
    }
    for (int i = 0; i < c.resnet_blocks; ++i) {
        const std::string p = "resnets." + std::to_string(i) + ".";
        LayerDef A; A.name = p + "conv_0"; A.wkey = p + "conv_0.weight"; A.bkey = bias_of(p + "conv_0");
        A.bn = bn ? p + "normalization" : ""; A.ric = ric; A.cout = f[2]; A.level_out = 2;
        A.segs = {{TT, 0, F[2], 0, f[2]}}; A.act = 1; A.out_buf = UU; A.inorm = inorm;
        add(A); add_norm();
        LayerDef Bl; Bl.name = p + "conv_1"; Bl.wkey = p + "conv_1.weight"; Bl.bkey = bias_of(p + "conv_1");
        Bl.ric = ric; Bl.cout = f[2]; Bl.level_out = 2;
        Bl.segs = {{UU, 0, F[2], 0, f[2]}}; Bl.act = 0; Bl.resid_in = 1; Bl.resid_out = 1;
        Bl.out_buf = TT; Bl.out_relu = (i + 1 < c.resnet_blocks) ? 1 : 0;
        add(Bl);
    }
    // plain (stage-2) up-convolutions run as four sub-pixel 2x2 convolutions on the low-resolution source (2.25x fewer
    // MACs); DSU_SUBPIXEL=0 at dsu_create restores the 3x3 form
    const bool subpixel = !ric && E->knobs.subpixel != 0;
    auto add_up = [&](LayerDef L) {
        L.inorm = inorm;
        if (!subpixel) { L.up = 1; add(L); add_norm(); return; }
        const std::string base = L.name;
        for (int cls = 0; cls < 4; ++cls) {
            LayerDef S = L;
            S.name = base + ".s" + std::to_string(cls);
            S.up = 0; S.sub = cls; S.wk = 3; S.k = 2; S.pad = 0;
            add(S);
        }
        add_norm();          // statistics over the whole output: after the fourth class
    };
    {
        LayerDef L; L.name = "upconv2"; L.wkey = "upconv2.1.weight"; L.bn = bn ? "upconv2.2" : "";
        L.ric = ric; L.cout = f[4]; L.level_out = 1;
        L.segs = {{has_res ? TT : O2, 0, F[2], 0, f[2]}, {O2, 0, F[2], f[3], f[2]}}; L.act = 1; L.out_buf = V2;
        add_up(L);
    }
    {
        LayerDef L; L.name = "upconv1"; L.wkey = "upconv1.1.weight"; L.bn = bn ? "upconv1.2" : "";
        L.ric = ric; L.cout = f[4]; L.level_out = 0;
        L.segs = {{V2, 0, F[4], 0, f[4]}, {O1, 0, F[1], f[4], f[1]}}; L.act = 1; L.out_buf = V1;
        add_up(L);
    }
    {
        LayerDef L; L.name = "conv_11"; L.wkey = "conv_11.0.weight"; L.bkey = bias_of("conv_11.0");
        L.k = k0; L.pad = k0 / 2; L.ric = ric; L.cout = f[5]; L.level_out = 0;
        L.segs = {{V1, 0, F[4], 0, f[4]}, {SK0, 0, F[0], f[4], f[0]}, {SK0, F[0], cp, f[4] + f[0], cin}};
        L.act = 1;
        if (c.append_smoothers) L.out_buf = C11; else L.final = 1;
        add(L);
    }
    if (c.append_smoothers) {
        if (!ric) {   // stage 1: this conv is dead code (models.py:348-350) and is skipped
            LayerDef L; L.name = "conv_11_a.0"; L.wkey = "conv_11_a.0.weight"; L.bkey = bias_of("conv_11_a.0");
            L.bn2 = "conv_11_a.2"; L.cout = f[5]; L.level_out = 0;
            L.segs = {{C11, 0, F[5], 0, f[5]}}; L.act = 1; L.out_buf = S0;
            add(L);
        }
        LayerDef L; L.name = "conv_11_a.3"; L.wkey = "conv_11_a.3.weight"; L.bkey = bias_of("conv_11_a.3");
        L.ric = ric; L.cout = f[5]; L.level_out = 0;
        L.segs = {{ric ? C11 : S0, 0, F[5], 0, f[5]}}; L.act = 1; L.final = 1;
        add(L);
    }
    return DSU_OK;
}

// ------------------------------------------------------------------ finalize: fold + pack
template <typename T>
int upload(T** dst, const std::vector<T>& src) {
    if (*dst) { cudaFree(*dst); *dst = nullptr; }
    if (src.empty()) return DSU_OK;
    CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(dst), src.size() * sizeof(T)));
    CUDA_TRY(cudaMemcpy(*dst, src.data(), src.size() * sizeof(T), cudaMemcpyHostToDevice));
    return DSU_OK;
}

int compile_layer(dsu_engine* E, LayerDef& L) {
    const bool exact = E->exact;
    const int C = L.cout, k = L.k;
    int cin_total = 0;
    for (const SegDef& s : L.segs) cin_total = std::max(cin_total, s.wch0 + s.wn);
    std::vector<float> Wsub;
    if (L.sub >= 0) {
        // 2x2 weights of sub-pixel class (py, px): tap a of an even output row (py = 0) collects kernel rows {0} / {1,2}, of an
        // odd row {0,1} / {2} (the rows of the nearest-x2 image that map to source row y+a-1+py); same for columns
        const std::vector<float>& W3 = E->w.at(L.wkey);
        if (L.wk != 3 || k != 2 || W3.size() != static_cast<size_t>(C) * cin_total * 9)
            return fail(DSU_E_INVALID, "weight size mismatch for " + L.wkey);
        const int py = L.sub >> 1, px = L.sub & 1;
        auto members = [](int parity, int tap, int* lo, int* hi) {
            if (parity == 0) { *lo = tap == 0 ? 0 : 1; *hi = tap == 0 ? 0 : 2; }
            else { *lo = tap == 0 ? 0 : 2; *hi = tap == 0 ? 1 : 2; }
        };
        Wsub.assign(static_cast<size_t>(C) * cin_total * 4, 0.0f);
        for (int o = 0; o < C; ++o)
            for (int c = 0; c < cin_total; ++c)
                for (int a = 0; a < 2; ++a)
                    for (int b = 0; b < 2; ++b) {
                        int r0, r1, c0, c1;
                        members(py, a, &r0, &r1);
                        members(px, b, &c0, &c1);
                        double acc = 0;
                        for (int kh = r0; kh <= r1; ++kh)
                            for (int kw = c0; kw <= c1; ++kw) acc += W3[((static_cast<size_t>(o) * cin_total + c) * 3 + kh) * 3 + kw];
                        Wsub[((static_cast<size_t>(o) * cin_total + c) * 2 + a) * 2 + b] = static_cast<float>(acc);
                    }
    }
    const std::vector<float>& Wt = L.sub >= 0 ? Wsub : E->w.at(L.wkey);
    if (Wt.size() != static_cast<size_t>(C) * cin_total * k * k) return fail(DSU_E_INVALID, "weight size mismatch for " + L.wkey);

    // A "data slot" is 8 input channels of one concat segment at one tap.  A chunk (8 smem slots =
    // 64 K elements) holds 8 data slots (fp16 mode) or 4 data slots as [hi x4 | lo x4] (exact mode).
    // plain conv: data slots are packed densely over (tap, segment, channel group);
    // RIC conv: channel groups are packed into blocks and every block spans the 9 taps (one chunk each).
    struct HSlot { int kh, kw, seg, choff, wch, nvalid, gi; };   // gi: channel group inside its block (halo mode)
    const int dpc = exact ? 4 : 8;            // data slots per chunk
    std::vector<std::vector<HSlot>> chunks;   // data slots of every chunk, in execution order
    std::vector<Slot> slots, hslots;
    double real_k = 0;
    for (const SegDef& s : L.segs) real_k += static_cast<double>(s.wn) * k * k;
    L.macs_per_px = real_k * L.live();
    // algorithmic work of a sub-pixel class = a quarter of the 3x3 layer's output pixels (flops are reported per output pixel of level_out)
    if (L.sub >= 0) L.macs_per_px = real_k / 4.0 * 9.0 / 4.0 * L.live();
    // a sub-pixel class (py, px) pads its 2x2 window by (1 - py, 1 - px) above and left; the slot taps and the halo origin both use it
    L.pad_y = L.sub >= 0 ? 1 - (L.sub >> 1) : L.pad;
    L.pad_x = L.sub >= 0 ? 1 - (L.sub & 1) : L.pad;
    const int pad_y = L.pad_y, pad_x = L.pad_x;
    auto dev_slot = [&](const HSlot& h, bool lo_plane) {
        Slot sl{};
        sl.dy = static_cast<int8_t>(h.kh - pad_y);
        sl.dx = static_cast<int8_t>(h.kw - pad_x);
        sl.seg = static_cast<uint8_t>(h.seg + (lo_plane ? kMaxSeg / 2 : 0));
        sl.valid = 1;
        sl.choff = static_cast<uint16_t>(h.choff);
        sl.hslot = static_cast<uint8_t>(h.gi + (lo_plane ? 4 : 0));
        return sl;
    };
    auto push_dev_slots = [&](const std::vector<HSlot>& ds, std::vector<Slot>& dst) {
        for (int j = 0; j < 8; ++j) {
            const int d = exact ? (j & 3) : j;
            if (d < static_cast<int>(ds.size())) dst.push_back(dev_slot(ds[d], exact && j >= 4));
            else dst.push_back(Slot{});
        }
    };
    // channel groups (8 channels of one segment) over the concat, packed into blocks of one 128-byte row (RIC / halo mode)
    std::vector<std::vector<HSlot>> blocks;
    for (size_t si = 0; si < L.segs.size(); ++si) {
        const SegDef& s = L.segs[si];
        for (int c8 = 0; c8 < s.nch; c8 += 8) {
            if (blocks.empty() || static_cast<int>(blocks.back().size()) == dpc) blocks.emplace_back();
            blocks.back().push_back(HSlot{0, 0, (int)si, s.choff + c8, s.wch0 + c8, std::max(0, std::min(8, s.wn - c8)), (int)blocks.back().size()});
        }
    }
    L.first = (!L.ric && L.stride == 1 && L.up == 0 && L.sub < 0 && L.segs.size() == 1 && L.segs[0].nch <= 8 && k > 3 && L.pad == (k - 1) / 2) ? 1 : 0;
    // Halo mode needs k >= 2: the halo of block b + 1 is loaded in the first chunk of block b and read k^2 - 1 chunks later.
    // The mode follows the layer's padded width, the same for every piece.
    L.mode = L.ric ? ConvMode::Ric
           : (L.stride == 1 && L.up == 0 && k >= 2 && (L.first || (E->knobs.halo && padded(C) <= 64))) ? ConvMode::Halo : ConvMode::Tap;
    L.nblocks = L.mode == ConvMode::Tap ? 0 : static_cast<int>(blocks.size());
    if (!L.ric) {
        std::vector<HSlot> all;
        if (L.mode == ConvMode::Halo) {
            // (block, tap, group): every full block is k^2 chunks of one tap each; the last block's groups are packed densely
            // over taps, so the chunk count equals tap mode's.  A one-group layer (conv0) gets the same chunks as in tap mode.
            for (const std::vector<HSlot>& blk : blocks) {
                push_dev_slots(blk, hslots);
                for (int kh = 0; kh < k; ++kh)
                    for (int kw = 0; kw < k; ++kw)
                        for (HSlot h : blk) { h.kh = kh; h.kw = kw; all.push_back(h); }
            }
        } else {
            for (int kh = 0; kh < k; ++kh) {
                for (int kw = 0; kw < k; ++kw)
                    for (size_t si = 0; si < L.segs.size(); ++si) {
                        const SegDef& s = L.segs[si];
                        for (int c8 = 0; c8 < s.nch; c8 += 8)
                            all.push_back(HSlot{kh, kw, (int)si, s.choff + c8, s.wch0 + c8, std::max(0, std::min(8, s.wn - c8)), 0});
                    }
            }
        }
        for (size_t i = 0; i < all.size(); i += dpc) {
            std::vector<HSlot> ds(all.begin() + i, all.begin() + std::min(all.size(), i + dpc));
            push_dev_slots(ds, slots);
            chunks.push_back(ds);
        }
    } else {
        for (const std::vector<HSlot>& blk : blocks) {
            push_dev_slots(blk, slots);                        // one slot row per BLOCK
            for (int tap = 0; tap < k * k; ++tap) {
                std::vector<HSlot> ds = blk;
                for (HSlot& h : ds) { h.kh = tap / k; h.kw = tap % k; }
                chunks.push_back(ds);
            }
        }
    }
    L.nchunks = static_cast<int>(chunks.size());
    const size_t tile = static_cast<size_t>(L.nw) * 128;   // the piece's output channels; rows past cout stay zero
    std::vector<uint8_t> pack(static_cast<size_t>(L.nchunks) * tile, 0);
    size_t off = 0;
    auto put = [&](size_t tile_off, int row, int slot, int ci, auto val) {     // val: __half or __nv_bfloat16
        static_assert(sizeof(val) == 2, "16-bit weight elements");
        const size_t b = tile_off + static_cast<size_t>(row) * 128 + ((static_cast<size_t>(slot) ^ (row & 7)) << 4) + ci * 2;
        std::memcpy(&pack[b], &val, 2);
    };
    for (int q = 0; q < L.nchunks; ++q) {
        const std::vector<HSlot>& ds = chunks[q];
        const int nd = static_cast<int>(ds.size());
        // B tile(s): row o = output channel, 128 B = 64 K elements, 16-byte slots XOR-swizzled by (row & 7)
        for (int o = 0; o < L.live(); ++o)
            for (int d = 0; d < nd; ++d) {
                const HSlot& h = ds[d];
                for (int ci = 0; ci < h.nvalid; ++ci) {
                    const float wv = Wt[((static_cast<size_t>(L.n0 + o) * cin_total + h.wch + ci) * k + h.kh) * k + h.kw];
                    if (E->bf16) {
                        const __nv_bfloat16 wb = __float2bfloat16_rn(wv);
                        put(off, o, d, ci, wb);
                        if (exact) put(off, o, d + 4, ci, __float2bfloat16_rn(wv - __bfloat162float(wb)));
                        continue;
                    }
                    const __half wh = __float2half_rn(wv);
                    put(off, o, d, ci, wh);
                    if (exact) put(off, o, d + 4, ci, __float2half_rn(wv - __half2float(wh)));   // [W_hi | W_lo] in one row
                }
            }
        off += tile;
    }
    pack.resize(off);
    // K-step masks (ConvParams) of a chunk of nd data slots; only the ragged last chunk (tap / halo mode) or the chunks of
    // the last channel block (RIC) have fewer data slots than the first chunk
    auto kmasks = [&](size_t nd, uint32_t* km, uint32_t* km2) {
        const uint32_t mask = (1u << ((nd + 1) / 2)) - 1;      // the K=16 steps covering the data slots
        *km = exact ? mask | (mask << 2) : mask;
        *km2 = exact ? mask : 0u;
    };
    kmasks(chunks.front().size(), &L.kmask_full, &L.kmask2_full);
    kmasks(chunks.back().size(), &L.kmask_last, &L.kmask2_last);
    int rc_up;
    if ((rc_up = upload(&L.d_slots, slots))) return rc_up;
    if ((rc_up = upload(&L.d_hslots, hslots))) return rc_up;
    if ((rc_up = upload(&L.d_wpack, pack))) return rc_up;
    int rc;

    // epilogue affine: y = act(acc * scale + shift) [* scale2 + shift2]; a padding channel gets zeros, so it stores exact zeros
    std::vector<float> scale(C, 1.0f), shift(C, 0.0f), scale2, shift2;
    const std::vector<float>* bias = L.bkey.empty() ? nullptr : &E->w.at(L.bkey);
    auto fold = [&](const std::string& p, std::vector<float>& sc, std::vector<float>& sh) {
        const auto& g = E->w.at(p + ".weight"); const auto& b = E->w.at(p + ".bias");
        const auto& m = E->w.at(p + ".running_mean"); const auto& v = E->w.at(p + ".running_var");
        sc.resize(C); sh.resize(C);
        for (int i = 0; i < C; ++i) {
            const double inv = 1.0 / std::sqrt(static_cast<double>(v[i]) + 1e-5);
            sc[i] = static_cast<float>(g[i] * inv);
            sh[i] = static_cast<float>(b[i] - m[i] * g[i] * inv);
        }
    };
    if (!L.bn.empty()) fold(L.bn, scale, shift);
    if (bias) for (int i = 0; i < C; ++i) shift[i] += scale[i] * (*bias)[i];
    if (!L.bn2.empty()) fold(L.bn2, scale2, shift2);
    // the piece's channels [n0, n0 + nw) of per-channel vectors with `rows` rows of `stride` channels
    auto piece = [&](const std::vector<float>& v, int rows, int stride) {
        std::vector<float> out;
        if (v.empty()) return out;
        out.assign(static_cast<size_t>(rows) * L.nw, 0.0f);
        for (int r = 0; r < rows; ++r)
            for (int o = 0; o < L.live(); ++o) out[static_cast<size_t>(r) * L.nw + o] = v[static_cast<size_t>(r) * stride + L.n0 + o];
        return out;
    };
    if ((rc = upload(&L.d_scale, piece(scale, 1, C)))) return rc;
    if ((rc = upload(&L.d_shift, piece(shift, 1, C)))) return rc;
    if ((rc = upload(&L.d_scale2, piece(scale2, 1, C)))) return rc;
    if ((rc = upload(&L.d_shift2, piece(shift2, 1, C)))) return rc;
    if (L.final && (rc = upload(&L.d_w12, piece(E->w.at(conv12_prefix(E->cfg) + ".weight"), 3, C)))) return rc;
    return DSU_OK;
}

// ------------------------------------------------------------------ RIC stencil tables
// generate_coordinates (models.py:551-604) restated in float; used when the host binding did not
// supply torch's own offsets through dsu_set_ric_offsets.
std::vector<float> default_offsets(int h, int w) {
    std::vector<float> off(static_cast<size_t>(18) * h * w, 0.0f);
    const float ch = static_cast<float>(h) / 2.0f - 0.5f, cw = static_cast<float>(w) / 2.0f - 0.5f;
    const float two_pi = static_cast<float>(M_PI) * 2.0f, step = two_pi / 8.0f;
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            float th = std::fmod(std::atan2(static_cast<float>(x) - cw, static_cast<float>(y) - ch), two_pi);
            if (th < 0) th += two_pi;
            th = std::nearbyint(10000.0f * th) / 10000.0f;
            for (int rot = 0; rot < 8; ++rot) {
                const int tap = rot < 4 ? rot : rot + 1;
                const float ang = th + step * static_cast<float>(rot);
                off[(static_cast<size_t>(2 * tap) * h + y) * w + x] = std::cos(ang) + static_cast<float>(1 - tap / 3);
                off[(static_cast<size_t>(2 * tap + 1) * h + y) * w + x] = std::sin(ang) + static_cast<float>(1 - tap % 3);
            }
        }
    return off;
}

// torchvision deform_conv2d bilinear rule (SURVEY.md 8a row T) for the RIC field.  Every non-centre
// tap k (rotation index 0..7) samples at pixel + (cos, sin)(theta + k*pi/4), i.e. inside the 3x3
// neighbourhood.  With o = octant of theta, tap k falls in the 45-degree sector m = (o + k) & 7, whose
// 2x2 corner set is fixed: rows {-1,0} if m in 2..5 else {0,+1}; cols {-1,0} if m >= 4 else {0,+1}.
// The table stores o and, in m order, the fractions (ly, lx) = sample - first corner, derived from
// the reference's own fp32 arithmetic (py = float(y-1+i) + offset; floor; subtract).  Corners outside
// the image contribute 0 in the kernel, which reproduces torchvision's border rule exactly.
int build_level(dsu_engine* E, Level& lv, int h, int w) {
    if (lv.h == h && lv.w == w && lv.lyx) return DSU_OK;
    std::vector<float> off;
    auto it = E->user_offsets.find({h, w});
    off = (it != E->user_offsets.end()) ? it->second : default_offsets(h, w);
    const size_t hw = static_cast<size_t>(h) * w;
    std::vector<float2> lyx(8 * hw);
    std::vector<uint8_t> oct(hw);
    std::vector<uint2> wh(8 * hw);
    float worst = 0.0f;
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            float dyv[8], dxv[8];
            for (int kq = 0; kq < 8; ++kq) {
                const int tap = kq < 4 ? kq : kq + 1, i = tap / 3, j = tap % 3;
                const float py = static_cast<float>(y - 1 + i) + off[(static_cast<size_t>(2 * tap) * h + y) * w + x];
                const float px = static_cast<float>(x - 1 + j) + off[(static_cast<size_t>(2 * tap + 1) * h + y) * w + x];
                const float fy = std::floor(py), fx = std::floor(px);
                dyv[kq] = (fy - static_cast<float>(y)) + (py - fy);     // integer part + the reference's lh
                dxv[kq] = (fx - static_cast<float>(x)) + (px - fx);
            }
            float th = std::atan2(dxv[0], dyv[0]);
            if (th < 0) th += 2.0f * static_cast<float>(M_PI);
            const int o0 = static_cast<int>(std::floor(th / (static_cast<float>(M_PI) / 4.0f))) & 7;
            int best_o = o0;
            float best_v = 1e9f;
            for (int cand = 0; cand < 3; ++cand) {
                const int o = (o0 + (cand == 0 ? 0 : (cand == 1 ? 7 : 1))) & 7;
                float viol = 0.0f;
                for (int kq = 0; kq < 8; ++kq) {
                    const int m = (o + kq) & 7;
                    const float ly = dyv[kq] - ((m >= 2 && m <= 5) ? -1.0f : 0.0f);
                    const float lx = dxv[kq] - ((m >= 4) ? -1.0f : 0.0f);
                    viol = std::max(viol, std::max(std::max(-ly, ly - 1.0f), std::max(-lx, lx - 1.0f)));
                }
                if (viol < best_v) { best_v = viol; best_o = o; }
            }
            worst = std::max(worst, best_v);
            const size_t e = static_cast<size_t>(y) * w + x;
            oct[e] = static_cast<uint8_t>(best_o);
            for (int kq = 0; kq < 8; ++kq) {
                const int m = (best_o + kq) & 7;
                const float ly = dyv[kq] - ((m >= 2 && m <= 5) ? -1.0f : 0.0f);
                const float lx = dxv[kq] - ((m >= 4) ? -1.0f : 0.0f);
                const float cy = std::min(1.0f, std::max(0.0f, ly)), cxl = std::min(1.0f, std::max(0.0f, lx));
                lyx[e * 8 + m] = make_float2(cy, cxl);
                const float hy = 1.0f - cy, hx = 1.0f - cxl;
                const __half w4[4] = {__float2half_rn(hy * hx), __float2half_rn(hy * cxl), __float2half_rn(cy * hx), __float2half_rn(cy * cxl)};
                uint2 packed;
                std::memcpy(&packed, w4, 8);
                wh[e * 8 + m] = packed;
            }
        }
    if (worst > 1e-3f)
        return fail(DSU_E_INVALID, "RIC offsets are not unit-circle samples (generate_coordinates, models.py:551-604): a tap "
                                   "misses its 45-degree sector by " + std::to_string(worst));
    int rc;
    if ((rc = upload(&lv.lyx, lyx))) return rc;
    if ((rc = upload(&lv.oct, oct))) return rc;
    if ((rc = upload(&lv.wh, wh))) return rc;
    lv.h = h; lv.w = w; lv.max_clamp = worst;
    return DSU_OK;
}

// ------------------------------------------------------------------ workspace
// Bytes of each workspace allocation at one shape: ensure_shape allocates them, dsu_workspace_bytes reports their sum
struct Workspace {
    size_t hi[NBUF], lo[NBUF];   // activation planes; f32_acts: one fp32 plane behind buf_hi, no lo plane
    size_t resid, inorm_x, inorm_stats, inorm_acc;
    size_t tail;                 // conv_12 partials of a final layer in pieces
    size_t ric[3];               // the RIC stencil tables of each level (Level: lyx, oct, wh)
    size_t total() const {
        size_t t = resid + inorm_x + inorm_stats + inorm_acc + tail;
        for (int b = 0; b < NBUF; ++b) t += hi[b] + lo[b];
        for (int l = 0; l < 3; ++l) t += ric[l];
        return t;
    }
};

Workspace workspace(const dsu_engine* E, int B, int H, int W) {
    Workspace ws{};
    for (int b = 0; b < NBUF; ++b) {
        if (!E->buf_used[b]) continue;
        const size_t n = static_cast<size_t>(B) * (H >> E->buf_level[b]) * (W >> E->buf_level[b]) * E->buf_C[b];
        ws.hi[b] = n * (E->f32_acts ? sizeof(float) : sizeof(__half));
        ws.lo[b] = E->exact && !E->f32_acts ? n * sizeof(__half) : 0;
    }
    if (E->cfg.resnet_blocks > 0) ws.resid = static_cast<size_t>(B) * (H >> 2) * (W >> 2) * padded(E->cfg.filters[2]) * sizeof(float);
    int cmax = 0;
    for (const LayerDef& L : E->layers)
        if (L.inorm) {
            const int C = padded(L.cout);
            ws.inorm_x = std::max(ws.inorm_x, static_cast<size_t>(B) * (H >> L.level_out) * (W >> L.level_out) * C * sizeof(float));
            cmax = std::max(cmax, C);
        }
    ws.inorm_stats = static_cast<size_t>(B) * cmax * sizeof(float2);
    ws.inorm_acc = static_cast<size_t>(B) * cmax * kInormMaxSlices * 2 * sizeof(double);   // one slot per statistics slice
    if (E->tail_pieces > 1) ws.tail = static_cast<size_t>(E->tail_pieces) * 3 * B * H * W * sizeof(float);
    if (E->cfg.kind == DSU_KIND_GENERATORJ_RIC)
        for (int l = 0; l < 3; ++l)
            ws.ric[l] = static_cast<size_t>(H >> l) * (W >> l) * (8 * sizeof(float2) + sizeof(uint8_t) + 8 * sizeof(uint2));
    return ws;
}

int ensure_shape(dsu_engine* E, int B, int H, int W) {
    if (B <= 0 || H <= 0 || W <= 0 || (H % 4) || (W % 4))
        return fail(DSU_E_INVALID, "frames must be [B>0, H, W] with H and W multiples of 4 (int(H/2), int(H/4) levels, models.py:296-300)");
    const Workspace ws = workspace(E, B, H, W);
    for (int b = 0; b < NBUF; ++b) {
        if (ws.hi[b] <= E->buf_cap[b]) continue;
        cudaFree(E->buf_hi[b]);
        cudaFree(E->buf_lo[b]);
        E->buf_hi[b] = E->buf_lo[b] = nullptr;
        CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&E->buf_hi[b]), ws.hi[b]));
        CUDA_TRY(cudaMemset(E->buf_hi[b], 0, ws.hi[b]));
        if (ws.lo[b]) {
            CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&E->buf_lo[b]), ws.lo[b]));
            CUDA_TRY(cudaMemset(E->buf_lo[b], 0, ws.lo[b]));
        }
        E->buf_cap[b] = ws.hi[b];
    }
    if (ws.resid > E->resid_cap) {
        if (E->resid) cudaFree(E->resid);
        CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&E->resid), ws.resid));
        E->resid_cap = ws.resid;
    }
    if (ws.inorm_x > E->inorm_cap) {
        if (E->inorm_x) cudaFree(E->inorm_x);
        E->inorm_x = nullptr;
        CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&E->inorm_x), ws.inorm_x));
        E->inorm_cap = ws.inorm_x;
    }
    if (ws.inorm_stats > E->inorm_stats_cap) {
        if (E->inorm_stats) cudaFree(E->inorm_stats);
        if (E->inorm_acc) cudaFree(E->inorm_acc);
        E->inorm_stats = nullptr; E->inorm_acc = nullptr;
        CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&E->inorm_stats), ws.inorm_stats));
        CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&E->inorm_acc), ws.inorm_acc));
        E->inorm_stats_cap = ws.inorm_stats;
    }
    if (ws.tail > E->tail_cap) {
        if (E->tail_part) cudaFree(E->tail_part);
        E->tail_part = nullptr;
        CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&E->tail_part), ws.tail));
        E->tail_cap = ws.tail;
    }
    if (E->cfg.kind == DSU_KIND_GENERATORJ_RIC)
        for (int l = 0; l < 3; ++l) {
            int rc = build_level(E, E->lv[l], H >> l, W >> l);
            if (rc) return rc;
        }
    E->B = B; E->H = H; E->W = W;
    return DSU_OK;
}

// The view of activation buffer `buf` from channel `choff` on, in the handle's storage form (act.cuh): where a kernel stores
// (or max-pool reads).  buf < 0: no store.
ActOut act_out(const dsu_engine* E, int buf, int choff) {
    if (buf < 0) return ActOut{};
    if (E->f32_acts) return ActOut{nullptr, nullptr, reinterpret_cast<float*>(E->buf_hi[buf]), E->buf_C[buf], choff};
    return ActOut{E->buf_hi[buf], E->buf_lo[buf], nullptr, E->buf_C[buf], choff, E->bf16 ? 1 : 0};
}

// The mode a layer runs under the run-time knobs `first` and `ric_halo` (the rule: conv.cuh ConvMode)
ConvMode conv_mode(const dsu_engine* E, const LayerDef& L) {
    if (L.mode == ConvMode::Halo && L.first && !E->knobs.first) return ConvMode::Tap;
    if (L.mode == ConvMode::Ric && E->knobs.ric_halo) return ConvMode::RicHalo;
    return L.mode;
}

int run_network(dsu_engine* E, int B, int H, int W, float* y_dev, uint8_t* y_rgba, const uint8_t* alpha_src,
                int alpha_stride, cudaStream_t st, std::vector<cudaEvent_t>* evs = nullptr) {
    size_t step_idx = 0;
    for (const Step& sp : E->steps) {
        if (evs) CUDA_TRY(cudaEventRecord((*evs)[step_idx], st));
        ++step_idx;
        if (sp.type == 1) {
            const int l = E->buf_level[sp.src];
            CUDA_TRY(maxpool2(act_out(E, sp.src, sp.src_choff), act_out(E, sp.dst, 0), B, H >> l, W >> l, sp.C, st));
            continue;
        }
        const LayerDef& L = E->layers[sp.layer];
        if (sp.type == 3) {
            CUDA_TRY(conv12_tail(E->tail_part, E->tail_pieces, E->d_b12, E->cfg.tanh, B, H, W, y_dev, y_rgba, alpha_src,
                                 alpha_stride, st));
            continue;
        }
        if (sp.type == 2) {
            // nn.InstanceNorm2d + activation + the stores of layer L's epilogue, from the raw output its launch(es) left in inorm_x
            InstNormApply a{};
            a.x = E->inorm_x; a.stats = E->inorm_stats;
            a.B = B; a.HW = (H >> L.level_out) * (W >> L.level_out); a.C = padded(L.cout); a.act = L.act;
            a.resid = L.resid_out ? E->resid : nullptr;
            a.out = act_out(E, L.out_buf, L.out_choff); a.out2 = act_out(E, L.out2_buf, 0); a.out_relu = L.out_relu;
            CUDA_TRY(instance_norm(a, E->inorm_acc, st));
            continue;
        }
        ConvParams p{};
        // a sub-pixel class iterates over the low-resolution grid (one level below its output buffer)
        const int grid_level = L.level_out + (L.sub >= 0 ? 1 : 0);
        p.B = B; p.Hout = H >> grid_level; p.Wout = W >> grid_level;
        const int src_level = E->buf_level[L.segs[0].buf];
        p.Hin = H >> src_level; p.Win = W >> src_level;
        p.up = L.up; p.Hv = p.Hin << L.up; p.Wv = p.Win << L.up;
        p.mode = conv_mode(E, L); p.stride = L.stride; p.exact = E->exact ? 1 : 0; p.bf16 = E->bf16 ? 1 : 0;
        p.nchunks = L.nchunks; p.nblocks = L.nblocks; p.Cout = L.nw;
        p.b_bytes = L.nw * 128;
        p.kmask_full = L.kmask_full; p.kmask_last = L.kmask_last; p.kmask2_full = L.kmask2_full; p.kmask2_last = L.kmask2_last;
        if (L.sub >= 0) { p.sub = 1; p.sub_py = L.sub >> 1; p.sub_px = L.sub & 1; }
        p.ksize = L.k; p.pad_y = L.pad_y; p.pad_x = L.pad_x;
        p.n128 = E->knobs.n128 != 0;
        p.hslots = L.d_hslots;
        p.slots = L.d_slots; p.wpack = L.d_wpack;
        for (size_t i = 0; i < L.segs.size(); ++i) {     // the producers read fp32 through the half-typed pointer (kEsz)
            const ActOut a = act_out(E, L.segs[i].buf, 0);
            p.seg[i].ptr = a.f32 ? reinterpret_cast<const __half*>(a.f32) : a.hi;
            p.seg[i + kMaxSeg / 2].ptr = a.lo;
            p.seg[i].pitch = p.seg[i + kMaxSeg / 2].pitch = a.pitch;
        }
        if (L.ric) { p.ric_lyx = E->lv[L.level_out].lyx; p.ric_oct = E->lv[L.level_out].oct; p.ric_wh = E->lv[L.level_out].wh; }
        EpiParams& e = p.epi;
        e.scale = L.d_scale; e.shift = L.d_shift; e.scale2 = L.d_scale2; e.shift2 = L.d_shift2;
        // a piece stores from its first channel n0; the residual stream and the instance-norm scratch keep the full pitch
        e.act = L.act; e.resid_in = L.resid_in; e.resid_out = L.resid_out; e.resid = E->resid ? E->resid + L.n0 : nullptr;
        e.resid_pitch = padded(L.cout);
        e.out = act_out(E, L.out_buf, L.out_choff + L.n0); e.out2 = act_out(E, L.out2_buf, L.n0); e.out_relu = L.out_relu;
        if (L.inorm) {
            // raw convolution output (+ bias) -> fp32 scratch through the residual-stream store; everything else happens in the type-2 step
            e.act = 0; e.resid_in = 0; e.resid_out = 1; e.resid = E->inorm_x + L.n0; e.out_relu = 0;
            e.out = e.out2 = ActOut{};
        }
        if (L.final) {
            e.w12 = L.d_w12; e.b12 = E->d_b12; e.tanh_flag = E->cfg.tanh;
            if (E->tail_pieces > 1) {       // conv_12 partials of this piece; the type-3 step finishes them
                e.y_part = E->tail_part + static_cast<size_t>(L.n0 / kMaxPiece(E->exact)) * 3 * B * H * W;
            } else {
                e.y_nchw = y_dev; e.y_rgba = y_rgba; e.alpha_src = alpha_src; e.alpha_stride = alpha_stride;
            }
        }
        CUDA_TRY(launch_conv(p, st));
    }
    if (evs) CUDA_TRY(cudaEventRecord((*evs)[step_idx], st));
    return DSU_OK;
}

int check_ready(dsu_handle h) {
    if (!h) return fail(DSU_E_INVALID, "null handle");
    if (!h->finalized) return fail(DSU_E_STATE, "dsu_finalize has not been called (weights not packed)");
    return DSU_OK;
}

// The network input of the uint8 frame path: RGB, then the mask when use_mask, then posXY when use_pos (data.py:36-40), so
// input_channels = 3 + use_mask + 2 * use_pos (test_stage1.py:33-39, test_stage2.py:37-43) and the checkpoint's input width
// alone fixes the layout.
struct FrameLayout {
    bool mask, pos;
};

// Checks the arguments of a uint8 frame forward and returns the layout: a NULL pos is allowed exactly when nothing reads it
int check_frame_args(dsu_handle h, const uint8_t* color, const uint8_t* pos, const uint8_t* out, FrameLayout* layout) {
    int rc = check_ready(h);
    if (rc) return rc;
    const int cin = h->cfg.input_channels;
    if (cin < 3 || cin > 6)
        return fail(DSU_E_INVALID, "the uint8 frame path needs input_channels = 3 + use_mask + 2 * use_pos, one of 3, 4, 5, 6 "
                                   "(RGB | mask | posXY, test_stage1.py:33-39); this handle has " + std::to_string(cin));
    *layout = FrameLayout{cin == 4 || cin == 6, cin >= 5};
    if (!color || !out) return fail(DSU_E_INVALID, "null frame pointer");
    if (!pos && layout->pos)
        return fail(DSU_E_INVALID, "pos is NULL but input_channels " + std::to_string(cin) + " reads posXY (use_pos); pos may "
                                   "be NULL only when input_channels is 3 or 4 and derive_edge is off");
    if (!pos && h->knobs.derive_edge)
        return fail(DSU_E_INVALID, "pos is NULL but derive_edge is set: derived edges come from the pos frames (pos2edge, "
                                   "run_render.py:31-57); pos may be NULL only when input_channels is 3 or 4 and derive_edge is off");
    return DSU_OK;
}

}  // namespace

// =================================================================== C ABI
extern "C" {

const char* dsu_last_error(void) { return g_err.c_str(); }
const char* dsu_version(void) { return "dsu_b200 0.2 (sm_90a, wgmma)"; }

int dsu_create(const dsu_config* cfg, dsu_handle* out) {
    if (!cfg || !out) return fail(DSU_E_INVALID, "null argument");
    *out = nullptr;
    if (cfg->kind != DSU_KIND_GENERATORJ_RIC && cfg->kind != DSU_KIND_GENERATORJ)
        return fail(DSU_E_INVALID, "kind must be DSU_KIND_GENERATORJ_RIC or DSU_KIND_GENERATORJ");
    if (cfg->norm != DSU_NORM_BATCH && cfg->norm != DSU_NORM_NONE && cfg->norm != DSU_NORM_INSTANCE) return fail(DSU_E_INVALID, "bad norm");
    if (cfg->precision != DSU_PREC_FP16 && cfg->precision != DSU_PREC_FP16X3 && cfg->precision != DSU_PREC_BF16 &&
        cfg->precision != DSU_PREC_BF16X3)
        return fail(DSU_E_INVALID, "bad precision");
    if (cfg->input_channels < 1 || cfg->input_channels > 16) return fail(DSU_E_INVALID, "input_channels must be in [1,16]");
    if (cfg->resnet_blocks < 0 || cfg->resnet_blocks > 64) return fail(DSU_E_INVALID, "resnet_blocks out of range");
    for (int i = 0; i < 6; ++i)
        if (cfg->filters[i] < 1 || cfg->filters[i] > 512)
            return fail(DSU_E_INVALID, "filters[" + std::to_string(i) + "] = " + std::to_string(cfg->filters[i]) +
                                       ": every width must be in [1, 512]");
    if (cfg->filters[3] != cfg->filters[2])
        return fail(DSU_E_INVALID, "filters[3] must equal filters[2] (upconv2 concatenates the residual trunk, models.py:72)");
    int ndev = 0;
    CUDA_TRY(cudaGetDeviceCount(&ndev));
    if (cfg->device < 0 || cfg->device >= ndev) return fail(DSU_E_INVALID, "no such CUDA device");
    cudaDeviceProp prop{};
    CUDA_TRY(cudaGetDeviceProperties(&prop, cfg->device));
    if (prop.major != 9 || prop.minor != 0)
        return fail(DSU_E_INVALID, std::string("device '") + prop.name + "' is not sm_90 (wgmma kernels built for sm_90a only, no fallback path)");
    dsu_engine* E = new dsu_engine();
    E->cfg = *cfg;
    E->knobs = knobs_from_env();
    E->cin_pad = (cfg->input_channels + 7) / 8 * 8;
    E->exact = cfg->precision == DSU_PREC_FP16X3 || cfg->precision == DSU_PREC_BF16X3;
    E->bf16 = cfg->precision == DSU_PREC_BF16 || cfg->precision == DSU_PREC_BF16X3;
    E->f32_acts = cfg->kind == DSU_KIND_GENERATORJ_RIC && E->exact;
    int rc = build_plan(E);
    if (rc) { delete E; return rc; }
    *out = E;
    return DSU_OK;
}

void dsu_destroy(dsu_handle h) {
    if (!h) return;
    DeviceGuard guard(h->cfg.device);
    for (LayerDef& L : h->layers) {
        cudaFree(L.d_slots); cudaFree(L.d_hslots); cudaFree(L.d_wpack);
        cudaFree(L.d_scale); cudaFree(L.d_shift); cudaFree(L.d_scale2); cudaFree(L.d_shift2); cudaFree(L.d_w12);
    }
    for (int b = 0; b < NBUF; ++b) { cudaFree(h->buf_hi[b]); cudaFree(h->buf_lo[b]); }
    for (int l = 0; l < 3; ++l) { cudaFree(h->lv[l].lyx); cudaFree(h->lv[l].oct); cudaFree(h->lv[l].wh); }
    cudaFree(h->resid); cudaFree(h->d_b12); cudaFree(h->tail_part);
    cudaFree(h->inorm_x); cudaFree(h->inorm_stats); cudaFree(h->inorm_acc);
    cudaFree(h->io_color); cudaFree(h->io_pos); cudaFree(h->io_edge); cudaFree(h->io_out);
    delete h;
}

int dsu_expected_keys(dsu_handle h) { return h ? static_cast<int>(h->expected.size()) : 0; }
int dsu_loaded_keys(dsu_handle h) { return h ? static_cast<int>(h->loaded.size()) : 0; }

int dsu_load_weights(dsu_handle h, const char* key, const void* data, const int64_t* shape, int32_t ndim,
                     int32_t dtype, int32_t location) {
    if (!h || !key || !data) return fail(DSU_E_INVALID, "null argument");
    auto it = h->expected.find(key);
    if (it == h->expected.end()) return fail(DSU_E_INVALID, std::string("unexpected key in state_dict: ") + key);
    const std::vector<int64_t>& es = it->second;
    bool same = static_cast<size_t>(ndim) == es.size();
    size_t n = 1;
    for (int i = 0; same && i < ndim; ++i) { same = shape[i] == es[i]; n *= static_cast<size_t>(es[i]); }
    if (!same) return fail(DSU_E_INVALID, std::string("size mismatch for ") + key);
    h->finalized = false;
    if (dtype == 1) { h->loaded.insert(key); return DSU_OK; }   // num_batches_tracked: accepted, unused in eval
    if (dtype != 0) return fail(DSU_E_INVALID, "dtype must be 0 (float32) or 1 (int64)");
    std::vector<float>& dst = h->w[key];
    dst.resize(n);
    if (location == 1) {
        DEVICE_GUARD(h);
        CUDA_TRY(cudaMemcpy(dst.data(), data, n * sizeof(float), cudaMemcpyDeviceToHost));
    } else {
        std::memcpy(dst.data(), data, n * sizeof(float));
    }
    h->loaded.insert(key);
    return DSU_OK;
}

int dsu_finalize(dsu_handle h, void* stream) {
    (void)stream;
    if (!h) return fail(DSU_E_INVALID, "null handle");
    for (const std::string& k : h->expected_order)
        if (!h->loaded.count(k)) return fail(DSU_E_STATE, "missing key in state_dict: " + k);
    DEVICE_GUARD(h);
    for (LayerDef& L : h->layers) {
        int rc = compile_layer(h, L);
        if (rc) return rc;
    }
    const std::string p12 = conv12_prefix(h->cfg);
    int rc;
    if ((rc = upload(&h->d_b12, h->w.at(p12 + ".bias")))) return rc;
    h->finalized = true;
    return DSU_OK;
}

int dsu_set_knob(dsu_handle h, const char* name, int32_t value) {
    if (!h || !name) return fail(DSU_E_INVALID, "null argument");
    for (const KnobName& kn : kKnobNames)
        if (std::strcmp(kn.name, name) == 0) {
            if (kn.field == &Knobs::subpixel && h->knobs.subpixel != value)
                return fail(DSU_E_STATE, "'subpixel' shapes the launch plan: set DSU_SUBPIXEL in the environment before dsu_create");
            if (kn.field == &Knobs::halo && h->knobs.halo != value)
                return fail(DSU_E_STATE, "'halo' shapes the weight packing: set DSU_HALO in the environment before dsu_create");
            h->knobs.*(kn.field) = value;
            return DSU_OK;
        }
    return fail(DSU_E_INVALID, std::string("unknown knob: ") + name);
}

int dsu_set_ric_offsets(dsu_handle h, int32_t height, int32_t width, const float* offsets_host) {
    if (!h || !offsets_host || height <= 0 || width <= 0) return fail(DSU_E_INVALID, "bad argument");
    h->user_offsets[{height, width}] = std::vector<float>(offsets_host, offsets_host + static_cast<size_t>(18) * height * width);
    for (int l = 0; l < 3; ++l)
        if (h->lv[l].h == height && h->lv[l].w == width) h->lv[l].h = h->lv[l].w = 0;   // rebuild on next forward
    return DSU_OK;
}

int dsu_forward(dsu_handle h, const float* x_dev, int32_t B, int32_t H, int32_t W, float* y_dev, void* stream) {
    int rc = check_ready(h);
    if (rc) return rc;
    if (!x_dev || !y_dev) return fail(DSU_E_INVALID, "null tensor pointer");
    DEVICE_GUARD(h);
    if ((rc = ensure_shape(h, B, H, W))) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CUDA_TRY(ingest_f32(x_dev, B, h->cfg.input_channels, h->cin_pad, H, W, act_out(h, SK0, padded(h->cfg.filters[0])), st));
    return run_network(h, B, H, W, y_dev, nullptr, nullptr, 0, st);
}

int dsu_forward_u8(dsu_handle h, const uint8_t* color_dev, const uint8_t* pos_dev, const uint8_t* edge_dev,
                   int32_t B, int32_t H, int32_t W, uint8_t* out_rgba_dev, float* y_dev, void* stream) {
    FrameLayout lay;
    int rc = check_frame_args(h, color_dev, pos_dev, out_rgba_dev, &lay);
    if (rc) return rc;
    DEVICE_GUARD(h);
    if ((rc = ensure_shape(h, B, H, W))) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CUDA_TRY(ingest_u8(color_dev, pos_dev, edge_dev, h->knobs.derive_edge, lay.mask, lay.pos, B, H, W,
                       act_out(h, SK0, padded(h->cfg.filters[0])), st));
    return run_network(h, B, H, W, y_dev, out_rgba_dev, color_dev + 3, 4, st);
}

int dsu_forward_u8_host(dsu_handle h, const uint8_t* color_host, const uint8_t* pos_host, const uint8_t* edge_host,
                        int32_t B, int32_t H, int32_t W, uint8_t* out_rgba_host, void* stream) {
    FrameLayout lay;
    int rc = check_frame_args(h, color_host, pos_host, out_rgba_host, &lay);
    if (rc) return rc;
    DEVICE_GUARD(h);
    const size_t np = static_cast<size_t>(B) * H * W;
    if (np * 4 > h->io_cap) {
        cudaFree(h->io_color); cudaFree(h->io_pos); cudaFree(h->io_edge); cudaFree(h->io_out);
        h->io_color = h->io_pos = h->io_edge = h->io_out = nullptr; h->io_cap = 0;
        CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&h->io_color), np * 4));
        CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&h->io_pos), np * 4));
        CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&h->io_edge), np));
        CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&h->io_out), np * 4));
        h->io_cap = np * 4;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CUDA_TRY(cudaMemcpyAsync(h->io_color, color_host, np * 4, cudaMemcpyHostToDevice, st));
    if (pos_host) CUDA_TRY(cudaMemcpyAsync(h->io_pos, pos_host, np * 4, cudaMemcpyHostToDevice, st));
    if (edge_host) CUDA_TRY(cudaMemcpyAsync(h->io_edge, edge_host, np, cudaMemcpyHostToDevice, st));
    rc = dsu_forward_u8(h, h->io_color, pos_host ? h->io_pos : nullptr, edge_host ? h->io_edge : nullptr, B, H, W, h->io_out,
                        nullptr, stream);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(out_rgba_host, h->io_out, np * 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return DSU_OK;
}

size_t dsu_workspace_bytes(dsu_handle h, int32_t B, int32_t H, int32_t W) {
    return h ? workspace(h, B, H, W).total() : 0;
}

int dsu_forward_launches(dsu_handle h, int32_t B, int32_t H, int32_t W) {
    (void)B; (void)H; (void)W;
    if (!h) return 0;
    int n = 1;                                      // ingest
    for (const Step& sp : h->steps) n += sp.type == 2 ? 3 : 1;     // instance norm = statistics + finish + apply
    return n;
}

double dsu_forward_flops(dsu_handle h, int32_t B, int32_t H, int32_t W) {
    if (!h) return 0;
    double macs = 0;
    for (const LayerDef& L : h->layers) {
        double mp = L.macs_per_px;
        if (mp == 0) {   // before finalize: derive from the plan
            double kk = 0;
            for (const SegDef& s : L.segs) kk += s.wn;
            mp = L.sub >= 0 ? kk * 9.0 / 4.0 * L.live() : kk * L.k * L.k * L.live();
        }
        macs += mp * static_cast<double>(H >> L.level_out) * (W >> L.level_out);
    }
    macs += 3.0 * h->cfg.filters[5] * static_cast<double>(H) * W;   // conv_12
    return 2.0 * macs * B;
}

int dsu_profile_forward(dsu_handle h, int32_t B, int32_t H, int32_t W, int32_t reps, void* stream,
                        double* ms_out, double* flops_out, int32_t capacity) {
    int rc = check_ready(h);
    if (rc) return rc;
    if (!ms_out || !flops_out || reps <= 0) return fail(DSU_E_INVALID, "bad argument");
    DEVICE_GUARD(h);
    if ((rc = ensure_shape(h, B, H, W))) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t n = h->steps.size();
    struct Events {                                   // destroyed on every exit path
        std::vector<cudaEvent_t> v;
        ~Events() { for (cudaEvent_t e : v) if (e) cudaEventDestroy(e); }
    } events;
    events.v.assign(n + 1, nullptr);
    std::vector<cudaEvent_t>& evs = events.v;
    for (auto& e : evs) CUDA_TRY(cudaEventCreate(&e));
    std::vector<double> acc(n, 0.0);
    for (int r = 0; r < reps; ++r) {
        if ((rc = run_network(h, B, H, W, nullptr, nullptr, nullptr, 0, st, &evs))) return rc;
        CUDA_TRY(cudaStreamSynchronize(st));
        for (size_t i = 0; i < n; ++i) {
            float ms = 0;
            CUDA_TRY(cudaEventElapsedTime(&ms, evs[i], evs[i + 1]));
            acc[i] += ms;
        }
    }
    for (size_t i = 0; i < n && i < static_cast<size_t>(capacity); ++i) {
        ms_out[i] = acc[i] / reps;
        const Step& sp = h->steps[i];
        if (sp.type == 0) {
            const LayerDef& L = h->layers[sp.layer];
            double f = 2.0 * L.macs_per_px * (H >> L.level_out) * (W >> L.level_out) * B;
            if (L.final) f += 2.0 * 3.0 * L.live() * static_cast<double>(H) * W * B;
            flops_out[i] = f;
        } else {
            flops_out[i] = 0;
        }
    }
    return static_cast<int>(n);
}

const char* dsu_step_name(dsu_handle h, int32_t index) {
    if (!h || index < 0 || index >= static_cast<int>(h->steps.size())) return "";
    const Step& sp = h->steps[index];
    static const char* const kStepNames[] = {"", "maxpool", "instance_norm", "conv_12"};    // Step::type order
    return sp.type == 0 ? h->layers[sp.layer].name.c_str() : kStepNames[sp.type];
}

const char* dsu_step_kernel(dsu_handle h, int32_t index) {
    if (!h || index < 0 || index >= static_cast<int>(h->steps.size())) return "";
    const Step& sp = h->steps[index];
    if (sp.type != 0) return dsu_step_name(h, index);
    static const char* const kModeNames[] = {"tap", "ric", "ric_halo", "halo"};    // ConvMode order
    return kModeNames[static_cast<int>(conv_mode(h, h->layers[sp.layer]))];
}

int dsu_frames_to_tensor(const uint8_t* color_dev, const uint8_t* pos_dev, const uint8_t* edge_dev,
                         int32_t B, int32_t H, int32_t W, float* pre_dev, float* mask_dev, void* stream) {
    if (!color_dev || !pos_dev || !pre_dev || B <= 0 || H <= 0 || W <= 0) return fail(DSU_E_INVALID, "bad argument");
    CUDA_TRY(frames_to_tensor(color_dev, pos_dev, edge_dev, B, H, W, pre_dev, mask_dev, static_cast<cudaStream_t>(stream)));
    return DSU_OK;
}
int dsu_to_image_space(const float* x_dev, uint8_t* out_dev, size_t n, void* stream) {
    if (!x_dev || !out_dev) return fail(DSU_E_INVALID, "null pointer");
    if (n) CUDA_TRY(to_image_space(x_dev, out_dev, n, static_cast<cudaStream_t>(stream)));
    return DSU_OK;
}
int dsu_overlap_edge(const uint8_t* edge_dev, uint8_t* rgba_dev, size_t npixels, void* stream) {
    if (!edge_dev || !rgba_dev) return fail(DSU_E_INVALID, "null pointer");
    if (npixels) CUDA_TRY(overlap_edge(edge_dev, rgba_dev, npixels, static_cast<cudaStream_t>(stream)));
    return DSU_OK;
}
int dsu_compose_rgba(const float* y_dev, const float* mask_dev, int32_t B, int32_t H, int32_t W,
                     uint8_t* out_rgba_dev, void* stream) {
    if (!y_dev || !mask_dev || !out_rgba_dev || B <= 0 || H <= 0 || W <= 0) return fail(DSU_E_INVALID, "bad argument");
    CUDA_TRY(compose_rgba(y_dev, mask_dev, B, H, W, out_rgba_dev, static_cast<cudaStream_t>(stream)));
    return DSU_OK;
}
int dsu_pos2edge(const uint8_t* pos_dev, int32_t B, int32_t H, int32_t W, uint8_t* edge_dev, void* stream) {
    if (!pos_dev || !edge_dev || B <= 0 || H <= 0 || W <= 0) return fail(DSU_E_INVALID, "bad argument");
    CUDA_TRY(pos2edge(pos_dev, B, H, W, edge_dev, static_cast<cudaStream_t>(stream)));
    return DSU_OK;
}

int dsu_debug_read(dsu_handle h, int32_t buffer, int32_t plane, void* dst_host, size_t bytes) {
    if (!h || !dst_host) return fail(DSU_E_INVALID, "null argument");
    DEVICE_GUARD(h);
    CUDA_TRY(cudaDeviceSynchronize());
    const void* src = nullptr;
    size_t have = 0;
    if (buffer == 100) { src = h->resid; have = h->resid_cap; }
    else if (buffer >= 0 && buffer < NBUF) { src = plane ? h->buf_lo[buffer] : h->buf_hi[buffer]; have = h->buf_cap[buffer]; }
    if (!src) return fail(DSU_E_INVALID, "no such buffer in this configuration");
    CUDA_TRY(cudaMemcpy(dst_host, src, std::min(bytes, have), cudaMemcpyDeviceToHost));
    return DSU_OK;
}

}  // extern "C"
