/* dsu_b200 - C ABI of the DrawingSpinUp stylization engine (CUDA, sm_90a).
 *
 * The reference (LordLiang/DrawingSpinUp, 100 % Python) has no FFI: its seam for this path is
 * `training.trainers.build_model` -> `getattr(training.models, type)(**args)`
 * (3_style_translator/training/trainers.py:33-35) followed by `load_state_dict`, `.eval()` and
 * `generator(x)` (test_stage1.py:43-63, test_stage2.py:50-70).  This header is the C boundary a
 * binding for that seam uses; each entry point cites the reference code it replaces.
 * `drawingspinup_b200/models.py` is the ctypes host side that mirrors the reference classes.
 *
 * Conventions: every function returns 0 on success or a negative DSU_E_* code; the message is
 * available from dsu_last_error() (thread-local).  Nothing aborts or throws across the boundary.
 * Pointers named *_dev are CUDA device pointers on the handle's device; *_host are host pointers.
 * All work is enqueued on the given stream (a cudaStream_t passed as void*); no hidden host syncs
 * except where stated.  A handle is single-stream and not thread-safe; distinct handles are
 * independent (one per GPU).  The caller owns inputs / outputs; the library owns packed weights,
 * stencil tables and workspace (grown on demand, released by dsu_destroy).
 */
#ifndef DSU_B200_H
#define DSU_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DSU_OK 0
#define DSU_E_INVALID (-1)     /* bad argument / unsupported configuration */
#define DSU_E_CUDA (-2)        /* CUDA runtime error, see dsu_last_error() */
#define DSU_E_STATE (-3)       /* call order violated (e.g. forward before finalize) */
#define DSU_E_NOTIMPL (-4)     /* legal reference option this engine does not implement */

/* generator kinds = class names resolved by build_model (trainers.py:33-35) */
#define DSU_KIND_GENERATORJ_RIC 1   /* stage 1, training/models.py:200-356 */
#define DSU_KIND_GENERATORJ 2       /* stage 2, training/models.py:24-129  */

/* operand precision of the tensor-core contractions */
#define DSU_PREC_FP16 0     /* fp16 operands, fp32 accumulate (1 MMA pass) */
#define DSU_PREC_FP16X3 1   /* split fp16 hi+lo operands, 3 MMA passes: fp32-grade, meets 1e-3 parity */
#define DSU_PREC_BF16 2     /* bf16 operands, fp32 accumulate (1 MMA pass): fp32's exponent range at fp16's width and rate */
/* split bf16 hi+lo operands, 3 MMA passes: a 16-bit significand with fp32's exponent range (value 3: the split of
 * DSU_PREC_FP16X3 combined with the element type of DSU_PREC_BF16) */
#define DSU_PREC_BF16X3 (DSU_PREC_BF16 | DSU_PREC_FP16X3)

#define DSU_NORM_NONE 0
#define DSU_NORM_BATCH 1
#define DSU_NORM_INSTANCE 2   /* nn.InstanceNorm2d defaults (models.py:34-35): statistics per (frame, channel), no state-dict keys */

typedef struct dsu_engine* dsu_handle;

/* Constructor arguments of GeneratorJ / GeneratorJ_RIC (models.py:25-27, 201-203). */
typedef struct dsu_config {
    int32_t kind;              /* DSU_KIND_* */
    int32_t input_channels;    /* after the +1 mask +2 pos of test_stage1.py:33-39 (6 in shipped configs) */
    int32_t filters[6];        /* each in [1, 512]; filters[3] == filters[2] (upconv2 concatenates the trunk) */
    int32_t resnet_blocks;
    int32_t use_bias;
    int32_t tanh;
    int32_t append_smoothers;
    int32_t norm;              /* DSU_NORM_* */
    int32_t precision;         /* DSU_PREC_* */
    int32_t device;            /* CUDA device ordinal */
} dsu_config;

const char* dsu_last_error(void);
const char* dsu_version(void);

/* models.py:24-111 / 200-291 (module construction) */
int dsu_create(const dsu_config* cfg, dsu_handle* out);
void dsu_destroy(dsu_handle h);

/* generator.load_state_dict(sd) (test_stage1.py:44-47): one call per state-dict entry.
 * dtype: 0 = float32, 1 = int64 (num_batches_tracked, accepted and ignored).
 * location: 0 = host pointer, 1 = device pointer.  Shapes are checked against the layout of
 * SURVEY.md section 8a row a8; unknown keys are DSU_E_INVALID. */
int dsu_load_weights(dsu_handle h, const char* key, const void* data, const int64_t* shape, int32_t ndim,
                     int32_t dtype, int32_t location);
/* Number of state-dict keys the configuration expects / has received so far. */
int dsu_expected_keys(dsu_handle h);
int dsu_loaded_keys(dsu_handle h);
/* Fold BatchNorm running stats into per-channel scale/shift, round + swizzle the conv weights into
 * tensor-core tiles, upload.  Requires every expected key (strict=True semantics). */
int dsu_finalize(dsu_handle h, void* stream);

/* Development / test hook, no counterpart in the reference: knobs of this handle ("first", "n128", "subpixel", "derive_edge",
 * "halo", "ric_halo" - engine.cu Knobs).  Their defaults are read once from the environment (DSU_<NAME>) by dsu_create; "subpixel" shapes the
 * launch plan and "halo" the weight packing, so those two can only be set through the environment (DSU_E_STATE otherwise). */
int dsu_set_knob(dsu_handle h, const char* name, int32_t value);

/* generate_coordinates (models.py:551-604) is data independent; by default the engine derives the
 * per-level bilinear stencil from its own float math.  A host binding that wants the offsets
 * bit-identical to torch's (the Python mirror does) supplies them: offsets_host = fp32 [18, h, w]. */
int dsu_set_ric_offsets(dsu_handle h, int32_t height, int32_t width, const float* offsets_host);

/* generator(x) under torch.no_grad() in eval mode (test_stage1.py:63, test_stage2.py:70,
 * trainers.py:223).  x_dev: fp32 NCHW [B, input_channels, H, W]; y_dev: fp32 NCHW [B, 3, H, W].
 * H and W must be multiples of 4. */
int dsu_forward(dsu_handle h, const float* x_dev, int32_t B, int32_t H, int32_t W, float* y_dev, void* stream);

/* Fused frame path: DatasetFullImages.__getitem__ (data.py:23-47) + forward + to_image_space +
 * alpha composite (test_stage1.py:68-70), all on device.
 * color_dev / pos_dev: uint8 RGBA [B,H,W,4]; edge_dev: uint8 [B,H,W] or NULL (stage 2 passes it:
 * overlap_edge_on_img, custom_transforms.py:30-35); out_rgba_dev: uint8 [B,H,W,4];
 * y_dev: optional fp32 NCHW network output (may be NULL).
 * The network input is RGB, then the mask when use_mask, then posXY when use_pos (data.py:36-40), so the handle's
 * input_channels = 3 + use_mask + 2*use_pos selects it: 3 RGB, 4 RGB|mask, 5 RGB|posXY, 6 RGB|mask|posXY (the
 * reference's --no_mask / --no_pos ablations).  The output alpha is always the colour alpha.  pos_dev may be NULL exactly
 * when the layout has no pos (3 or 4) and the derive_edge knob is off.  Any other input_channels, or a NULL pos_dev that
 * would be read, returns DSU_E_INVALID before any launch. */
int dsu_forward_u8(dsu_handle h, const uint8_t* color_dev, const uint8_t* pos_dev, const uint8_t* edge_dev,
                   int32_t B, int32_t H, int32_t W, uint8_t* out_rgba_dev, float* y_dev, void* stream);

/* Same as dsu_forward_u8 with HOST buffers (pinned memory recommended): copies the inputs to the
 * device, runs, copies the RGBA result back, and synchronizes the stream before returning.  The same
 * layouts and rules: pos_host may be NULL exactly when dsu_forward_u8 allows a NULL pos_dev, and is then
 * not uploaded. */
int dsu_forward_u8_host(dsu_handle h, const uint8_t* color_host, const uint8_t* pos_host, const uint8_t* edge_host,
                        int32_t B, int32_t H, int32_t W, uint8_t* out_rgba_host, void* stream);

/* Bytes of device workspace the engine holds / would need for a [B,*,H,W] forward. */
size_t dsu_workspace_bytes(dsu_handle h, int32_t B, int32_t H, int32_t W);
/* Convolution kernel launches and algorithmic FLOPs (2 x live MACs) of one forward of this shape. */
int dsu_forward_launches(dsu_handle h, int32_t B, int32_t H, int32_t W);
double dsu_forward_flops(dsu_handle h, int32_t B, int32_t H, int32_t W);

/* Measurement hook: re-run the launches of one forward of this shape `reps` times on the current
 * workspace contents with a CUDA event pair around every launch; ms_out[i] = mean milliseconds of
 * launch i, flops_out[i] = its algorithmic FLOPs (0 for non-convolution launches).  Returns the
 * number of launches (<= capacity are written) or a negative error.  Synchronizes the stream. */
int dsu_profile_forward(dsu_handle h, int32_t B, int32_t H, int32_t W, int32_t reps, void* stream,
                        double* ms_out, double* flops_out, int32_t capacity);
/* Name of launch i of a forward ("ingest", "conv0", "maxpool", "resnets.3.conv_1", ...).  A layer wider than one launch
 * computes (128 channels in DSU_PREC_FP16X3 and DSU_PREC_BF16X3, 256 in DSU_PREC_FP16 and DSU_PREC_BF16) runs as
 * output-channel pieces "<layer>.n0", "<layer>.n1", ...; a final layer in pieces is followed by "conv_12", which sums their conv_12 partial dot products. */
const char* dsu_step_name(dsu_handle h, int32_t index);
/* Mainloop launch i runs with the handle's current plan and knobs: "halo" (A fragments from a shared-memory input halo),
 * "tap" (A tiles gathered per tap), "ric_halo" (stage-1 deformable, stencil and corners from shared memory), "ric" (stage-1
 * deformable, gathered from global memory: knob "ric_halo" = 0), or "maxpool" / "instance_norm" / "conv_12" for the other steps.  Valid after dsu_finalize. */
const char* dsu_step_kernel(dsu_handle h, int32_t index);

/* ---- stand-alone uint8 / fp32 frame steps (device pointers) -------------------------------- */
/* DatasetFullImages.__getitem__ (data.py:23-47) in the default layout (use_mask and use_pos):
 * pre_dev fp32 [B,6,H,W] = RGB(3) | mask | posXY(2), mask_dev fp32 [B,1,H,W] (may be NULL).
 * edge_dev NULL = stage 1.  The ablation layouts run only inside dsu_forward_u8. */
int dsu_frames_to_tensor(const uint8_t* color_dev, const uint8_t* pos_dev, const uint8_t* edge_dev,
                         int32_t B, int32_t H, int32_t W, float* pre_dev, float* mask_dev, void* stream);
/* to_image_space (custom_transforms.py:7-8), n elements. */
int dsu_to_image_space(const float* x_dev, uint8_t* out_dev, size_t n, void* stream);
/* overlap_edge_on_img (custom_transforms.py:30-35) in place on rgba_dev [B,H,W,4]. */
int dsu_overlap_edge(const uint8_t* edge_dev, uint8_t* rgba_dev, size_t npixels, void* stream);
/* Result image of test_stage1.py:68-70: y fp32 NCHW [B,3,H,W] + mask fp32 [B,1,H,W] -> RGBA. */
int dsu_compose_rgba(const float* y_dev, const float* mask_dev, int32_t B, int32_t H, int32_t W,
                     uint8_t* out_rgba_dev, void* stream);
/* pos2edge (run_render.py:31-57): pos RGBA [B,H,W,4] -> edge [B,H,W] (255 on edges). */
int dsu_pos2edge(const uint8_t* pos_dev, int32_t B, int32_t H, int32_t W, uint8_t* edge_dev, void* stream);

/* Test hook: copy an internal activation buffer of the last forward to the host (synchronous).
 * buffer: 0 SK0(o0|x) 1 P0 2 O1 3 P1 4 O2 5 T 6 U 7 V2 8 V1 9 C11 10 S0 (fp16 NHWC; bf16 bits for a DSU_PREC_BF16 or
 * DSU_PREC_BF16X3 handle; fp32 in stage 1 of DSU_PREC_FP16X3 and DSU_PREC_BF16X3), 100 = fp32 residual stream;
 * plane 0 = hi, 1 = lo (stage 2 of DSU_PREC_FP16X3 and DSU_PREC_BF16X3 only).  Copies min(bytes, buffer size). */
int dsu_debug_read(dsu_handle h, int32_t buffer, int32_t plane, void* dst_host, size_t bytes);

#ifdef __cplusplus
}
#endif
#endif /* DSU_B200_H */
