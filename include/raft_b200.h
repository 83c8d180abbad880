/* raft_b200.h -- C ABI of the H100-native (sm_90a) RAFT forward/update hot path.
 *
 * Drop-in boundary for daigo0927/tf-raft (reference @ 3c85f54).  The reference has no FFI of
 * its own: its boundary is the Python object API of tf_raft/layers/corr.py, tf_raft/layers/update.py
 * and tf_raft/model.py.  Each entry point below replaces the TensorFlow op sequence behind one of
 * those Python calls (cited as file:line); the host-side mirror (tf_raft_b200/) keeps the reference's
 * class / method names and binds these symbols with ctypes (INTEGRATION.md shows the stub).
 *
 * Conventions
 *   - every pointer is DEVICE memory, dense row-major, NHWC, float32 unless stated;
 *     coordinates are (x, y) in the last dimension, exactly as in the reference;
 *   - the caller owns every buffer; the library never allocates or frees device memory;
 *   - its global state is the per-thread launch counter (raft_b200_launch_count), the
 *     process-wide loop profiler (raft_b200_profile_loop, off by default) and caches filled
 *     once: kernel shared-memory attributes, SM counts and the resolved driver entry point
 *     for cuTensorMapEncodeTiled;
 *   - every call is asynchronous on `stream` (a cudaStream_t passed as void*); nothing
 *     synchronises the device, so a sequence of calls can be captured into a CUDA graph;
 *   - return value: 0 = ok, < 0 = raft_status (argument / shape / workspace error, detected on
 *     the host before anything is launched), > 0 = cudaError_t of a failed launch;
 *   - re-entrant across host threads as long as streams and buffers differ and the loop
 *     profiler is off;
 *   - there is NO CPU path: without an sm_90 device every compute entry point returns
 *     RAFT_ERR_NO_DEVICE or the CUDA error.
 */
#ifndef RAFT_B200_H_
#define RAFT_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RAFT_B200_ABI_VERSION 2
#define RAFT_MAX_LEVELS 8

typedef enum raft_status {
  RAFT_OK = 0,
  RAFT_ERR_BAD_ARG = -1,     /* null pointer, unknown enum value                          */
  RAFT_ERR_BAD_SHAPE = -2,   /* non-positive dims, C not a multiple of 8, level too small */
  RAFT_ERR_WORKSPACE = -3,   /* workspace / prepared-weights buffer too small             */
  RAFT_ERR_NO_DEVICE = -4,   /* no CUDA device of compute capability 9.0                  */
  RAFT_ERR_DRIVER = -5,      /* cuTensorMapEncodeTiled unavailable or rejected a map       */
  RAFT_ERR_UNSUPPORTED = -6  /* valid request this build does not implement               */
} raft_status;

/* Arithmetic of the contraction kernels (correlation GEMM and update-block convolutions).
 * Both are fp32-grade: the final-flow parity gate (<= 1e-3 max-abs) holds for either.
 *   FP32   CUDA-core FFMA, fp32 operands, fp32 accumulate.
 *   F16X2  wgmma tensor cores: every fp32 operand v is split into fp16 (hi, lo) with
 *          v ~= hi + lo (22-bit significand), the product is hi*hi + lo*hi + hi*lo
 *          with fp32 accumulation (DESIGN.md "Precision").                                  */
typedef enum raft_precision { RAFT_PREC_FP32 = 0, RAFT_PREC_F16X2 = 1 } raft_precision;

/* model.py:10-30 (RAFT, BasicUpdateBlock) / model.py:173-188 (SmallRAFT, SmallUpdateBlock). */
typedef enum raft_variant { RAFT_VARIANT_BASIC = 0, RAFT_VARIANT_SMALL = 1 } raft_variant;

const char* raft_b200_strerror(int status);
int raft_b200_abi_version(void);
/* 0 if device `device` can run the kernels (compute capability 9.0), else RAFT_ERR_NO_DEVICE.  */
int raft_b200_device_ok(int device);

/* ---------------------------------------------------------------------------------------------
 * CorrBlock  (tf_raft/layers/corr.py:99-162)
 * ------------------------------------------------------------------------------------------- */

/* Bytes of each pyramid level for CorrBlock(fmap1, fmap2, num_levels): level l is
 * (B*h*w, h>>l, w>>l, 1) float32 -- corr.py:108-114 (avg_pool2d 2x2 VALID floors odd dims).   */
int raft_b200_corr_pyramid_sizes(int B, int h, int w, int levels, size_t bytes_per_level[]);

/* Scratch needed by raft_b200_corr_pyramid_build.                                              */
int raft_b200_corr_workspace_bytes(int B, int h, int w, int C, int levels, int precision, size_t* bytes);

/* CorrBlock.__init__ = correlation() + pyramid: corr.py:100-114 and :154-162.
 *   fmap1, fmap2 : (B, h, w, C);  pyr[l] : (B*h*w, h>>l, w>>l, 1), l < levels.
 *   pyr[0][b*h*w + q][y2][x2] = <fmap1[b,q,:], fmap2[b,y2,x2,:]> / sqrt(C); level l is the
 *   2^l x 2^l block mean of level 0 over (y2, x2).                                              */
int raft_b200_corr_pyramid_build(const float* fmap1, const float* fmap2, int B, int h, int w, int C, int levels,
                                 float* const pyr[], void* workspace, size_t workspace_bytes, int precision,
                                 void* stream);

/* CorrBlock.retrieve: corr.py:116-152 with bilinear_sampler corr.py:28-69.
 *   coords : (B, h, w, 2) (x, y);  out : (B, h, w, out_stride) with the first
 *   levels*(2r+1)^2 channels written; channel = level*(2r+1)^2 + a*(2r+1) + b, tap (a, b) has
 *   x-offset a-r and y-offset b-r (corr.py:133-143).  A tap whose clamped x or y coordinate is
 *   an integer is exactly 0 (floor/ceil corners, corr.py:45-60) -- reproduced bit for bit.      */
int raft_b200_corr_lookup(const float* const pyr[], const float* coords, int B, int h, int w, int levels,
                          int radius, float* out, int out_stride, void* stream);

/* Backward of CorrBlock.retrieve for the training step (tf_raft/model.py:133: tape.gradient through corr.py:116-152;
 * the reference does not detach coords1, model.py:102).  grad_out (B, h, w, levels*(2r+1)^2) -> grad_coords (B, h, w, 2)
 * and grad_pyr[l] (same shapes as pyr[l]); both outputs are ACCUMULATED into (zero them first).  TensorFlow gradient
 * rules: floor / ceil / indices carry no gradient, clip_by_value passes it inside [0, dim-1].                        */
int raft_b200_corr_lookup_backward(const float* const pyr[], const float* coords, const float* grad_out, int B, int h, int w,
                                   int levels, int radius, float* grad_coords, float* const grad_pyr[], void* stream);

/* tf.linalg.global_norm over a flat gradient buffer (model.py:135): out[0] = sum g^2 (deterministic two-stage
 * reduction; `partials` holds one float per block, at most npartials blocks are used).                               */
int raft_b200_sumsq(const float* g, size_t n, float* partials, size_t npartials, float* out, void* stream);

/* tf.clip_by_global_norm (model.py:135) + tfa.optimizers.AdamW.apply_gradients (model.py:136, train_chairs.py:87-90)
 * on flat buffers: g' = g * clip / max(sqrt(*sumsq), clip) (clip_norm <= 0: no clipping); var -= wd * var;
 * m = b1 m + (1-b1) g'; v = b2 v + (1-b2) g'^2; var -= lr_t * m / (sqrt(v) + eps), lr_t already bias-corrected.        */
int raft_b200_adamw_step(float* param, const float* grad, float* m, float* v, size_t n, const float* sumsq, float clip_norm,
                         float lr_t, float beta1, float beta2, float epsilon, float weight_decay, void* stream);

/* bilinear_sampler(image, coords): corr.py:28-69.  image (M, H, W, 1), coords (M, P, 2),
 * out (M, P).  Same floor/ceil semantics as above.                                             */
int raft_b200_bilinear_sampler(const float* image, const float* coords, int M, int H, int W, int P, float* out,
                               void* stream);

/* coords_grid(B, h, w): corr.py:72-90 -> (B, h, w, 2), out[b,y,x] = (x, y).                    */
int raft_b200_coords_grid(int B, int h, int w, float* out, void* stream);

/* RAFT's warm start: forward interpolation of a (B,h,w,2) low-resolution flow (an addition beyond the reference, whose
 * loop always starts from zero flow).  Per image, source pixel (x, y) lands at (x1, y1) = (x + fx, y + fy) in fp64 and is
 * valid iff 0 < x1 < w and 0 < y1 < h (NaN / inf never are); target (X, Y) receives a copy of the flow of the valid
 * source minimising (x1 - X)^2 + (y1 - Y)^2 (fp64, each operation rounded, no FMA), ties to the lowest source index;
 * an image without a valid source gets zero flow.  out (B,h,w,2) must not alias flow.  O((h*w)^2) per image;
 * h*w must stay below 2^31 - 512 (RAFT_ERR_BAD_SHAPE otherwise).                                                    */
int raft_b200_forward_interpolate(const float* flow, int B, int h, int w, float* out, void* stream);

/* coords1 = coords_grid(B,h,w) + flow_init (fp32, one rounding per component): the loop's warm-start entry state.
 * coords1 may alias flow_init.                                                                                      */
int raft_b200_coords_init(const float* flow_init, int B, int h, int w, float* coords1, void* stream);

/* Forward-backward consistency (an addition beyond the reference).  flow_fw, flow_bw: (B, H, W, 2) float32, the flow
 * a->b and b->a of B image pairs, 8-byte aligned.  occ_fw[b,y,x] = 1 where pixel (x,y) of image a has no consistent
 * correspondence in b, occ_bw likewise for image b; else 0.  One launch covers both directions.  For direction fw,
 * with F = flow_fw[b], G = flow_bw[b] (bw swaps them), every operation a rounded fp32 one in this order, no FMA:
 *   p = (x + Fx, y + Fy); occluded unless 0 <= px <= W-1 and 0 <= py <= H-1 (NaN never is inside);
 *   g = bilinear sample of G at p (x0 = floor(px), x1 = min(x0+1, W-1), ax = px - x0, bx = 1 - ax, y likewise;
 *       g = by*(bx*G[y0,x0] + ax*G[y0,x1]) + ay*(bx*G[y1,x0] + ax*G[y1,x1]));
 *   consistent iff |F + g|^2 <= alpha1*(|F|^2 + |g|^2) + alpha2; anything else (NaN included) is occluded.
 * A non-finite texel makes g non-finite even at weight 0.  alpha1, alpha2 finite and >= 0 (RAFT_ERR_BAD_ARG otherwise);
 * Sundaram et al. use 0.01 and 0.5 (DESIGN.md section 3.5).                                                         */
int raft_b200_fb_occlusion(const float* flow_fw, const float* flow_bw, int B, int H, int W, float alpha1, float alpha2,
                           uint8_t* occ_fw, uint8_t* occ_bw, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Training augmentation  (tf_raft/datasets/augmentor.py FlowAugmentor :9-129, SparseFlowAugmentor :132-267, given
 * their random draws; dataset.py:102's dense valid)
 * ------------------------------------------------------------------------------------------- */

/* One sample.  Every pointer is device memory; sources and outputs are HWC and contiguous.  Per image k (0 = img1):
 * lut[k][0] is albumentations' brightness/contrast LUT (identity when that transform is skipped); when hsv[k] is set
 * the image then goes RGB->HSV (cv2, uint8), through lut[k][1..3] (hue, sat, val) and back (augmentor.py:42-59).
 * rect[0..n_rects) = (x0, y0, dx, dy) eraser rectangles of img2 at source resolution, filled with the truncated mean of
 * the colour-transformed img2 (:61-74).  spatial: cv2.resize by (scale_x, scale_y), INTER_LINEAR, to
 * (rint(H*scale_y), rint(W*scale_x)), the flow then scaled in fp64 (:93-98); otherwise a copy.  Then h/v flips and the
 * (crop_h, crop_w) window at (y0, x0) of the flipped image (:100-116).  ws_offset is filled by
 * raft_b200_augment_workspace_bytes.                                                                                */
typedef struct raft_augment_sample {
  const uint8_t* img1;
  const uint8_t* img2;          /* (H, W, 3)                                                                       */
  const float* flow;            /* (H, W, 2)                                                                       */
  const float* valid;           /* (H, W), sparse samples only (a source counts where valid >= 1)                 */
  uint8_t* out_img1;
  uint8_t* out_img2;            /* (crop_h, crop_w, 3)                                                             */
  float* out_flow;              /* (crop_h, crop_w, 2)                                                             */
  float* out_valid;             /* (crop_h, crop_w)                                                                */
  double scale_x, scale_y;
  size_t ws_offset;
  int H, W, crop_h, crop_w, y0, x0;
  int spatial, hflip, vflip;
  int hsv[2];
  int n_rects;
  int rect[2][4];
  uint8_t lut[2][4][256];
} raft_augment_sample;

/* Workspace of one raft_b200_augment_dense / _sparse call over samples[0..B) (host array); fills each sample's
 * ws_offset.  RAFT_ERR_BAD_SHAPE if a crop does not fit the (resized) image or a size is out of range.               */
int raft_b200_augment_workspace_bytes(raft_augment_sample* samples, int B, int sparse, size_t* bytes);

/* FlowAugmentor.__call__ + dataset.py:102 for B samples of any source sizes in one launch set (3 kernels): out_flow is
 * float32 of the fp64 flow, out_valid = |fx| < 1000 && |fy| < 1000 evaluated on the fp64 flow.  samples_host and
 * samples_dev hold the same array (host copy for checks and grid sizes, device copy read by the kernels).
 * Asynchronous on `stream`, no allocation: graph-capturable.                                                         */
int raft_b200_augment_dense(const raft_augment_sample* samples_host, const raft_augment_sample* samples_dev, int B,
                            void* workspace, size_t workspace_bytes, void* stream);

/* SparseFlowAugmentor.__call__ likewise (4 kernels).  A spatial sample's flow goes through resize_sparse_flow_map
 * (:183-215): source (x, y) with valid >= 1 lands at (rint(x*fx), rint(y*fy)) in fp64, half to even, kept iff
 * 0 < xx < rw and 0 < yy < rh; the last source in index order wins a target; flow = float32(fp64 flow * scale), valid 1.
 * A non-spatial sample copies flow and valid.                                                                        */
int raft_b200_augment_sparse(const raft_augment_sample* samples_host, const raft_augment_sample* samples_dev, int B,
                             void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Flow visualisation  (tf_raft/datasets/flow_viz.py: make_colorwheel :20-67, flow_uv_to_colors :70-106,
 * flow_to_image :109-132)
 * ------------------------------------------------------------------------------------------- */

/* Per-image status bits of raft_b200_flow_to_image.                                                                 */
enum {
  RAFT_FLOWVIZ_INF = 1,          /* a component is +-inf (after the clip)                                            */
  RAFT_FLOWVIZ_NAN = 2,          /* a component is NaN (after the clip)                                              */
  RAFT_FLOWVIZ_BAD_RAD_MAX = 4   /* the caller's rad_max of this image is negative or not finite                    */
};

/* The Middlebury colour wheel of B flow fields of H x W pixels -> image (B, H, W, 3) uint8, RGB (BGR when bgr != 0).
 * Component k of pixel p (flat over B*H*W) is u[p*stride], v[p*stride]: stride 2 with v = u + 1 reads (B, H, W, 2)
 * flows, stride 1 reads separate (B, H, W) planes.  Per pixel, NumPy 2 dtypes (NEP 50):
 *   clip != 0: u, v = np.clip(., 0, clip_flow) in float32 (NaN propagates, -0.0 stays -0.0)            (:123-124)
 *   normalize != 0: u, v /= rad_max[b] + float32(1e-5), float32; rad_max[b] is the caller's (rad_max != NULL) or
 *     max over image b of sqrt(u*u + v*v) (float32, each operation rounded, no FMA)                      (:127-131)
 *   rad = sqrt(u*u + v*v); a = float32(atan2((double)-v, (double)-u)) / float32(pi) (correctly rounded atan2);
 *   fk = (a + 1) / 2 * 54, k0 = floor(fk), k1 = k0 + 1 wrapping 55 to 0 (float32); f = fk - k0 in float64;
 *   col = (1 - f) * cw[k0] / 255 + f * cw[k1] / 255, then 1 - rad * (1 - col) if rad <= 1 else col * 0.75, and
 *   floor(255 * col), all float64                                                                          (:85-106)
 * status[b] (int) collects RAFT_FLOWVIZ_* bits of image b; the reference raises for NaN, and flow_to_image for +-inf
 * too (an infinite rad_max makes u / rad_max NaN).  A pixel whose angle is NaN is written (0, 0, 0).  work (B
 * unsigned words) holds the reduction; it is needed only when normalize != 0 and rad_max == NULL.  The call zeroes
 * work and status on `stream` first.  image must be 4-byte aligned.  RAFT_ERR_BAD_ARG for a null pointer, stride not
 * 1 or 2, or clip != 0 with a negative or non-finite clip_flow; RAFT_ERR_BAD_SHAPE unless 1 <= B <= 65535, H, W >= 1
 * and H*W < 2^31.  Two kernels (one without the reduction), asynchronous, no allocation: graph-capturable.           */
int raft_b200_flow_to_image(const float* u, const float* v, int stride, int B, int H, int W, int clip, float clip_flow,
                            int normalize, const float* rad_max, int bgr, uint8_t* image, unsigned int* work,
                            int* status, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Evaluation data  (tf_raft/datasets/frame_utils.py:102-107 readFlowKITTI; tf_raft/losses/losses.py:24-43
 * end_point_error, with the KITTI outlier rule of RAFT's evaluate.py)
 * ------------------------------------------------------------------------------------------- */

/* One 16-bit RGB, non-interlaced PNG (a KITTI / HD1K flow map) after zlib inflation: h rows of 1 filter byte + 6 * w
 * bytes start at data + offset.  flow (h, w, 2) float32, 8-byte aligned; valid (h, w) float32.  Device pointers.     */
typedef struct raft_png16_image {
  size_t offset;
  int h, w;
  float* flow;
  float* valid;
} raft_png16_image;

/* Decodes n such images in one launch, one CTA per image, rows in order: PNG filters 0-4 undone per byte lane (bpp 6),
 * then flow = (RGB16 - 2^15) / 64 and valid = B16, exactly readFlowKITTI's float32 values.  status[i] (int, device) is
 * 0, or 1 + the first row of image i whose filter byte is not 0-4 (decoding of that image stops there).  The call
 * zeroes status on `stream` first.  images_host and images_dev hold the same array (host copy for checks and the grid,
 * device copy read by the kernel).  RAFT_ERR_BAD_ARG for a null pointer or a misaligned flow; RAFT_ERR_BAD_SHAPE
 * unless 1 <= n <= 2^31 - 1, 1 <= h, 1 <= w <= 16384, h * w < 2^31 and every image's rows lie inside data_bytes.
 * Asynchronous, no allocation: graph-capturable.                                                                     */
int raft_b200_png16_flow_decode(const uint8_t* data, size_t data_bytes, const raft_png16_image* images_host,
                                const raft_png16_image* images_dev, int n, int* status, void* stream);

/* Per-image record of raft_b200_flow_metrics: counts[b][k] over the pixels of image b that the mask keeps.             */
enum {
  RAFT_METRIC_N = 0,             /* pixels kept                                                                        */
  RAFT_METRIC_LT1 = 1,           /* epe < 1                                                                            */
  RAFT_METRIC_LT3 = 2,           /* epe < 3                                                                            */
  RAFT_METRIC_LT5 = 3,           /* epe < 5                                                                            */
  RAFT_METRIC_OUTLIER = 4,       /* epe > 3 and epe / mag > float32(0.05)                                              */
  RAFT_METRIC_COUNTS = 5
};

/* Workspace of raft_b200_flow_metrics for B images of H x W pixels.                                                 */
int raft_b200_flow_metrics_workspace_bytes(int B, int H, int W, size_t* bytes);

/* End-point-error records of B flow pairs.  pred, gt (B, H, W, 2) float32, 8-byte aligned; valid (B, H, W) float32 or
 * NULL (every pixel valid).  Per pixel, float32 with every operation rounded and none fused:
 *   mag = sqrt(g0*g0 + g1*g1); kept = valid != 0 (NaN counts as nonzero) && (!use_max_flow || mag < max_flow);
 *   epe = sqrt(d0*d0 + d1*d1), d = pred - gt; outlier = epe > 3 && epe / mag > float32(0.05).
 * counts (B, RAFT_METRIC_COUNTS) int64 and sums (B) float64 (the sum of epe over kept pixels; a NaN epe enters it and
 * fails every comparison).  The reduction has a fixed order that depends on H * W only: runs are bit-identical and an
 * image's record does not depend on the rest of the batch.  RAFT_ERR_BAD_ARG for a null or misaligned pointer;
 * RAFT_ERR_BAD_SHAPE unless 1 <= B <= 65535, H, W >= 1 and H * W < 2^31; RAFT_ERR_WORKSPACE if workspace_bytes is
 * below raft_b200_flow_metrics_workspace_bytes.  Two kernels, asynchronous, no allocation: graph-capturable.          */
int raft_b200_flow_metrics(const float* pred, const float* gt, const float* valid, int B, int H, int W, int use_max_flow,
                           float max_flow, void* workspace, size_t workspace_bytes, long long* counts, double* sums,
                           void* stream);

/* ---------------------------------------------------------------------------------------------
 * Update blocks  (tf_raft/layers/update.py)
 * ------------------------------------------------------------------------------------------- */

/* One keras Conv2D: HWIO kernel (kh, kw, cin, cout) and bias (cout), device pointers.           */
typedef struct raft_conv {
  const float* kernel;
  const float* bias;
  int kh, kw, cin, cout;
} raft_conv;

/* BasicUpdateBlock (update.py:128-141): BasicMotionEncoder :88-95, SepConvGRU :38-49,
 * FlowHead(256) :5-11, mask head :137-141.                                                      */
typedef struct raft_basic_weights {
  raft_conv convc1, convc2, convf1, convf2, conv;                 /* encoder    */
  raft_conv convz1, convr1, convq1, convz2, convr2, convq2;       /* gru        */
  raft_conv fh_conv1, fh_conv2;                                   /* flow_head  */
  raft_conv mask0, mask2;                                         /* mask[0], mask[2] */
} raft_basic_weights;

/* SmallUpdateBlock (update.py:109-116): SmallMotionEncoder :70-76, ConvGRU :17-24, FlowHead(128). */
typedef struct raft_small_weights {
  raft_conv convc1, convf1, convf2, conv;                         /* encoder    */
  raft_conv convz, convr, convq;                                  /* gru        */
  raft_conv fh_conv1, fh_conv2;                                   /* flow_head  */
} raft_small_weights;

/* Weights are re-laid-out once per model (tap-major; for F16X2 also split into scaled fp16
 * hi/lo planes) into a caller-owned device buffer that the update calls then read.              */
int raft_b200_update_prepared_bytes(int variant, int corr_channels, int precision, size_t* bytes);
int raft_b200_update_prepare(int variant, const void* weights /* raft_basic_weights* | raft_small_weights* */,
                             void* prepared, size_t prepared_bytes, int precision, void* stream);

/* Activation scratch for one update call (and for raft_b200_forward_loop) at this shape.        */
int raft_b200_update_workspace_bytes(int variant, int B, int h, int w, int precision, size_t* bytes);

/* BasicUpdateBlock.call([net, inp, corr, flow]) -> (net, 0.25*mask, delta_flow): update.py:143-153.
 *   net, inp : (B,h,w,128); corr : (B,h,w,324); flow : (B,h,w,2)
 *   net_out (B,h,w,128) may alias net; mask (B,h,w,576) may be NULL (skips the mask head);
 *   delta_flow (B,h,w,2).                                                                        */
int raft_b200_update_basic(const void* prepared, const float* net, const float* inp, const float* corr,
                           const float* flow, float* net_out, float* mask_or_null, float* delta_flow, int B,
                           int h, int w, void* workspace, size_t workspace_bytes, int precision, void* stream);

/* SmallUpdateBlock.call -> (net, None, delta_flow): update.py:118-125.
 *   net (B,h,w,96), inp (B,h,w,64), corr (B,h,w,196), flow (B,h,w,2).                            */
int raft_b200_update_small(const void* prepared, const float* net, const float* inp, const float* corr,
                           const float* flow, float* net_out, float* delta_flow, int B, int h, int w,
                           void* workspace, size_t workspace_bytes, int precision, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Encoders  (tf_raft/layers/extractor.py) -- SURVEY.md section 8(f) rank 1
 * ------------------------------------------------------------------------------------------- */

/* One normalisation layer: tfa InstanceNormalization (gamma, beta) or keras BatchNormalization (+ moving
 * statistics); all (C,) device pointers; NULL members for norm_type NONE.  eps = 1e-3 (extractor.py:6-16).   */
typedef struct raft_norm {
  const float* gamma;
  const float* beta;
  const float* moving_mean;
  const float* moving_variance;
} raft_norm;

/* ResBlock (extractor.py:19-49); downsample.kernel == NULL when strides == 1.                              */
typedef struct raft_resblock {
  raft_conv conv1, conv2;
  raft_norm norm1, norm2;
  raft_conv downsample;
  raft_norm downsample_norm;
} raft_resblock;

/* BasicEncoder / SmallEncoder (extractor.py:88-175): conv1 7x7 s2, norm1, layer1..3 (2 ResBlocks each,
 * in order layer1.0, layer1.1, layer2.0, ...), conv2 1x1.                                                   */
typedef struct raft_encoder_weights {
  raft_conv conv1;
  raft_norm norm1;
  raft_resblock block[6];
  raft_conv conv2;
} raft_encoder_weights;

typedef enum raft_norm_type { RAFT_NORM_NONE = 0, RAFT_NORM_INSTANCE = 1, RAFT_NORM_BATCH = 2 } raft_norm_type;

int raft_b200_encoder_prepared_bytes(int variant, int out_dim, size_t* bytes);
int raft_b200_encoder_prepare(int variant, int norm_type, int out_dim, const raft_encoder_weights* weights,
                              void* prepared, size_t prepared_bytes, void* stream);
int raft_b200_encoder_workspace_bytes(int variant, int N, int H, int W, size_t* bytes);

/* BasicEncoder.call / SmallEncoder.call (extractor.py:113-130 / 158-175) on N images.
 *   images : (N, H, W, 3); image_norm != 0: values are 0..255 and the 2*(x/255)-1 of model.py:70-71 is
 *            fused into the first load; image_norm == 0: already normalised (the encoder layer on its own)
 *   out    : (N, ceil(H/8), ceil(W/8), out_dim)
 *   training != 0 selects batch statistics for RAFT_NORM_BATCH (moving statistics are not updated here).   */
int raft_b200_encoder_forward(int variant, int norm_type, int out_dim, const void* prepared, const float* images,
                              int N, int H, int W, int training, int image_norm, float* out, void* workspace,
                              size_t workspace_bytes, void* stream);

/* model.py:84-86: net = tanh(cnet[..., :hidden]), inp = relu(cnet[..., hidden:]).                          */
int raft_b200_context_split(const float* cnet, int npix, int hidden, int context, float* net, float* inp,
                            void* stream);

/* The encoders of one inference forward, model.py:74-86, as concurrent branches forked from `stream` and joined back
 * into it before the call returns:
 *   A: fnet(image1);
 *   B: fnet(image2);
 *   C: cnet(image1), then the context split into net / inp.
 * fnet runs at the device's greatest stream priority, cnet at its least.  image1's stem im2col planes are built once, by
 * A, and read by C.  Every output equals, bit for bit, what raft_b200_encoder_forward (training = 0, image_norm = 1) on
 * each image batch and raft_b200_context_split compute.
 *   image1, image2 : (N, H, W, 3), values 0..255
 *   fmap1, fmap2   : (N, ceil(H/8), ceil(W/8), fnet_dim);  net : (..., hidden);  inp : (..., context)
 *   workspace      : raft_b200_encode_pair_workspace_bytes(variant, N, H, W, hidden + context)
 * The side streams and events are created on a host thread's first call for a device; that call must not be under
 * CUDA-graph capture (RAFT_ERR_UNSUPPORTED).  Later calls allocate, create and synchronise nothing, so a capture
 * records the call as a graph with three parallel branches.                                                        */
int raft_b200_encode_pair_workspace_bytes(int variant, int N, int H, int W, int cnet_dim, size_t* bytes);
int raft_b200_encode_pair(int variant, const void* fnet_prepared, int fnet_norm, int fnet_dim, const void* cnet_prepared,
                          int cnet_norm, int hidden, int context, const float* image1, const float* image2, int N, int H,
                          int W, float* fmap1, float* fmap2, float* net, float* inp, void* workspace, size_t workspace_bytes,
                          void* stream);

/* One keras Conv2D(cout, (kh, kw), 1, 'same') + optional activation on its own (fp32 FFMA path): the building block
 * behind the stand-alone FlowHead / ConvGRU / SepConvGRU / *MotionEncoder layers of update.py:5-106 when they are
 * used outside the fused update block.  x (B,H,W,cin), kernel HWIO, out (B,H,W,out_stride) written at channel out_c0.
 * act: 0 none, 1 relu, 2 sigmoid, 3 tanh.                                                                        */
int raft_b200_conv2d(const float* x, const float* kernel, const float* bias, int B, int H, int W, int cin, int kh,
                     int kw, int cout, int act, float* out, int out_stride, int out_c0, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Model loop  (tf_raft/model.py)
 * ------------------------------------------------------------------------------------------- */

/* RAFT.upsample_flow(flow, mask): model.py:39-66.  flow (B,h,w,2), mask (B,h,w,576) with channel
 * (by*8+bx)*9 + ky*3+kx -> out (B,8h,8w,2): softmax over the 9 taps of the zero-padded 3x3
 * neighbourhood of 8*flow, depth_to_space(8).                                                    */
int raft_b200_upsample_convex(const float* flow, const float* mask, int B, int h, int w, float* out, void* stream);

/* upflow8(flow): corr.py:93-96 = 8 * bilinear resize with half-pixel centres.                    */
int raft_b200_upflow8(const float* flow, int B, int h, int w, float* out, void* stream);

/* The iteration loop of RAFT.call / SmallRAFT.call: model.py:93-106 / :212-224.
 *   for i < iters:  corr = retrieve(coords1); flow = coords1 - coords0;
 *                   net, mask, delta = update_block([net, inp, corr, flow]);
 *                   coords1 += delta;  flow_up[i] = upsample(coords1 - coords0, mask)
 *   pyr          : the CorrBlock pyramid (levels entries)
 *   net          : (B,h,w,hidden) in/out -- the tanh() half of cnet's output on entry
 *   inp          : (B,h,w,context)       -- the relu() half
 *   coords1      : (B,h,w,2) in/out; holds coords_grid(B,h,w) plus an initial flow on entry: zero flow in the
 *                  reference (model.py:89), raft_b200_coords_init for a warm start; the loop's first
 *                  flow is coords1 - coords_grid
 *   flow_up      : iters pointers to (B,8h,8w,2) outputs; entries may be NULL to skip that
 *                  iteration's upsampling (predict_step keeps only the last, model.py:166);
 *                  for BASIC a skipped iteration also skips the mask head.                        */
int raft_b200_forward_loop(int variant, const void* prepared, const float* const pyr[], int levels, int radius,
                           float* net, const float* inp, float* coords1, float* const flow_up[], int iters,
                           int B, int h, int w, void* workspace, size_t workspace_bytes, int precision,
                           void* stream);

/* Number of kernels launched on this host thread since the last raft_b200_launch_count_reset (bench.py's gpu_launches). */
long long raft_b200_launch_count(void);
void raft_b200_launch_count_reset(void);
/* Profiling aid for bench.py's roofline objects: while enabled, raft_b200_forward_loop (F16X2, <= 64 iterations, not
 * under CUDA-graph capture) records CUDA events on its stream around the lookup and around the update-block kernel(s)
 * of every iteration; _read waits for the last one and returns the summed durations of the most recent call.      */
void raft_b200_profile_loop(int enable);
int raft_b200_profile_read(float* lookup_ms, float* update_ms, int* iterations);

#ifdef __cplusplus
}
#endif
#endif /* RAFT_B200_H_ */
