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

/* model.py:10-30 (RAFT, BasicUpdateBlock) / model.py:173-188 (SmallRAFT, SmallUpdateBlock).
 * SMALL_PYTORCH is the original PyTorch RAFT-small: its encoders are built from bottleneck blocks
 * (raft_b200_encoder_prepare_bottleneck) and its loop upsamples with raft_b200_upflow8_align_corners.  The encoder
 * entry points (encoder_prepared_bytes / _workspace_bytes / _forward, encode_pair_workspace_bytes, encode_pair) and
 * forward_loop / forward_loop_ex accept it; the loop treats it as RAFT_VARIANT_SMALL (same update-block blob, prepared
 * as SMALL, same workspace, same lookup) except for the upsampling.  Every other entry point returns RAFT_ERR_BAD_ARG. */
typedef enum raft_variant {
  RAFT_VARIANT_BASIC = 0,
  RAFT_VARIANT_SMALL = 1,
  RAFT_VARIANT_SMALL_PYTORCH = 2
} raft_variant;

/* Lookup sampler (raft_b200_corr_lookup_ex, raft_b200_forward_loop_ex).
 *   TF    tf-raft's bilinear_sampler (corr.py:28-69): clamp to [0, S-1], floor / ceil corners.
 *   GRID  the original PyTorch RAFT's: F.grid_sample(align_corners=True, padding_mode='zeros') after RAFT's
 *         normalisation 2*x/(S-1) - 1.  Per axis of size S, level coordinate v = fl(fl(c * 2^-l) + d), op by op in
 *         fp32 with no FMA: g = fl(fl(fl(2v) * fl(1 / (S-1))) - 1) (the division as ATen's CUDA kernel does it for
 *         a scalar divisor, a product with the reciprocal); ix = fl(fl(fl(g + 1) / 2) * (S-1)); ix = -100 unless
 *         -2^31 <= ix <= 2^31 (NaN included); corners x0 = floor(ix), x1 = x0 + 1 with weights fl(x1 - ix),
 *         fl(ix - x0).  A corner outside [0, S-1] is never read and adds nothing, so a level with S = 1 gives 0 for
 *         every tap.  Sum order of a tap: acc = +0, then for (y0,x0), (y0,x1), (y1,x0), (y1,x1) in that order, if the
 *         corner is in the level, acc = fl(acc + fl(fl(wy * wx) * texel)) -- weight 0 included.                    */
typedef enum raft_sampler { RAFT_SAMPLER_TF = 0, RAFT_SAMPLER_GRID = 1 } raft_sampler;

/* Arithmetic conventions of the encoders (raft_b200_encoder_prepare_ex).
 *   TF       tf-raft: Keras 'same' padding, asymmetric at stride 2 on even inputs (7x7/s2 pads 2 before, 3 after;
 *            3x3/s2 0 / 1), norm epsilon 1e-3.
 *   PYTORCH  the original PyTorch RAFT: symmetric padding (7x7/s2 p=3, 3x3/s2 p=1, 1x1/s2 p=0), epsilon 1e-5.
 * Both give ceil(H/2) outputs at stride 2, so workspaces do not depend on the convention.                        */
typedef enum raft_conventions { RAFT_CONVENTIONS_TF = 0, RAFT_CONVENTIONS_PYTORCH = 1 } raft_conventions;

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
/* raft_b200_corr_lookup with the sampler chosen (raft_sampler); RAFT_SAMPLER_TF is raft_b200_corr_lookup.        */
int raft_b200_corr_lookup_ex(const float* const pyr[], const float* coords, int B, int h, int w, int levels,
                             int radius, float* out, int out_stride, int sampler, void* stream);

/* Backward of CorrBlock.retrieve for the training step (tf_raft/model.py:133: tape.gradient through corr.py:116-152;
 * the reference does not detach coords1, model.py:102).  grad_out (B, h, w, levels*(2r+1)^2) -> grad_coords (B, h, w, 2)
 * and grad_pyr[l] (same shapes as pyr[l]); both outputs are ACCUMULATED into (zero them first).  TensorFlow gradient
 * rules: floor / ceil / indices carry no gradient, clip_by_value passes it inside [0, dim-1]; terms with a zero
 * grad_out, and pyramid terms with a zero bilinear weight, are skipped.
 * Deterministic: no atomics, and every sum has a fixed order that depends on the shape and the data only, with each
 * operation one rounded fp32 operation (no FMA).  With t = a*(2r+1) + b:
 *   grad_pyr : a touched cell ends as in + term_1 + term_2 + ... left to right, terms fl(fl(wy*wx) * grad_out) in
 *              ascending t (then corner 00, 01, 10, 11); cells no term reaches are not written;
 *   grad_coords : per level l, 32 lane sums (lane j adds taps j, j+32, ... in order, from +0) combined by the xor
 *              butterfly with strides 16, 8, 4, 2, 1 give G_l; grad_coords ends as in + fl(G_0 * 2^0) + fl(G_1 * 2^-1)
 *              + ... in ascending level.  Two calls on the same inputs give the same bits (DESIGN.md section 9).  */
int raft_b200_corr_lookup_backward(const float* const pyr[], const float* coords, const float* grad_out, int B, int h, int w,
                                   int levels, int radius, float* grad_coords, float* const grad_pyr[], void* stream);
/* raft_b200_corr_lookup_backward with the sampler chosen (raft_sampler); RAFT_SAMPLER_TF is
 * raft_b200_corr_lookup_backward.  RAFT_SAMPLER_GRID is the backward of the grid_sample lookup with respect to the
 * pyramid only, as the original RAFT, which detaches the sampling position, computes it: grad_coords must be NULL
 * (RAFT_ERR_BAD_ARG otherwise) and pyr is not read.  ATen's grid_sampler_2d_backward with the forward's per-axis
 * set-up: every in-frame corner of a tap adds fl(fl(wy*wx) * grad_out) to its cell, a zero weight or a zero grad_out
 * included (so a non-finite grad_out reaches the cells ATen's backward reaches); corners outside the level add nothing.
 * grad_pyr is ACCUMULATED, in the same order as above: a touched cell ends as in + term_1 + term_2 + ... left to right,
 * in ascending t, then corner 00, 01, 10, 11; cells no in-frame corner reaches are not written (a level with S = 1
 * receives nothing).  No atomics; two calls on the same inputs give the same bits.                                 */
int raft_b200_corr_lookup_backward_ex(const float* const pyr[], const float* coords, const float* grad_out, int B, int h,
                                      int w, int levels, int radius, float* grad_coords, float* const grad_pyr[],
                                      int sampler, void* stream);

/* tf.linalg.global_norm over a flat gradient buffer (model.py:135): out[0] = sum g^2 (deterministic two-stage
 * reduction; `partials` holds one float per block, at most npartials blocks are used).                               */
int raft_b200_sumsq(const float* g, size_t n, float* partials, size_t npartials, float* out, void* stream);

/* tf.clip_by_global_norm (model.py:135) + tfa.optimizers.AdamW.apply_gradients (model.py:136, train_chairs.py:87-90)
 * on flat buffers: g' = g * clip / max(sqrt(*sumsq), clip) (clip_norm <= 0: no clipping); var -= wd * var;
 * m = b1 m + (1-b1) g'; v = b2 v + (1-b2) g'^2; var -= lr_t * m / (sqrt(v) + eps), lr_t already bias-corrected.        */
int raft_b200_adamw_step(float* param, const float* grad, float* m, float* v, size_t n, const float* sumsq, float clip_norm,
                         float lr_t, float beta1, float beta2, float epsilon, float weight_decay, void* stream);

/* Optimiser rule of raft_b200_adamw_step_ex.
 *   TFA    tf.clip_by_global_norm + tfa AdamW: raft_b200_adamw_step (lr = the bias-corrected lr_t; bias_correction1/2
 *          are not read).
 *   TORCH  the original PyTorch RAFT's: torch.nn.utils.clip_grad_norm_ then torch.optim.AdamW,
 *          g' = g * min(1, clip / (sqrt(*sumsq) + 1e-6)) (clip_norm <= 0: no clipping); var *= 1 - lr*wd;
 *          m = b1 m + (1-b1) g'; v = b2 v + (1-b2) g'^2; var -= (lr / bias_correction1) * m / (sqrt(v) /
 *          sqrt(bias_correction2) + eps), with the scheduled lr and bias_correction1 = 1 - b1^t, bias_correction2 =
 *          1 - b2^t of step t from the caller.                                                                     */
typedef enum raft_adamw_rule { RAFT_ADAMW_TFA = 0, RAFT_ADAMW_TORCH = 1 } raft_adamw_rule;
int raft_b200_adamw_step_ex(float* param, const float* grad, float* m, float* v, size_t n, const float* sumsq,
                            float clip_norm, float lr, float beta1, float beta2, float epsilon, float weight_decay,
                            float bias_correction1, float bias_correction2, int rule, void* stream);

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

/* Flow warping and composition (additions beyond the reference; DESIGN.md section 3.9).  Both use
 * raft_b200_fb_occlusion's conventions: flows (B, H, W, 2) float32, 8-byte aligned; pixel (x, y) lands at
 * p = (x + fx, y + fy); p is inside a (Hs, Ws) grid iff 0 <= px <= Ws-1 and 0 <= py <= Hs-1 (NaN never is);
 *   bilinear(T, p): x0 = floor(px), x1 = min(x0+1, Ws-1), ax = px - x0, bx = 1 - ax (y likewise),
 *                   by*(bx*T[y0,x0] + ax*T[y0,x1]) + ay*(bx*T[y1,x0] + ax*T[y1,x1]);
 *   nearest(p):     xi = min(floor(px + 0.5), Ws-1), yi = min(floor(py + 0.5), Hs-1).
 * Every operation is one rounded fp32 operation in the order written, no FMA; a non-finite texel makes a bilinear
 * sample non-finite even at weight 0.  Each call is one asynchronous launch with no allocation and no host
 * synchronisation.                                                                                                   */
typedef enum raft_warp_mode { RAFT_WARP_BILINEAR = 0, RAFT_WARP_NEAREST = 1 } raft_warp_mode;
typedef enum raft_warp_dtype { RAFT_WARP_F32 = 0, RAFT_WARP_U8 = 1 } raft_warp_dtype;

/* Backward warping: out[b,y,x,:] = sample of src[b] at the landing of flow[b,y,x] (bilinear or nearest, raft_warp_mode).
 * src (B, Hs, Ws, C) of raft_warp_dtype (float32 4-byte aligned, or uint8 with RAFT_WARP_NEAREST only, which copies
 * labels unchanged); flow (B, H, W, 2) sets the output grid: out is (B, H, W, C) of src's dtype.  The flow is in pixels
 * of src and is not rescaled when (Hs, Ws) differs from (H, W).  Where the landing is outside src's frame or not
 * finite, out is `fill` (for uint8 an integer 0..255) and occ[b,y,x] = 1; elsewhere occ is 0.  occ (B, H, W) uint8 may
 * be NULL.  out and occ must not overlap each other, src or flow.  RAFT_ERR_BAD_ARG: NULL src / flow / out, unknown
 * mode or dtype, uint8 with BILINEAR, a bad uint8 fill, misalignment or overlap; RAFT_ERR_BAD_SHAPE: a non-positive
 * dimension, C outside 1..1024, or H*W*C or Hs*Ws*C above 2^31 - 1.                                                 */
int raft_b200_warp(const void* src, int dtype, int Hs, int Ws, int C, const float* flow, int B, int H, int W, int mode,
                   float fill, void* out, uint8_t* occ, void* stream);

/* Flow composition, the chaining step of tracking.  With p the landing of f1 at pixel x of image b, on one (H, W) grid:
 *   out(x)     = f1(x) + bilinear(f2[b], p)   (the sum one fp32 addition per component),
 *   occ_out(x) = occ1(x) || !inside(p) || occ2[b](nearest(p)) || !finite(out(x)),
 * and out(x) = f1(x) unchanged wherever occ_out(x) is set, so a lost track keeps its last position.  occ1, occ2,
 * occ_out: (B, H, W) uint8, nonzero = no correspondence; occ1 and occ2 may be NULL (no mask).  out may be f1 itself and
 * occ_out may be occ1 itself; any other overlap of an output with another buffer is RAFT_ERR_BAD_ARG, as are NULL
 * f1 / f2 / out / occ_out and misaligned flows.  RAFT_ERR_BAD_SHAPE: a non-positive dimension or H*W above 2^31 - 1.
 *   forward chaining  (frame 0 -> t): acc, lost = compose(acc, F_{t-1->t}, lost, occ_fw);
 *   backward chaining (frame t -> 0): acc, lost = compose(B_{t->t-1}, acc, occ_bw, lost).                             */
int raft_b200_compose_flow(const float* f1, const float* f2, const uint8_t* occ1, const uint8_t* occ2, int B, int H,
                           int W, float* out, uint8_t* occ_out, void* stream);

/* Self-supervised training (an addition beyond the reference; DESIGN.md section 9.1).
 *
 * raft_b200_census: images (B, H, W, 3) float32 in 0..255 -> out (B, H, W, 48) float32, 16-byte aligned.  With
 * g = (0.2989 R + 0.5870 G + 0.1140 B) / 255 (0 outside the frame) and the offsets (dy, dx) of [-3, 3]^2 \ {(0, 0)} in
 * row-major order, channel k of pixel (x, y) is t / sqrt(0.81 + t^2), t = g(y + dy, x + dx) - g(y, x).  Every
 * operation is one rounded fp32 operation in that order, no FMA.                                                    */
int raft_b200_census(const float* images, int B, int H, int W, float* out, void* stream);

/* raft_b200_unsup_loss: one direction's share of the self-supervised loss and its gradient, all n predictions in one
 * pass.  census_t / census_s: raft_b200_census of the target (the image the flows start from) and of the source;
 * image_t: the target image (B, H, W, 3); occ: (B, H, W) forward-backward occlusion of the target's pixels
 * (raft_b200_fb_occlusion); flows: (n, B, H, W, 2) predictions, 8-byte aligned.  With m = !occ and the pixel at least
 * 3 px from every border, gamma_i = gamma^(n-1-i), and for prediction i at pixel x:
 *   D_i(x) = sum_c d^2 / (0.1 + d^2), d = census_t(x) - bilinear sample of census_s at x + F_i(x) (fb_occlusion's
 *            corner rule; a landing outside the closed frame contributes 0),
 *   L_c = sum_i gamma_i sum_x m (D_i + 0.01)^0.4 / max(sum_x m, 1),
 *   L_s = sum_i gamma_i (S_h + S_v) / 2, S_h (S_v) the mean over horizontal (vertical) neighbour pairs of
 *         exp(-edge_weight * mean_c |I_c(x') - I_c(x)| / 255) * (|dFx| + |dFy|) / 2,
 * it writes sums[0] = L_c, sums[1] = L_s, sums[2] = sum_x m, sums[3] = census_weight / 2 * L_c +
 * smoothness_weight / 2 * L_s (fp64), and grad (n, B, H, W, 2) = d sums[3] / d flows (d|u|/du = 0 at 0).
 * partials: device scratch of npartials doubles, at least 4; the call uses 4 per CTA of a grid of
 * min(npartials / 4, ceil(B*H*W / 256), 1056) CTAs and adds them in a fixed order, so two calls with the same
 * inputs and npartials give the same bits.  H, W >= 2 (RAFT_ERR_BAD_SHAPE otherwise); weights and gamma finite and
 * >= 0 (RAFT_ERR_BAD_ARG otherwise).                                                                                */
int raft_b200_unsup_loss(const float* census_t, const float* census_s, const float* image_t, const uint8_t* occ,
                         const float* flows, int n, int B, int H, int W, float census_weight, float smoothness_weight,
                         float edge_weight, float gamma, double* partials, size_t npartials, double* sums, float* grad,
                         void* stream);

/* raft_b200_unsup_loss_norm: raft_b200_unsup_loss with L_c = sum_i gamma_i sum_x m (D_i + 0.01)^0.4 / N.
 * census_norm: NULL (N = max(sum_x m, 1): the same launches and bits as raft_b200_unsup_loss) or a device pointer to
 * one double N > 0, 8-byte aligned (RAFT_ERR_BAD_ARG otherwise); sums[2] is still this call's own mask count.
 * Under data parallelism over R equal shards, with C the mask count of the whole batch, a rank passes
 * N = max(C, 1) / R: its census share is then R times its part of the whole batch's, and the gradients summed over
 * the ranks and divided by R are the whole batch's.                                                                 */
int raft_b200_unsup_loss_norm(const float* census_t, const float* census_s, const float* image_t, const uint8_t* occ,
                              const float* flows, int n, int B, int H, int W, float census_weight,
                              float smoothness_weight, float edge_weight, float gamma, double* partials,
                              size_t npartials, double* sums, float* grad, const double* census_norm, void* stream);

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
 * Colour jitter  (the original RAFT's core/utils/augmentor.py colour step: torchvision ColorJitter on RGB PIL images,
 * Pillow's arithmetic, given ColorJitter.get_params' draws)
 * ------------------------------------------------------------------------------------------- */

/* Ops of raft_colour_jitter_sample.order, torchvision's fn_idx values.                                               */
enum { RAFT_JITTER_NONE = -1, RAFT_JITTER_BRIGHTNESS = 0, RAFT_JITTER_CONTRAST = 1, RAFT_JITTER_SATURATION = 2,
       RAFT_JITTER_HUE = 3 };

/* One sample: two (H, W, 3) uint8 images, device memory, HWC and contiguous, jittered into out_img1 / out_img2 (which
 * may be the sources).  stacked != 0: parameter set 0 jitters img1 stacked above img2 as one (2H, W) image;
 * otherwise set k jitters image k.  A set applies order[0..3] to every pixel, each op at most once; RAFT_JITTER_NONE
 * stands for an op that ColorJitter skips (a strength of 0 makes get_params return None for its factor):
 *   brightness  c = blend(0, c, factor[0])
 *   contrast    c = blend(m, c, factor[1]), m = int(S / n + 0.5) in float64, S the integer sum of L over the set's
 *               n pixels after the ops before contrast
 *   saturation  c = blend(L, c, factor[2]), L the pixel's own L
 *   hue         Pillow RGB->HSV, H = (H + hue) mod 256, Pillow HSV->RGB (the round trip also runs for hue = 0)
 * with blend(a, b, f) = clip(trunc(fl32(a + fl32(f * (b - a)))), 0, 255) and L = (19595 R + 38470 G + 7471 B + 0x8000)
 * >> 16.  Pillow's RGB<->HSV mixes float32 and float64 as its C source promotes them (DESIGN.md section 3.8).       */
typedef struct raft_colour_jitter_sample {
  const uint8_t* img1;
  const uint8_t* img2;
  uint8_t* out_img1;
  uint8_t* out_img2;
  int H, W;
  int stacked;
  int order[2][4];              /* per set: the ops in application order, or RAFT_JITTER_NONE                      */
  float factor[2][3];           /* per set: brightness, contrast and saturation factors, finite                    */
  int hue[2];                   /* per set: the byte added to H, 0..255: uint8(int32(hue_factor * 255))            */
} raft_colour_jitter_sample;

/* ColorJitter on B samples of any sizes in one launch pair (2 kernels after a memset of sums).  samples_host and
 * samples_dev hold the same array (host copy for checks and grid sizes, device copy read by the kernels).
 * sums: device, 2 * B unsigned 64-bit words, overwritten (the L sums of each sample's two sets).  Set 1 of a stacked
 * sample is neither checked nor read.  Asynchronous on `stream`, no allocation: graph-capturable.                    */
int raft_b200_colour_jitter(const raft_colour_jitter_sample* samples_host, const raft_colour_jitter_sample* samples_dev,
                            int B, unsigned long long* sums, void* stream);

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

/* Element type and fill of one raft_b200_pad_batch plane.                                                           */
typedef enum raft_pad_dtype { RAFT_PAD_U8 = 0, RAFT_PAD_F32 = 1 } raft_pad_dtype;
typedef enum raft_pad_mode { RAFT_PAD_ZERO = 0, RAFT_PAD_REPLICATE = 1 } raft_pad_mode;

/* One plane of an evaluation batch: src (h, w, c) is placed with its pixel (0, 0) at (top, left) of dst (H, W, c);
 * a negative top or left crops.  Both dense row-major, of element type dtype, device memory.                         */
typedef struct raft_pad_plane {
  const void* src;
  void* dst;
  int h, w, c;
  int H, W;
  int top, left;
  int dtype;                    /* raft_pad_dtype                                                                   */
  int mode;                     /* raft_pad_mode                                                                    */
} raft_pad_plane;

/* Writes n planes of any sizes in one launch (RAFT's InputPadder and the reference's CropOrPadder, evaluate.py /
 * dataset.py:323-334).  For every destination pixel, with sy = y - top, sx = x - left:
 *   RAFT_PAD_REPLICATE: dst(y, x) = src(clamp(sy, 0, h-1), clamp(sx, 0, w-1))   (F.pad mode='replicate', np.pad 'edge')
 *   RAFT_PAD_ZERO:      dst(y, x) = src(sy, sx) inside the source, 0 outside it
 * Pure copies: the output is bit-exact.  dst must not overlap any src.  planes_host and planes_dev hold the same array
 * (host copy for checks and the grid, device copy read by the kernel).  RAFT_ERR_BAD_ARG for a null pointer, an
 * unknown dtype or mode, or a float32 plane that is not 4-byte aligned; RAFT_ERR_BAD_SHAPE unless 1 <= n <= 65535,
 * h, w, c, H, W >= 1 and h * w * c, H * W * c <= 2^31 - 1.  Asynchronous, no allocation: graph-capturable.         */
int raft_b200_pad_batch(const raft_pad_plane* planes_host, const raft_pad_plane* planes_dev, int n, void* stream);

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
/* raft_b200_encoder_prepare under the given conventions (raft_conventions), which the blob records: the BatchNorm
 * fold uses its epsilon now, and raft_b200_encoder_forward / raft_b200_encode_pair take its padding and epsilon from
 * the blob.  raft_b200_encoder_prepare is this call with RAFT_CONVENTIONS_TF.  The convention is bound to the blob's
 * device address by the last prepare call at that address, and forward calls look it up there without touching the
 * device.  A blob copied to an address no prepare call has used has its convention read back from the device once
 * (never under CUDA-graph capture: RAFT_ERR_UNSUPPORTED).  A blob copied onto an address a prepare call used is taken
 * to have that call's convention: prepare a blob where it is used instead of copying one there.                  */
int raft_b200_encoder_prepare_ex(int variant, int norm_type, int out_dim, const raft_encoder_weights* weights,
                                 int conventions, void* prepared, size_t prepared_bytes, void* stream);
int raft_b200_encoder_workspace_bytes(int variant, int N, int H, int W, size_t* bytes);

/* The original PyTorch RAFT's BottleneckBlock(in, planes, stride): y = relu(norm1(conv1 1x1, in -> planes/4));
 * y = relu(norm2(conv2 3x3, padding 1, stride, planes/4 -> planes/4)); y = relu(norm3(conv3 1x1, planes/4 -> planes));
 * x = norm4(downsample 1x1, stride, in -> planes) when stride != 1, else x = the block input; out = relu(x + y).
 * downsample.kernel == NULL when stride == 1.                                                                     */
typedef struct raft_bottleneck {
  raft_conv conv1, conv2, conv3;
  raft_norm norm1, norm2, norm3;
  raft_conv downsample;
  raft_norm downsample_norm;
} raft_bottleneck;

/* The original RAFT-small's SmallEncoder: conv1 7x7 s2 3 -> 32, norm1, layer1 = 2 x Bottleneck(32), layer2 =
 * Bottleneck(32 -> 64, s2), Bottleneck(64), layer3 = Bottleneck(64 -> 96, s2), Bottleneck(96) (block[0..5] in that
 * order; bottleneck widths 8, 16, 24), conv2 1x1 96 -> out_dim.                                                 */
typedef struct raft_bottleneck_encoder_weights {
  raft_conv conv1;
  raft_norm norm1;
  raft_bottleneck block[6];
  raft_conv conv2;
} raft_bottleneck_encoder_weights;

/* Prepares a RAFT_VARIANT_SMALL_PYTORCH encoder blob (raft_b200_encoder_prepared_bytes(RAFT_VARIANT_SMALL_PYTORCH,
 * out_dim)).  The blob always records RAFT_CONVENTIONS_PYTORCH (bound to its address as raft_b200_encoder_prepare_ex
 * describes).  norm_type: RAFT_NORM_INSTANCE (gamma / beta of every norm given) or RAFT_NORM_NONE; RAFT_NORM_BATCH
 * returns RAFT_ERR_BAD_ARG.                                                                                      */
int raft_b200_encoder_prepare_bottleneck(int norm_type, int out_dim, const raft_bottleneck_encoder_weights* weights,
                                         void* prepared, size_t prepared_bytes, void* stream);

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

/* Tensor-core convolutions of the training step (RAFT.compile(train_precision='f16x2')): a stride-1 Conv2D with odd
 * kh, kw <= 7 and symmetric 'same' padding ((kh-1)/2, (kw-1)/2; a 1x1 'valid' convolution is the 1x1 case), 16 <= cin
 * <= 1024, 1 <= cout <= 1024, B*H*W < 2^31 (RAFT_ERR_BAD_SHAPE otherwise).  NHWC fp32 activations, HWIO fp32 kernel, fp16
 * hi/lo three-pass arithmetic with IEEE-fp32 promotion (DESIGN.md section 9).
 *
 * Workspace: with workspace == NULL either call writes the bytes the shape needs to *workspace_bytes and runs nothing;
 * otherwise *workspace_bytes is the buffer's size (RAFT_ERR_WORKSPACE if smaller).  One buffer of that size serves the
 * forward and the backward of a shape.  x_planes and workspace 256-byte aligned, out and grad_x 32-byte aligned
 * (RAFT_ERR_BAD_ARG otherwise).
 *
 * forward: out (B,H,W,cout) = conv(x (B,H,W,cin)) + bias.  Writes x_planes, what the backward reads of x: the fp16
 * hi/lo split of x * 2^k_x (hi plane, then lo plane, B*H*W * round_up(cin, 64) halves each; max finite |x| * 2^k_x in
 * [2^12, 2^13), k_x in [-100, 100]) followed by 256 bytes holding the scale: 4 * B*H*W * round_up(cin, 64) + 256 bytes.
 * backward: from x_planes and grad_out (B,H,W,cout): grad_kernel (kh,kw,cin,cout) and, unless grad_x is NULL, grad_x
 * (B,H,W,cin).  grad_out is scaled by 2^k_g before its split, max finite |grad_out| * 2^k_g in [2^12, 2^13), k_g in
 * [-100, 100]; a NaN or inf in grad_out or x makes every output whose sum includes it NaN, and no other (image
 * edges included).  The weight gradient adds
 * per-slice partial sums in a fixed order (slices depend on the shape only; no atomics): two calls give the same bits. */
int raft_b200_conv_tc_forward(const float* x, const float* kernel, const float* bias, int B, int H, int W, int cin, int kh,
                              int kw, int cout, float* out, void* x_planes, void* workspace, size_t* workspace_bytes,
                              void* stream);
int raft_b200_conv_tc_backward(const void* x_planes, const float* kernel, const float* grad_out, int B, int H, int W,
                               int cin, int kh, int kw, int cout, float* grad_x, float* grad_kernel, void* workspace,
                               size_t* workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Model loop  (tf_raft/model.py)
 * ------------------------------------------------------------------------------------------- */

/* RAFT.upsample_flow(flow, mask): model.py:39-66.  flow (B,h,w,2), mask (B,h,w,576) with channel
 * (by*8+bx)*9 + ky*3+kx -> out (B,8h,8w,2): softmax over the 9 taps of the zero-padded 3x3
 * neighbourhood of 8*flow, depth_to_space(8).                                                    */
int raft_b200_upsample_convex(const float* flow, const float* mask, int B, int h, int w, float* out, void* stream);

/* upflow8(flow): corr.py:93-96 = 8 * bilinear resize with half-pixel centres.                    */
int raft_b200_upflow8(const float* flow, int B, int h, int w, float* out, void* stream);

/* The original RAFT-small's upflow8: 8 * F.interpolate(flow, size=(8h, 8w), mode='bilinear', align_corners=True), as
 * ATen's upsample_bilinear2d computes it.  flow (B,h,w,2) -> out (B,8h,8w,2).  Per axis of n input cells, in fp32,
 * each operation one rounded operation, no FMA:
 *   scale = fl((n-1) / (8n-1)) (0 when 8n = 1, never the case here);  src = fl(scale * X);  i0 = (int)src;
 *   i1 = i0 + (i0 < n-1);  l1 = fl(src - i0);  l0 = fl(1 - l1);
 * and per output pixel and channel, with a = f[y0][x0], b = f[y0][x1], c = f[y1][x0], d = f[y1][x1]:
 *   val = fl(fl(ly0 * fl(fl(lx0 * a) + fl(lx1 * b))) + fl(ly1 * fl(fl(lx0 * c) + fl(lx1 * d))));  out = fl(8 * val)
 * (the factor 8 is exact).  All four corners are read even at weight 0, so a NaN or inf reaches the outputs ATen's
 * kernel gives it.                                                                                               */
int raft_b200_upflow8_align_corners(const float* flow, int B, int h, int w, float* out, void* stream);

/* Backward of F.interpolate(scale_factor=8, mode='bilinear', align_corners=False), the upsampling of SmallRAFT's
 * training graph (without upflow8's factor 8).  grad_up (B, 8h, 8w, 2) -> grad_flow (B, h, w, 2), WRITTEN (not
 * accumulated); both 8-byte aligned (RAFT_ERR_BAD_ARG otherwise).  PyTorch's upsample_bilinear2d weights: per output
 * coordinate X of an axis of n input cells, src = max(0.125 (X + 0.5) - 0.5, 0), i0 = (int)src, i1 = i0 + (i0 < n-1),
 * l1 = src - i0, l0 = 1 - l1; y likewise.  Every output pixel contributes to all four of its corners, zero weights
 * included (so NaN reaches the cells PyTorch's backward gives it), term fl(fl(ly * lx) * grad_up).  Deterministic, no
 * atomics: a cell is +0 + its terms, added left to right in ascending output pixel (row-major), then corner 00, 01, 10,
 * 11, each operation one rounded fp32 operation.                                                                      */
int raft_b200_upflow8_backward(const float* grad_up, int B, int h, int w, float* grad_flow, void* stream);

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
 *                  for BASIC a skipped iteration also skips the mask head.  Upsampling: BASIC convex,
 *                  SMALL raft_b200_upflow8, SMALL_PYTORCH raft_b200_upflow8_align_corners.        */
int raft_b200_forward_loop(int variant, const void* prepared, const float* const pyr[], int levels, int radius,
                           float* net, const float* inp, float* coords1, float* const flow_up[], int iters,
                           int B, int h, int w, void* workspace, size_t workspace_bytes, int precision,
                           void* stream);
/* raft_b200_forward_loop with the lookup's sampler chosen (raft_sampler); RAFT_SAMPLER_TF is raft_b200_forward_loop. */
int raft_b200_forward_loop_ex(int variant, const void* prepared, const float* const pyr[], int levels, int radius,
                              float* net, const float* inp, float* coords1, float* const flow_up[], int iters,
                              int B, int h, int w, void* workspace, size_t workspace_bytes, int precision,
                              int sampler, void* stream);

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
