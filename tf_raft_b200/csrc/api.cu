// extern "C" entry points of libraft_b200.so (see include/raft_b200.h for the contract and the
// reference file:line each one replaces).  Host code only decides shapes and launches kernels;
// there is no CPU compute path.
#include <float.h>
#include <limits.h>
#include <stdlib.h>

#include <algorithm>

#include "augment.cuh"
#include "conv_train.cuh"
#include "corr_tc.cuh"
#include "dataset.cuh"
#include "encoder.cuh"
#include "flow_viz.cuh"
#include "pad.cuh"
#include "train.cuh"
#include "unsup.cuh"
#include "video.cuh"

namespace raft {
thread_local long long g_launches = 0;

static int check_dims(int B, int h, int w) { return (B > 0 && h > 0 && w > 0) ? 0 : RAFT_ERR_BAD_SHAPE; }
static int check_variant(int v) { return (v == RAFT_VARIANT_BASIC || v == RAFT_VARIANT_SMALL) ? 0 : RAFT_ERR_BAD_ARG; }
static int check_precision(int p) { return (p == RAFT_PREC_FP32 || p == RAFT_PREC_F16X2) ? 0 : RAFT_ERR_BAD_ARG; }

// Per-kernel timing of raft_b200_forward_loop for bench.py's roofline objects: CUDA events on the launching stream around
// the lookup and around the update-block kernel(s) of every iteration (raft_b200_profile_loop / _read).  Off by default;
// never armed while a CUDA graph is being captured.
struct LoopProfile {
  bool on = false;
  int n = 0;                                   // iterations recorded by the last forward_loop call
  cudaEvent_t ev[64][3];                       // [iteration]: before lookup, after lookup (+ im2col), after the update block
  bool created = false;
};
static LoopProfile g_prof;

// ------------------------------------------------------------------------------------------------
// Correlation pyramid
// ------------------------------------------------------------------------------------------------
struct CorrWs {
  float* f2_lvl[RAFT_MAX_LEVELS];            // pooled fmap2 per level (level 0 = fmap2 itself, not stored)
  __half *f1_hi, *f1_lo;
  __half *f2_hi[RAFT_MAX_LEVELS], *f2_lo[RAFT_MAX_LEVELS];
  size_t total;
};
static CorrWs corr_ws_layout(void* base, int B, int h, int w, int C, int levels, int precision) {
  CorrWs W;
  memset(&W, 0, sizeof(W));
  if (precision != RAFT_PREC_F16X2) return W;
  uint8_t* b8 = reinterpret_cast<uint8_t*>(base);
  size_t off = 0;
  auto take = [&](size_t bytes) {
    uint8_t* p = b8 + off;
    off = align_up(off + bytes, 1024);
    return p;
  };
  W.f1_hi = reinterpret_cast<__half*>(take((size_t)B * h * w * C * 2));
  W.f1_lo = reinterpret_cast<__half*>(take((size_t)B * h * w * C * 2));
  int lh = h, lw = w;
  for (int l = 0; l < levels; ++l) {
    if (l > 0) W.f2_lvl[l] = reinterpret_cast<float*>(take((size_t)B * lh * lw * C * 4));
    W.f2_hi[l] = reinterpret_cast<__half*>(take((size_t)B * lh * lw * C * 2));
    W.f2_lo[l] = reinterpret_cast<__half*>(take((size_t)B * lh * lw * C * 2));
    lh /= 2;
    lw /= 2;
  }
  W.total = off;
  return W;
}

static int corr_build_fp32(const float* f1, const float* f2, int B, int h, int w, int C, int levels, float* const pyr[],
                           cudaStream_t st) {
  const int N = h * w;
  dim3 grid((unsigned)ceil_div(N, 64), (unsigned)ceil_div(N, 64), (unsigned)B);
  RAFT_TRY(launch(corr_fp32_kernel, grid, 256, 0, st, f1, f2, pyr[0], N, C, sqrtf((float)C)));
  int lh = h, lw = w;
  for (int l = 1; l < levels; ++l) {        // corr.py:112-114: pool the volume itself
    const size_t M = (size_t)B * N;
    const size_t total = M * (lh / 2) * (lw / 2);
    RAFT_TRY(launch(avgpool2x2_kernel, grid_for(total), 256, 0, st, pyr[l - 1], pyr[l], M, lh, lw, 1));
    lh /= 2;
    lw /= 2;
  }
  return 0;
}

// Tensor-core path: level l = fmap1 . avgpool^l(fmap2)^T / sqrt(C).  Pooling is linear, so pooling
// the 256-channel features (a few MB) before the GEMM equals pooling the N x N volume after it
// (up to fp32 summation order) and every level is written exactly once, straight from the accumulator registers.
// Two launches: corr_prep_kernel (pool + hi/lo split of both feature maps) and corr_tc_kernel (all levels).
static int corr_build_tc(const float* f1, const float* f2, int B, int h, int w, int C, int levels, float* const pyr[],
                         void* ws, cudaStream_t st) {
  if (C % kChunkK != 0) return RAFT_ERR_BAD_SHAPE;
  CorrWs W = corr_ws_layout(ws, B, h, w, C, levels, RAFT_PREC_F16X2);
  const int N = h * w;
  const size_t npix = (size_t)B * N;
  if (levels <= 4) {
    CorrPrepParams q;
    memset(&q, 0, sizeof(q));
    q.f1 = f1; q.f2 = f2; q.f1_hi = W.f1_hi; q.f1_lo = W.f1_lo;
    for (int l = 0; l < levels; ++l) { q.f2_hi[l] = W.f2_hi[l]; q.f2_lo[l] = W.f2_lo[l]; }
    q.B = B; q.h = h; q.w = w; q.C = C; q.levels = levels;
    q.patches_x = ceil_div(w, 8); q.patches_y = ceil_div(h, 8);
    q.npatch = B * q.patches_x * q.patches_y;
    const int split_blocks = (int)std::min<size_t>((npix * C / 4 + 127) / 128, (size_t)kNumSMs * 8);
    RAFT_TRY(launch(corr_prep_kernel, q.npatch + split_blocks, 128, 0, st, q));
  } else {                                   // deeper pyramids: generic pooling / split kernels, level by level
    RAFT_TRY(launch(split_plane_kernel, grid_for(npix * C), 256, 0, st, f1, C, 0, C, C, W.f1_hi, W.f1_lo, C, 0, npix, 1.0f));
    int lh = h, lw = w;
    const float* src = f2;
    for (int l = 0; l < levels; ++l) {
      if (l > 0) {
        const size_t total = (size_t)B * (lh / 2) * (lw / 2) * C;
        RAFT_TRY(launch(avgpool2x2_kernel, grid_for(total), 256, 0, st, src, W.f2_lvl[l], (size_t)B, lh, lw, C));
        src = W.f2_lvl[l];
        lh /= 2;
        lw /= 2;
      }
      const size_t np2 = (size_t)B * lh * lw;
      RAFT_TRY(launch(split_plane_kernel, grid_for(np2 * C), 256, 0, st, src, C, 0, C, C, W.f2_hi[l], W.f2_lo[l], C, 0, np2,
                      1.0f));
    }
  }

  CorrTcParams p;
  memset(&p, 0, sizeof(p));
  // A: fmap1 as a (B, 1, N, C) "image" -> 128 consecutive queries per tile
  RAFT_TRY(make_tmap_act2(&p.a_map, W.f1_hi, W.f1_lo, B, 1, N, C, 128, 1));
  p.levels = levels; p.B = B; p.N = N; p.chunks = C / kChunkK;
  p.mtiles_img = ceil_div(N, kTileM);
  const int mtiles = B * p.mtiles_img;
  int lh = h, lw = w;
  for (int l = 0; l < levels; ++l) {
    const int N2 = lh * lw;
    const int ntn = ceil_div(N2, kCorrBn);
    const int bn = round_up(ceil_div(N2, ntn), 16);
    // B: level-l features [B][N2][C] -> the batch index rides in the "tap" coordinate
    RAFT_TRY(make_tmap_wgt2(&p.b_map[l], W.f2_hi[l], W.f2_lo[l], B, N2, C, bn));
    p.out[l] = pyr[l];
    p.n2[l] = N2; p.bn[l] = bn;
    p.tile0[l + 1] = p.tile0[l] + mtiles * ntn;
    lh /= 2;
    lw /= 2;
  }
  p.corr_div = sqrtf((float)C);
  {
    int e = 0;
    const float m = frexpf(p.corr_div, &e);          // sqrt(C) = m * 2^e; m == 0.5 <=> exact power of two
    p.corr_mul = (m == 0.5f && p.corr_div * p.corr_div == (float)C) ? 1.0f / p.corr_div : 0.0f;
  }
  unsigned grid = 0;
  RAFT_TRY(persistent_grid<corr_tc_kernel>(kCorrSmemBytes, p.tile0[levels], &grid));
  return launch(corr_tc_kernel, grid, kTcThreads, kCorrSmemBytes, st, p);
}

// ------------------------------------------------------------------------------------------------
// Concurrent encode of an image pair (raft_b200_encode_pair)
// ------------------------------------------------------------------------------------------------
// Workspace: one encoder workspace per branch, then cnet's raw output (before the context split).
struct PairWs {
  void* enc[3];
  size_t enc_bytes;
  const __half *stem_hi, *stem_lo;           // image1's stem planes, built in branch A's workspace
  float* cnet_out;
  size_t total;
};
static PairWs pair_ws_layout(void* base, int variant, int N, int H, int W, int cnet_dim) {
  PairWs P;
  memset(&P, 0, sizeof(P));
  uint8_t* b8 = reinterpret_cast<uint8_t*>(base);
  P.enc_bytes = align_up(enc_ws_layout(nullptr, variant, N, H, W).total, 1024);
  for (int i = 0; i < 3; ++i) P.enc[i] = b8 + i * P.enc_bytes;
  const EncWs E = enc_ws_layout(P.enc[0], variant, N, H, W);
  P.stem_hi = E.Ih; P.stem_lo = E.Il;
  P.cnet_out = reinterpret_cast<float*>(b8 + 3 * P.enc_bytes);
  P.total = 3 * P.enc_bytes + (size_t)N * ceil_div(H, 8) * ceil_div(W, 8) * cnet_dim * sizeof(float);
  return P;
}

// The three side streams (two at the device's greatest priority for fnet, one at its least for cnet) and the fork / join
// events, created on first use per host thread and device -- never inside a call that is being captured, so that a
// captured call contains no stream or event creation.  Per thread, so that two threads never interleave their records
// and waits on the same events.
struct PairStreams { cudaStream_t s[3]; cudaEvent_t fork, stem, a, b, c; bool ready; };
static int pair_streams(cudaStream_t caller, PairStreams** out) {
  static thread_local PairStreams tab[64];
  int dev = 0;
  RAFT_CUDA_TRY(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64) return RAFT_ERR_UNSUPPORTED;
  PairStreams& ps = tab[dev];
  if (!ps.ready) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    RAFT_CUDA_TRY(cudaStreamIsCapturing(caller, &cs));
    if (cs != cudaStreamCaptureStatusNone) return RAFT_ERR_UNSUPPORTED;      // the first call must run eagerly
    int least = 0, greatest = 0;
    RAFT_CUDA_TRY(cudaDeviceGetStreamPriorityRange(&least, &greatest));
    for (int i = 0; i < 3; ++i)
      RAFT_CUDA_TRY(cudaStreamCreateWithPriority(&ps.s[i], cudaStreamNonBlocking, i < 2 ? greatest : least));
    for (cudaEvent_t* e : {&ps.fork, &ps.stem, &ps.a, &ps.b, &ps.c})
      RAFT_CUDA_TRY(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    ps.ready = true;
  }
  *out = &ps;
  return RAFT_OK;
}

// Per-pair setup shared by the update_* entry points and the loop: zero the fp16 planes (their
// padded channels must hold exact zeros), stage inp and the hidden state in operand format.
static int update_begin(const UpdateCtx& c, const float* h, const float* inp) {
  const Workspace& W = c.W;
  const VariantDims d = variant_dims(c.variant);
  const size_t npix = (size_t)c.B * c.h * c.w;
  if (c.precision == RAFT_PREC_F16X2) {
    RAFT_CUDA_TRY(cudaMemsetAsync(W.f16_begin, 0, W.f16_bytes, c.stream));
    RAFT_TRY(launch(split_plane_kernel, grid_for(npix * d.ctx), 256, 0, c.stream, inp, d.ctx, 0, d.ctx, d.ctx, W.x_hi, W.x_lo,
                    d.s_x, 0, npix, 1.0f));
    return launch(split_plane_kernel, grid_for(npix * d.hid), 256, 0, c.stream, h, d.hid, 0, d.hid, d.hid, W.h_hi, W.h_lo,
                  d.s_h, 0, npix, 1.0f);
  }
  RAFT_CUDA_TRY(cudaMemsetAsync(W.x, 0, npix * d.c_x * sizeof(float), c.stream));
  return launch(copy_channels_kernel, grid_for(npix * d.ctx), 256, 0, c.stream, inp, d.ctx, 0, W.x, d.c_x, 0, d.ctx, npix);
}

static int make_ctx(UpdateCtx& c, int variant, const void* prepared, int B, int h, int w, void* ws, size_t ws_bytes,
                    int precision, void* stream) {
  RAFT_TRY(check_variant(variant));
  RAFT_TRY(check_precision(precision));
  if (!prepared || !ws) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_dims(B, h, w));
  c.variant = variant; c.precision = precision; c.B = B; c.h = h; c.w = w;
  c.prepared = reinterpret_cast<const uint8_t*>(prepared);
  c.PL = prepared_layout(variant, precision);
  c.W = workspace_layout(ws, variant, B, h, w, precision);
  if (c.W.total > ws_bytes) return RAFT_ERR_WORKSPACE;
  c.stream = reinterpret_cast<cudaStream_t>(stream);
  c.plan = nullptr;
  c.fim_ready = false;
  return 0;
}

// One update_mega_kernel launch for all tensor-core layers of an update-block application (default), or one launch per
// layer (RAFT_B200_MEGA=0: A/B timing and bisecting).
static bool mega_enabled() {
  static const int v = [] { const char* e = getenv("RAFT_B200_MEGA"); return e ? atoi(e) : 1; }();
  return v != 0;
}
static int update_block_tc(UpdateCtx& c, float* h, float* delta, float* mask, float* adv_coords) {
  MegaPlan plan;
  c.plan = mega_enabled() ? &plan : nullptr;
  const int st = update_core_tc(c, h, delta, mask, adv_coords);
  c.plan = nullptr;
  RAFT_TRY(st);
  if (!mega_enabled()) return 0;
  return mega_launch(plan, c.W.mega_flags, c.W.mega_flag_words, true, c.stream);
}

static int update_once(int variant, const void* prepared, const float* net, const float* inp, const float* corr,
                       const float* flow, float* net_out, float* mask, float* delta, int B, int h, int w, void* ws,
                       size_t ws_bytes, int precision, void* stream) {
  if (!net || !inp || !corr || !flow || !net_out || !delta) return RAFT_ERR_BAD_ARG;
  UpdateCtx c;
  RAFT_TRY(make_ctx(c, variant, prepared, B, h, w, ws, ws_bytes, precision, stream));
  const VariantDims d = variant_dims(variant);
  const size_t npix = (size_t)B * h * w;
  if (net_out != net)
    RAFT_CUDA_TRY(cudaMemcpyAsync(net_out, net, npix * d.hid * sizeof(float), cudaMemcpyDeviceToDevice, c.stream));
  RAFT_CUDA_TRY(cudaMemcpyAsync(c.W.flow, flow, npix * 2 * sizeof(float), cudaMemcpyDeviceToDevice, c.stream));
  RAFT_TRY(update_begin(c, net_out, inp));
  if (precision == RAFT_PREC_F16X2) {
    RAFT_TRY(launch(split_plane_kernel, grid_for(npix * d.s_corr), 256, 0, c.stream, corr, d.corr_ch, 0, d.corr_ch, d.s_corr,
                    c.W.corr_hi, c.W.corr_lo, d.s_corr, 0, npix, 1.0f));
    return update_block_tc(c, net_out, delta, mask, nullptr);
  }
  RAFT_CUDA_TRY(cudaMemcpyAsync(c.W.corr, corr, npix * d.corr_ch * sizeof(float), cudaMemcpyDeviceToDevice, c.stream));
  return update_core_fp32(c, net_out, delta, mask);
}

// im_flow != null (iteration loop, tensor-core path): the convf1 im2col planes im_hi / im_lo are produced too -- by the
// window kernel itself when it runs, else by flow_im2col_kernel.
static int lookup_launch(const float* const pyr[], const float* coords, int B, int h, int w, int levels, int radius,
                         float* out, int out_stride, __half* out_hi, __half* out_lo, int h_stride, int h_pad,
                         cudaStream_t st, const float* im_flow = nullptr, __half* im_hi = nullptr, __half* im_lo = nullptr) {
  LookupParams p;
  memset(&p, 0, sizeof(p));
  int lh = h, lw = w;
  for (int l = 0; l < levels; ++l) {
    if (lh < 1 || lw < 1) return RAFT_ERR_BAD_SHAPE;
    p.pyr[l] = pyr[l];
    p.lh[l] = lh;
    p.lw[l] = lw;
    lh /= 2;
    lw /= 2;
  }
  p.coords = coords;
  p.out = out; p.out_stride = out_stride;
  p.out_hi = out_hi; p.out_lo = out_lo; p.h_stride = h_stride; p.h_pad = h_pad;
  p.nq = B * h * w; p.levels = levels; p.radius = radius;
  p.im_flow = im_flow; p.im_hi = im_hi; p.im_lo = im_lo; p.im_B = B; p.im_h = h; p.im_w = w;
  const size_t nwork = (size_t)p.nq * levels;
  static const int gather = [] { const char* e = getenv("RAFT_B200_LOOKUP_GATHER"); return e ? atoi(e) : 0; }();   // A/B: force the generic kernel
  const LookupKernel win = gather ? nullptr : lookup_win_kernel(p, levels, radius);   // the model's (radius, levels)
  if (win) return launch(win, grid_for(nwork * 32, 256, kNumSMs * 4), 256, 0, st, p);   // 4 resident blocks per SM: one wave
  RAFT_TRY(launch(corr_lookup_kernel, grid_for(nwork * 32, 256, kNumSMs * 32), 256, 0, st, p));
  if (!im_flow) return RAFT_OK;
  return launch(flow_im2col_kernel, grid_for((size_t)p.nq * 128), 256, 0, st, im_flow, B, h, w, im_hi, im_lo);
}

}  // namespace raft

using namespace raft;

// =================================================================================================
extern "C" {

const char* raft_b200_strerror(int status) {
  switch (status) {
    case RAFT_OK: return "ok";
    case RAFT_ERR_BAD_ARG: return "bad argument (null pointer or unknown enum)";
    case RAFT_ERR_BAD_SHAPE: return "bad shape";
    case RAFT_ERR_WORKSPACE: return "workspace or prepared-weights buffer too small";
    case RAFT_ERR_NO_DEVICE: return "no sm_90 CUDA device";
    case RAFT_ERR_DRIVER: return "cuTensorMapEncodeTiled unavailable or failed";
    case RAFT_ERR_UNSUPPORTED: return "unsupported configuration";
    default: return status > 0 ? cudaGetErrorString((cudaError_t)status) : "unknown raft_status";
  }
}

int raft_b200_abi_version(void) { return RAFT_B200_ABI_VERSION; }

int raft_b200_device_ok(int device) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || device < 0 || device >= n) {
    (void)cudaGetLastError();
    return RAFT_ERR_NO_DEVICE;
  }
  int major = 0, minor = 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device) != cudaSuccess ||
      cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device) != cudaSuccess)
    return RAFT_ERR_NO_DEVICE;
  return major == 9 && minor == 0 ? RAFT_OK : RAFT_ERR_NO_DEVICE;       // the library holds sm_90a code only
}

void raft_b200_profile_loop(int enable) { g_prof.on = enable != 0; g_prof.n = 0; }
int raft_b200_profile_read(float* lookup_ms, float* update_ms, int* iterations) {
  if (!lookup_ms || !update_ms || !iterations) return RAFT_ERR_BAD_ARG;
  *lookup_ms = 0.f; *update_ms = 0.f; *iterations = g_prof.n;
  for (int i = 0; i < g_prof.n; ++i) {
    float a = 0.f, b = 0.f;
    RAFT_CUDA_TRY(cudaEventSynchronize(g_prof.ev[i][2]));
    RAFT_CUDA_TRY(cudaEventElapsedTime(&a, g_prof.ev[i][0], g_prof.ev[i][1]));
    RAFT_CUDA_TRY(cudaEventElapsedTime(&b, g_prof.ev[i][1], g_prof.ev[i][2]));
    *lookup_ms += a;
    *update_ms += b;
  }
  return RAFT_OK;
}

long long raft_b200_launch_count(void) { return g_launches; }
void raft_b200_launch_count_reset(void) { g_launches = 0; }

int raft_b200_corr_pyramid_sizes(int B, int h, int w, int levels, size_t bytes_per_level[]) {
  if (!bytes_per_level || levels < 1 || levels > RAFT_MAX_LEVELS) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_dims(B, h, w));
  int lh = h, lw = w;
  for (int l = 0; l < levels; ++l) {
    if (lh < 1 || lw < 1) return RAFT_ERR_BAD_SHAPE;
    bytes_per_level[l] = (size_t)B * h * w * lh * lw * sizeof(float);
    lh /= 2;
    lw /= 2;
  }
  return RAFT_OK;
}

int raft_b200_corr_workspace_bytes(int B, int h, int w, int C, int levels, int precision, size_t* bytes) {
  if (!bytes || levels < 1 || levels > RAFT_MAX_LEVELS) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_dims(B, h, w));
  if (C < 1) return RAFT_ERR_BAD_SHAPE;
  *bytes = corr_ws_layout(nullptr, B, h, w, C, levels, precision).total + 1024;
  return RAFT_OK;
}

int raft_b200_corr_pyramid_build(const float* fmap1, const float* fmap2, int B, int h, int w, int C, int levels,
                                 float* const pyr[], void* workspace, size_t workspace_bytes, int precision,
                                 void* stream) {
  if (!fmap1 || !fmap2 || !pyr || levels < 1 || levels > RAFT_MAX_LEVELS) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_dims(B, h, w));
  if (C < 1 || (h >> (levels - 1)) < 1 || (w >> (levels - 1)) < 1) return RAFT_ERR_BAD_SHAPE;
  for (int l = 0; l < levels; ++l)
    if (!pyr[l]) return RAFT_ERR_BAD_ARG;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (precision == RAFT_PREC_FP32) return corr_build_fp32(fmap1, fmap2, B, h, w, C, levels, pyr, st);
  if (precision != RAFT_PREC_F16X2) return RAFT_ERR_BAD_ARG;
  if (!workspace || corr_ws_layout(nullptr, B, h, w, C, levels, precision).total > workspace_bytes)
    return RAFT_ERR_WORKSPACE;
  return corr_build_tc(fmap1, fmap2, B, h, w, C, levels, pyr, workspace, st);
}

int raft_b200_corr_lookup(const float* const pyr[], const float* coords, int B, int h, int w, int levels, int radius,
                          float* out, int out_stride, void* stream) {
  if (!pyr || !coords || !out || levels < 1 || levels > RAFT_MAX_LEVELS || radius < 0) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_dims(B, h, w));
  const int side = 2 * radius + 1;
  if (out_stride < levels * side * side) return RAFT_ERR_BAD_SHAPE;
  return lookup_launch(pyr, coords, B, h, w, levels, radius, out, out_stride, nullptr, nullptr, 0, 0,
                       reinterpret_cast<cudaStream_t>(stream));
}

int raft_b200_corr_lookup_backward(const float* const pyr[], const float* coords, const float* grad_out, int B, int h, int w,
                                   int levels, int radius, float* grad_coords, float* const grad_pyr[], void* stream) {
  if (!pyr || !coords || !grad_out || !grad_coords || !grad_pyr || levels < 1 || levels > RAFT_MAX_LEVELS || radius < 0)
    return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_dims(B, h, w));
  LookupBwdParams p;
  memset(&p, 0, sizeof(p));
  int lh = h, lw = w;
  for (int l = 0; l < levels; ++l) {
    if (lh < 1 || lw < 1) return RAFT_ERR_BAD_SHAPE;
    if (!pyr[l] || !grad_pyr[l]) return RAFT_ERR_BAD_ARG;
    p.pyr[l] = pyr[l]; p.gpyr[l] = grad_pyr[l]; p.lh[l] = lh; p.lw[l] = lw;
    lh /= 2;
    lw /= 2;
  }
  const int side = 2 * radius + 1;
  p.coords = coords; p.gout = grad_out; p.gout_stride = levels * side * side; p.gcoords = grad_coords;
  p.nq = B * h * w; p.levels = levels; p.radius = radius;
  const int qpb = lookup_bwd_queries_per_block(levels);
  return launch(corr_lookup_bwd_kernel, grid_for((size_t)p.nq, qpb, kNumSMs * 32), 32 * levels * qpb, 0,
                reinterpret_cast<cudaStream_t>(stream), p);
}

int raft_b200_sumsq(const float* g, size_t n, float* partials, size_t npartials, float* out, void* stream) {
  if (!g || !partials || !out || npartials < 1) return RAFT_ERR_BAD_ARG;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int blocks = (int)std::min<size_t>(std::min<size_t>(npartials, (size_t)kNumSMs * 4), (n + 255) / 256);
  if (blocks < 1) blocks = 1;
  RAFT_TRY(launch(sumsq_partial_kernel, blocks, 256, 0, st, g, n, partials));
  return launch(sumsq_final_kernel, 1, 256, 0, st, partials, blocks, out);
}

int raft_b200_adamw_step(float* param, const float* grad, float* m, float* v, size_t n, const float* sumsq, float clip_norm,
                         float lr_t, float beta1, float beta2, float epsilon, float weight_decay, void* stream) {
  if (!param || !grad || !m || !v || (clip_norm > 0.0f && !sumsq)) return RAFT_ERR_BAD_ARG;
  return launch(adamw_kernel, grid_for(n), 256, 0, reinterpret_cast<cudaStream_t>(stream), param, grad, m, v, n, sumsq,
                clip_norm, lr_t, beta1, beta2, epsilon, weight_decay);
}

int raft_b200_bilinear_sampler(const float* image, const float* coords, int M, int H, int W, int P, float* out,
                               void* stream) {
  if (!image || !coords || !out) return RAFT_ERR_BAD_ARG;
  if (M < 1 || H < 1 || W < 1 || P < 1) return RAFT_ERR_BAD_SHAPE;
  return launch(bilinear_sampler_kernel, grid_for((size_t)M * P), 256, 0, reinterpret_cast<cudaStream_t>(stream), image,
                coords, M, H, W, P, out);
}

int raft_b200_coords_grid(int B, int h, int w, float* out, void* stream) {
  if (!out) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_dims(B, h, w));
  return launch(coords_grid_kernel, grid_for((size_t)B * h * w), 256, 0, reinterpret_cast<cudaStream_t>(stream), out, B, h, w);
}

int raft_b200_forward_interpolate(const float* flow, int B, int h, int w, float* out, void* stream) {
  if (!flow || !out) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_dims(B, h, w));
  if ((size_t)h * w > (size_t)INT_MAX - kFiChunk) return RAFT_ERR_BAD_SHAPE;     // pixel indices are int
  dim3 grid((unsigned)ceil_div(h * w, kFiThreads), (unsigned)std::min(B, 65535));
  return launch(forward_interpolate_kernel, grid, kFiThreads, 0, reinterpret_cast<cudaStream_t>(stream), flow, out, B, h, w);
}

int raft_b200_coords_init(const float* flow_init, int B, int h, int w, float* coords1, void* stream) {
  if (!flow_init || !coords1) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_dims(B, h, w));
  return launch(coords_init_kernel, grid_for((size_t)B * h * w), 256, 0, reinterpret_cast<cudaStream_t>(stream), flow_init,
                coords1, B, h, w);
}

int raft_b200_fb_occlusion(const float* flow_fw, const float* flow_bw, int B, int H, int W, float alpha1, float alpha2,
                           uint8_t* occ_fw, uint8_t* occ_bw, void* stream) {
  if (!flow_fw || !flow_bw || !occ_fw || !occ_bw) return RAFT_ERR_BAD_ARG;
  if (!(alpha1 >= 0.0f && alpha1 <= FLT_MAX) || !(alpha2 >= 0.0f && alpha2 <= FLT_MAX)) return RAFT_ERR_BAD_ARG;
  if ((reinterpret_cast<uintptr_t>(flow_fw) | reinterpret_cast<uintptr_t>(flow_bw)) % sizeof(float2)) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_dims(B, H, W));
  return launch(fb_occlusion_kernel, grid_for(2 * (size_t)B * H * W), 256, 0, reinterpret_cast<cudaStream_t>(stream),
                reinterpret_cast<const float2*>(flow_fw), reinterpret_cast<const float2*>(flow_bw), B, H, W, alpha1, alpha2,
                occ_fw, occ_bw);
}

int raft_b200_census(const float* images, int B, int H, int W, float* out, void* stream) {
  if (!images || !out || reinterpret_cast<uintptr_t>(out) % 16) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_dims(B, H, W));
  return launch(census_kernel, grid_for((size_t)B * H * W), 256, 0, reinterpret_cast<cudaStream_t>(stream), images, B, H,
                W, out);
}

int raft_b200_unsup_loss_norm(const float* census_t, const float* census_s, const float* image_t, const uint8_t* occ,
                              const float* flows, int n, int B, int H, int W, float census_weight,
                              float smoothness_weight, float edge_weight, float gamma, double* partials,
                              size_t npartials, double* sums, float* grad, const double* census_norm, void* stream) {
  if (!census_t || !census_s || !image_t || !occ || !flows || !partials || !sums || !grad || npartials < 4)
    return RAFT_ERR_BAD_ARG;
  for (float v : {census_weight, smoothness_weight, edge_weight, gamma})
    if (!(v >= 0.0f && v <= FLT_MAX)) return RAFT_ERR_BAD_ARG;
  if ((reinterpret_cast<uintptr_t>(census_t) | reinterpret_cast<uintptr_t>(census_s)) % 16 ||
      (reinterpret_cast<uintptr_t>(flows) | reinterpret_cast<uintptr_t>(grad)) % sizeof(float2) ||
      (reinterpret_cast<uintptr_t>(partials) | reinterpret_cast<uintptr_t>(sums) |
       reinterpret_cast<uintptr_t>(census_norm)) % sizeof(double))
    return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_dims(B, H, W));
  if (n < 1 || H < 2 || W < 2) return RAFT_ERR_BAD_SHAPE;
  const size_t npix = (size_t)B * H * W;
  const int blocks = (int)std::min<size_t>(std::min<size_t>(npartials / 4, (npix + kUnsupThreads - 1) / kUnsupThreads),
                                           (size_t)kUnsupMaxBlocks);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  RAFT_TRY(launch(unsup_mask_count_kernel, blocks, kUnsupThreads, 0, st, occ, B, H, W, partials));
  UnsupParams p;
  p.ct = census_t; p.cs = census_s; p.img = image_t; p.occ = occ; p.census_norm = census_norm;
  p.flows = reinterpret_cast<const float2*>(flows); p.grad = reinterpret_cast<float2*>(grad); p.partials = partials;
  p.n = n; p.B = B; p.H = H; p.W = W;
  p.gamma = gamma; p.edge = edge_weight; p.census_half = 0.5f * census_weight;
  const double n_h = (double)B * H * (W - 1), n_v = (double)B * (H - 1) * W;
  p.sh_scale = (float)(0.25 * smoothness_weight / n_h);
  p.sv_scale = (float)(0.25 * smoothness_weight / n_v);
  RAFT_TRY(launch(unsup_loss_partial_kernel, blocks, kUnsupThreads, 0, st, p));
  return launch(unsup_loss_final_kernel, 1, kUnsupThreads, 0, st, partials, blocks, n_h, n_v, 0.5 * census_weight,
                0.5 * smoothness_weight, census_norm, sums);
}

int raft_b200_unsup_loss(const float* census_t, const float* census_s, const float* image_t, const uint8_t* occ,
                         const float* flows, int n, int B, int H, int W, float census_weight, float smoothness_weight,
                         float edge_weight, float gamma, double* partials, size_t npartials, double* sums, float* grad,
                         void* stream) {
  return raft_b200_unsup_loss_norm(census_t, census_s, image_t, occ, flows, n, B, H, W, census_weight,
                                   smoothness_weight, edge_weight, gamma, partials, npartials, sums, grad, nullptr,
                                   stream);
}

// Checks every sample of an augmentation call and lays out its workspace: fills (fill) or verifies each ws_offset.
static int augment_layout(raft_augment_sample* samples, const raft_augment_sample* check, int B, int sparse,
                          size_t* bytes, int* max_src, int* max_map, int* max_out) {
  if ((!samples && !check) || !bytes || (sparse != 0 && sparse != 1)) return RAFT_ERR_BAD_ARG;
  if (B < 1 || B > 65535) return RAFT_ERR_BAD_SHAPE;
  size_t off = 0;
  *max_src = *max_map = *max_out = 1;
  for (int b = 0; b < B; ++b) {
    const raft_augment_sample& s = check ? check[b] : samples[b];
    if (!s.img1 || !s.img2 || !s.flow || !s.out_img1 || !s.out_img2 || !s.out_flow || !s.out_valid) return RAFT_ERR_BAD_ARG;
    if ((sparse && !s.valid) || (sparse && s.vflip) || s.n_rects < 0 || s.n_rects > 2) return RAFT_ERR_BAD_ARG;
    for (int r = 0; r < s.n_rects; ++r)
      for (int k = 0; k < 4; ++k)
        if (s.rect[r][k] < 0) return RAFT_ERR_BAD_ARG;
    if (s.H < 1 || s.W < 1 || s.crop_h < 1 || s.crop_w < 1) return RAFT_ERR_BAD_SHAPE;
    if ((size_t)s.H * s.W * 3 > (size_t)INT_MAX) return RAFT_ERR_BAD_SHAPE;
    int rh = s.H, rw = s.W;
    if (s.spatial) {
      if (!(s.scale_x > 0.0 && s.scale_x <= 64.0 && s.scale_y > 0.0 && s.scale_y <= 64.0)) return RAFT_ERR_BAD_ARG;
      rh = aug_resized(s.H, s.scale_y);
      rw = aug_resized(s.W, s.scale_x);
      if (rh < 1 || rw < 1 || (size_t)rh * rw > (size_t)INT_MAX) return RAFT_ERR_BAD_SHAPE;
    }
    if (s.y0 < 0 || s.x0 < 0 || s.y0 > rh - s.crop_h || s.x0 > rw - s.crop_w) return RAFT_ERR_BAD_SHAPE;
    const bool map = sparse && s.spatial;
    if (check ? s.ws_offset != off : false) return RAFT_ERR_BAD_ARG;
    if (!check) samples[b].ws_offset = off;
    off += aug_layout(s.H, s.W, rh, rw, map).total;
    *max_src = std::max(*max_src, 2 * s.H * s.W);
    if (map) *max_map = std::max(*max_map, rh * rw);
    *max_out = std::max(*max_out, s.crop_h * s.crop_w);
  }
  *bytes = off;
  return RAFT_OK;
}

int raft_b200_augment_workspace_bytes(raft_augment_sample* samples, int B, int sparse, size_t* bytes) {
  int a, b, c;
  return augment_layout(samples, nullptr, B, sparse, bytes, &a, &b, &c);
}

static int augment_run(const raft_augment_sample* host, const raft_augment_sample* dev, int B, int sparse, void* workspace,
                       size_t workspace_bytes, void* stream) {
  size_t need;
  int max_src, max_map, max_out;
  if (!host) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(augment_layout(nullptr, host, B, sparse, &need, &max_src, &max_map, &max_out));
  if (!dev || !workspace || reinterpret_cast<uintptr_t>(workspace) % 256) return RAFT_ERR_BAD_ARG;
  if (workspace_bytes < need) return RAFT_ERR_WORKSPACE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  auto blocks = [](int n) { return (unsigned)std::min(ceil_div(n, kAugThreads), 4096); };
  RAFT_TRY(launch(augment_init_kernel, dim3(blocks(max_map), B), kAugThreads, 0, st, dev, ws, sparse));
  RAFT_TRY(launch(augment_colour_kernel, dim3(blocks(max_src), B), kAugThreads, 0, st, dev, ws));
  if (sparse) RAFT_TRY(launch(augment_scatter_kernel, dim3(blocks(max_src / 2), B), kAugThreads, 0, st, dev, ws));
  return launch(augment_gather_kernel, dim3(blocks(max_out), B), kAugThreads, 0, st, dev, ws, sparse);
}

int raft_b200_augment_dense(const raft_augment_sample* samples_host, const raft_augment_sample* samples_dev, int B,
                            void* workspace, size_t workspace_bytes, void* stream) {
  return augment_run(samples_host, samples_dev, B, 0, workspace, workspace_bytes, stream);
}

int raft_b200_augment_sparse(const raft_augment_sample* samples_host, const raft_augment_sample* samples_dev, int B,
                             void* workspace, size_t workspace_bytes, void* stream) {
  return augment_run(samples_host, samples_dev, B, 1, workspace, workspace_bytes, stream);
}

int raft_b200_flow_to_image(const float* u, const float* v, int stride, int B, int H, int W, int clip, float clip_flow,
                            int normalize, const float* rad_max, int bgr, uint8_t* image, unsigned int* work,
                            int* status, void* stream) {
  const bool reduce = normalize && !rad_max;
  if (!u || !v || !image || !status || (reduce && !work) || (stride != 1 && stride != 2)) return RAFT_ERR_BAD_ARG;
  if (clip && !(clip_flow >= 0.0f && clip_flow <= FLT_MAX)) return RAFT_ERR_BAD_ARG;
  if (reinterpret_cast<uintptr_t>(image) % 4) return RAFT_ERR_BAD_ARG;
  if (B < 1 || B > 65535 || H < 1 || W < 1 || (size_t)H * W > (size_t)INT_MAX) return RAFT_ERR_BAD_SHAPE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int hw = H * W;
  RAFT_CUDA_TRY(cudaMemsetAsync(status, 0, (size_t)B * sizeof(int), st));
  if (reduce) {
    RAFT_CUDA_TRY(cudaMemsetAsync(work, 0, (size_t)B * sizeof(unsigned), st));
    const unsigned gx = (unsigned)std::min(ceil_div(hw, kVizThreads * 8), std::max(1, kNumSMs * 8 / B));
    RAFT_TRY(launch(flow_radmax_kernel, dim3(gx, B), kVizThreads, 0, st, u, v, stride, hw, clip, clip_flow, work));
  }
  VizParams p;
  p.u = u; p.v = v; p.stride = stride; p.hw = hw; p.npix = (size_t)B * hw;
  p.clip = clip != 0; p.clip_flow = clip_flow; p.normalize = normalize != 0; p.rad_max = rad_max; p.work = work;
  p.bgr = bgr != 0; p.out = image; p.status = status;
  const size_t nblk = (p.npix + kVizPixPerBlock - 1) / kVizPixPerBlock;
  return launch(flow_colour_kernel, dim3((unsigned)nblk), kVizThreads, 0, st, p);
}

int raft_b200_png16_flow_decode(const uint8_t* data, size_t data_bytes, const raft_png16_image* images_host,
                                const raft_png16_image* images_dev, int n, int* status, void* stream) {
  if (!data || !images_host || !images_dev || !status) return RAFT_ERR_BAD_ARG;
  if (n < 1) return RAFT_ERR_BAD_SHAPE;
  int max_w = 1;
  for (int i = 0; i < n; ++i) {
    const raft_png16_image& im = images_host[i];
    if (!im.flow || !im.valid || reinterpret_cast<uintptr_t>(im.flow) % sizeof(float2)) return RAFT_ERR_BAD_ARG;
    if (im.h < 1 || im.w < 1 || im.w > kPngMaxWidth || (size_t)im.h * im.w > (size_t)INT_MAX) return RAFT_ERR_BAD_SHAPE;
    const size_t rows = (size_t)im.h * (1 + 6 * (size_t)im.w);
    if (im.offset > data_bytes || rows > data_bytes - im.offset) return RAFT_ERR_BAD_SHAPE;
    max_w = std::max(max_w, im.w);
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  PngParams p;
  p.data = data; p.images = images_dev; p.status = status; p.row_bytes = round_up(6 * max_w, 16);
  const size_t smem = 2 * (size_t)p.row_bytes;
  RAFT_CUDA_TRY(cudaFuncSetAttribute(png16_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  RAFT_CUDA_TRY(cudaMemsetAsync(status, 0, (size_t)n * sizeof(int), st));
  return launch(png16_decode_kernel, dim3((unsigned)n), kPngThreads, smem, st, p);
}

int raft_b200_flow_metrics_workspace_bytes(int B, int H, int W, size_t* bytes) {
  if (!bytes) return RAFT_ERR_BAD_ARG;
  if (B < 1 || B > 65535 || H < 1 || W < 1 || (size_t)H * W > (size_t)INT_MAX - kMetChunk) return RAFT_ERR_BAD_SHAPE;
  *bytes = (size_t)B * ceil_div(H * W, kMetChunk) * sizeof(MetricPartial);
  return RAFT_OK;
}

int raft_b200_flow_metrics(const float* pred, const float* gt, const float* valid, int B, int H, int W, int use_max_flow,
                           float max_flow, void* workspace, size_t workspace_bytes, long long* counts, double* sums,
                           void* stream) {
  if (!pred || !gt || !workspace || !counts || !sums) return RAFT_ERR_BAD_ARG;
  if ((reinterpret_cast<uintptr_t>(pred) | reinterpret_cast<uintptr_t>(gt)) % sizeof(float2) ||
      reinterpret_cast<uintptr_t>(workspace) % alignof(MetricPartial) || reinterpret_cast<uintptr_t>(counts) % 8 ||
      reinterpret_cast<uintptr_t>(sums) % 8)
    return RAFT_ERR_BAD_ARG;
  size_t need;
  RAFT_TRY(raft_b200_flow_metrics_workspace_bytes(B, H, W, &need));
  if (workspace_bytes < need) return RAFT_ERR_WORKSPACE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int hw = H * W, nchunk = ceil_div(hw, kMetChunk);
  MetricPartial* part = reinterpret_cast<MetricPartial*>(workspace);
  RAFT_TRY(launch(flow_metrics_partial_kernel, dim3((unsigned)nchunk, (unsigned)B), kMetThreads, 0, st,
                  reinterpret_cast<const float2*>(pred), reinterpret_cast<const float2*>(gt), valid, hw, use_max_flow != 0,
                  max_flow, part));
  return launch(flow_metrics_final_kernel, dim3((unsigned)B), kMetThreads, 0, st, part, nchunk, counts, sums);
}

int raft_b200_pad_batch(const raft_pad_plane* planes_host, const raft_pad_plane* planes_dev, int n, void* stream) {
  if (!planes_host || !planes_dev) return RAFT_ERR_BAD_ARG;
  if (n < 1 || n > 65535) return RAFT_ERR_BAD_SHAPE;
  int max_h = 1;
  for (int i = 0; i < n; ++i) {
    const raft_pad_plane& p = planes_host[i];
    if (!p.src || !p.dst || (p.dtype != RAFT_PAD_U8 && p.dtype != RAFT_PAD_F32)) return RAFT_ERR_BAD_ARG;
    if (p.mode != RAFT_PAD_ZERO && p.mode != RAFT_PAD_REPLICATE) return RAFT_ERR_BAD_ARG;
    if (p.dtype == RAFT_PAD_F32 &&
        (reinterpret_cast<uintptr_t>(p.src) | reinterpret_cast<uintptr_t>(p.dst)) % sizeof(float))
      return RAFT_ERR_BAD_ARG;
    if (p.h < 1 || p.w < 1 || p.c < 1 || p.H < 1 || p.W < 1) return RAFT_ERR_BAD_SHAPE;
    if ((size_t)p.h * p.w * p.c > (size_t)INT_MAX || (size_t)p.H * p.W * p.c > (size_t)INT_MAX) return RAFT_ERR_BAD_SHAPE;
    max_h = std::max(max_h, p.H);
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return launch(pad_planes_kernel, dim3((unsigned)std::min(max_h, kPadMaxRowBlocks), (unsigned)n), kPadThreads, 0, st,
                planes_dev);
}

int raft_b200_update_prepared_bytes(int variant, int corr_channels, int precision, size_t* bytes) {
  if (!bytes) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_variant(variant));
  RAFT_TRY(check_precision(precision));
  if (corr_channels != variant_dims(variant).corr_ch) return RAFT_ERR_BAD_SHAPE;
  *bytes = prepared_layout(variant, precision).total;
  return RAFT_OK;
}

int raft_b200_update_prepare(int variant, const void* weights, void* prepared, size_t prepared_bytes, int precision,
                             void* stream) {
  if (!weights || !prepared) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_variant(variant));
  RAFT_TRY(check_precision(precision));
  const PreparedLayout L = prepared_layout(variant, precision);
  if (L.total > prepared_bytes) return RAFT_ERR_WORKSPACE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const raft_conv* convs = reinterpret_cast<const raft_conv*>(weights);   // both structs are arrays of raft_conv
  const ConvDim* cd = conv_dims(variant);
  uint8_t* base = reinterpret_cast<uint8_t*>(prepared);
  for (int i = 0; i < n_convs(variant); ++i) {
    const raft_conv& cv = convs[i];
    if (!cv.kernel || !cv.bias) return RAFT_ERR_BAD_ARG;
    if (cv.kh != cd[i].kh || cv.kw != cd[i].kw || cv.cin != cd[i].cin || cv.cout != cd[i].cout) return RAFT_ERR_BAD_SHAPE;
  }
  RAFT_CUDA_TRY(cudaMemsetAsync(base, 0, L.total, st));
  for (int i = 0; i < n_convs(variant); ++i) {
    const size_t nw = (size_t)cd[i].kh * cd[i].kw * cd[i].cin * cd[i].cout;
    RAFT_CUDA_TRY(cudaMemcpyAsync(base + L.raw_w[i], convs[i].kernel, nw * sizeof(float), cudaMemcpyDeviceToDevice, st));
    RAFT_CUDA_TRY(cudaMemcpyAsync(base + L.raw_b[i], convs[i].bias, cd[i].cout * sizeof(float), cudaMemcpyDeviceToDevice, st));
  }
  if (precision == RAFT_PREC_F16X2) {
    const TcLayer* tl = tc_layers(variant);
    for (int li = 0; li < n_tc_layers(variant); ++li) {
      const TcLayer& T = tl[li];
      const raft_conv* src[2] = {&convs[T.src[0]], T.nsrc > 1 ? &convs[T.src[1]] : nullptr};
      RAFT_TRY(tc_pack_weights(base, L.tc[li], src, T.nsrc, T.cin_map.nrange ? &T.cin_map : nullptr, T.flatten != 0, st));
    }
  }
  return raft_launch_status();
}

int raft_b200_update_workspace_bytes(int variant, int B, int h, int w, int precision, size_t* bytes) {
  if (!bytes) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_variant(variant));
  RAFT_TRY(check_precision(precision));
  RAFT_TRY(check_dims(B, h, w));
  *bytes = workspace_layout(nullptr, variant, B, h, w, precision).total;
  return RAFT_OK;
}

int raft_b200_update_basic(const void* prepared, const float* net, const float* inp, const float* corr,
                           const float* flow, float* net_out, float* mask_or_null, float* delta_flow, int B, int h,
                           int w, void* workspace, size_t workspace_bytes, int precision, void* stream) {
  return update_once(RAFT_VARIANT_BASIC, prepared, net, inp, corr, flow, net_out, mask_or_null, delta_flow, B, h, w,
                     workspace, workspace_bytes, precision, stream);
}

int raft_b200_update_small(const void* prepared, const float* net, const float* inp, const float* corr,
                           const float* flow, float* net_out, float* delta_flow, int B, int h, int w, void* workspace,
                           size_t workspace_bytes, int precision, void* stream) {
  return update_once(RAFT_VARIANT_SMALL, prepared, net, inp, corr, flow, net_out, nullptr, delta_flow, B, h, w,
                     workspace, workspace_bytes, precision, stream);
}

int raft_b200_upsample_convex(const float* flow, const float* mask, int B, int h, int w, float* out, void* stream) {
  if (!flow || !mask || !out) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_dims(B, h, w));
  const size_t npix = (size_t)B * h * w;
  return launch(upsample_convex_kernel, grid_for(npix, 4, kNumSMs * 32), 256, 0, reinterpret_cast<cudaStream_t>(stream), flow,
                mask, B, h, w, out);
}

int raft_b200_upflow8(const float* flow, int B, int h, int w, float* out, void* stream) {
  if (!flow || !out) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_dims(B, h, w));
  return launch(upflow8_kernel, grid_for((size_t)B * h * w * 64), 256, 0, reinterpret_cast<cudaStream_t>(stream), flow, B, h,
                w, out);
}

int raft_b200_upflow8_backward(const float* grad_up, int B, int h, int w, float* grad_flow, void* stream) {
  if (!grad_up || !grad_flow || (reinterpret_cast<uintptr_t>(grad_up) & 7) || (reinterpret_cast<uintptr_t>(grad_flow) & 7))
    return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_dims(B, h, w));
  return launch(upflow8_bwd_kernel, grid_for((size_t)B * h * w, 128), 128, 0, reinterpret_cast<cudaStream_t>(stream),
                grad_up, B, h, w, grad_flow);
}

int raft_b200_encoder_prepared_bytes(int variant, int out_dim, size_t* bytes) {
  if (!bytes) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_variant(variant));
  if (out_dim < 32 || out_dim > 256 || out_dim % 32) return RAFT_ERR_BAD_SHAPE;
  *bytes = enc_layout(variant, out_dim).total;
  return RAFT_OK;
}

int raft_b200_encoder_prepare(int variant, int norm_type, int out_dim, const raft_encoder_weights* weights,
                              void* prepared, size_t prepared_bytes, void* stream) {
  if (!weights || !prepared) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_variant(variant));
  if (norm_type < 0 || norm_type > 2) return RAFT_ERR_BAD_ARG;
  if (out_dim < 32 || out_dim > 256 || out_dim % 32) return RAFT_ERR_BAD_SHAPE;
  return encoder_prepare(variant, norm_type, out_dim, weights, prepared, prepared_bytes, reinterpret_cast<cudaStream_t>(stream));
}

int raft_b200_encoder_workspace_bytes(int variant, int N, int H, int W, size_t* bytes) {
  if (!bytes) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_variant(variant));
  RAFT_TRY(check_dims(N, H, W));
  *bytes = enc_ws_layout(nullptr, variant, N, H, W).total;
  return RAFT_OK;
}

int raft_b200_encoder_forward(int variant, int norm_type, int out_dim, const void* prepared, const float* images,
                              int N, int H, int W, int training, int image_norm, float* out, void* workspace,
                              size_t workspace_bytes, void* stream) {
  if (!prepared || !images || !out || !workspace) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_variant(variant));
  if (norm_type < 0 || norm_type > 2) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_dims(N, H, W));
  if (out_dim < 32 || out_dim > 256 || out_dim % 32 || H < 8 || W < 8) return RAFT_ERR_BAD_SHAPE;
  return encoder_forward(variant, norm_type, out_dim, prepared, images, N, H, W, training, image_norm, out, workspace, workspace_bytes,
                         reinterpret_cast<cudaStream_t>(stream));
}

int raft_b200_context_split(const float* cnet, int npix, int hidden, int context, float* net, float* inp,
                            void* stream) {
  if (!cnet || !net || !inp) return RAFT_ERR_BAD_ARG;
  if (npix < 1 || hidden < 1 || context < 1) return RAFT_ERR_BAD_SHAPE;
  return launch(context_split_kernel, grid_for((size_t)npix * (hidden + context)), 256, 0, reinterpret_cast<cudaStream_t>(stream),
                cnet, (size_t)npix, hidden, context, net, inp);
}

int raft_b200_encode_pair_workspace_bytes(int variant, int N, int H, int W, int cnet_dim, size_t* bytes) {
  if (!bytes) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_variant(variant));
  RAFT_TRY(check_dims(N, H, W));
  if (cnet_dim < 1) return RAFT_ERR_BAD_SHAPE;
  *bytes = pair_ws_layout(nullptr, variant, N, H, W, cnet_dim).total;
  return RAFT_OK;
}

int raft_b200_encode_pair(int variant, const void* fnet_prepared, int fnet_norm, int fnet_dim, const void* cnet_prepared,
                          int cnet_norm, int hidden, int context, const float* image1, const float* image2, int N, int H,
                          int W, float* fmap1, float* fmap2, float* net, float* inp, void* workspace, size_t workspace_bytes,
                          void* stream) {
  if (!fnet_prepared || !cnet_prepared || !image1 || !image2 || !fmap1 || !fmap2 || !net || !inp || !workspace)
    return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_variant(variant));
  if (fnet_norm < 0 || fnet_norm > 2 || cnet_norm < 0 || cnet_norm > 2) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_dims(N, H, W));
  const int cnet_dim = hidden + context;
  for (int d : {fnet_dim, cnet_dim})
    if (d < 32 || d > 256 || d % 32) return RAFT_ERR_BAD_SHAPE;
  if (hidden < 1 || context < 1 || H < 8 || W < 8) return RAFT_ERR_BAD_SHAPE;
  const int h = ceil_div(H, 8), w = ceil_div(W, 8);
  const PairWs P = pair_ws_layout(workspace, variant, N, H, W, cnet_dim);
  if (P.total > workspace_bytes) return RAFT_ERR_WORKSPACE;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  PairStreams* ps = nullptr;
  RAFT_TRY(pair_streams(st, &ps));
  cudaStream_t sa = ps->s[0], sb = ps->s[1], sc = ps->s[2];
  const size_t enc_bytes = P.enc_bytes;

  // Fork.  Branch A: fnet(image1); B: fnet(image2); C: cnet(image1) and the context split.  A builds image1's stem planes
  // first and C reads them from A's workspace.
  RAFT_CUDA_TRY(cudaEventRecord(ps->fork, st));
  for (cudaStream_t s : {sa, sb, sc}) RAFT_CUDA_TRY(cudaStreamWaitEvent(s, ps->fork, 0));
  int status = encoder_stem_im2col(variant, image1, N, H, W, 1, P.enc[0], sa);
  if (!status) status = (int)cudaEventRecord(ps->stem, sa);
  if (!status) status = encoder_forward(variant, fnet_norm, fnet_dim, fnet_prepared, image2, N, H, W, 0, 1, fmap2, P.enc[1],
                                        enc_bytes, sb);
  if (!status) status = (int)cudaStreamWaitEvent(sc, ps->stem, 0);
  if (!status) status = encoder_forward(variant, cnet_norm, cnet_dim, cnet_prepared, image1, N, H, W, 0, 1, P.cnet_out, P.enc[2],
                                        enc_bytes, sc, P.stem_hi, P.stem_lo);
  if (!status) status = launch(context_split_kernel, grid_for((size_t)N * h * w * cnet_dim), 256, 0, sc, P.cnet_out,
                               (size_t)N * h * w, hidden, context, net, inp);
  if (!status) status = encoder_forward(variant, fnet_norm, fnet_dim, fnet_prepared, image1, N, H, W, 0, 1, fmap1, P.enc[0],
                                        enc_bytes, sa, P.stem_hi, P.stem_lo);
  // Join every branch back into the caller's stream, also after an error: a capture must not be left forked.
  RAFT_CUDA_TRY(cudaEventRecord(ps->a, sa));
  RAFT_CUDA_TRY(cudaEventRecord(ps->b, sb));
  RAFT_CUDA_TRY(cudaEventRecord(ps->c, sc));
  for (cudaEvent_t e : {ps->a, ps->b, ps->c}) RAFT_CUDA_TRY(cudaStreamWaitEvent(st, e, 0));
  return status ? status : raft_launch_status();
}

int raft_b200_conv2d(const float* x, const float* kernel, const float* bias, int B, int H, int W, int cin, int kh,
                     int kw, int cout, int act, float* out, int out_stride, int out_c0, void* stream) {
  if (!x || !kernel || !out) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(check_dims(B, H, W));
  if (cin < 1 || cout < 1 || kh < 1 || kw < 1 || !(kh & 1) || !(kw & 1) || act < 0 || act > 3) return RAFT_ERR_BAD_SHAPE;
  if (out_stride < out_c0 + cout) return RAFT_ERR_BAD_SHAPE;
  SimtConvParams p;
  memset(&p, 0, sizeof(p));
  p.src[0] = x; p.src_stride[0] = cin; p.src_c0[0] = 0; p.src_n[0] = cin; p.nsrc = 1;
  p.w = kernel; p.bias = bias;
  p.kh = kh; p.kw = kw; p.cin = cin; p.cout = cout;
  p.B = B; p.H = H; p.W = W;
  p.out = out; p.out_stride = out_stride; p.out_c0 = out_c0;
  p.act = act; p.out_scale = 1.0f;
  dim3 grid((unsigned)ceil_div(B * H * W, 64), (unsigned)ceil_div(cout, 64));
  return launch(conv_simt_kernel, grid, 256, 0, reinterpret_cast<cudaStream_t>(stream), p);
}

int raft_b200_forward_loop(int variant, const void* prepared, const float* const pyr[], int levels, int radius,
                           float* net, const float* inp, float* coords1, float* const flow_up[], int iters, int B,
                           int h, int w, void* workspace, size_t workspace_bytes, int precision, void* stream) {
  if (!pyr || !net || !inp || !coords1 || !flow_up || iters < 0) return RAFT_ERR_BAD_ARG;
  if (levels < 1 || levels > RAFT_MAX_LEVELS || radius < 0) return RAFT_ERR_BAD_ARG;
  UpdateCtx c;
  RAFT_TRY(make_ctx(c, variant, prepared, B, h, w, workspace, workspace_bytes, precision, stream));
  const VariantDims d = variant_dims(variant);
  const int side = 2 * radius + 1;
  if (levels * side * side != d.corr_ch) return RAFT_ERR_BAD_SHAPE;
  const size_t npix = (size_t)B * h * w;
  const Workspace& W = c.W;
  RAFT_TRY(update_begin(c, net, inp));
  RAFT_TRY(launch(flow_advance_kernel, grid_for(npix), 256, 0, c.stream, coords1, nullptr, W.flow, B, h, w));   // model.py:97
  const bool prof = g_prof.on && iters <= 64;
  if (prof && !g_prof.created) {
    for (int i = 0; i < 64; ++i)
      for (int k = 0; k < 3; ++k) RAFT_CUDA_TRY(cudaEventCreate(&g_prof.ev[i][k]));
    g_prof.created = true;
  }
  if (prof) g_prof.n = iters;
  for (int i = 0; i < iters; ++i) {
    float* mask = (variant == RAFT_VARIANT_BASIC && flow_up[i]) ? W.mask : nullptr;
    if (precision == RAFT_PREC_F16X2) {
      if (prof) RAFT_CUDA_TRY(cudaEventRecord(g_prof.ev[i][0], c.stream));
      RAFT_TRY(lookup_launch(pyr, coords1, B, h, w, levels, radius, nullptr, 0, W.corr_hi, W.corr_lo, d.s_corr, d.s_corr,
                             c.stream, W.flow, W.fim_hi, W.fim_lo));                                // model.py:95 (+ convf1's im2col)
      if (prof) RAFT_CUDA_TRY(cudaEventRecord(g_prof.ev[i][1], c.stream));
      c.fim_ready = true;
      RAFT_TRY(update_block_tc(c, net, W.delta, mask, coords1));                                    // :99, :102 (fused advance)
      c.fim_ready = false;
      if (prof) RAFT_CUDA_TRY(cudaEventRecord(g_prof.ev[i][2], c.stream));
    } else {
      RAFT_TRY(lookup_launch(pyr, coords1, B, h, w, levels, radius, W.corr, d.corr_ch, nullptr, nullptr, 0, 0, c.stream));
      RAFT_TRY(update_core_fp32(c, net, W.delta, mask));
      RAFT_TRY(launch(flow_advance_kernel, grid_for(npix), 256, 0, c.stream, coords1, W.delta, W.flow, B, h, w));  // :102
    }
    if (flow_up[i]) {                                                                               // :105 / :223
      if (variant == RAFT_VARIANT_BASIC)
        RAFT_TRY(raft_b200_upsample_convex(W.flow, W.mask, B, h, w, flow_up[i], stream));
      else
        RAFT_TRY(raft_b200_upflow8(W.flow, B, h, w, flow_up[i], stream));
    }
  }
  return raft_launch_status();
}

// Training convolutions (conv_train.cuh).  workspace == null: *workspace_bytes = the size the shape needs, nothing runs.
static int conv_train_prologue(int B, int H, int W, int cin, int kh, int kw, int cout, const void* planes, const void* ws,
                               size_t* ws_bytes, ConvTrainLayout& L) {
  if (!ws_bytes) return RAFT_ERR_BAD_ARG;
  RAFT_TRY(conv_train_check(B, H, W, cin, kh, kw, cout));
  RAFT_TRY(conv_train_layout(B, H, W, cin, kh, kw, cout, L));
  if (!ws) return RAFT_OK;
  if (!planes || (reinterpret_cast<uintptr_t>(planes) | reinterpret_cast<uintptr_t>(ws)) % 256) return RAFT_ERR_BAD_ARG;
  return *ws_bytes < L.total ? RAFT_ERR_WORKSPACE : RAFT_OK;
}

int raft_b200_conv_tc_forward(const float* x, const float* kernel, const float* bias, int B, int H, int W, int cin, int kh,
                              int kw, int cout, float* out, void* x_planes, void* workspace, size_t* workspace_bytes,
                              void* stream) {
  ConvTrainLayout L;
  RAFT_TRY(conv_train_prologue(B, H, W, cin, kh, kw, cout, x_planes, workspace, workspace_bytes, L));
  if (!workspace) { *workspace_bytes = L.total; return RAFT_OK; }
  if (!x || !kernel || !bias || !out || reinterpret_cast<uintptr_t>(out) % 32) return RAFT_ERR_BAD_ARG;
  return conv_train_forward(x, kernel, bias, B, H, W, cin, kh, kw, cout, out, static_cast<__half*>(x_planes),
                            static_cast<uint8_t*>(workspace), L, reinterpret_cast<cudaStream_t>(stream));
}

int raft_b200_conv_tc_backward(const void* x_planes, const float* kernel, const float* grad_out, int B, int H, int W,
                               int cin, int kh, int kw, int cout, float* grad_x, float* grad_kernel, void* workspace,
                               size_t* workspace_bytes, void* stream) {
  ConvTrainLayout L;
  RAFT_TRY(conv_train_prologue(B, H, W, cin, kh, kw, cout, x_planes, workspace, workspace_bytes, L));
  if (!workspace) { *workspace_bytes = L.total; return RAFT_OK; }
  if (!kernel || !grad_out || !grad_kernel || (grad_x && reinterpret_cast<uintptr_t>(grad_x) % 32)) return RAFT_ERR_BAD_ARG;
  return conv_train_backward(static_cast<const __half*>(x_planes), kernel, grad_out, B, H, W, cin, kh, kw, cout, grad_x,
                             grad_kernel, static_cast<uint8_t*>(workspace), L, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
