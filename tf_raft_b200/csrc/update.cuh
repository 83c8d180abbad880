// Host-side plan of the update blocks (update.py:109-153): prepared-weight layout, activation
// workspace layout, and the per-iteration launch sequence for both arithmetic paths.
#pragma once
#include <string.h>

#include "conv_tc.cuh"
#include "kernels.cuh"
#include "mega.cuh"

namespace raft {

// ------------------------------------------------------------------------------------------------
// Reference convolutions, in raft_basic_weights / raft_small_weights member order.
// ------------------------------------------------------------------------------------------------
struct ConvDim { int kh, kw, cin, cout; };

static const ConvDim kBasicConvs[15] = {
    {1, 1, 324, 256}, {3, 3, 256, 192}, {7, 7, 2, 128}, {3, 3, 128, 64}, {3, 3, 256, 126},   // encoder
    {1, 5, 384, 128}, {1, 5, 384, 128}, {1, 5, 384, 128},                                    // gru horizontal
    {5, 1, 384, 128}, {5, 1, 384, 128}, {5, 1, 384, 128},                                    // gru vertical
    {3, 3, 128, 256}, {3, 3, 256, 2},                                                        // flow head
    {3, 3, 128, 256}, {1, 1, 256, 576}};                                                     // mask head
enum BasicConv { BC1 = 0, BC2, BF1, BF2, BCV, BZ1, BR1, BQ1, BZ2, BR2, BQ2, BFH1, BFH2, BM0, BM2 };

static const ConvDim kSmallConvs[9] = {
    {1, 1, 196, 96}, {7, 7, 2, 64}, {3, 3, 64, 32}, {3, 3, 128, 80},
    {3, 3, 242, 96}, {3, 3, 242, 96}, {3, 3, 242, 96},
    {3, 3, 96, 128}, {3, 3, 128, 2}};
enum SmallConv { SC1 = 0, SF1, SF2, SCV, SZ, SR, SQ, SFH1, SFH2 };

inline int n_convs(int variant) { return variant == RAFT_VARIANT_BASIC ? 15 : 9; }
inline const ConvDim* conv_dims(int variant) { return variant == RAFT_VARIANT_BASIC ? kBasicConvs : kSmallConvs; }

// ------------------------------------------------------------------------------------------------
// Tensor-core layers (precision F16X2), one table per variant in work-list order: the order in which update_mega_kernel
// hands out their tiles (list order is priority order), and the order of the per-layer launches.  A row is everything
// about one layer: how its weights are packed, its tiling, the planes it reads, its epilogue and the rows it waits on.
// ------------------------------------------------------------------------------------------------
// Operands: fp16 hi/lo planes of the workspace (channel stride from VariantDims; fim: 128), and the caller's fp32
// outputs, which only an epilogue writes.
enum TcPlane : int { PL_CORR, PL_COR1, PL_CF, PL_FLO1, PL_X, PL_H, PL_RH, PL_FM, PL_FIM, OUT_DELTA, OUT_MASK };

struct TcSeg { int plane, c0, chunks; };   // K segment: `chunks` 64-channel chunks of a plane, from channel c0

enum TcLayerFlags : int {
  TC_CONCAT_FLOW = 1,   // the epilogue appends the 2 flow channels after column n_total (the motion encoder's output)
  TC_ADVANCE = 2,       // inside the iteration loop the epilogue also applies coords1 += delta and flow = coords1 - grid
  TC_MASK_ONLY = 4,     // runs only when the mask is wanted (only the last row may: a row's index is its plan position)
  TC_MASK_TAIL = 8,     // the last table column tile (bn columns) feeds only the mask head: dropped without a mask
};

struct TcLayer {
  int nsrc, src[2];               // packing: reference convs merged along cout,
  int kh, kw, cin_pad, cout_pad;  //   packed dims,
  int flatten;                    //   1: (kh,kw,cin) flattened into the channel axis, read as a 1x1 conv of im2col planes,
  TcCinMap cin_map;               //   where the input channels land (nrange == 0: where they are)
  int bn, ntn;                    // tiling: N per column tile, column tiles (split further when bn > kMaxTileN)
  TcSeg seg[2];                   // inputs: one or two K segments (seg[1].chunks == 0: one)
  int mode, act, n_total;         // epilogue (the GRU modes read z and update the caller's hidden state),
  float out_scale;
  int out, out_c0;                //   output plane and its first channel,
  int flags;                      //   TcLayerFlags
  int ndep;                       // rows read by this one, with the columns read: update_mega_kernel waits for their tiles
  MegaDep dep[2];                 //   over the halo, which also covers the write-after-read hazards
};

// Fields per row: nsrc, convs, kh, kw, cin_pad, cout_pad, flatten, cin map, bn, ntn, inputs,
//                 mode, act, n_total, out_scale, out, out_c0, flags, ndep, deps.
// The flow branch (convf1, convf2) needs only the current flow, so it is interleaved with the correlation branch.
static const TcLayer kBasicTc[12] = {
    /*  0 convc1 */ {1, {BC1}, 1, 1, 384, 256, 0, {}, 256, 1, {{PL_CORR, 0, 6}},
                     EPI_LINEAR, ACT_RELU, 256, 1.0f, PL_COR1, 0, 0, 0, {}},
    /*  1 convf1 */ {1, {BF1}, 1, 1, 128, 128, 1, {}, 128, 1, {{PL_FIM, 0, 2}},
                     EPI_LINEAR, ACT_RELU, 128, 1.0f, PL_FLO1, 0, 0, 0, {}},
    /*  2 convc2 */ {1, {BC2}, 3, 3, 256, 192, 0, {}, 192, 1, {{PL_COR1, 0, 4}},
                     EPI_LINEAR, ACT_RELU, 192, 1.0f, PL_CF, 0, 0, 1, {{0}}},
    /*  3 convf2 */ {1, {BF2}, 3, 3, 128, 64, 0, {}, 64, 1, {{PL_FLO1, 0, 2}},
                     EPI_LINEAR, ACT_RELU, 64, 1.0f, PL_CF, 192, 0, 1, {{1}}},
    /*  4 conv   */ {1, {BCV}, 3, 3, 256, 128, 0, {}, 128, 1, {{PL_CF, 0, 4}},
                     EPI_LINEAR, ACT_RELU, 126, 1.0f, PL_X, 128, TC_CONCAT_FLOW, 2, {{2}, {3}}},
    /*  5 z|r1   */ {2, {BZ1, BR1}, 1, 5, 384, 256, 0, {}, 256, 1, {{PL_H, 0, 2}, {PL_X, 0, 4}},
                     EPI_GRU_ZR, ACT_NONE, 256, 1.0f, PL_RH, 0, 0, 1, {{4}}},
    /*  6 q1     */ {1, {BQ1}, 1, 5, 384, 128, 0, {}, 128, 1, {{PL_RH, 0, 2}, {PL_X, 0, 4}},
                     EPI_GRU_Q, ACT_NONE, 128, 1.0f, PL_H, 0, 0, 1, {{5}}},
    /*  7 z|r2   */ {2, {BZ2, BR2}, 5, 1, 384, 256, 0, {}, 256, 1, {{PL_H, 0, 2}, {PL_X, 0, 4}},
                     EPI_GRU_ZR, ACT_NONE, 256, 1.0f, PL_RH, 0, 0, 1, {{6}}},
    /*  8 q2     */ {1, {BQ2}, 5, 1, 384, 128, 0, {}, 128, 1, {{PL_RH, 0, 2}, {PL_X, 0, 4}},
                     EPI_GRU_Q, ACT_NONE, 128, 1.0f, PL_H, 0, 0, 1, {{7}}},
    /*  9 fh1|m0 */ {2, {BFH1, BM0}, 3, 3, 128, 512, 0, {}, 256, 2, {{PL_H, 0, 2}},
                     EPI_LINEAR, ACT_RELU, 512, 1.0f, PL_FM, 0, TC_MASK_TAIL, 1, {{8}}},
    /* 10 fh2    */ {1, {BFH2}, 3, 3, 256, 16, 0, {}, 16, 1, {{PL_FM, 0, 4}},
                     EPI_LINEAR, ACT_NONE, 2, 1.0f, OUT_DELTA, 0, TC_ADVANCE, 1, {{9, 0, 256}}},
    /* 11 mask2  */ {1, {BM2}, 1, 1, 256, 576, 0, {}, 192, 3, {{PL_FM, 256, 4}},
                     EPI_LINEAR, ACT_NONE, 576, 0.25f, OUT_MASK, 0, TC_MASK_ONLY, 1, {{9, 256, 512}}}};

static const TcLayer kSmallTc[8] = {
    /* 0 convc1 */ {1, {SC1}, 1, 1, 256, 96, 0, {}, 96, 1, {{PL_CORR, 0, 4}},
                    EPI_LINEAR, ACT_RELU, 96, 1.0f, PL_CF, 0, 0, 0, {}},
    /* 1 convf1 */ {1, {SF1}, 1, 1, 128, 64, 1, {}, 64, 1, {{PL_FIM, 0, 2}},
                    EPI_LINEAR, ACT_RELU, 64, 1.0f, PL_FLO1, 0, 0, 0, {}},
    /* 2 convf2 */ {1, {SF2}, 3, 3, 64, 32, 0, {}, 32, 1, {{PL_FLO1, 0, 1}},
                    EPI_LINEAR, ACT_RELU, 32, 1.0f, PL_CF, 96, 0, 1, {{1}}},
    /* 3 conv   */ {1, {SCV}, 3, 3, 128, 96, 0, {}, 96, 1, {{PL_CF, 0, 2}},
                    EPI_LINEAR, ACT_RELU, 80, 1.0f, PL_X, 64, TC_CONCAT_FLOW, 2, {{0}, {2}}},
    /* 4 z|r    */ {2, {SZ, SR}, 3, 3, 320, 192, 0, {2, {0, 96}, {96, 146}, {0, 128}}, 192, 1, {{PL_H, 0, 2}, {PL_X, 0, 3}},
                    EPI_GRU_ZR, ACT_NONE, 192, 1.0f, PL_RH, 0, 0, 1, {{3}}},
    /* 5 q      */ {1, {SQ}, 3, 3, 320, 96, 0, {2, {0, 96}, {96, 146}, {0, 128}}, 96, 1, {{PL_RH, 0, 2}, {PL_X, 0, 3}},
                    EPI_GRU_Q, ACT_NONE, 96, 1.0f, PL_H, 0, 0, 1, {{4}}},
    /* 6 fh1    */ {1, {SFH1}, 3, 3, 128, 128, 0, {}, 128, 1, {{PL_H, 0, 2}},
                    EPI_LINEAR, ACT_RELU, 128, 1.0f, PL_FM, 0, 0, 1, {{5}}},
    /* 7 fh2    */ {1, {SFH2}, 3, 3, 128, 16, 0, {}, 16, 1, {{PL_FM, 0, 2}},
                    EPI_LINEAR, ACT_NONE, 2, 1.0f, OUT_DELTA, 0, TC_ADVANCE, 1, {{6}}}};

inline int n_tc_layers(int variant) { return variant == RAFT_VARIANT_BASIC ? 12 : 8; }
inline const TcLayer* tc_layers(int variant) { return variant == RAFT_VARIANT_BASIC ? kBasicTc : kSmallTc; }

// ------------------------------------------------------------------------------------------------
// Prepared-weights blob (device).  Offsets are a pure function of (variant, precision).
// ------------------------------------------------------------------------------------------------
struct PreparedLayout {
  size_t raw_w[15], raw_b[15];                 // fp32 copies of every reference conv (HWIO) + bias
  TcWeightSlot tc[12];                         // packed weights of every tensor-core layer (F16X2 only)
  size_t total;
};

inline PreparedLayout prepared_layout(int variant, int precision) {
  PreparedLayout L;
  memset(&L, 0, sizeof(L));
  size_t off = 0;
  const ConvDim* cd = conv_dims(variant);
  for (int i = 0; i < n_convs(variant); ++i) {
    L.raw_w[i] = off;
    off = align_up(off + sizeof(float) * cd[i].kh * cd[i].kw * cd[i].cin * cd[i].cout, 256);
    L.raw_b[i] = off;
    off = align_up(off + sizeof(float) * cd[i].cout, 256);
  }
  if (precision == RAFT_PREC_F16X2) {
    const TcLayer* tl = tc_layers(variant);
    for (int i = 0; i < n_tc_layers(variant); ++i)
      L.tc[i] = tc_weight_slot(off, tl[i].kh, tl[i].kw, tl[i].cin_pad, tl[i].cout_pad);
  }
  L.total = off;
  return L;
}

// ------------------------------------------------------------------------------------------------
// Activation workspace.
// ------------------------------------------------------------------------------------------------
struct VariantDims {
  int hid, ctx, corr_ch;
  int c_cor1, c_cf, c_flo1, c_x, c_fm;        // fp32-path plane widths
  int s_corr, s_cor1, s_cf, s_flo1, s_x, s_h, s_fm;   // fp16-plane channel strides (multiples of 64)
};
inline VariantDims variant_dims(int variant) {
  if (variant == RAFT_VARIANT_BASIC)
    return {.hid = 128, .ctx = 128, .corr_ch = 324,
            .c_cor1 = 256, .c_cf = 256, .c_flo1 = 128, .c_x = 256, .c_fm = 512,
            .s_corr = 384, .s_cor1 = 256, .s_cf = 256, .s_flo1 = 128, .s_x = 256, .s_h = 128, .s_fm = 512};
  return {.hid = 96, .ctx = 64, .corr_ch = 196,
          .c_cor1 = 0, .c_cf = 128, .c_flo1 = 64, .c_x = 148, .c_fm = 128,
          .s_corr = 256, .s_cor1 = 0, .s_cf = 128, .s_flo1 = 64, .s_x = 192, .s_h = 128, .s_fm = 128};
}

struct Workspace {
  // fp32 planes
  float *corr, *cor1, *cf, *flo1, *x, *z, *r, *rh, *q, *fm, *flow, *delta, *mask;
  // fp16 hi/lo planes (tensor-core path)
  __half *corr_hi, *corr_lo, *cor1_hi, *cor1_lo, *cf_hi, *cf_lo, *flo1_hi, *flo1_lo, *x_hi, *x_lo, *h_hi, *h_lo,
      *rh_hi, *rh_lo, *fm_hi, *fm_lo, *fim_hi, *fim_lo;
  uint8_t* f16_begin; size_t f16_bytes;
  unsigned int* mega_flags; size_t mega_flag_words;   // per-(layer, tile) completion counters of update_mega_kernel
  size_t total;
};

inline Workspace workspace_layout(void* base, int variant, int B, int h, int w, int precision) {
  Workspace W;
  memset(&W, 0, sizeof(W));
  const VariantDims d = variant_dims(variant);
  const size_t npix = (size_t)B * h * w;
  size_t off = 0;
  uint8_t* b8 = reinterpret_cast<uint8_t*>(base);
  auto f32 = [&](int ch) {
    float* p = reinterpret_cast<float*>(b8 + off);
    off = align_up(off + npix * ch * sizeof(float), 1024);
    return p;
  };
  auto f16 = [&](int ch) {
    __half* p = reinterpret_cast<__half*>(b8 + off);
    off = align_up(off + npix * ch * sizeof(__half), 1024);
    return p;
  };
  W.flow = f32(2);
  W.delta = f32(2);
  W.mask = f32(576);
  W.z = f32(d.hid);
  if (precision == RAFT_PREC_FP32) {
    W.corr = f32(d.corr_ch);
    if (d.c_cor1) W.cor1 = f32(d.c_cor1);
    W.cf = f32(d.c_cf);
    W.flo1 = f32(d.c_flo1);
    W.x = f32(d.c_x);
    W.r = f32(d.hid);
    W.rh = f32(d.hid);
    W.q = f32(d.hid);
    W.fm = f32(d.c_fm);
  } else {
    W.f16_begin = b8 + off;
    W.corr_hi = f16(d.s_corr); W.corr_lo = f16(d.s_corr);
    if (d.s_cor1) { W.cor1_hi = f16(d.s_cor1); W.cor1_lo = f16(d.s_cor1); }
    W.cf_hi = f16(d.s_cf); W.cf_lo = f16(d.s_cf);
    W.flo1_hi = f16(d.s_flo1); W.flo1_lo = f16(d.s_flo1);
    W.x_hi = f16(d.s_x); W.x_lo = f16(d.s_x);
    W.h_hi = f16(d.s_h); W.h_lo = f16(d.s_h);
    W.rh_hi = f16(d.s_h); W.rh_lo = f16(d.s_h);
    W.fm_hi = f16(d.s_fm); W.fm_lo = f16(d.s_fm);
    W.fim_hi = f16(128); W.fim_lo = f16(128);      // im2col of the 7x7 flow window (98 -> 128 channels)
    W.f16_bytes = (size_t)((b8 + off) - W.f16_begin);
    // any 128-pixel tile shape covers an h x w plane with at most h*w/128 + h + w + 1 tiles
    W.mega_flag_words = (size_t)mega_flag_words(B, h * w / 128 + h + w + 1);
    W.mega_flags = reinterpret_cast<unsigned int*>(b8 + off);
    off = align_up(off + W.mega_flag_words * sizeof(unsigned int), 1024);
  }
  W.total = off;
  return W;
}

// ------------------------------------------------------------------------------------------------
// Launch helpers
// ------------------------------------------------------------------------------------------------
struct UpdateCtx {
  int variant, precision, B, h, w;
  const uint8_t* prepared;
  PreparedLayout PL;
  Workspace W;
  cudaStream_t stream;
  bool fim_ready;      // the convf1 im2col planes of the current flow already exist (written by the loop's lookup kernel)
  MegaPlan* plan;      // non-null: tensor-core layers are collected here and run as ONE update_mega_kernel launch
};

inline int launch_simt_conv(const UpdateCtx& c, int conv_idx, int nsrc, const float* const src[], const int src_stride[],
                            const int src_c0[], const int src_n[], float* out, int out_stride, int out_c0, int act,
                            float out_scale, __half* out_hi = nullptr, __half* out_lo = nullptr, int h_stride = 0,
                            int h_c0 = 0) {
  const ConvDim cd = conv_dims(c.variant)[conv_idx];
  SimtConvParams p;
  memset(&p, 0, sizeof(p));
  int cin = 0;
  for (int i = 0; i < nsrc; ++i) {
    p.src[i] = src[i];
    p.src_stride[i] = src_stride[i];
    p.src_c0[i] = src_c0[i];
    p.src_n[i] = src_n[i];
    cin += src_n[i];
  }
  if (cin != cd.cin) return RAFT_ERR_BAD_SHAPE;
  p.nsrc = nsrc;
  p.w = reinterpret_cast<const float*>(c.prepared + c.PL.raw_w[conv_idx]);
  p.bias = reinterpret_cast<const float*>(c.prepared + c.PL.raw_b[conv_idx]);
  p.kh = cd.kh; p.kw = cd.kw; p.cin = cd.cin; p.cout = cd.cout;
  p.B = c.B; p.H = c.h; p.W = c.w;
  p.out = out; p.out_stride = out_stride; p.out_c0 = out_c0;
  p.out_hi = out_hi; p.out_lo = out_lo; p.h_stride = h_stride; p.h_c0 = h_c0;
  p.act = act; p.out_scale = out_scale;
  const int npix = c.B * c.h * c.w;
  dim3 grid((unsigned)ceil_div(npix, 64), (unsigned)ceil_div(cd.cout, 64));
  return launch(conv_simt_kernel, grid, 256, 0, c.stream, p);
}

inline int simt1(const UpdateCtx& c, int conv_idx, const float* src, int stride, int c0, int n, float* out, int out_stride,
                 int out_c0, int act, float scale = 1.0f) {
  const float* s[1] = {src};
  int st[1] = {stride}, o[1] = {c0}, nn[1] = {n};
  return launch_simt_conv(c, conv_idx, 1, s, st, o, nn, out, out_stride, out_c0, act, scale);
}
inline int simt2(const UpdateCtx& c, int conv_idx, const float* s0, int st0, int n0, const float* s1, int st1, int n1,
                 float* out, int out_stride, int act) {
  const float* s[2] = {s0, s1};
  int st[2] = {st0, st1}, o[2] = {0, 0}, nn[2] = {n0, n1};
  return launch_simt_conv(c, conv_idx, 2, s, st, o, nn, out, out_stride, 0, act, 1.0f);
}

// ------------------------------------------------------------------------------------------------
// Update block, fp32 FFMA path: the reference's op sequence, one launch per Conv2D.
// ------------------------------------------------------------------------------------------------
inline int gru_fp32(const UpdateCtx& c, float* h, int iz, int ir, int iq, int hid, int xs, int xn) {
  const Workspace& W = c.W;
  const size_t n = (size_t)c.B * c.h * c.w * hid;
  RAFT_TRY(simt2(c, iz, h, hid, hid, W.x, xs, xn, W.z, hid, SACT_SIGMOID));
  RAFT_TRY(simt2(c, ir, h, hid, hid, W.x, xs, xn, W.r, hid, SACT_SIGMOID));
  RAFT_TRY(launch(gru_rh_kernel, grid_for(n), 256, 0, c.stream, W.r, h, W.rh, n));
  RAFT_TRY(simt2(c, iq, W.rh, hid, hid, W.x, xs, xn, W.q, hid, SACT_TANH));
  return launch(gru_update_kernel, grid_for(n), 256, 0, c.stream, W.z, W.q, h, n);
}

inline int update_core_fp32(const UpdateCtx& c, float* h, float* delta, float* mask) {
  const Workspace& W = c.W;
  const VariantDims d = variant_dims(c.variant);
  const size_t npix = (size_t)c.B * c.h * c.w;
  if (c.variant == RAFT_VARIANT_BASIC) {
    RAFT_TRY(simt1(c, BC1, W.corr, 324, 0, 324, W.cor1, 256, 0, SACT_RELU));           // update.py:98
    RAFT_TRY(simt1(c, BC2, W.cor1, 256, 0, 256, W.cf, 256, 0, SACT_RELU));              // :99
    RAFT_TRY(simt1(c, BF1, W.flow, 2, 0, 2, W.flo1, 128, 0, SACT_RELU));                // :100
    RAFT_TRY(simt1(c, BF2, W.flo1, 128, 0, 128, W.cf, 256, 192, SACT_RELU));            // :101,104
    RAFT_TRY(simt1(c, BCV, W.cf, 256, 0, 256, W.x, 256, 128, SACT_RELU));               // :105
    RAFT_TRY(launch(copy_channels_kernel, grid_for(npix * 2), 256, 0, c.stream, W.flow, 2, 0, W.x, 256, 254, 2, npix));  // :106
    RAFT_TRY(gru_fp32(c, h, BZ1, BR1, BQ1, 128, 256, 256));                             // :53-58
    RAFT_TRY(gru_fp32(c, h, BZ2, BR2, BQ2, 128, 256, 256));                             // :60-65
    RAFT_TRY(simt1(c, BFH1, h, 128, 0, 128, W.fm, 512, 0, SACT_RELU));                  // :14
    RAFT_TRY(simt1(c, BFH2, W.fm, 512, 0, 256, delta, 2, 0, SACT_NONE));
    if (mask) {
      RAFT_TRY(simt1(c, BM0, h, 128, 0, 128, W.fm, 512, 256, SACT_RELU));               // :137-141
      RAFT_TRY(simt1(c, BM2, W.fm, 512, 256, 256, mask, 576, 0, SACT_NONE, 0.25f));     // :152
    }
  } else {
    RAFT_TRY(simt1(c, SC1, W.corr, 196, 0, 196, W.cf, 128, 0, SACT_RELU));              // update.py:80
    RAFT_TRY(simt1(c, SF1, W.flow, 2, 0, 2, W.flo1, 64, 0, SACT_RELU));                 // :81
    RAFT_TRY(simt1(c, SF2, W.flo1, 64, 0, 64, W.cf, 128, 96, SACT_RELU));               // :82-83
    RAFT_TRY(simt1(c, SCV, W.cf, 128, 0, 128, W.x, d.c_x, 64, SACT_RELU));              // :84
    RAFT_TRY(launch(copy_channels_kernel, grid_for(npix * 2), 256, 0, c.stream, W.flow, 2, 0, W.x, d.c_x, 144, 2, npix));  // :85
    RAFT_TRY(gru_fp32(c, h, SZ, SR, SQ, 96, d.c_x, 146));                               // :26-35
    RAFT_TRY(simt1(c, SFH1, h, 96, 0, 96, W.fm, 128, 0, SACT_RELU));
    RAFT_TRY(simt1(c, SFH2, W.fm, 128, 0, 128, delta, 2, 0, SACT_NONE));
  }
  return raft_launch_status();
}

// ------------------------------------------------------------------------------------------------
// Update block, tensor-core path: the rows of tc_layers(variant), in order.  Operands travel between layers as fp16
// hi/lo planes written by the producing layer's epilogue.  h: the caller's hidden state, updated in place; mask == null:
// no mask head; adv_coords != null (iteration loop): the flow head's epilogue also advances coords1 and the flow.
// With c.plan the layers are appended to the plan (one update_mega_kernel launch), else launched one by one.
// ------------------------------------------------------------------------------------------------
inline int update_core_tc(const UpdateCtx& c, float* h, float* delta, float* mask, float* adv_coords) {
  const Workspace& W = c.W;
  const VariantDims d = variant_dims(c.variant);
  struct Plane { __half *hi, *lo; int stride; };
  const Plane planes[] = {{W.corr_hi, W.corr_lo, d.s_corr}, {W.cor1_hi, W.cor1_lo, d.s_cor1}, {W.cf_hi, W.cf_lo, d.s_cf},
                          {W.flo1_hi, W.flo1_lo, d.s_flo1}, {W.x_hi, W.x_lo, d.s_x},          {W.h_hi, W.h_lo, d.s_h},
                          {W.rh_hi, W.rh_lo, d.s_h},        {W.fm_hi, W.fm_lo, d.s_fm},       {W.fim_hi, W.fim_lo, 128}};
  int tw, th;
  tc_pick_tile(c.w, c.h, &tw, &th);
  const TcLayer* rows = tc_layers(c.variant);
  for (int i = 0; i < n_tc_layers(c.variant); ++i) {
    const TcLayer& L = rows[i];
    if ((L.flags & TC_MASK_ONLY) && !mask) continue;
    const bool no_tail = (L.flags & TC_MASK_TAIL) && !mask;
    if (L.flatten && !c.fim_ready)           // (in the iteration loop the lookup kernel has already produced the planes)
      RAFT_TRY(launch(flow_im2col_kernel, grid_for((size_t)c.B * c.h * c.w * 128), 256, 0, c.stream, W.flow, c.B, c.h, c.w,
                      W.fim_hi, W.fim_lo));
    TcConvParams p;
    memset(&p, 0, sizeof(p));
    int chunks = 0;
    for (int s = 0; s < 2 && L.seg[s].chunks; ++s) {
      const Plane& a = planes[L.seg[s].plane];
      RAFT_TRY(make_tmap_act2(&p.a_map[s], a.hi, a.lo, c.B, c.h, c.w, a.stride, tw, th));
      p.seg_chunks[s] = L.seg[s].chunks;
      p.seg_c0[s] = L.seg[s].c0;
      chunks += L.seg[s].chunks;
      p.nseg = s + 1;
    }
    if (chunks * kChunkK != L.cin_pad) return RAFT_ERR_BAD_SHAPE;
    const int nsplit = tc_n_split(L.bn);                // layers wider than kMaxTileN run as more column tiles
    if (!nsplit) return RAFT_ERR_BAD_SHAPE;
    RAFT_TRY(tc_use_weights(p, c.prepared, c.PL.tc[i], L.bn / nsplit));
    p.ph = (L.kh - 1) / 2; p.pw = (L.kw - 1) / 2;
    p.B = c.B; p.H = c.h; p.W = c.w; p.TH = th; p.TW = tw;
    // Promotion group of the update-block layers: 2 chunks (24-MMA chains).  Their K = 1920 GRU contractions feed a
    // 12-iteration recurrence (DESIGN.md section 4).
    p.group_chunks = 2;
    p.mode = L.mode; p.act = L.act; p.out_scale = L.out_scale;
    p.n_total = no_tail ? L.n_total - L.bn : L.n_total;
    if (L.out == OUT_DELTA) { p.out_f32 = delta; p.f32_stride = 2; }
    else if (L.out == OUT_MASK) { p.out_f32 = mask; p.f32_stride = 576; }
    else { p.out_hi = planes[L.out].hi; p.out_lo = planes[L.out].lo; p.h_stride = planes[L.out].stride; p.h_c0 = L.out_c0; }
    if (L.flags & TC_CONCAT_FLOW) { p.concat_src = W.flow; p.concat_n = 2; }
    if (L.mode != EPI_LINEAR) { p.z = W.z; p.h = h; p.hid = d.hid; }
    if ((L.flags & TC_ADVANCE) && adv_coords) { p.adv_coords = adv_coords; p.adv_flow = W.flow; }
    const int n_tiles_n = (no_tail ? L.ntn - 1 : L.ntn) * nsplit;
    if (c.plan && c.plan->P.nlayers != i) return RAFT_ERR_UNSUPPORTED;   // a dependency names its source by row index
    RAFT_TRY(c.plan ? mega_add(*c.plan, p, n_tiles_n, L.ndep, L.dep) : tc_launch(p, n_tiles_n, c.stream));
  }
  return 0;
}

}  // namespace raft
