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
// Tensor-core layers: one or two reference convs merged along cout, cin remapped onto the
// 64-channel-aligned operand planes.
// ------------------------------------------------------------------------------------------------
struct TcLayerSpec {
  int nsrc, src[2];            // reference conv indices merged along cout
  int kh, kw;
  int cin_pad, cout_pad;       // packed dims
  TcCinMap cin_map;
  int bn, ntn;                 // N per column tile, column tiles (launch_tc_layer splits bn > kMaxTileN further)
  int flatten;                 // 1: (kh,kw,cin) flattened into the channel axis -- the layer runs as a 1x1 conv on im2col planes
};

static const TcLayerSpec kBasicTc[12] = {
    /*T0 convc1 */ {1, {BC1, -1}, 1, 1, 384, 256, {1, {0, 0}, {324, 0}, {0, 0}}, 256, 1},
    /*T1 convc2 */ {1, {BC2, -1}, 3, 3, 256, 192, {1, {0, 0}, {256, 0}, {0, 0}}, 192, 1},
    /*T2 convf2 */ {1, {BF2, -1}, 3, 3, 128, 64, {1, {0, 0}, {128, 0}, {0, 0}}, 64, 1},
    /*T3 conv   */ {1, {BCV, -1}, 3, 3, 256, 128, {1, {0, 0}, {256, 0}, {0, 0}}, 128, 1},
    /*T4 zr1    */ {2, {BZ1, BR1}, 1, 5, 384, 256, {1, {0, 0}, {384, 0}, {0, 0}}, 256, 1},
    /*T5 q1     */ {1, {BQ1, -1}, 1, 5, 384, 128, {1, {0, 0}, {384, 0}, {0, 0}}, 128, 1},
    /*T6 zr2    */ {2, {BZ2, BR2}, 5, 1, 384, 256, {1, {0, 0}, {384, 0}, {0, 0}}, 256, 1},
    /*T7 q2     */ {1, {BQ2, -1}, 5, 1, 384, 128, {1, {0, 0}, {384, 0}, {0, 0}}, 128, 1},
    /*T8 fh1|m0 */ {2, {BFH1, BM0}, 3, 3, 128, 512, {1, {0, 0}, {128, 0}, {0, 0}}, 256, 2},
    /*T9 fh2    */ {1, {BFH2, -1}, 3, 3, 256, 16, {1, {0, 0}, {256, 0}, {0, 0}}, 16, 1},
    /*T10 mask2 */ {1, {BM2, -1}, 1, 1, 256, 576, {1, {0, 0}, {256, 0}, {0, 0}}, 192, 3},
    /*T11 convf1*/ {1, {BF1, -1}, 1, 1, 128, 128, {1, {0, 0}, {98, 0}, {0, 0}}, 128, 1, 1}};

static const TcLayerSpec kSmallTc[8] = {
    /*S0 convc1 */ {1, {SC1, -1}, 1, 1, 256, 96, {1, {0, 0}, {196, 0}, {0, 0}}, 96, 1},
    /*S1 convf2 */ {1, {SF2, -1}, 3, 3, 64, 32, {1, {0, 0}, {64, 0}, {0, 0}}, 32, 1},
    /*S2 conv   */ {1, {SCV, -1}, 3, 3, 128, 96, {1, {0, 0}, {128, 0}, {0, 0}}, 96, 1},
    /*S3 zr     */ {2, {SZ, SR}, 3, 3, 320, 192, {2, {0, 96}, {96, 146}, {0, 128}}, 192, 1},
    /*S4 q      */ {1, {SQ, -1}, 3, 3, 320, 96, {2, {0, 96}, {96, 146}, {0, 128}}, 96, 1},
    /*S5 fh1    */ {1, {SFH1, -1}, 3, 3, 128, 128, {1, {0, 0}, {96, 0}, {0, 0}}, 128, 1},
    /*S6 fh2    */ {1, {SFH2, -1}, 3, 3, 128, 16, {1, {0, 0}, {128, 0}, {0, 0}}, 16, 1},
    /*S7 convf1 */ {1, {SF1, -1}, 1, 1, 128, 64, {1, {0, 0}, {98, 0}, {0, 0}}, 64, 1, 1}};

inline int n_tc_layers(int variant) { return variant == RAFT_VARIANT_BASIC ? 12 : 8; }
inline const TcLayerSpec* tc_layers(int variant) { return variant == RAFT_VARIANT_BASIC ? kBasicTc : kSmallTc; }

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
    const TcLayerSpec* tl = tc_layers(variant);
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

// One tensor-core layer.  Operand planes: up to two K segments (hi/lo plane pair, channel stride,
// first channel, number of 64-channel chunks).
struct TcSeg { const __half* hi; const __half* lo; int stride, c0, chunks; };

inline int launch_tc_layer(const UpdateCtx& c, int layer, int nseg, const TcSeg* segs, TcConvParams& p, int ntn = -1,
                           const TcDeps& deps = TcDeps{0, {-1, -1}, {-1, -1}}) {
  const TcLayerSpec& L = tc_layers(c.variant)[layer];
  int tw, th;
  tc_pick_tile(c.w, c.h, &tw, &th);
  p.nseg = nseg;
  int chunks = 0;
  for (int i = 0; i < nseg; ++i) {
    RAFT_TRY(make_tmap_act2(&p.a_map[i], segs[i].hi, segs[i].lo, c.B, c.h, c.w, segs[i].stride, tw, th));
    p.seg_chunks[i] = segs[i].chunks;
    p.seg_c0[i] = segs[i].c0;
    chunks += segs[i].chunks;
  }
  if (chunks * kChunkK != L.cin_pad) return RAFT_ERR_BAD_SHAPE;
  const int nsplit = tc_n_split(L.bn);                // layers wider than kMaxTileN run as more column tiles
  if (!nsplit) return RAFT_ERR_BAD_SHAPE;
  RAFT_TRY(tc_use_weights(p, c.prepared, c.PL.tc[layer], L.bn / nsplit));
  p.ph = (L.kh - 1) / 2; p.pw = (L.kw - 1) / 2;
  p.B = c.B; p.H = c.h; p.W = c.w; p.TH = th; p.TW = tw;
  if (p.out_scale == 0.0f) p.out_scale = 1.0f;
  // Promotion group of the update-block layers: 2 chunks (24-MMA chains).  Their K = 1920 GRU contractions feed a
  // 12-iteration recurrence (DESIGN.md section 4).
  p.group_chunks = 2;
  const int n_tiles_n = (ntn > 0 ? ntn : L.ntn) * nsplit;
  if (c.plan) return mega_add(*c.plan, layer, p, n_tiles_n, nsplit, deps);
  return tc_launch(p, n_tiles_n, c.stream);
}

}  // namespace raft
