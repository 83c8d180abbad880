// Feature / context encoders (tf_raft/layers/extractor.py:88-175) on the tensor-core path.
//   conv1 7x7 s2 (Cin = 3, K = 147: CUDA cores, image normalisation 2*(x/255)-1 fused into the load)
//   6 ResBlocks (extractor.py:19-49): 3x3 convs on conv_tc_kernel; stride-2 convs fetch their A operand with
//   TMA elementStrides = 2 (Keras 'same' is asymmetric there: pad 0 before / 1 after); 1x1 s2 downsample.
//   conv2 1x1.
// Norms: 'batch' in inference is a per-channel affine folded into the conv epilogue (everything fuses);
// 'instance' (and 'batch' in training) need statistics of the raw conv output: two deterministic reduction
// passes + one apply kernel that also does ReLU, the residual add and the fp16 hi/lo re-split.
#pragma once
#include <algorithm>

#include "lookup.cuh"
#include "update.cuh"

namespace raft {

enum { NORM_NONE = 0, NORM_INSTANCE = 1, NORM_BATCH = 2 };

struct EncSpec { int c0; int c[3]; int s[3]; };
inline EncSpec enc_spec(int variant) {
  if (variant == RAFT_VARIANT_BASIC) return {64, {64, 96, 128}, {1, 2, 2}};
  return {32, {32, 64, 96}, {1, 2, 2}};
}
inline int pad64(int c) { return round_up(c, 64); }

struct EncNormSlot { size_t gamma, beta, fscale, fshift; int C; };
struct EncLayout {
  TcWeightSlot conv1;                         // stem as a 1x1 conv over the 147 (->192) im2col channels
  EncNormSlot norm1;
  TcWeightSlot bc1[6], bc2[6], bds[6];
  EncNormSlot bn1[6], bn2[6], bnd[6];
  int has_ds[6], bc[6], bstride[6];
  TcWeightSlot conv2;
  size_t total;
};

inline EncLayout enc_layout(int variant, int out_dim) {
  EncLayout L;
  memset(&L, 0, sizeof(L));
  const EncSpec S = enc_spec(variant);
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
  auto conv_slot = [&](int kh, int kw, int cin, int cout) { return tc_weight_slot(off, kh, kw, pad64(cin), round_up(cout, 32)); };
  auto norm_slot = [&](int C) {
    EncNormSlot n;
    n.C = C;
    n.gamma = take(sizeof(float) * (C + 64)); n.beta = take(sizeof(float) * (C + 64));
    n.fscale = take(sizeof(float) * (C + 64)); n.fshift = take(sizeof(float) * (C + 64));
    return n;
  };
  L.conv1 = conv_slot(1, 1, 147, S.c0);
  L.norm1 = norm_slot(S.c0);
  int cin = S.c0;
  for (int k = 0; k < 6; ++k) {
    const int c = S.c[k / 2], st = (k % 2 == 0) ? S.s[k / 2] : 1;
    L.bc[k] = c; L.bstride[k] = st;
    L.bc1[k] = conv_slot(3, 3, cin, c);
    L.bc2[k] = conv_slot(3, 3, c, c);
    L.bn1[k] = norm_slot(c);
    L.bn2[k] = norm_slot(c);
    L.has_ds[k] = st != 1;
    if (L.has_ds[k]) { L.bds[k] = conv_slot(1, 1, cin, c); L.bnd[k] = norm_slot(c); }
    cin = c;
  }
  L.conv2 = conv_slot(1, 1, cin, out_dim);
  L.total = off;
  return L;
}

struct EncWs {
  float *X32, *O32, *Y32, *D32;
  __half *Xh, *Xl, *Oh, *Ol, *Fh, *Fl, *Ih, *Il;
  float *part, *mean, *mult;
  size_t total;
};
constexpr int kNormSplit = 64;
inline EncWs enc_ws_layout(void* base, int variant, int N, int H, int W) {
  EncWs E;
  memset(&E, 0, sizeof(E));
  const EncSpec S = enc_spec(variant);
  size_t max32 = 0, max16 = 0;
  for (int l = 0; l < 3; ++l) {
    const int d = 2 << l;
    const size_t np = (size_t)N * ((H + d - 1) / d) * ((W + d - 1) / d);
    const int c = l == 0 ? (S.c0 > S.c[0] ? S.c0 : S.c[0]) : S.c[l];
    if (np * c > max32) max32 = np * c;
    if (np * pad64(c) > max16) max16 = np * pad64(c);
  }
  uint8_t* b8 = reinterpret_cast<uint8_t*>(base);
  size_t off = 0;
  auto take = [&](size_t bytes) { uint8_t* p = b8 + off; off = align_up(off + bytes, 1024); return p; };
  E.X32 = (float*)take(max32 * 4); E.O32 = (float*)take(max32 * 4);
  E.Y32 = (float*)take(max32 * 4); E.D32 = (float*)take(max32 * 4);
  E.Xh = (__half*)take(max16 * 2); E.Xl = (__half*)take(max16 * 2);
  E.Oh = (__half*)take(max16 * 2); E.Ol = (__half*)take(max16 * 2);
  E.Fh = (__half*)take(max16 * 2); E.Fl = (__half*)take(max16 * 2);
  {
    const size_t np1 = (size_t)N * ((H + 1) / 2) * ((W + 1) / 2);
    E.Ih = (__half*)take(np1 * 192 * 2); E.Il = (__half*)take(np1 * 192 * 2);
  }
  E.part = (float*)take((size_t)N * kNormSplit * 3 * 256 * 4);
  E.mean = (float*)take((size_t)N * 256 * 4);
  E.mult = (float*)take((size_t)N * 256 * 4);
  E.total = off;
  return E;
}

// ---- prepare ----------------------------------------------------------------------------------
// Packs one convolution after checking that it has the shape (kh, kw, cin, cout); flatten: the 7x7 stem, as a 1x1 conv.
inline int enc_pack_conv(const raft_conv& cv, int kh, int kw, int cin, int cout, const TcWeightSlot& s, bool flatten,
                         uint8_t* base, cudaStream_t st) {
  if (!cv.kernel || !cv.bias) return RAFT_ERR_BAD_ARG;
  if (cv.kh != kh || cv.kw != kw || cv.cin != cin || cv.cout != cout) return RAFT_ERR_BAD_SHAPE;
  const raft_conv* src[1] = {&cv};
  return tc_pack_weights(base, s, src, 1, nullptr, flatten, st);
}

inline int enc_pack_norm(const raft_norm& nm, const EncNormSlot& s, int norm_type, uint8_t* base, cudaStream_t st) {
  if (norm_type == NORM_NONE) return 0;
  if (!nm.gamma || !nm.beta) return RAFT_ERR_BAD_ARG;
  float* g = reinterpret_cast<float*>(base + s.gamma);
  float* b = reinterpret_cast<float*>(base + s.beta);
  RAFT_CUDA_TRY(cudaMemcpyAsync(g, nm.gamma, s.C * sizeof(float), cudaMemcpyDeviceToDevice, st));
  RAFT_CUDA_TRY(cudaMemcpyAsync(b, nm.beta, s.C * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (norm_type == NORM_BATCH) {
    if (!nm.moving_mean || !nm.moving_variance) return RAFT_ERR_BAD_ARG;
    return launch(bn_fold_kernel, ceil_div(s.C, 128), 128, 0, st, nm.gamma, nm.beta, nm.moving_mean, nm.moving_variance,
                  1e-3f, s.C, reinterpret_cast<float*>(base + s.fscale), reinterpret_cast<float*>(base + s.fshift));
  }
  return raft_launch_status();
}

inline int encoder_prepare(int variant, int norm_type, int out_dim, const raft_encoder_weights* w, void* prepared,
                           size_t bytes, cudaStream_t st) {
  const EncLayout L = enc_layout(variant, out_dim);
  if (L.total > bytes) return RAFT_ERR_WORKSPACE;
  const EncSpec S = enc_spec(variant);
  uint8_t* base = reinterpret_cast<uint8_t*>(prepared);
  RAFT_CUDA_TRY(cudaMemsetAsync(base, 0, L.total, st));
  RAFT_TRY(enc_pack_conv(w->conv1, 7, 7, 3, S.c0, L.conv1, true, base, st));
  RAFT_TRY(enc_pack_norm(w->norm1, L.norm1, norm_type, base, st));
  int cin = S.c0;
  for (int k = 0; k < 6; ++k) {
    const int c = L.bc[k];
    RAFT_TRY(enc_pack_conv(w->block[k].conv1, 3, 3, cin, c, L.bc1[k], false, base, st));
    RAFT_TRY(enc_pack_conv(w->block[k].conv2, 3, 3, c, c, L.bc2[k], false, base, st));
    RAFT_TRY(enc_pack_norm(w->block[k].norm1, L.bn1[k], norm_type, base, st));
    RAFT_TRY(enc_pack_norm(w->block[k].norm2, L.bn2[k], norm_type, base, st));
    if (L.has_ds[k]) {
      RAFT_TRY(enc_pack_conv(w->block[k].downsample, 1, 1, cin, c, L.bds[k], false, base, st));
      RAFT_TRY(enc_pack_norm(w->block[k].downsample_norm, L.bnd[k], norm_type, base, st));
    }
    cin = c;
  }
  RAFT_TRY(enc_pack_conv(w->conv2, 1, 1, cin, out_dim, L.conv2, false, base, st));
  return raft_launch_status();
}

// ---- forward ----------------------------------------------------------------------------------
struct EncCtx {
  const uint8_t* prep; EncLayout L; EncWs W; cudaStream_t st;
  int N, norm_type, stats;    // stats: 1 = statistics from the data (instance, or batch in training)
  int per_image;              // instance: one group per image; batch-training: one group
};

// y (npix, C) raw conv output -> normalised, activated, (+skip), re-split.
inline int enc_norm_apply(const EncCtx& c, const EncNormSlot& ns, const float* y, size_t npix, int P, int relu,
                          const float* skip32, const __half* skip_hi, const __half* skip_lo, float* out32, __half* hi,
                          __half* lo) {
  const int C = ns.C, G = c.per_image ? c.N : 1;
  const int Pg = c.per_image ? P : (int)npix;
  const float* gamma = reinterpret_cast<const float*>(c.prep + ns.gamma);
  const float* beta = reinterpret_cast<const float*>(c.prep + ns.beta);
  // (Finalisation is a separate launch: inside norm_stats_kernel the merge of C channels by the last block of a group would
  //  be serial, where norm_final_kernel spreads it over G*C warps.)
  RAFT_TRY(launch(norm_stats_kernel, dim3((unsigned)G, kNormSplit), 256, 0, c.st, y, Pg, C, kNormSplit, c.W.part));
  RAFT_TRY(launch(norm_final_kernel, ceil_div(G * C * 32, 256), 256, 0, c.st, c.W.part, G, C, kNormSplit, gamma, 1e-3f,
                  c.W.mean, c.W.mult));
  return launch(norm_apply_kernel, grid_for(npix * (pad64(C) / 8)), 256, 0, c.st, y, npix, P, C, c.per_image, c.W.mean,
                c.W.mult, beta, relu, skip32, skip_hi, skip_lo, out32, hi, lo, pad64(C));
}

// One tensor-core convolution of the encoder, cout output channels.  When the norm needs data statistics the raw output
// goes to `raw32` (bias only); otherwise the folded affine, activation and skip are applied in the epilogue.
inline int enc_conv_tc(const EncCtx& c, const TcWeightSlot& cs, int cout, const EncNormSlot* ns, const __half* ahi,
                       const __half* alo, int Hin, int Win, int Hout, int Wout, int stride, int relu, const float* skip,
                       float* out32, __half* ohi, __half* olo) {
  TcConvParams p;
  memset(&p, 0, sizeof(p));
  int tw, th;
  tc_pick_tile(Wout, Hout, &tw, &th);
  if (tw * stride > 256) tw = 128 / stride, th = 128 / tw;
  const int nsplit = tc_n_split(cs.cout_pad);          // layers wider than kMaxTileN run as more column tiles
  if (!nsplit) return RAFT_ERR_BAD_SHAPE;
  RAFT_TRY(make_tmap_act2(&p.a_map[0], ahi, alo, c.N, Hin, Win, cs.cin_pad, tw, th, stride));
  RAFT_TRY(tc_use_weights(p, c.prep, cs, cs.cout_pad / nsplit));
  p.nseg = 1; p.seg_chunks[0] = cs.cin_pad / kChunkK; p.seg_c0[0] = 0;
  p.stride = stride;
  // Keras 'same': stride 1 -> (k-1)/2 before; stride 2 on even input -> total k-2, before = (k-2)/2 (0 for 3x3);
  // 1x1 convs are 'valid' (no padding).
  if (stride == 1) { p.ph = (cs.kh - 1) / 2; p.pw = (cs.kw - 1) / 2; }
  else {
    const int tot_h = (Hout - 1) * stride + cs.kh - Hin, tot_w = (Wout - 1) * stride + cs.kw - Win;
    p.ph = (tot_h > 0 ? tot_h : 0) / 2; p.pw = (tot_w > 0 ? tot_w : 0) / 2;
  }
  p.B = c.N; p.H = Hout; p.W = Wout; p.TH = th; p.TW = tw;
  p.n_total = cout;
  p.mode = EPI_LINEAR; p.out_scale = 1.0f;
  p.out_f32 = out32; p.f32_stride = cout; p.f32_c0 = 0;
  p.out_hi = ohi; p.out_lo = olo; p.h_stride = pad64(cout); p.h_c0 = 0;
  if (ns && !c.stats && c.norm_type == NORM_BATCH) {
    p.post_scale = reinterpret_cast<const float*>(c.prep + ns->fscale);
    p.post_shift = reinterpret_cast<const float*>(c.prep + ns->fshift);
  }
  const bool fused = !(ns && c.stats);
  if (fused) {
    p.act = relu ? ACT_RELU : ACT_NONE;
    p.residual = skip; p.res_stride = cout; p.res_c0 = 0;
  } else {
    p.act = ACT_NONE; p.out_hi = nullptr; p.out_lo = nullptr;
  }
  // Promotion group of the encoder convolutions: their contractions are short (K <= 1152, 18 chunks), so the tensor-core
  // accumulator may run for 5 chunks (60 MMA steps) between IEEE promotions instead of the update block's 2 (its
  // K = 1920 GRU contractions feed a 12-iteration recurrence).
  p.group_chunks = 5;
  return tc_launch(p, nsplit, c.st);
}

// The stem's operand: the 7x7 s2 input window of every output pixel as 192-channel fp16 planes (E.Ih / E.Il of `ws`).
// It depends on the images alone, so encoders of the same images can share it (raft_b200_encode_pair).
inline int encoder_stem_im2col(int variant, const float* images, int N, int H, int W, int image_norm, void* ws,
                               cudaStream_t st) {
  const EncWs E = enc_ws_layout(ws, variant, N, H, W);
  const int h = (H + 1) / 2, w = (W + 1) / 2;
  const size_t npix = (size_t)N * h * w;
  const int tot_h = (h - 1) * 2 + 7 - H, tot_w = (w - 1) * 2 + 7 - W;
  const float* src = images;
  if (image_norm) {                                 // normalise once (O32 is free until the first ResBlock finishes)
    const size_t nimg = (size_t)N * H * W * 3;
    RAFT_TRY(launch(image_norm_kernel, grid_for(nimg), 256, 0, st, images, E.O32, nimg));
    src = E.O32;
  }
  return launch(stem_im2col_kernel, grid_for(npix * 24), 256, 0, st, src, N, H, W, h, w, (tot_h > 0 ? tot_h : 0) / 2,
                (tot_w > 0 ? tot_w : 0) / 2, 0, E.Ih, E.Il);
}

// stem_hi / stem_lo: the stem planes encoder_stem_im2col built for these images (in this or another workspace of the same
// shape), or null to build them here.
inline int encoder_forward(int variant, int norm_type, int out_dim, const void* prepared, const float* images, int N,
                           int H, int W, int training, int image_norm, float* out, void* ws, size_t ws_bytes, cudaStream_t st,
                           const __half* stem_hi = nullptr, const __half* stem_lo = nullptr) {
  EncCtx c;
  c.prep = reinterpret_cast<const uint8_t*>(prepared);
  c.L = enc_layout(variant, out_dim);
  c.W = enc_ws_layout(ws, variant, N, H, W);
  if (c.W.total > ws_bytes) return RAFT_ERR_WORKSPACE;
  c.st = st; c.N = N; c.norm_type = norm_type;
  c.stats = (norm_type == NORM_INSTANCE) || (norm_type == NORM_BATCH && training);
  c.per_image = norm_type == NORM_INSTANCE;
  const EncSpec S = enc_spec(variant);
  const EncLayout& L = c.L;
  const EncWs& E = c.W;

  // ---- stem: conv1 7x7 s2 + norm1 + relu (extractor.py:120) ----
  // K = 7*7*3 = 147: gather the (normalised) input window of every output pixel into 192-channel fp16 planes
  // and run the stem as a 1x1 tensor-core convolution.
  int h = (H + 1) / 2, w = (W + 1) / 2;
  {
    const size_t npix = (size_t)N * h * w;
    if (!stem_hi) {
      RAFT_TRY(encoder_stem_im2col(variant, images, N, H, W, image_norm, ws, st));
      stem_hi = E.Ih; stem_lo = E.Il;
    }
    if (!c.stats && pad64(S.c0) != S.c0) {
      RAFT_CUDA_TRY(cudaMemsetAsync(E.Xh, 0, npix * pad64(S.c0) * 2, st));
      RAFT_CUDA_TRY(cudaMemsetAsync(E.Xl, 0, npix * pad64(S.c0) * 2, st));
    }
    RAFT_TRY(enc_conv_tc(c, L.conv1, S.c0, &L.norm1, stem_hi, stem_lo, h, w, h, w, 1, 1, nullptr, c.stats ? E.Y32 : E.X32, E.Xh, E.Xl));
    if (c.stats) RAFT_TRY(enc_norm_apply(c, L.norm1, E.Y32, npix, h * w, 1, nullptr, nullptr, nullptr, nullptr, E.Xh, E.Xl));
  }

  float *X32 = E.X32, *O32 = E.O32;
  __half *Xh = E.Xh, *Xl = E.Xl, *Oh = E.Oh, *Ol = E.Ol;
  for (int k = 0; k < 6; ++k) {
    const int st2 = L.bstride[k], cc = L.bc[k];
    const int ho = (h + st2 - 1) / st2, wo = (w + st2 - 1) / st2;
    const size_t npo = (size_t)N * ho * wo;
    const bool zero_pad_out = pad64(cc) != cc;     // fused epilogues write 32-column chunks: clear the 64-pad tail
    // conv1 + norm1 + relu -> F
    if (!c.stats && zero_pad_out) {
      RAFT_CUDA_TRY(cudaMemsetAsync(E.Fh, 0, npo * pad64(cc) * 2, st));
      RAFT_CUDA_TRY(cudaMemsetAsync(E.Fl, 0, npo * pad64(cc) * 2, st));
      RAFT_CUDA_TRY(cudaMemsetAsync(Oh, 0, npo * pad64(cc) * 2, st));
      RAFT_CUDA_TRY(cudaMemsetAsync(Ol, 0, npo * pad64(cc) * 2, st));
    }
    RAFT_TRY(enc_conv_tc(c, L.bc1[k], cc, &L.bn1[k], Xh, Xl, h, w, ho, wo, st2, 1, nullptr, c.stats ? E.Y32 : nullptr, E.Fh, E.Fl));
    if (c.stats) RAFT_TRY(enc_norm_apply(c, L.bn1[k], E.Y32, npo, ho * wo, 1, nullptr, nullptr, nullptr, nullptr, E.Fh, E.Fl));
    // skip branch
    const float* skip = X32;
    if (L.has_ds[k]) {
      RAFT_TRY(enc_conv_tc(c, L.bds[k], cc, &L.bnd[k], Xh, Xl, h, w, ho, wo, st2, 0, nullptr, c.stats ? E.Y32 : E.D32, nullptr, nullptr));
      if (c.stats) RAFT_TRY(enc_norm_apply(c, L.bnd[k], E.Y32, npo, ho * wo, 0, nullptr, nullptr, nullptr, E.D32, nullptr, nullptr));
      skip = E.D32;
    }
    // conv2 + norm2 + relu, then relu(skip + fx) -> O
    RAFT_TRY(enc_conv_tc(c, L.bc2[k], cc, &L.bn2[k], E.Fh, E.Fl, ho, wo, ho, wo, 1, 1, skip, c.stats ? E.Y32 : O32, Oh, Ol));
    if (c.stats) {   // skip = block input: from D32 after a downsample, else from the block's own fp16 operand planes
      if (L.has_ds[k]) RAFT_TRY(enc_norm_apply(c, L.bn2[k], E.Y32, npo, ho * wo, 1, E.D32, nullptr, nullptr, nullptr, Oh, Ol));
      else RAFT_TRY(enc_norm_apply(c, L.bn2[k], E.Y32, npo, ho * wo, 1, nullptr, Xh, Xl, nullptr, Oh, Ol));
    }
    // next block reads O
    float* t32 = X32; X32 = O32; O32 = t32;
    __half* th_ = Xh; Xh = Oh; Oh = th_;
    __half* tl_ = Xl; Xl = Ol; Ol = tl_;
    h = ho; w = wo;
  }
  // conv2 1x1 -> (N, H/8, W/8, out_dim), bias only (extractor.py:125)
  RAFT_TRY(enc_conv_tc(c, L.conv2, out_dim, nullptr, Xh, Xl, h, w, h, w, 1, 0, nullptr, out, nullptr, nullptr));
  return raft_launch_status();
}

}  // namespace raft
