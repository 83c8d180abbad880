// CorrBlock.retrieve (tf_raft/layers/corr.py:116-152) for the model's configurations (radius 4 / 3, 4 levels): the
// HBM gather of the recurrent loop.
//
// One warp per (query pixel, pyramid level).  The (2r+1)^2 floor/ceil-bilinear taps of one such item read a footprint
// of at most (2r+2) x (2r+2) texels of the query's H x W correlation plane, so the warp
//   1. computes the 2*(2r+1) per-axis tap set-ups (clamp, floor, ceil, weights -- corr.py:40-60) once, lanes 0..2S-1;
//   2. copies the footprint (<= 11 rows x 16 columns, 16-byte aligned row segments) from global to shared memory with
//      two 128-bit loads per lane -- every texel is fetched once, coalesced, instead of four scalar gathers per tap;
//   3. evaluates the taps from shared memory: lane = (x offset a, b mod 3), three taps per lane, the x set-up of the
//      lane is read once.  Each tap is the reference expression op by op with individually rounded fp32 operations
//      (__fmul_rn / __fadd_rn), so the output is bit-identical to the oracle, quirks included (integer or clamped
//      coordinate => 0, x-major tap order, fl(fl(c / 2^l) + d)).
// About 140 warp instructions per item instead of the 469 of the gather-per-tap kernel (kernels.cuh, kept for other
// radii / level counts and as the per-item escape when a footprint does not fit the window).
//
// corr_lookup_win_grid_kernel is the same kernel with the grid_sample sampler (RAFT_SAMPLER_GRID, kernels.cuh): the
// set-up lanes compute RAFT's normalisation and ATen's unnormalisation op by op, a corner outside the level is marked
// (offset -1) and never read, and the footprint is the intersection of the taps' corners with the level -- it may be
// empty.  Its corners still span at most 2r+2 texels per axis, so the window bound holds.  Sum order of one tap: acc =
// +0, then (y0,x0), (y0,x1), (y1,x0), (y1,x1), each in-frame corner adding fl(fl(wy * wx) * texel) (weight 0 included,
// so a NaN texel there reaches the tap as in ATen).
#pragma once
#include "kernels.cuh"

namespace raft {

constexpr int kWinPitch = 20;     // floats per window row: 16 columns + 4 (banks of the three row groups stay apart)
constexpr int kWinRows = 11;

// Per-item state that travels from the set-up / load phase to the tap phase one loop iteration later.
struct LookupItem {
  float w1, w0;          // this lane's axis set-up (lanes [0,S): x, [S,2S): y): weights of the floor / ceil corner
  int off0, off1;        // ... and window offsets of the two corners (x: columns, y: rows * pitch)
  int ok;                // footprint fits the window (always, by construction; else the item takes the gather escape)
  float cx, cy;          // level coordinates (escape path only)
};

template <int R, int L, bool kVec, bool kHalf, bool kGrid>
__device__ __forceinline__ void corr_lookup_win_body(const LookupParams& p) {
  constexpr int S = 2 * R + 1, NT = S * S;
  constexpr int NJ = (S + 2) / 3;                                   // taps per lane
  constexpr int NV = kVec ? 2 : 6;                                  // window registers per lane (float4 / float)
  static_assert(S <= 10 && 3 * S <= 32, "lane = (a, b mod 3) needs 3 * (2r+1) lanes");
  static_assert((L & (L - 1)) == 0, "level = work item mod L must be constant per warp (grid stride is a multiple of L)");
  __shared__ float4 ax_s[8][32];                                    // per warp: [0,16) x set-ups, [16,32) y set-ups
  __shared__ __align__(16) float win_s[8][kWinRows * kWinPitch];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  float4* ax = ax_s[wib];
  float* win = win_s[wib];
  const int a = lane / 3, bq = lane - 3 * a;                        // this lane's taps: (a, bq + 3j)
  // The grid stride (8 warps per block) is a multiple of L, so a warp meets ONE level: everything that depends on the
  // level only is computed once, and the per-query pointers advance by constants.
  const int l = wib % L;
  const int H = p.lh[l], W = p.lw[l];
  const float inv = 1.0f / (float)(1 << l);                         // exact power of two
  const unsigned q0 = (blockIdx.x * 8u + wib) / L, qstep = gridDim.x * (8u / L);
  // element offsets stay below 2^31 (host-checked), so the per-query advance is one 32-bit add per pointer
  const float* const img_base = p.pyr[l];
  unsigned img_off = q0 * (unsigned)(H * W);
  const unsigned img_step = qstep * (unsigned)(H * W);
  const float2* cptr = reinterpret_cast<const float2*>(p.coords) + q0;
  const unsigned ostride = (unsigned)(kHalf ? p.h_stride : p.out_stride);
  unsigned o_off = q0 * ostride + (unsigned)(l * NT);
  const unsigned o_step = qstep * ostride;
  const int npad = (kHalf && l == L - 1) ? p.h_pad - L * NT : 0;   // zero channels behind the last level (operand planes)
  // set-up lanes: [0,S) x, [S,2S) y (the other lanes compute a harmless duplicate)
  const bool isy = lane >= S;
  const int i = min(isy ? lane - S : lane, S - 1);
  const float fi = (float)(i - R), fmax_dim = (float)((isy ? H : W) - 1);
  const int t0 = a * S + bq;                                        // x-major tap order (corr.py:133-143): t = a * S + b
  // window element k of this lane sits at (row, column) = (wrow(k), wcol(k)) of the footprint: its global offset from the
  // footprint origin and its shared-memory offset are per-lane constants of the level
  auto wrow = [&](int k) { const int e = lane + 32 * k; return kVec ? e >> 2 : e >> 4; };
  auto wcol = [&](int k) { const int e = lane + 32 * k; return kVec ? (e & 3) << 2 : e & 15; };
  int goff[NV], soff[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    goff[k] = wrow(k) * W + wcol(k);
    soff[k] = wrow(k) < kWinRows ? wrow(k) * kWinPitch + wcol(k) : -1;      // -1: this lane has no element k
  }

  // Software pipeline: the set-up and the footprint LOADS of item n+1 are issued before the taps of item n are
  // evaluated, so every warp has one footprint in flight while it computes (the kernel is latency-bound otherwise:
  // ~10 items per warp, each a DRAM round trip).
  LookupItem it;
  float4 wv4[kVec ? NV : 1];
  float wv1[kVec ? 1 : NV];
  unsigned wmask = 0;                                               // which of this lane's window elements are loaded

  auto stage = [&](float2 c, const float* img_q) {                  // set-up + loads of one item
    const float cx = __fmul_rn(c.x, inv), cy = __fmul_rn(c.y, inv); // coords / 2**i  (corr.py:141)
    int i0, i1, lo, hi;                                             // corners; this lane's share of the footprint
    float g, g0, g1;                                                // coordinate and its floor / ceil corners
    if constexpr (kGrid) {
      // the taps' ix are non-decreasing in the tap index wherever a corner can lie in the level (-100 only stands for
      // values far outside or NaN, which are so for every tap): tap 0's x0 and tap S-1's x0 + 1, clipped to the level,
      // bound every in-frame corner.  lo > hi: no corner of this axis is in the frame.
      g = grid_unnormalize(__fadd_rn(isy ? cy : cx, fi), fmax_dim);
      g0 = floorf(g);
      g1 = __fadd_rn(g0, 1.0f);
      i0 = (g0 >= 0.0f && g0 <= fmax_dim) ? (int)g0 : -1;
      i1 = (g1 >= 0.0f && g1 <= fmax_dim) ? (int)g1 : -1;
      lo = (int)fminf(fmaxf(g0, 0.0f), __fadd_rn(fmax_dim, 1.0f));
      hi = (int)fmaxf(fminf(g1, fmax_dim), -1.0f);
    } else {
      g = fminf(fmaxf(__fadd_rn(isy ? cy : cx, fi), 0.0f), fmax_dim);   // centroid + delta, clamp
      g0 = floorf(g);
      g1 = ceilf(g);
      i0 = (int)g0; i1 = (int)g1;
      lo = i0; hi = i1;
    }
    const int bx = __shfl_sync(0xffffffffu, lo, 0), by = __shfl_sync(0xffffffffu, lo, S);
    const int ex = __shfl_sync(0xffffffffu, hi, S - 1), ey = __shfl_sync(0xffffffffu, hi, 2 * S - 1);
    const int bxa = kVec ? (bx & ~3) : bx;                          // first window column (16-byte aligned when vectorised)
    it.w1 = __fsub_rn(g1, g);                                       // weights of the floor / ceil corner
    it.w0 = __fsub_rn(g, g0);
    it.off0 = (isy ? (i0 - by) * kWinPitch : i0 - bxa) * 4;           // BYTE offsets inside the window
    it.off1 = (isy ? (i1 - by) * kWinPitch : i1 - bxa) * 4;
    if constexpr (kGrid) {                                          // -1: the corner lies outside the level
      if (i0 < 0) it.off0 = -1;
      if (i1 < 0) it.off1 = -1;
    }
    it.ok = (ex - bxa < 16 && ey - by < kWinRows) ? 1 : 0;
    it.cx = cx;
    it.cy = cy;
    wmask = 0;
    if (it.ok) {
      const float* src = img_q + by * W + bxa;
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        if (soff[k] >= 0 && wrow(k) <= ey - by && wcol(k) <= ex - bxa) {
          wmask |= 1u << k;
          if constexpr (kVec) wv4[k] = __ldg(reinterpret_cast<const float4*>(src + goff[k]));
          else wv1[k] = __ldg(src + goff[k]);
        }
      }
    }
  };

  if (q0 < (unsigned)p.nq) stage(__ldg(cptr), img_base + img_off);
  float2 cnext = make_float2(0.f, 0.f);
  if (q0 + qstep < (unsigned)p.nq) cnext = __ldg(cptr + qstep);
  for (unsigned q = q0; q < (unsigned)p.nq; q += qstep) {
    // ---- publish the staged item (set-ups, footprint) to shared memory ----
    const int ok = it.ok;
    const float ecx = it.cx, ecy = it.cy;
    __syncwarp();                                                   // previous item's readers are done with ax / win
    if (lane < 2 * S) ax[(isy ? 16 : 0) + i] = make_float4(it.w1, it.w0, __int_as_float(it.off0), __int_as_float(it.off1));
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      if ((wmask >> k) & 1u) {
        if constexpr (kVec) *reinterpret_cast<float4*>(win + soff[k]) = wv4[k];
        else win[soff[k]] = wv1[k];
      }
    }
    __syncwarp();
    // ---- stage the next item: its loads are in flight while this one's taps are evaluated ----
    const unsigned img_cur = img_off;
    img_off += img_step;
    if (q + qstep < (unsigned)p.nq) {
      const float2 c = cnext;
      cptr += qstep;
      if (q + 2 * qstep < (unsigned)p.nq) cnext = __ldg(cptr + qstep);
      stage(c, img_base + img_off);
    }
    // ---- taps of the current item ----
    if (ok) {
      if (a < S) {
        const float4 sx = ax[a];                                    // (w1, w0, byte off0, byte off1)
        const char* w0p = reinterpret_cast<const char*>(win) + __float_as_int(sx.z);
        const char* w1p = reinterpret_cast<const char*>(win) + __float_as_int(sx.w);
        __half* ohq = kHalf ? p.out_hi + o_off + t0 : nullptr;
        __half* olq = kHalf ? p.out_lo + o_off + t0 : nullptr;
        float* oq = kHalf ? nullptr : p.out + o_off + t0;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          if (S % 3 == 0 || bq + 3 * j < S) {
            const float4 sy = ax[16 + bq + 3 * j];
            const int oy0 = __float_as_int(sy.z), oy1 = __float_as_int(sy.w);
            float v;
            if constexpr (kGrid) {
              const int ox0 = __float_as_int(sx.z), ox1 = __float_as_int(sx.w);
              v = 0.0f;
              if (oy0 >= 0 && ox0 >= 0) v = __fadd_rn(v, __fmul_rn(__fmul_rn(sy.x, sx.x), *reinterpret_cast<const float*>(w0p + oy0)));
              if (oy0 >= 0 && ox1 >= 0) v = __fadd_rn(v, __fmul_rn(__fmul_rn(sy.x, sx.y), *reinterpret_cast<const float*>(w1p + oy0)));
              if (oy1 >= 0 && ox0 >= 0) v = __fadd_rn(v, __fmul_rn(__fmul_rn(sy.y, sx.x), *reinterpret_cast<const float*>(w0p + oy1)));
              if (oy1 >= 0 && ox1 >= 0) v = __fadd_rn(v, __fmul_rn(__fmul_rn(sy.y, sx.y), *reinterpret_cast<const float*>(w1p + oy1)));
            } else {
              v = __fmul_rn(__fmul_rn(sy.x, sx.x), *reinterpret_cast<const float*>(w0p + oy0));   // corr.py:68, left to right
              v = __fadd_rn(v, __fmul_rn(__fmul_rn(sy.x, sx.y), *reinterpret_cast<const float*>(w1p + oy0)));
              v = __fadd_rn(v, __fmul_rn(__fmul_rn(sy.y, sx.x), *reinterpret_cast<const float*>(w0p + oy1)));
              v = __fadd_rn(v, __fmul_rn(__fmul_rn(sy.y, sx.y), *reinterpret_cast<const float*>(w1p + oy1)));
            }
            if constexpr (kHalf) {
              __half hh, ll;
              split_f16(v, hh, ll);
              ohq[3 * j] = hh;
              olq[3 * j] = ll;
            } else {
              oq[3 * j] = v;
            }
          }
        }
      }
    } else {                                                        // escape: gather per tap (never taken in practice)
      for (int t = lane; t < NT; t += 32) {
        const int ta = t / S, tb = t - ta * S;
        const float v = sample_tap<kGrid>(img_base + img_cur, H, W, __fadd_rn(ecx, (float)(ta - R)), __fadd_rn(ecy, (float)(tb - R)));
        if constexpr (kHalf) {
          __half hh, ll;
          split_f16(v, hh, ll);
          p.out_hi[o_off + t] = hh;
          p.out_lo[o_off + t] = ll;
        } else {
          p.out[o_off + t] = v;
        }
      }
    }
    if constexpr (kHalf) {
      const __half zero = __float2half_rn(0.f);
      for (int cpad = NT + lane; cpad < NT + npad; cpad += 32) {    // channels [levels * ntap, h_pad) of the operand planes
        p.out_hi[o_off + cpad] = zero;
        p.out_lo[o_off + cpad] = zero;
      }
    }
    o_off += o_step;
  }
  if (p.im_flow)
    flow_im2col_rider(p.im_flow, p.im_B, p.im_h, p.im_w, p.im_hi, p.im_lo, (size_t)blockIdx.x * blockDim.x + threadIdx.x,
                      (size_t)gridDim.x * blockDim.x);
}
template <int R, int L, bool kVec, bool kHalf>
__global__ void __launch_bounds__(256, 4) corr_lookup_win_kernel(const LookupParams p) {
  corr_lookup_win_body<R, L, kVec, kHalf, false>(p);
}
template <int R, int L, bool kVec, bool kHalf>
__global__ void __launch_bounds__(256, 4) corr_lookup_win_grid_kernel(const LookupParams p) {
  corr_lookup_win_body<R, L, kVec, kHalf, true>(p);
}

// The window kernel instantiation for (radius, levels) in {(4,4), (3,4)} and the sampler (RAFT_SAMPLER_*); null when
// the configuration has none.
using LookupKernel = void (*)(LookupParams);
template <template <int, int, bool, bool> class K>
struct WinKernels {
  static LookupKernel pick(int radius, bool vec, bool half) {
    if (radius == 4) {
      if (vec) return half ? K<4, 4, true, true>::fn : K<4, 4, true, false>::fn;
      return half ? K<4, 4, false, true>::fn : K<4, 4, false, false>::fn;
    }
    if (vec) return half ? K<3, 4, true, true>::fn : K<3, 4, true, false>::fn;
    return half ? K<3, 4, false, true>::fn : K<3, 4, false, false>::fn;
  }
};
template <int R, int L, bool V, bool H> struct WinTf { static constexpr LookupKernel fn = corr_lookup_win_kernel<R, L, V, H>; };
template <int R, int L, bool V, bool H> struct WinGrid { static constexpr LookupKernel fn = corr_lookup_win_grid_kernel<R, L, V, H>; };
inline LookupKernel lookup_win_kernel(const LookupParams& p, int levels, int radius, int sampler) {
  const size_t nwork = (size_t)p.nq * levels;
  if (levels != 4 || (radius != 4 && radius != 3) || nwork >= (1u << 31)) return nullptr;
  if ((size_t)p.nq * p.lh[0] * p.lw[0] >= (1u << 31) || (size_t)p.nq * (size_t)(p.out_hi ? p.h_stride : p.out_stride) >= (1u << 31))
    return nullptr;                                                  // 32-bit element offsets inside the kernel
  bool vec = true;                                                  // 128-bit loads need 16-byte aligned rows on every level
  for (int l = 0; l < levels; ++l)
    vec = vec && (p.lw[l] % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.pyr[l]) & 15) == 0);
  const bool half = p.out_hi != nullptr;
  if (half == (p.out != nullptr)) return nullptr;                    // exactly one of the two output forms
  return sampler == RAFT_SAMPLER_GRID ? WinKernels<WinGrid>::pick(radius, vec, half) : WinKernels<WinTf>::pick(radius, vec, half);
}

}  // namespace raft
