// Training-step kernels (tf_raft/model.py:126-144): backward of the pyramid lookup, global gradient norm, AdamW.
#pragma once
#include "kernels.cuh"

namespace raft {

// ------------------------------------------------------------------------------------------------
// Backward of CorrBlock.retrieve (corr.py:116-152 with bilinear_sampler corr.py:28-69).
//   out[q, l, a, b] = sum over the 4 floor/ceil corners of  wy * wx * P_l[q, iy, ix],
//   gx = clip(cx / 2^l + (a - r), 0, W-1),  wx1 = ceil(gx) - gx (corner x0), wx0 = gx - floor(gx) (corner x1), same in y.
// TensorFlow's gradients: floor / ceil / gather indices contribute nothing; clip_by_value passes the gradient where the
// value lies inside [lo, hi]; so with go = d loss / d out[q, l, a, b]
//   d P_l[q, iy, ix] += wy * wx * go                                  (4 scatter-adds)
//   d gx = go * ( wy1 * (P01 - P00) + wy0 * (P11 - P10) ),  d cx += d gx / 2^l  when 0 <= cx/2^l + (a-r) <= W-1
//   d gy = go * ( wx1 * (P10 - P00) + wx0 * (P11 - P01) ),  d cy likewise.
// Terms are skipped where go == 0 and, for the pyramid, where c = wy * wx == 0; the coordinate terms are gated by the
// clip as above.
//
// Fixed order, no atomics: every result depends on the shape and the data only, so two calls give the same bits.  Each
// operation is one rounded fp32 operation (__fmul_rn / __fadd_rn / __fsub_rn, never contracted into an FMA), so
// oracle/determinism_np.py reproduces every bit in NumPy float32.  With t = a*(2r+1) + b the tap index:
//   d P_l[q] : a touched cell ends as v_in + term_1 + term_2 + ..., added left to right, its terms fl(fl(wy*wx) * go) in
//              ascending t and, within a tap, in corner order 00, 01, 10, 11 (a tap reaches a cell through one corner at
//              most).  Untouched cells are neither read nor written.
//   d coords : per level, lane j (0..31) sums, left to right from +0, the gated d gx of taps j, j+32, j+64, ...; the 32
//              lane sums are combined by the butterfly s_j <- s_j + s_{j xor o}, o = 16, 8, 4, 2, 1, giving G_l (lane 0's
//              value; d gy likewise).  grad_coords[q] ends as in + fl(G_0 * inv_0) + fl(G_1 * inv_1) + ..., added in
//              ascending level l, inv_l = 2^-l.
// One warp per (query, level) owns grad_pyr[l]'s private h_l x w_l slice of that query: first its lanes stride over the
// taps for G_l, then over the (2r+2)^2 cells of the window, each lane gathering a cell's terms in order.  A tap with a
// non-zero x weight has x0 = floor(fl(cx + a - r)) = floor(cx) + a - r exactly (rounding cannot move a non-integer sum
// past an integer), so window column s (0..2r+1) is reached by tap a = s-1 through its x1 corner and by a = s through its
// x0 corner, and by no other tap; rows likewise.  The warps of one query share a block, and one thread per query adds
// their G_l to grad_coords after a barrier.
// ------------------------------------------------------------------------------------------------
struct LookupBwdParams {
  const float* pyr[RAFT_MAX_LEVELS];
  float* gpyr[RAFT_MAX_LEVELS];
  int lh[RAFT_MAX_LEVELS], lw[RAFT_MAX_LEVELS];
  const float* coords;
  const float* gout; int gout_stride;
  float* gcoords;
  int nq, levels, radius;
};

// One axis of one tap: u = c + offset before the clip, g = clip(u, 0, n-1); corner 0 = floor(g) with weight w1 =
// ceil(g) - g, corner 1 = ceil(g) with weight w0 = g - floor(g); `in` is the clip's gradient gate.
struct LookupAxis {
  int i0, i1;
  float w0, w1;
  bool in;
};

__device__ __forceinline__ LookupAxis lookup_axis(float c, int offset, int n) {
  const float u = __fadd_rn(c, (float)offset);
  const float g = fminf(fmaxf(u, 0.0f), (float)(n - 1));
  const float f0 = floorf(g), f1 = ceilf(g);
  LookupAxis ax;
  ax.i0 = (int)f0;
  ax.i1 = (int)f1;
  ax.w1 = __fsub_rn(f1, g);
  ax.w0 = __fsub_rn(g, f0);
  ax.in = u >= 0.0f && u <= (float)(n - 1);
  return ax;
}

// Queries per block for `levels` levels: one warp per (query, level), at most 8 warps.
inline int lookup_bwd_queries_per_block(int levels) { return levels >= 8 ? 1 : 8 / levels; }

__global__ void __launch_bounds__(256) corr_lookup_bwd_kernel(const LookupBwdParams p) {
  __shared__ float level_sum[8][2];                              // G_l of each warp of the block
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qpb = blockDim.x / (32 * p.levels);
  const int l = warp % p.levels;
  const int side = 2 * p.radius + 1, ntap = side * side, ncell = (side + 1) * (side + 1);
  for (size_t q0 = (size_t)blockIdx.x * qpb; q0 < (size_t)p.nq; q0 += (size_t)gridDim.x * qpb) {
    const size_t q = q0 + warp / p.levels;
    if (q < (size_t)p.nq) {
      const int H = p.lh[l], W = p.lw[l];
      const float* img = p.pyr[l] + q * H * W;
      float* gimg = p.gpyr[l] + q * H * W;
      const float* go_row = p.gout + q * p.gout_stride + (size_t)l * ntap;
      const float inv = 1.0f / (float)(1 << l);
      const float cx = __fmul_rn(__ldg(p.coords + 2 * q), inv), cy = __fmul_rn(__ldg(p.coords + 2 * q + 1), inv);
      // coordinate gradient: lanes stride over the taps
      float gcx = 0.0f, gcy = 0.0f;
      for (int t = lane; t < ntap; t += 32) {
        const float go = __ldg(go_row + t);
        if (go == 0.0f) continue;
        const int a = t / side, b = t - a * side;
        const LookupAxis X = lookup_axis(cx, a - p.radius, W), Y = lookup_axis(cy, b - p.radius, H);
        const float p00 = __ldg(img + (size_t)Y.i0 * W + X.i0), p01 = __ldg(img + (size_t)Y.i0 * W + X.i1);
        const float p10 = __ldg(img + (size_t)Y.i1 * W + X.i0), p11 = __ldg(img + (size_t)Y.i1 * W + X.i1);
        const float dgx = __fmul_rn(go, __fadd_rn(__fmul_rn(Y.w1, __fsub_rn(p01, p00)), __fmul_rn(Y.w0, __fsub_rn(p11, p10))));
        const float dgy = __fmul_rn(go, __fadd_rn(__fmul_rn(X.w1, __fsub_rn(p10, p00)), __fmul_rn(X.w0, __fsub_rn(p11, p01))));
        if (X.in) gcx = __fadd_rn(gcx, dgx);
        if (Y.in) gcy = __fadd_rn(gcy, dgy);
      }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        gcx = __fadd_rn(gcx, __shfl_xor_sync(0xffffffffu, gcx, off));
        gcy = __fadd_rn(gcy, __shfl_xor_sync(0xffffffffu, gcy, off));
      }
      if (lane == 0) {
        level_sum[warp][0] = gcx;
        level_sum[warp][1] = gcy;
      }
      // pyramid gradient: lanes stride over the window's cells, x fastest; cell (sx, sy) gathers taps a = sx-1 (x1
      // corner), a = sx (x0 corner) and b = sy-1 (y1 corner), b = sy (y0 corner), in ascending t
      for (int k = lane; k < ncell; k += 32) {
        const int sy = k / (side + 1), sx = k - sy * (side + 1);
        LookupAxis Ys[2];
#pragma unroll
        for (int ib = 0; ib < 2; ++ib) Ys[ib] = lookup_axis(cy, sy - 1 + ib - p.radius, H);
        float v = 0.0f;
        size_t off = 0;
        bool touched = false;
#pragma unroll
        for (int ia = 0; ia < 2; ++ia) {
          const int a = sx - 1 + ia;
          if (a < 0 || a >= side) continue;
          const LookupAxis X = lookup_axis(cx, a - p.radius, W);
          const float wx = ia == 0 ? X.w0 : X.w1;
          const int xi = ia == 0 ? X.i1 : X.i0;
#pragma unroll
          for (int ib = 0; ib < 2; ++ib) {
            const int b = sy - 1 + ib;
            if (b < 0 || b >= side) continue;
            const float go = __ldg(go_row + a * side + b);
            if (go == 0.0f) continue;
            const float wy = ib == 0 ? Ys[0].w0 : Ys[1].w1;
            const float c = __fmul_rn(wy, wx);
            if (c == 0.0f) continue;
            if (!touched) {
              off = (size_t)(ib == 0 ? Ys[0].i1 : Ys[1].i0) * W + xi;
              v = gimg[off];
              touched = true;
            }
            v = __fadd_rn(v, __fmul_rn(c, go));
          }
        }
        if (touched) gimg[off] = v;
      }
    }
    __syncthreads();
    if (threadIdx.x < qpb && q0 + threadIdx.x < (size_t)p.nq) {       // one owner per query: levels in ascending order
      const size_t qq = q0 + threadIdx.x;
      float gx = p.gcoords[2 * qq], gy = p.gcoords[2 * qq + 1];
      for (int k = 0; k < p.levels; ++k) {
        const float inv = 1.0f / (float)(1 << k);
        gx = __fadd_rn(gx, __fmul_rn(level_sum[threadIdx.x * p.levels + k][0], inv));
        gy = __fadd_rn(gy, __fmul_rn(level_sum[threadIdx.x * p.levels + k][1], inv));
      }
      p.gcoords[2 * qq] = gx;
      p.gcoords[2 * qq + 1] = gy;
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------
// Backward of the grid_sample lookup (RAFT_SAMPLER_GRID, kernels.cuh) with respect to the pyramid only: the original
// RAFT detaches the sampling position, so there is no coordinate gradient.  ATen's grid_sampler_2d_backward
// (align_corners, zeros padding) with the same per-axis set-up as the forward (grid_axis): with go = d loss / d out[q,
// l, a, b], every IN-FRAME corner of the tap adds fl(fl(wy * wx) * go) to its cell -- zero weights and zero go included,
// so a non-finite go reaches every cell ATen's backward reaches -- and a corner outside the level adds nothing.
//
// Fixed order, no atomics, each operation one rounded fp32 operation (no FMA), as in corr_lookup_bwd_kernel: a touched
// cell ends as v_in + term_1 + term_2 + ..., added left to right, its terms in ascending tap t = a*(2r+1) + b and, within
// a tap, in corner order 00, 01, 10, 11 (a tap reaches a cell through one corner at most, since x1 = x0 + 1).  Cells
// that no in-frame corner reaches are neither read nor written, so a level of height or width 1 receives nothing.
//
// Unlike the tf-raft sampler's, consecutive taps' unnormalised ix are not exactly 1 apart (the normalisation rounds),
// so a column can be reached by taps other than s-1 and s.  One warp per (query, level) owns that query's private
// slice of grad_pyr[l]: its lanes first compute the 2(2r+1) per-axis set-ups once (shared memory), then stride over
// the cells of the in-frame corners' bounding box, each cell gathering from the taps whose corners hit it.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) corr_lookup_grid_bwd_kernel(const LookupBwdParams p) {
  extern __shared__ GridAxis grid_bwd_axes[];                    // per warp: [0, S) x set-up of tap column a, [S, 2S) y of b
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const int side = 2 * p.radius + 1;
  GridAxis* ax = grid_bwd_axes + (threadIdx.x >> 5) * 2 * side;
  const size_t nwork = (size_t)p.nq * p.levels;
  for (size_t wi = (size_t)blockIdx.x * wpb + (threadIdx.x >> 5); wi < nwork; wi += (size_t)gridDim.x * wpb) {
    const size_t q = wi / p.levels;
    const int l = (int)(wi % p.levels);
    const int H = p.lh[l], W = p.lw[l];
    float* gimg = p.gpyr[l] + q * H * W;
    const float* go_row = p.gout + q * p.gout_stride + (size_t)l * side * side;
    const float inv = 1.0f / (float)(1 << l);                    // exact power of two
    const float cx = __fmul_rn(__ldg(p.coords + 2 * q), inv), cy = __fmul_rn(__ldg(p.coords + 2 * q + 1), inv);
    int lox = INT_MAX, hix = -1, loy = INT_MAX, hiy = -1;        // bounding box of the in-frame corners
    __syncwarp();                                                // the previous item's readers are done with ax
    for (int i = lane; i < 2 * side; i += 32) {
      const bool isy = i >= side;
      const int k = isy ? i - side : i;
      const GridAxis g = grid_axis(__fadd_rn(isy ? cy : cx, (float)(k - p.radius)), isy ? H : W);
      ax[i] = g;
      const int lo = g.i0 >= 0 ? g.i0 : (g.i1 >= 0 ? g.i1 : INT_MAX);
      const int hi = g.i1 >= 0 ? g.i1 : g.i0;
      if (isy) { loy = min(loy, lo); hiy = max(hiy, hi); }
      else { lox = min(lox, lo); hix = max(hix, hi); }
    }
    lox = __reduce_min_sync(0xffffffffu, lox);
    loy = __reduce_min_sync(0xffffffffu, loy);
    hix = __reduce_max_sync(0xffffffffu, hix);
    hiy = __reduce_max_sync(0xffffffffu, hiy);
    __syncwarp();
    if (lox > hix || loy > hiy) continue;                        // no in-frame corner (warp-uniform)
    const int nx = hix - lox + 1;
    const size_t ncell = (size_t)nx * (hiy - loy + 1);
    for (size_t k = lane; k < ncell; k += 32) {
      const int y = loy + (int)(k / nx), x = lox + (int)(k % nx);
      const size_t off = (size_t)y * W + x;
      float v = 0.0f;
      bool touched = false;
      for (int a = 0; a < side; ++a) {
        const GridAxis X = ax[a];
        if (X.i0 != x && X.i1 != x) continue;
        const float wx = X.i0 == x ? X.wf : X.wc;
        for (int b = 0; b < side; ++b) {
          const GridAxis Y = ax[side + b];
          if (Y.i0 != y && Y.i1 != y) continue;
          const float wy = Y.i0 == y ? Y.wf : Y.wc;
          if (!touched) {
            v = gimg[off];
            touched = true;
          }
          v = __fadd_rn(v, __fmul_rn(__fmul_rn(wy, wx), __ldg(go_row + a * side + b)));
        }
      }
      if (touched) gimg[off] = v;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// tf.linalg.global_norm / tf.clip_by_global_norm (model.py:135) and tfa AdamW (train_chairs.py:87-90) on a flat buffer.
// sumsq: deterministic two-stage reduction (fixed grid, fixed tree) -> out[0] = sum g^2.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) sumsq_partial_kernel(const float* __restrict__ g, size_t n, float* __restrict__ part) {
  __shared__ float red[8];
  float s = 0.0f;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) s += g[i] * g[i];
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.0f;
    for (int i = 0; i < 8; ++i) t += red[i];
    part[blockIdx.x] = t;
  }
}
__global__ void __launch_bounds__(256) sumsq_final_kernel(const float* __restrict__ part, int nparts, float* __restrict__ out) {
  __shared__ float red[8];
  float s = 0.0f;
  for (int i = threadIdx.x; i < nparts; i += blockDim.x) s += part[i];
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.0f;
    for (int i = 0; i < 8; ++i) t += red[i];
    out[0] = t;
  }
}

// g <- g * clip / max(||g||, clip)   (clip_norm > 0; tf.clip_by_global_norm), then
// var -= wd * var;  m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;  var -= lr_t * m / (sqrt(v) + eps)
// with lr_t = lr * sqrt(1 - b2^t) / (1 - b1^t) computed by the caller (Keras Adam, non-amsgrad).
__global__ void adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                             size_t n, const float* __restrict__ sumsq, float clip_norm, float lr_t, float b1, float b2,
                             float eps, float wd) {
  float scale = 1.0f;
  if (clip_norm > 0.0f) {
    const float norm = sqrtf(*sumsq);
    scale = clip_norm / fmaxf(norm, clip_norm);
  }
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float gi = g[i] * scale;
    float w = p[i];
    w -= wd * w;
    const float mi = b1 * m[i] + (1.0f - b1) * gi;
    const float vi = b2 * v[i] + (1.0f - b2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    p[i] = w - lr_t * mi / (sqrtf(vi) + eps);
  }
}

// The original RAFT's optimiser step (RAFT_ADAMW_TORCH): torch.nn.utils.clip_grad_norm_ then torch.optim.AdamW,
//   g <- g * min(1, clip / (||g|| + 1e-6))   (clip_norm > 0)
//   var *= 1 - lr * wd;  m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;  var -= (lr / bc1) * m / (sqrt(v) / sqrt(bc2) + eps)
// with the scheduled lr and the bias corrections bc1 = 1 - b1^t, bc2 = 1 - b2^t from the caller.
__global__ void adamw_torch_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                   float* __restrict__ v, size_t n, const float* __restrict__ sumsq, float clip_norm,
                                   float lr, float b1, float b2, float eps, float wd, float bc1, float bc2) {
  float scale = 1.0f;
  if (clip_norm > 0.0f) scale = fminf(1.0f, clip_norm / (sqrtf(*sumsq) + 1e-6f));
  const float decay = 1.0f - lr * wd, step = lr / bc1, bc2_sqrt = sqrtf(bc2);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float gi = g[i] * scale;
    const float mi = b1 * m[i] + (1.0f - b1) * gi;
    const float vi = b2 * v[i] + (1.0f - b2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    p[i] = p[i] * decay - step * (mi / (sqrtf(vi) / bc2_sqrt + eps));
  }
}

}  // namespace raft
