// Warm start for video inference: RAFT's forward interpolation of the previous pair's low-resolution flow onto the new
// frame, and the loop's entry state coords1 = coords_grid + flow_init.  Both are additions beyond tf-raft, whose
// model.py:89 always starts from zero flow.  Also the forward-backward occlusion check of bidirectional flow.
#pragma once
#include <math_constants.h>

#include "kernels.cuh"

namespace raft {

// ------------------------------------------------------------------------------------------------
// forward_interpolate: per image b of a (B, h, w, 2) flow, source pixel i = y*w + x lands at
//   x1 = x + fx, y1 = y + fy                              (fp64, one rounding each)
// and is valid iff 0 < x1 < w and 0 < y1 < h (strict; NaN / +-inf flow is never valid).  Target pixel (X, Y) receives
// the flow of the valid source minimising d = (x1 - X)^2 + (y1 - Y)^2 (fp64, every operation rounded on its own, no FMA
// contraction), ties to the lowest source index; zero flow when the image has no valid source.  That is
// scipy.interpolate.griddata((x1, y1), f, (X, Y), method='nearest') with a deterministic tie rule.
//
// Brute force, one thread per target holding (best d, best index).  The CTA stages chunks of the image's sources in
// shared memory as (x1, y1) pairs, an invalid source as (NaN, NaN): its distance is NaN and `d < best` is false, so it
// never wins.  Sources are scanned in index order and only a strictly smaller d replaces the best: ties keep the lowest
// index.  The output is a copy of the chosen source's two floats.  Cost: (h*w)^2 fp64 distance evaluations per image.
// grid (ceil(h*w / kFiThreads), min(B, 65535)); `out` must not alias `flow` (targets read sources other threads write).
// ------------------------------------------------------------------------------------------------
constexpr int kFiThreads = 128;
constexpr int kFiChunk = 512;

__global__ void __launch_bounds__(kFiThreads) forward_interpolate_kernel(const float* __restrict__ flow,
                                                                         float* __restrict__ out, int B, int h, int w) {
  __shared__ double2 src[kFiChunk];
  const int n = h * w;
  const int t = blockIdx.x * kFiThreads + threadIdx.x;
  const double X = (double)(t % w), Y = (double)(t / w);
  const double dw = (double)w, dh = (double)h;
  for (int b = blockIdx.y; b < B; b += gridDim.y) {
    const float* fb = flow + (size_t)b * n * 2;
    double best = CUDART_INF;
    int best_i = -1;
    for (int c0 = 0; c0 < n; c0 += kFiChunk) {
      __syncthreads();                                   // the previous chunk has been read by every thread
      for (int j = threadIdx.x; j < kFiChunk; j += kFiThreads) {
        const int i = c0 + j;
        double2 s = make_double2(CUDART_NAN, CUDART_NAN);
        if (i < n) {
          const double x1 = __dadd_rn((double)(i % w), (double)fb[2 * (size_t)i]);
          const double y1 = __dadd_rn((double)(i / w), (double)fb[2 * (size_t)i + 1]);
          if (x1 > 0.0 && x1 < dw && y1 > 0.0 && y1 < dh) s = make_double2(x1, y1);
        }
        src[j] = s;
      }
      __syncthreads();
      const int m = min(kFiChunk, n - c0);
#pragma unroll 4
      for (int j = 0; j < m; ++j) {
        const double2 s = src[j];
        const double dx = __dsub_rn(s.x, X), dy = __dsub_rn(s.y, Y);
        const double d = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
        if (d < best) {
          best = d;
          best_i = c0 + j;
        }
      }
    }
    if (t < n) {
      float* ob = out + (size_t)b * n * 2;
      ob[2 * (size_t)t] = best_i >= 0 ? fb[2 * (size_t)best_i] : 0.0f;
      ob[2 * (size_t)t + 1] = best_i >= 0 ? fb[2 * (size_t)best_i + 1] : 0.0f;
    }
  }
}

// coords1 = coords_grid(B, h, w) + flow_init, one fp32 rounding per component (model.py:89 with an initial flow; the
// reference's is zero).  flow_init may alias coords1.
__global__ void coords_init_kernel(const float* flow_init, float* coords1, int B, int h, int w) {
  const size_t total = (size_t)B * h * w;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const float gx = (float)(i % w), gy = (float)((i / w) % h);
    const float fx = flow_init[2 * i], fy = flow_init[2 * i + 1];
    coords1[2 * i] = __fadd_rn(gx, fx);
    coords1[2 * i + 1] = __fadd_rn(gy, fy);
  }
}

// ------------------------------------------------------------------------------------------------
// fb_occlusion: the forward-backward consistency check (Sundaram, Brox and Keutzer, ECCV 2010; UnFlow's boundary), an
// addition beyond tf-raft.  Thread i < n = B*H*W handles pixel i of direction fw (F = flow_fw, G = flow_bw), thread
// n + i pixel i of direction bw (the roles swapped).  Pixel (x, y) of image b:
//   p = (x + fx, y + fy); occluded unless 0 <= px <= W-1 and 0 <= py <= H-1 (closed; NaN never passes);
//   g = bilinear sample of G[b] at p: x0 = floor(px), x1 = min(x0 + 1, W-1), ax = px - x0, bx = 1 - ax (y likewise),
//       g = by*(bx*G[y0,x0] + ax*G[y0,x1]) + ay*(bx*G[y1,x0] + ax*G[y1,x1]);
//   consistent iff |f + g|^2 <= alpha1*(|f|^2 + |g|^2) + alpha2, every other outcome (NaN included) occluded.
// Every operation is an explicitly rounded fp32 intrinsic in the order written, so no FMA is contracted and NumPy float32
// reproduces each bit (oracle/occlusion_np.py).  A non-finite texel reaches g even at weight 0 (0 * inf = NaN).
// ------------------------------------------------------------------------------------------------
__global__ void fb_occlusion_kernel(const float2* __restrict__ flow_fw, const float2* __restrict__ flow_bw, int B, int H,
                                    int W, float alpha1, float alpha2, uint8_t* __restrict__ occ_fw,
                                    uint8_t* __restrict__ occ_bw) {
  const size_t hw = (size_t)H * W, n = (size_t)B * hw;
  const float xmax = (float)(W - 1), ymax = (float)(H - 1);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < 2 * n; i += (size_t)gridDim.x * blockDim.x) {
    const bool bw = i >= n;
    const size_t p = bw ? i - n : i;
    const float2* F = bw ? flow_bw : flow_fw;
    const float2* G = (bw ? flow_fw : flow_bw) + (p / hw) * hw;
    const size_t q = p % hw;
    const float2 f = F[p];
    const float px = __fadd_rn((float)(q % W), f.x), py = __fadd_rn((float)(q / W), f.y);
    bool occ = true;
    if (px >= 0.0f && px <= xmax && py >= 0.0f && py <= ymax) {
      const float fx0 = floorf(px), fy0 = floorf(py);
      const int x0 = (int)fx0, y0 = (int)fy0;
      const size_t x1 = (size_t)min(x0 + 1, W - 1), y1 = (size_t)min(y0 + 1, H - 1);
      const float ax = __fsub_rn(px, fx0), bx = __fsub_rn(1.0f, ax);
      const float ay = __fsub_rn(py, fy0), by = __fsub_rn(1.0f, ay);
      const float2 g00 = G[(size_t)y0 * W + x0], g01 = G[(size_t)y0 * W + x1];
      const float2 g10 = G[y1 * W + x0], g11 = G[y1 * W + x1];
      const float gx = __fadd_rn(__fmul_rn(by, __fadd_rn(__fmul_rn(bx, g00.x), __fmul_rn(ax, g01.x))),
                                 __fmul_rn(ay, __fadd_rn(__fmul_rn(bx, g10.x), __fmul_rn(ax, g11.x))));
      const float gy = __fadd_rn(__fmul_rn(by, __fadd_rn(__fmul_rn(bx, g00.y), __fmul_rn(ax, g01.y))),
                                 __fmul_rn(ay, __fadd_rn(__fmul_rn(bx, g10.y), __fmul_rn(ax, g11.y))));
      const float sx = __fadd_rn(f.x, gx), sy = __fadd_rn(f.y, gy);
      const float lhs = __fadd_rn(__fmul_rn(sx, sx), __fmul_rn(sy, sy));
      const float mag = __fadd_rn(__fadd_rn(__fmul_rn(f.x, f.x), __fmul_rn(f.y, f.y)),
                                  __fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)));
      const float rhs = __fadd_rn(__fmul_rn(alpha1, mag), alpha2);
      occ = !(lhs <= rhs);
    }
    (bw ? occ_bw : occ_fw)[p] = occ ? 1 : 0;
  }
}

}  // namespace raft
