// Self-supervised training loss (an addition beyond tf-raft, which trains with ground truth only): the census transform
// of the images and, per direction of a bidirectional prediction sequence, an occlusion-masked census penalty plus an
// edge-aware first-order smoothness term, with its gradient with respect to every prediction (DESIGN.md section 9.1).
//
//   census_kernel              images (B, H, W, 3) in 0..255 -> (B, H, W, 48) census features, every operation an
//                              explicitly rounded fp32 one (NumPy float32 reproduces each bit, oracle/unsup_np.py)
//   unsup_mask_count_kernel    per CTA of the loss kernel's grid: its pixels' mask count (the census normaliser unless
//                              the caller supplies one)
//   unsup_loss_partial_kernel  one thread per pixel, all n predictions: the gradient of the direction's share of the loss
//                              and per-CTA fp64 partial sums in a fixed order
//   unsup_loss_final_kernel    one CTA: the partials added in index order, the normalised terms
// No atomics: each pixel's smoothness gradient gathers its up-to-four neighbour pairs itself, so two calls on the same
// inputs give the same bits.
#pragma once
#include "kernels.cuh"

namespace raft {

constexpr int kCensusRadius = 3;
constexpr int kCensusCh = 48;                    // (2 * 3 + 1)^2 - 1 offsets
constexpr int kUnsupThreads = 256;
constexpr int kUnsupMaxBlocks = kNumSMs * 8;

// grey = (0.2989 R + 0.5870 G + 0.1140 B) / 255, 0 outside the frame.
__device__ __forceinline__ float census_grey(const float* __restrict__ img, size_t b, int H, int W, int y, int x) {
  if (y < 0 || y >= H || x < 0 || x >= W) return 0.0f;
  const float* p = img + ((b * H + y) * (size_t)W + x) * 3;
  const float s = __fadd_rn(__fadd_rn(__fmul_rn(0.2989f, p[0]), __fmul_rn(0.5870f, p[1])), __fmul_rn(0.1140f, p[2]));
  return __fdiv_rn(s, 255.0f);
}

// out[b, y, x, k] = t / sqrt(0.81 + t^2), t = grey(y + dy, x + dx) - grey(y, x), (dy, dx) the k-th offset of
// [-3, 3]^2 \ {(0, 0)} in row-major order.  `out` 16-byte aligned.
__global__ void __launch_bounds__(256) census_kernel(const float* __restrict__ img, int B, int H, int W,
                                                    float* __restrict__ out) {
  const size_t hw = (size_t)H * W, n = (size_t)B * hw;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const size_t b = i / hw, q = i % hw;
    const int y = (int)(q / W), x = (int)(q % W);
    const float gc = census_grey(img, b, H, W, y, x);
    float4* o = reinterpret_cast<float4*>(out + i * kCensusCh);
    float v[4];
    int k = 0;
#pragma unroll
    for (int dy = -kCensusRadius; dy <= kCensusRadius; ++dy)
#pragma unroll
      for (int dx = -kCensusRadius; dx <= kCensusRadius; ++dx) {
        if (dy == 0 && dx == 0) continue;
        const float t = __fsub_rn(census_grey(img, b, H, W, y + dy, x + dx), gc);
        v[k & 3] = __fdiv_rn(t, __fsqrt_rn(__fadd_rn(0.81f, __fmul_rn(t, t))));
        if ((k & 3) == 3) o[k >> 2] = make_float4(v[0], v[1], v[2], v[3]);
        ++k;
      }
  }
}

// m(x): not occluded and the whole 7x7 census window inside the frame.
__device__ __forceinline__ bool unsup_masked(const uint8_t* __restrict__ occ, size_t p, int H, int W, int y, int x) {
  return occ[p] == 0 && x >= kCensusRadius && x < W - kCensusRadius && y >= kCensusRadius && y < H - kCensusRadius;
}

// Fixed-order block sum of kUnsupThreads doubles (shuffle tree per warp, warps in index order); the result in thread 0.
template <int N>
__device__ __forceinline__ void unsup_block_sum(double (&v)[N]) {
  __shared__ double warp_sum[kUnsupThreads / 32][N];
#pragma unroll
  for (int k = 0; k < N; ++k)
    for (int d = 16; d > 0; d >>= 1) v[k] = __dadd_rn(v[k], __shfl_down_sync(0xffffffffu, v[k], d));
  __syncthreads();                                // warp_sum of a previous call has been read
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int k = 0; k < N; ++k) warp_sum[threadIdx.x >> 5][k] = v[k];
  __syncthreads();
  if (threadIdx.x == 0)
#pragma unroll
    for (int k = 0; k < N; ++k) {
      double s = 0.0;
      for (int w = 0; w < kUnsupThreads / 32; ++w) s = __dadd_rn(s, warp_sum[w][k]);
      v[k] = s;
    }
}

// partials[3 * nblocks + blk] = number of masked pixels of CTA blk's pixels (the loss kernel's grid-stride split).
__global__ void __launch_bounds__(kUnsupThreads) unsup_mask_count_kernel(const uint8_t* __restrict__ occ, int B, int H,
                                                                         int W, double* __restrict__ partials) {
  const size_t hw = (size_t)H * W, n = (size_t)B * hw;
  long long c = 0;
  for (size_t p = blockIdx.x * (size_t)kUnsupThreads + threadIdx.x; p < n; p += (size_t)gridDim.x * kUnsupThreads) {
    const size_t q = p % hw;
    c += unsup_masked(occ, p, H, W, (int)(q / W), (int)(q % W)) ? 1 : 0;
  }
  double v[1] = {(double)c};                      // exact: every count stays below 2^53
  unsup_block_sum(v);
  if (threadIdx.x == 0) partials[3 * (size_t)gridDim.x + blockIdx.x] = v[0];
}

// The direction's mask count: the count partials added up (integers, exact in any order); every thread gets it.
__device__ __forceinline__ double unsup_mask_total(const double* __restrict__ partials, int nblocks) {
  __shared__ double total;
  double v[1] = {0.0};
  for (int c = threadIdx.x; c < nblocks; c += kUnsupThreads) v[0] += partials[3 * (size_t)nblocks + c];
  unsup_block_sum(v);
  if (threadIdx.x == 0) total = v[0];
  __syncthreads();
  return total;
}

struct UnsupParams {
  const float* ct;         // target census (B, H, W, 48): the image the flows start from
  const float* cs;         // source census (B, H, W, 48): the image the flows point into
  const float* img;        // target image (B, H, W, 3), 0..255: edge weights
  const uint8_t* occ;      // (B, H, W) occlusion of the target's pixels
  const float2* flows;     // (n, B, H, W) predictions
  float2* grad;            // (n, B, H, W) d(direction's loss share) / d flows
  double* partials;        // 3 per CTA: census, horizontal and vertical smoothness sums, gamma-weighted; then one mask
                           // count per CTA (unsup_mask_count_kernel)
  const double* census_norm;  // NULL: max(mask count, 1); else the caller's normaliser (> 0), e.g. of a global batch
  int n, B, H, W;
  double gamma;
  float edge;              // lambda of the edge weight
  float census_half;       // census_weight / 2
  float sh_scale, sv_scale;  // smoothness_weight / 2 * 1/2 * 1 / (number of horizontal / vertical pairs)
};

// Edge weight of the pair (a, b) of target pixels: exp(-lambda * mean_c |I_c(b) - I_c(a)| / 255).
__device__ __forceinline__ float unsup_edge(const float* __restrict__ img, size_t a, size_t b, float lambda) {
  const float* pa = img + a * 3;
  const float* pb = img + b * 3;
  const float d = fabsf(pb[0] - pa[0]) + fabsf(pb[1] - pa[1]) + fabsf(pb[2] - pa[2]);
  return expf(-lambda * (d / 3.0f) / 255.0f);
}

// d|u|/du with autograd's conventions: 0 at 0, and 0 for NaN too (torch's abs backward).  The loss itself keeps the NaN.
__device__ __forceinline__ float unsup_sgn(float u) { return u > 0.0f ? 1.0f : (u < 0.0f ? -1.0f : 0.0f); }

__global__ void __launch_bounds__(kUnsupThreads) unsup_loss_partial_kernel(const UnsupParams P) {
  const int H = P.H, W = P.W;
  const size_t hw = (size_t)H * W, npix = (size_t)P.B * hw;
  const float xmax = (float)(W - 1), ymax = (float)(H - 1);
  const double norm = P.census_norm ? *P.census_norm : fmax(unsup_mask_total(P.partials, gridDim.x), 1.0);
  const float census_scale = (float)(P.census_half / norm);
  double acc[3] = {0.0, 0.0, 0.0};
  for (size_t p = blockIdx.x * (size_t)kUnsupThreads + threadIdx.x; p < npix; p += (size_t)gridDim.x * kUnsupThreads) {
    const size_t bi = p / hw, q = p % hw;
    const int y = (int)(q / W), x = (int)(q % W);
    const float m = unsup_masked(P.occ, p, H, W, y, x) ? 1.0f : 0.0f;
    const bool has_l = x > 0, has_r = x < W - 1, has_u = y > 0, has_d = y < H - 1;
    const float wl = has_l ? unsup_edge(P.img, p - 1, p, P.edge) : 0.0f;
    const float wr = has_r ? unsup_edge(P.img, p, p + 1, P.edge) : 0.0f;
    const float wu = has_u ? unsup_edge(P.img, p - W, p, P.edge) : 0.0f;
    const float wd = has_d ? unsup_edge(P.img, p, p + W, P.edge) : 0.0f;
    const float4* ct = reinterpret_cast<const float4*>(P.ct + p * kCensusCh);
    const float* cs_img = P.cs + bi * hw * kCensusCh;
    for (int i = 0; i < P.n; ++i) {
      const double wgt = pow(P.gamma, (double)(P.n - 1 - i));
      const float wf = (float)wgt;
      const float2* F = P.flows + (size_t)i * npix;
      const float2 f = F[p];
      float2 g = make_float2(0.0f, 0.0f);
      // census: bilinear sample of the source census at p = (x, y) + f, closed frame, fb_occlusion_kernel's corner rule
      const float px = __fadd_rn((float)x, f.x), py = __fadd_rn((float)y, f.y);
      if (px >= 0.0f && px <= xmax && py >= 0.0f && py <= ymax) {
        const float fx0 = floorf(px), fy0 = floorf(py);
        const int x0 = (int)fx0, y0 = (int)fy0;
        const int x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);
        const float ax = px - fx0, bx = 1.0f - ax, ay = py - fy0, by = 1.0f - ay;
        const float4* c00 = reinterpret_cast<const float4*>(cs_img + ((size_t)y0 * W + x0) * kCensusCh);
        const float4* c01 = reinterpret_cast<const float4*>(cs_img + ((size_t)y0 * W + x1) * kCensusCh);
        const float4* c10 = reinterpret_cast<const float4*>(cs_img + ((size_t)y1 * W + x0) * kCensusCh);
        const float4* c11 = reinterpret_cast<const float4*>(cs_img + ((size_t)y1 * W + x1) * kCensusCh);
        float D = 0.0f, gpx = 0.0f, gpy = 0.0f;
#pragma unroll 2
        for (int k = 0; k < kCensusCh / 4; ++k) {
          const float4 t4 = __ldg(ct + k), a4 = __ldg(c00 + k), b4 = __ldg(c01 + k), e4 = __ldg(c10 + k), d4 = __ldg(c11 + k);
          const float tv[4] = {t4.x, t4.y, t4.z, t4.w}, v00[4] = {a4.x, a4.y, a4.z, a4.w};
          const float v01[4] = {b4.x, b4.y, b4.z, b4.w}, v10[4] = {e4.x, e4.y, e4.z, e4.w};
          const float v11[4] = {d4.x, d4.y, d4.z, d4.w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float top = bx * v00[j] + ax * v01[j], bot = bx * v10[j] + ax * v11[j];
            const float s = by * top + ay * bot;
            const float dsx = by * (v01[j] - v00[j]) + ay * (v11[j] - v10[j]);   // d s / d px
            const float dsy = bot - top;                                          // d s / d py
            const float d = tv[j] - s, e = 0.1f + d * d;
            D += d * d / e;
            const float q = 0.2f * d / (e * e);                                   // d/dd of d^2 / (0.1 + d^2)
            gpx -= q * dsx;
            gpy -= q * dsy;
          }
        }
        const float r = powf(D + 0.01f, 0.4f);
        acc[0] += wgt * (double)(m * r);
        const float s = census_scale * wf * m * 0.4f * r / (D + 0.01f);          // d rho / dD = 0.4 (D + 0.01)^-0.6
        g.x = s * gpx;
        g.y = s * gpy;
      }
      // smoothness: this pixel owns its right and lower pairs in the sums and gathers all four pairs in the gradient
      float hx = 0.0f, hy = 0.0f, vx = 0.0f, vy = 0.0f;
      if (has_r) {
        const float2 o = F[p + 1];
        const float dx = o.x - f.x, dy = o.y - f.y;
        acc[1] += wgt * (double)(wr * (fabsf(dx) + fabsf(dy)) * 0.5f);
        hx -= wr * unsup_sgn(dx);
        hy -= wr * unsup_sgn(dy);
      }
      if (has_l) {
        const float2 o = F[p - 1];
        hx += wl * unsup_sgn(f.x - o.x);
        hy += wl * unsup_sgn(f.y - o.y);
      }
      if (has_d) {
        const float2 o = F[p + W];
        const float dx = o.x - f.x, dy = o.y - f.y;
        acc[2] += wgt * (double)(wd * (fabsf(dx) + fabsf(dy)) * 0.5f);
        vx -= wd * unsup_sgn(dx);
        vy -= wd * unsup_sgn(dy);
      }
      if (has_u) {
        const float2 o = F[p - W];
        vx += wu * unsup_sgn(f.x - o.x);
        vy += wu * unsup_sgn(f.y - o.y);
      }
      const float sh = 0.5f * wf * P.sh_scale, sv = 0.5f * wf * P.sv_scale;
      g.x += sh * hx + sv * vx;
      g.y += sh * hy + sv * vy;
      P.grad[(size_t)i * npix + p] = g;
    }
  }
  unsup_block_sum(acc);
  if (threadIdx.x == 0)
#pragma unroll
    for (int k = 0; k < 3; ++k) P.partials[(size_t)blockIdx.x * 3 + k] = acc[k];
}

// One CTA.  sums[2] = mask count, sums[0] = L_c = census sum / norm, norm = *census_norm or max(count, 1); sums[1] = L_s =
// (S_h + S_v) / 2 with S_h, S_v the smoothness sums over the numbers of pairs; sums[3] = census_weight / 2 * L_c +
// smoothness_weight / 2 * L_s.
__global__ void __launch_bounds__(kUnsupThreads) unsup_loss_final_kernel(const double* __restrict__ partials, int nblocks,
                                                                         double n_h, double n_v, double census_half,
                                                                         double smooth_half,
                                                                         const double* __restrict__ census_norm,
                                                                         double* __restrict__ sums) {
  const double count = unsup_mask_total(partials, nblocks);
  double v[3] = {0.0, 0.0, 0.0};
  for (int c = threadIdx.x; c < nblocks; c += kUnsupThreads)
#pragma unroll
    for (int k = 0; k < 3; ++k) v[k] = __dadd_rn(v[k], partials[(size_t)c * 3 + k]);
  unsup_block_sum(v);
  if (threadIdx.x == 0) {
    const double lc = v[0] / (census_norm ? *census_norm : fmax(count, 1.0));
    const double ls = (v[1] / n_h + v[2] / n_v) / 2.0;
    sums[0] = lc;
    sums[1] = ls;
    sums[2] = count;
    sums[3] = census_half * lc + smooth_half * ls;
  }
}

}  // namespace raft
