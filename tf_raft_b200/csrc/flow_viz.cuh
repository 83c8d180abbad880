// Flow visualisation: tf_raft/datasets/flow_viz.py's Middlebury colour wheel (make_colorwheel, flow_uv_to_colors,
// flow_to_image) with NumPy 2's dtype chain (DESIGN.md section 3.5, oracle/flow_viz_np.py).
//   flow_radmax_kernel   grid (x, B): max over image b of rad = sqrt(u*u + v*v) after the clip, as an atomicMax on the
//                        bits of the non-negative float (exact, independent of the order)
//   flow_colour_kernel   1024 consecutive pixels of the flat (B*H*W) range per CTA: clip, normalise, the colour wheel,
//                        staged in shared memory and written as 32-bit words; non-finite inputs set status bits
// float32 steps are explicitly rounded intrinsics and the float64 ones too, so nothing is contracted into an FMA.
#pragma once
#include <float.h>

#include "kernels.cuh"

namespace raft {

constexpr int kVizThreads = 256;
constexpr int kVizPixPerThread = 4;
constexpr int kVizPixPerBlock = kVizThreads * kVizPixPerThread;
constexpr int kWheelCols = 55;                 // RY + YG + GC + CB + BM + MR of make_colorwheel
constexpr float kPiF = 3.14159274101257324f;   // float32(np.pi): `/ np.pi` on a float32 array stays float32 (NEP 50)

// make_colorwheel()[k][c] (flow_viz.py:20-67).  floor(255*j/n) of the reference is float64 arithmetic on small
// integers; the quotient is never within half an ulp of an integer, so it equals the integer division.
__device__ __forceinline__ int viz_wheel(int k, int c) {
  int j;
  if (k < 15) { j = k;      return c == 0 ? 255 : c == 1 ? 255 * j / 15 : 0; }             // RY
  if (k < 21) { j = k - 15; return c == 0 ? 255 - 255 * j / 6 : c == 1 ? 255 : 0; }       // YG
  if (k < 25) { j = k - 21; return c == 0 ? 0 : c == 1 ? 255 : 255 * j / 4; }             // GC
  if (k < 36) { j = k - 25; return c == 0 ? 0 : c == 1 ? 255 - 255 * j / 11 : 255; }      // CB
  if (k < 49) { j = k - 36; return c == 0 ? 255 * j / 13 : c == 1 ? 0 : 255; }            // BM
  j = k - 49;               return c == 0 ? 255 : c == 1 ? 0 : 255 - 255 * j / 6;         // MR
}

// np.clip(x, 0, c) on float32: NaN propagates, -0.0 stays -0.0 (NumPy's max keeps its first operand on a tie),
// -inf -> 0, +inf -> c.  Not fmaxf / fminf, which drop NaN.
__device__ __forceinline__ float viz_clip(float x, float c) {
  if (x != x) return x;
  x = x < 0.0f ? 0.0f : x;
  return x > c ? c : x;
}

__device__ __forceinline__ float viz_rad(float u, float v) {
  return __fsqrt_rn(__fadd_rn(__fmul_rn(u, u), __fmul_rn(v, v)));
}

__device__ __forceinline__ float viz_load(const float* __restrict__ p, size_t i, int stride) { return __ldg(p + i * stride); }

__global__ void __launch_bounds__(kVizThreads) flow_radmax_kernel(const float* __restrict__ u, const float* __restrict__ v,
                                                                  int stride, int hw, int clip, float clip_flow,
                                                                  unsigned* __restrict__ work) {
  const int b = blockIdx.y;
  const size_t base = (size_t)b * hw;
  unsigned m = 0u;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)hw; i += (size_t)gridDim.x * blockDim.x) {
    float x = viz_load(u, base + i, stride), y = viz_load(v, base + i, stride);
    if (clip) { x = viz_clip(x, clip_flow); y = viz_clip(y, clip_flow); }
    m = max(m, __float_as_uint(viz_rad(x, y)));     // rad >= +0, so its bits order as the floats do (NaN: status)
  }
  __shared__ unsigned warp_max[kVizThreads / 32];
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0) warp_max[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {                                        // one atomic per CTA
    m = __reduce_max_sync(0xffffffffu, threadIdx.x < kVizThreads / 32 ? warp_max[threadIdx.x] : 0u);
    if (threadIdx.x == 0 && m) atomicMax(work + b, m);
  }
}

struct VizParams {
  const float* u;
  const float* v;
  int stride;                 // component of pixel p at u[p * stride], v[p * stride]
  int hw;
  size_t npix;                // B * hw
  int clip;
  float clip_flow;
  int normalize;
  const float* rad_max;       // per-image divisor base given by the caller, or null: the reduced max in work
  const unsigned* work;
  int bgr;
  uint8_t* out;               // (B, H, W, 3), 4-byte aligned
  int* status;
};

// One pixel of flow_to_image / flow_uv_to_colors (flow_viz.py:85-106, 123-132).  Returns its status bits.
__device__ __forceinline__ int viz_pixel(float x, float y, float div, const VizParams& p, const double* wheel,
                                         uint8_t rgb[3]) {
  if (p.clip) { x = viz_clip(x, p.clip_flow); y = viz_clip(y, p.clip_flow); }
  int st = 0;
  if (isinf(x) || isinf(y)) st |= RAFT_FLOWVIZ_INF;
  if (isnan(x) || isnan(y)) st |= RAFT_FLOWVIZ_NAN;
  if (p.normalize) { x = __fdiv_rn(x, div); y = __fdiv_rn(y, div); }                 // u / (rad_max + 1e-5)
  const float rad = viz_rad(x, y);
  // arctan2(-v, -u) / np.pi: negate first (signed zeros pick the half plane), correctly rounded atan2 from fp64
  const float a = __fdiv_rn(__double2float_rn(atan2((double)(-y), (double)(-x))), kPiF);
  const float fk = __fmul_rn(__fdiv_rn(__fadd_rn(a, 1.0f), 2.0f), (float)(kWheelCols - 1));
  if (!(fk >= 0.0f && fk <= (float)(kWheelCols - 1))) {          // NaN only: the reference fails here (IndexError)
    rgb[0] = rgb[1] = rgb[2] = 0;
    return st;
  }
  const int k0 = (int)floorf(fk);
  const int k1 = k0 + 1 == kWheelCols ? 0 : k0 + 1;
  const double f = __dsub_rn((double)fk, (double)k0);            // float32 - int32 promotes to float64: exact
  const double g = __dsub_rn(1.0, f);
  for (int i = 0; i < 3; ++i) {
    double col = __dadd_rn(__dmul_rn(g, wheel[k0 * 3 + i]), __dmul_rn(f, wheel[k1 * 3 + i]));
    col = rad <= 1.0f ? __dsub_rn(1.0, __dmul_rn((double)rad, __dsub_rn(1.0, col))) : __dmul_rn(col, 0.75);
    rgb[p.bgr ? 2 - i : i] = (uint8_t)(int)floor(__dmul_rn(255.0, col));
  }
  return st;
}

__global__ void __launch_bounds__(kVizThreads) flow_colour_kernel(const VizParams p) {
  __shared__ double wheel[kWheelCols * 3];                       // make_colorwheel() / 255.0, IEEE float64 division
  __shared__ __align__(16) uint8_t stage[kVizPixPerBlock * 3];
  for (int i = threadIdx.x; i < kWheelCols * 3; i += blockDim.x) wheel[i] = __ddiv_rn((double)viz_wheel(i / 3, i % 3), 255.0);
  __syncthreads();
  const size_t first = (size_t)blockIdx.x * kVizPixPerBlock;
  const int n = (int)min((size_t)kVizPixPerBlock, p.npix - first);
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const size_t px = first + j;
    const int b = (int)(px / (size_t)p.hw);
    float div = 0.0f;
    int st = 0;
    if (p.normalize) {
      const float rm = p.rad_max ? p.rad_max[b] : __uint_as_float(p.work[b]);
      if (p.rad_max && !(rm >= 0.0f && rm <= FLT_MAX)) st |= RAFT_FLOWVIZ_BAD_RAD_MAX;
      div = __fadd_rn(rm, 1e-5f);                                // float32(1e-5) under NEP 50
    }
    uint8_t rgb[3];
    st |= viz_pixel(viz_load(p.u, px, p.stride), viz_load(p.v, px, p.stride), div, p, wheel, rgb);
    if (st) atomicOr(p.status + b, st);
    stage[j * 3 + 0] = rgb[0];
    stage[j * 3 + 1] = rgb[1];
    stage[j * 3 + 2] = rgb[2];
  }
  __syncthreads();
  uint8_t* out = p.out + first * 3;
  if (n == kVizPixPerBlock) {                                    // 3072 bytes as coalesced 32-bit words
    const uint32_t* s32 = reinterpret_cast<const uint32_t*>(stage);
    uint32_t* o32 = reinterpret_cast<uint32_t*>(out);
    for (int w = threadIdx.x; w < kVizPixPerBlock * 3 / 4; w += blockDim.x) o32[w] = s32[w];
  } else {
    for (int i = threadIdx.x; i < n * 3; i += blockDim.x) out[i] = stage[i];
  }
}

}  // namespace raft
