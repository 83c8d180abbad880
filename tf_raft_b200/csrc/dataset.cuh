// Evaluation data path (DESIGN.md section 3.5):
//   png16_decode_kernel          one CTA per KITTI / HD1K flow PNG: the zlib-inflated, still filtered scanlines go
//                                through the five PNG filters row by row in shared memory, then flow = (RGB16 - 2^15)
//                                / 64 and valid = B16 (tf_raft/datasets/frame_utils.py:102-107 readFlowKITTI)
//   flow_metrics_partial_kernel  grid (chunks, B): kMetChunk consecutive pixels of one image per CTA -> counts and an
//                                fp64 EPE sum in a fixed order
//   flow_metrics_final_kernel    one CTA per image: the CTA partials added in index order
#pragma once
#include "kernels.cuh"

namespace raft {

constexpr int kPngThreads = 256;
constexpr int kPngMaxWidth = 16384;            // two rows of 6 * W bytes in shared memory: 192 KB at most

// Bytes 0..3 and 4..5 of pixel x of a row as two words of byte lanes (the 6 interleaved R16 G16 B16 byte lanes).
__device__ __forceinline__ void png_load6(const uint8_t* row, int x, uint32_t& lo, uint32_t& hi) {
  const uint8_t* p = row + 6 * x;
  lo = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
  hi = (uint32_t)p[4] | ((uint32_t)p[5] << 8);
}

__device__ __forceinline__ void png_store6(uint8_t* row, int x, uint32_t lo, uint32_t hi) {
  uint8_t* p = row + 6 * x;
  p[0] = (uint8_t)lo; p[1] = (uint8_t)(lo >> 8); p[2] = (uint8_t)(lo >> 16); p[3] = (uint8_t)(lo >> 24);
  p[4] = (uint8_t)hi; p[5] = (uint8_t)(hi >> 8);
}

// PNG Paeth predictor (ISO/IEC 15948 section 9.4) on byte values; ties go to a, then b.
__device__ __forceinline__ int png_paeth(int a, int b, int c) {
  const int pa = abs(b - c), pb = abs(a - c), pc = abs(a + b - 2 * c);
  return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

// Sub: per byte lane, a prefix sum mod 256 along the row.  Each thread owns a contiguous run of pixels; __vadd4 adds
// four byte lanes at once without carries between them, so the six lanes travel as two words through a block scan.
__device__ __forceinline__ void png_sub_row(uint8_t* cur, int W) {
  __shared__ uint32_t warp_lo[kPngThreads / 32], warp_hi[kPngThreads / 32];
  const int per = ceil_div(W, kPngThreads);
  const int x0 = min(W, threadIdx.x * per), x1 = min(W, x0 + per);
  uint32_t lo = 0, hi = 0, a, b;
  for (int x = x0; x < x1; ++x) {
    png_load6(cur, x, a, b);
    lo = __vadd4(lo, a);
    hi = __vadd4(hi, b);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t ilo = lo, ihi = hi;                                   // inclusive scan over the warp
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t tlo = __shfl_up_sync(0xffffffffu, ilo, d), thi = __shfl_up_sync(0xffffffffu, ihi, d);
    if (lane >= d) { ilo = __vadd4(ilo, tlo); ihi = __vadd4(ihi, thi); }
  }
  if (lane == 31) { warp_lo[warp] = ilo; warp_hi[warp] = ihi; }
  __syncthreads();
  uint32_t run_lo = __vsub4(ilo, lo), run_hi = __vsub4(ihi, hi);  // exclusive within the warp
  for (int k = 0; k < warp; ++k) { run_lo = __vadd4(run_lo, warp_lo[k]); run_hi = __vadd4(run_hi, warp_hi[k]); }
  for (int x = x0; x < x1; ++x) {
    png_load6(cur, x, a, b);
    run_lo = __vadd4(run_lo, a);
    run_hi = __vadd4(run_hi, b);
    png_store6(cur, x, run_lo, run_hi);
  }
}

// Average (ft 3) and Paeth (ft 4): byte lane `lane` of the row as one serial chain over the W pixels.  The operands of
// eight pixels are read before any of them is written back, so the loads leave the dependent chain.
template <int FT>
__device__ __forceinline__ void png_chain_row(uint8_t* cur, const uint8_t* prev, int W, int lane) {
  int a = 0, c = 0;
  for (int x = 0; x < W; x += 8) {
    int f[8], up[8];
    const int n = min(8, W - x);
#pragma unroll
    for (int k = 0; k < 8; ++k)
      if (k < n) { f[k] = cur[6 * (x + k) + lane]; up[k] = prev[6 * (x + k) + lane]; }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (k < n) {
        const int pred = FT == 3 ? (a + up[k]) >> 1 : png_paeth(a, up[k], c);
        a = (f[k] + pred) & 255;
        c = up[k];
        cur[6 * (x + k) + lane] = (uint8_t)a;
      }
    }
  }
}

struct PngParams {
  const uint8_t* data;
  const raft_png16_image* images;
  int* status;
  int row_bytes;              // shared-memory bytes of one row buffer (6 * max w, rounded up to 16)
};

__global__ void __launch_bounds__(kPngThreads) png16_decode_kernel(const PngParams p) {
  extern __shared__ __align__(16) uint8_t png_smem[];
  const raft_png16_image im = p.images[blockIdx.x];
  const int W = im.w, stride = 6 * W;
  uint8_t* prev = png_smem;
  uint8_t* cur = png_smem + p.row_bytes;
  for (int i = threadIdx.x; i < stride; i += kPngThreads) prev[i] = 0;   // the row above the first is zero
  const uint8_t* src = p.data + im.offset;
  float2* flow = reinterpret_cast<float2*>(im.flow);
  for (int y = 0; y < im.h; ++y) {
    const uint8_t* line = src + (size_t)y * (stride + 1);
    const int ft = line[0];                                      // the same byte in every thread of the CTA
    if (ft > 4) {
      if (threadIdx.x == 0) p.status[blockIdx.x] = y + 1;
      return;
    }
    for (int i = threadIdx.x; i < stride; i += kPngThreads) cur[i] = line[1 + i];
    __syncthreads();
    if (ft == 1) {
      png_sub_row(cur, W);
    } else if (ft == 2) {
      for (int i = threadIdx.x; i < stride; i += kPngThreads) cur[i] = (uint8_t)(cur[i] + prev[i]);
    } else if (ft == 3) {
      if (threadIdx.x < 6) png_chain_row<3>(cur, prev, W, threadIdx.x);
    } else if (ft == 4) {
      if (threadIdx.x < 6) png_chain_row<4>(cur, prev, W, threadIdx.x);
    }
    __syncthreads();
    const size_t row0 = (size_t)y * W;
    for (int x = threadIdx.x; x < W; x += kPngThreads) {
      const uint8_t* q = cur + 6 * x;
      const float r = (float)(((int)q[0] << 8) | q[1]), g = (float)(((int)q[2] << 8) | q[3]);
      // (v - 2^15) / 64: both steps are exact in float32 for 16-bit v, as in the reference's float32 arithmetic
      flow[row0 + x] = make_float2(__fdiv_rn(__fsub_rn(r, 32768.0f), 64.0f), __fdiv_rn(__fsub_rn(g, 32768.0f), 64.0f));
      im.valid[row0 + x] = (float)(((int)q[4] << 8) | q[5]);
    }
    uint8_t* t = prev;                                           // the next row's copy writes the old `prev`, which
    prev = cur;                                                  // nothing reads after the __syncthreads above
    cur = t;
  }
}

// ------------------------------------------------------------------------------------------------
// Flow metrics
// ------------------------------------------------------------------------------------------------
constexpr int kMetThreads = 256;
constexpr int kMetChunk = 8192;                // pixels per CTA of the first pass; depends on nothing but this constant

struct MetricPartial {
  long long count[RAFT_METRIC_COUNTS];
  double sum;
};

__global__ void __launch_bounds__(kMetThreads) flow_metrics_partial_kernel(
    const float2* __restrict__ pred, const float2* __restrict__ gt, const float* __restrict__ valid, int hw,
    int use_max_flow, float max_flow, MetricPartial* __restrict__ part) {
  const int b = blockIdx.y, chunk = blockIdx.x;
  const size_t base = (size_t)b * hw;
  const int end = min(hw, (chunk + 1) * kMetChunk);
  int cnt[RAFT_METRIC_COUNTS] = {0, 0, 0, 0, 0};
  double sum = 0.0;
  for (int i = chunk * kMetChunk + threadIdx.x; i < end; i += kMetThreads) {
    const float2 g = __ldg(gt + base + i);
    const float mag = __fsqrt_rn(__fadd_rn(__fmul_rn(g.x, g.x), __fmul_rn(g.y, g.y)));
    const bool v = valid ? __ldg(valid + base + i) != 0.0f : true;            // NaN is nonzero, as tf.cast(., bool)
    if (!(v && (!use_max_flow || mag < max_flow))) continue;
    const float2 q = __ldg(pred + base + i);
    const float d0 = __fsub_rn(q.x, g.x), d1 = __fsub_rn(q.y, g.y);
    const float epe = __fsqrt_rn(__fadd_rn(__fmul_rn(d0, d0), __fmul_rn(d1, d1)));
    cnt[0] += 1;
    cnt[1] += epe < 1.0f;
    cnt[2] += epe < 3.0f;
    cnt[3] += epe < 5.0f;
    cnt[4] += epe > 3.0f && __fdiv_rn(epe, mag) > 0.05f;                       // mag = 0: epe / 0 = +inf > 0.05
    sum = __dadd_rn(sum, (double)epe);
  }
  // Fixed-shape trees: the same operations in the same order on every run.
  __shared__ double warp_sum[kMetThreads / 32];
  __shared__ int warp_cnt[kMetThreads / 32][RAFT_METRIC_COUNTS];
  for (int d = 16; d > 0; d >>= 1) sum = __dadd_rn(sum, __shfl_down_sync(0xffffffffu, sum, d));
#pragma unroll
  for (int k = 0; k < RAFT_METRIC_COUNTS; ++k) cnt[k] = __reduce_add_sync(0xffffffffu, cnt[k]);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    warp_sum[warp] = sum;
#pragma unroll
    for (int k = 0; k < RAFT_METRIC_COUNTS; ++k) warp_cnt[warp][k] = cnt[k];
  }
  __syncthreads();
  if (threadIdx.x < RAFT_METRIC_COUNTS) {                        // thread k adds count k of the 8 warps
    long long c = 0;
    for (int w = 0; w < kMetThreads / 32; ++w) c += warp_cnt[w][threadIdx.x];
    part[(size_t)b * gridDim.x + chunk].count[threadIdx.x] = c;
  }
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < kMetThreads / 32; ++w) s = __dadd_rn(s, warp_sum[w]);
    part[(size_t)b * gridDim.x + chunk].sum = s;
  }
}

__global__ void __launch_bounds__(kMetThreads) flow_metrics_final_kernel(const MetricPartial* __restrict__ part, int nchunk,
                                                                         long long* __restrict__ counts,
                                                                         double* __restrict__ sums) {
  __shared__ double stage[kMetThreads];
  __shared__ unsigned long long total[RAFT_METRIC_COUNTS];
  const int b = blockIdx.x;
  const MetricPartial* pb = part + (size_t)b * nchunk;
  if (threadIdx.x < RAFT_METRIC_COUNTS) total[threadIdx.x] = 0ull;
  unsigned long long cnt[RAFT_METRIC_COUNTS] = {0, 0, 0, 0, 0};
  double sum = 0.0;                                              // thread 0's running sum over chunks 0, 1, 2, ...
  for (int c0 = 0; c0 < nchunk; c0 += kMetThreads) {
    const int c = c0 + threadIdx.x;
    if (c < nchunk) {
      stage[threadIdx.x] = pb[c].sum;
#pragma unroll
      for (int k = 0; k < RAFT_METRIC_COUNTS; ++k) cnt[k] += (unsigned long long)pb[c].count[k];
    }
    __syncthreads();
    if (threadIdx.x == 0)
      for (int i = 0; i < min(kMetThreads, nchunk - c0); ++i) sum = __dadd_rn(sum, stage[i]);
    __syncthreads();
  }
#pragma unroll
  for (int k = 0; k < RAFT_METRIC_COUNTS; ++k) atomicAdd(&total[k], cnt[k]);   // integers: exact in any order
  __syncthreads();
  if (threadIdx.x < RAFT_METRIC_COUNTS) counts[(size_t)b * RAFT_METRIC_COUNTS + threadIdx.x] = (long long)total[threadIdx.x];
  if (threadIdx.x == 0) sums[b] = sum;
}

}  // namespace raft
