// Colour jitter: torchvision's ColorJitter on an RGB PIL image, as the original RAFT's augmentor applies it, given its
// random draws (the draws live on the host, tf_raft_b200/datasets/augmentor.py).  One launch pair serves a batch whose
// samples have different sizes: both kernels read a device array of raft_colour_jitter_sample and run grid (x, B),
// blockIdx.y = sample, grid-striding over the 2*H*W pixels of the sample's two images.
//   colour_jitter_sum_kernel    the ops before contrast, then the integer sum of Pillow's L per parameter set
//   colour_jitter_apply_kernel  the ops before contrast again, contrast towards int(sum / n + 0.5), the ops after it
// A parameter set covers img1 stacked above img2 (one sum over 2*H*W pixels) or one image.  The arithmetic is Pillow's
// (DESIGN.md section 3.8, oracle/pil_colour_np.py): every float32 and float64 operation is one explicitly rounded
// intrinsic, so no contraction can change a byte.
#pragma once
#include "kernels.cuh"

namespace raft {

constexpr int kJitterThreads = 256;
enum { kJitBrightness = 0, kJitContrast = 1, kJitSaturation = 2, kJitHue = 3 };

// Image.blend(a, b, f) on uint8: fl32(a + fl32(f * (b - a))), clipped to [0, 255] and truncated.
__device__ __forceinline__ int pil_blend(int a, int b, float f) {
  const float t = __fadd_rn((float)a, __fmul_rn(f, (float)(b - a)));
  return min(max(__float2int_rz(t), 0), 255);
}

// Image.convert('L')
__device__ __forceinline__ int pil_luma(int r, int g, int b) { return (19595 * r + 38470 * g + 7471 * b + 0x8000) >> 16; }

// Pillow's RGB->HSV.  float32: cr, s = cr / max, rc, gc, bc; the hue sums 2.0 + rc - bc and 4.0 + gc - rc are float64
// (C promotes them) rounded to float32, then h = fl32(fmod(h / 6.0 + 1.0, 1.0)).  h / 6 + 1 lies in [5/6, 11/6), where
// fmod(x, 1) is x - 1 for x >= 1, exact.  H and S are int(h * 255.0) and int(s * 255.0) in float64.
__device__ __forceinline__ void pil_rgb2hsv(int r, int g, int b, int& H, int& S, int& V) {
  const int mx = max(max(r, g), b), mn = min(min(r, g), b);
  V = mx;
  if (mx == mn) {
    H = S = 0;
    return;
  }
  const float cr = (float)(mx - mn);
  const float s = __fdiv_rn(cr, (float)mx);
  const float rc = __fdiv_rn((float)(mx - r), cr), gc = __fdiv_rn((float)(mx - g), cr), bc = __fdiv_rn((float)(mx - b), cr);
  float h;
  if (r == mx) h = __fsub_rn(bc, gc);
  else if (g == mx) h = __double2float_rn(__dsub_rn(__dadd_rn(2.0, (double)rc), (double)bc));
  else h = __double2float_rn(__dsub_rn(__dadd_rn(4.0, (double)gc), (double)rc));
  double x = __dadd_rn(__ddiv_rn((double)h, 6.0), 1.0);
  if (x >= 1.0) x = __dsub_rn(x, 1.0);
  h = __double2float_rn(x);
  H = min(max(__double2int_rz(__dmul_rn((double)h, 255.0)), 0), 255);
  S = min(max(__double2int_rz(__dmul_rn((double)s, 255.0)), 0), 255);
}

__device__ __forceinline__ int pil_round8(double x) { return min(max(__double2int_rz(round(x)), 0), 255); }

// Pillow's HSV->RGB.  float64 a = H * 6.0 / 255.0, i = floor(a), f = fl32(a - i), fs = fl32(S / 255.0);
// p = round(V (1 - fs)), q = round(V (1 - fl32(fs f))), t = round(V (1 - fs (1 - f))), float64 but for fs * f, round
// half away from zero; sector i % 6 picks (V,t,p), (q,V,p), (p,V,t), (p,q,V), (t,p,V), (V,p,q).
__device__ __forceinline__ void pil_hsv2rgb(int H, int S, int V, int& r, int& g, int& b) {
  if (S == 0) {
    r = g = b = V;
    return;
  }
  const double a = __ddiv_rn(__dmul_rn((double)H, 6.0), 255.0);
  const int i = (int)floor(a);
  const float f = __double2float_rn(__dsub_rn(a, (double)i));
  const float fs = __double2float_rn(__ddiv_rn((double)S, 255.0));
  const double v = (double)V;
  const int p = pil_round8(__dmul_rn(v, __dsub_rn(1.0, (double)fs)));
  const int q = pil_round8(__dmul_rn(v, __dsub_rn(1.0, (double)__fmul_rn(fs, f))));
  const int t = pil_round8(__dmul_rn(v, __dsub_rn(1.0, __dmul_rn((double)fs, __dsub_rn(1.0, (double)f)))));
  switch (i % 6) {
    case 0: r = V, g = t, b = p; break;
    case 1: r = q, g = V, b = p; break;
    case 2: r = p, g = V, b = t; break;
    case 3: r = p, g = q, b = V; break;
    case 4: r = t, g = p, b = V; break;
    default: r = V, g = p, b = q; break;
  }
}

// One parameter set, unpacked into registers: ops holds the order three bits per position (kJitNone: no op), cut the
// contrast position (4 without contrast).
constexpr int kJitNone = 4;

struct JitterSet {
  unsigned ops;
  int cut, hue;
  float fb, fc, fs;
};

__device__ __forceinline__ JitterSet jitter_set(const raft_colour_jitter_sample& s, int k) {
  JitterSet j;
  j.ops = 0;
  j.cut = 4;
  for (int q = 0; q < 4; ++q) {
    const int op = s.order[k][q];
    j.ops |= (unsigned)(op < 0 ? kJitNone : op) << (3 * q);
    if (op == kJitContrast) j.cut = q;
  }
  j.hue = s.hue[k];
  j.fb = s.factor[k][0];
  j.fc = s.factor[k][1];
  j.fs = s.factor[k][2];
  return j;
}

// The ops at positions [from, to) of a set; contrast blends towards the grey level m.
__device__ __forceinline__ void jitter_ops(const JitterSet& j, int from, int to, int m, int c[3]) {
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    if (q < from || q >= to) continue;
    const int op = (j.ops >> (3 * q)) & 7;
    if (op == kJitNone) {
    } else if (op == kJitBrightness) {
      for (int k = 0; k < 3; ++k) c[k] = pil_blend(0, c[k], j.fb);
    } else if (op == kJitContrast) {
      for (int k = 0; k < 3; ++k) c[k] = pil_blend(m, c[k], j.fc);
    } else if (op == kJitSaturation) {
      const int l = pil_luma(c[0], c[1], c[2]);
      for (int k = 0; k < 3; ++k) c[k] = pil_blend(l, c[k], j.fs);
    } else if (op == kJitHue) {
      int h, sa, v;
      pil_rgb2hsv(c[0], c[1], c[2], h, sa, v);
      pil_hsv2rgb((h + j.hue) & 255, sa, v, c[0], c[1], c[2]);
    }
  }
}

__global__ void __launch_bounds__(kJitterThreads) colour_jitter_sum_kernel(const raft_colour_jitter_sample* __restrict__ samples,
                                                                           unsigned long long* __restrict__ sums) {
  const raft_colour_jitter_sample& s = samples[blockIdx.y];
  const JitterSet j0 = jitter_set(s, 0), j1 = jitter_set(s, s.stacked ? 0 : 1);
  if (j0.cut == 4 && j1.cut == 4) return;                    // no contrast: no mean needed
  const size_t hw = (size_t)s.H * s.W;
  unsigned long long acc0 = 0ull, acc1 = 0ull;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < 2 * hw; i += (size_t)gridDim.x * blockDim.x) {
    const bool second = i >= hw;
    const uint8_t* src = (second ? s.img2 : s.img1) + 3 * (second ? i - hw : i);
    int c[3] = {src[0], src[1], src[2]};
    const JitterSet j = second ? j1 : j0;
    jitter_ops(j, 0, j.cut, 0, c);
    const unsigned long long l = (unsigned long long)pil_luma(c[0], c[1], c[2]);
    if (second && !s.stacked) acc1 += l;
    else acc0 += l;
  }
  for (int o = 16; o > 0; o >>= 1) {
    acc0 += __shfl_down_sync(0xffffffffu, acc0, o);
    acc1 += __shfl_down_sync(0xffffffffu, acc1, o);
  }
  if ((threadIdx.x & 31) == 0) {                              // integer sums: the order does not matter
    if (acc0) atomicAdd(sums + 2 * blockIdx.y, acc0);
    if (acc1) atomicAdd(sums + 2 * blockIdx.y + 1, acc1);
  }
}

// ImageEnhance.Contrast's grey level: int(ImageStat mean + 0.5), the mean sum / n in float64 (both exact as doubles).
__device__ __forceinline__ int jitter_grey(unsigned long long sum, size_t n) {
  return __double2int_rz(__dadd_rn(__ddiv_rn((double)sum, (double)n), 0.5));
}

__global__ void __launch_bounds__(kJitterThreads) colour_jitter_apply_kernel(const raft_colour_jitter_sample* __restrict__ samples,
                                                                             const unsigned long long* __restrict__ sums) {
  const raft_colour_jitter_sample& s = samples[blockIdx.y];
  const JitterSet j0 = jitter_set(s, 0), j1 = jitter_set(s, s.stacked ? 0 : 1);
  const size_t hw = (size_t)s.H * s.W;
  const int m0 = s.stacked ? jitter_grey(sums[2 * blockIdx.y], 2 * hw) : jitter_grey(sums[2 * blockIdx.y], hw);
  const int m1 = s.stacked ? m0 : jitter_grey(sums[2 * blockIdx.y + 1], hw);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < 2 * hw; i += (size_t)gridDim.x * blockDim.x) {
    const bool second = i >= hw;
    const size_t p = 3 * (second ? i - hw : i);
    const uint8_t* src = (second ? s.img2 : s.img1) + p;
    int c[3] = {src[0], src[1], src[2]};
    jitter_ops(second ? j1 : j0, 0, 4, second ? m1 : m0, c);
    uint8_t* dst = (second ? s.out_img2 : s.out_img1) + p;
    dst[0] = (uint8_t)c[0];
    dst[1] = (uint8_t)c[1];
    dst[2] = (uint8_t)c[2];
  }
}

}  // namespace raft
