// Training augmentation: tf_raft/datasets/augmentor.py's FlowAugmentor and SparseFlowAugmentor given their random draws
// (the draws themselves live on the host, tf_raft_b200/datasets/augmentor.py).  One launch set serves a batch whose
// samples have different source sizes: every kernel reads a device array of raft_augment_sample and runs
// grid (x, B), blockIdx.y = sample, grid-striding over that sample's pixels.
//   augment_init_kernel     zero the eraser channel sums; sparse: fill the target maps with -1
//   augment_colour_kernel   LUTs + RGB<->HSV of both sources into the workspace, uint64 channel sums of img2
//   augment_scatter_kernel  sparse only: atomicMax of the source index per resized target (the last source wins)
//   augment_gather_kernel   one thread per output pixel: flips and crop, cv2 INTER_LINEAR resize of both images with the
//                           eraser applied to fetched texels, the flow (dense: resized, fp64-scaled, valid) or its map
// The arithmetic is cv2's (DESIGN.md section 3.5, oracle/augment_np.py): explicitly rounded intrinsics, no FMA except the
// one HSV->RGB rounds once.
#pragma once
#include "kernels.cuh"

namespace raft {

constexpr int kAugThreads = 256;

// Per-sample workspace: colour-transformed img1 and img2 (H*W*3 bytes each), 3 uint64 channel sums of img2, and for a
// sparse spatial sample the (rh, rw) int32 target map.
struct AugLayout {
  size_t img1, img2, sums, map, total;
};
__host__ __device__ inline AugLayout aug_layout(int H, int W, int rh, int rw, bool map) {
  AugLayout L;
  const size_t px = (size_t)H * W * 3;
  L.img1 = 0;
  L.img2 = px;
  L.sums = (2 * px + 7) / 8 * 8;
  L.map = L.sums + 3 * sizeof(unsigned long long);
  L.total = (L.map + (map ? (size_t)rh * rw * sizeof(int) : 0) + 255) / 256 * 256;
  return L;
}

// cv2's output size of a spatial sample: saturate_cast<int>(n * scale), round half to even.
__host__ __device__ inline int aug_resized(int n, double scale) {
#ifdef __CUDA_ARCH__
  return __double2int_rn(__dmul_rn((double)n, scale));
#else
  return (int)nearbyint((double)n * scale);
#endif
}

__global__ void augment_init_kernel(const raft_augment_sample* __restrict__ samples, uint8_t* __restrict__ ws, int sparse) {
  const raft_augment_sample& s = samples[blockIdx.y];
  const bool map = sparse && s.spatial;
  const int rh = map ? aug_resized(s.H, s.scale_y) : 0, rw = map ? aug_resized(s.W, s.scale_x) : 0;
  const AugLayout L = aug_layout(s.H, s.W, rh, rw, map);
  uint8_t* base = ws + s.ws_offset;
  if (blockIdx.x == 0 && threadIdx.x < 3) reinterpret_cast<unsigned long long*>(base + L.sums)[threadIdx.x] = 0ull;
  int* m = reinterpret_cast<int*>(base + L.map);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)rh * rw; i += (size_t)gridDim.x * blockDim.x)
    m[i] = -1;
}

// ------------------------------------------------------------------------------------------------
// Colour.  RGB->HSV is cv2's uint8 RGB2HSV_b: hsv_shift = 12 fixed point with sdiv[v] = rint((255 << 12) / v) and
// hdiv[d] = rint((180 << 12) / (6 d)) (computed here in exact integers, equal to cv2's double rounding).  HSV->RGB is
// cv2's HSV2RGB_b: s, v scaled by 1/255 and h by 6/180 in float32, sector = floor, and the table v, v(1-s),
// v*fma(-s, f, 1), v*fma(-s, 1-f, 1), then *255.  cv2 converts each row in blocks of kHsvBlock pixels (4 float32
// vectors of its x86 AVX2 dispatch, also taken on AVX-512 CPUs), which truncate, and the last W mod kHsvBlock pixels of
// the row in a scalar loop, which rounds half to even.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int rint_div(int n, int d) {        // round-half-even n / d, n, d > 0
  const int q = n / d, r2 = 2 * (n - q * d);
  return q + ((r2 > d || (r2 == d && (q & 1))) ? 1 : 0);
}

__device__ __forceinline__ void rgb2hsv_u8(int r, int g, int b, const int* sdiv, const int* hdiv, int& h, int& s, int& v) {
  v = max(max(r, g), b);
  const int diff = v - min(min(r, g), b);
  s = (diff * sdiv[v] + (1 << 11)) >> 12;
  h = v == r ? g - b : (v == g ? b - r + 2 * diff : r - g + 4 * diff);
  h = (h * hdiv[diff] + (1 << 11)) >> 12;
  if (h < 0) h += 180;
}

constexpr int kHsvBlock = 32;

__device__ __forceinline__ int hsv_out(float x, bool tail) {
  const float y = __fmul_rn(x, 255.0f);
  return min(tail ? __float2int_rn(y) : (int)y, 255);
}

__device__ __forceinline__ void hsv2rgb_u8(int H, int S, int V, bool tail, int& r, int& g, int& b) {
  const float s = __fmul_rn((float)S, 1.0f / 255.0f), v = __fmul_rn((float)V, 1.0f / 255.0f);
  const float hs = __fmul_rn((float)H, 6.0f / 180.0f);
  const float sec = floorf(hs), f = __fsub_rn(hs, sec);
  const float t1 = __fmul_rn(v, __fsub_rn(1.0f, s));
  const float t2 = __fmul_rn(v, __fmaf_rn(-s, f, 1.0f));
  const float t3 = __fmul_rn(v, __fmaf_rn(-s, __fsub_rn(1.0f, f), 1.0f));
  auto pick = [&](int e) { return e == 0 ? v : e == 1 ? t1 : e == 2 ? t2 : t3; };
  // cv2's sector table, (b, g, r) entries {1,3,0},{1,0,2},{3,0,1},{0,2,1},{0,1,3},{2,1,0}, two bits per sector
  constexpr unsigned kB = 1u | 1u << 2 | 3u << 4 | 0u << 6 | 0u << 8 | 2u << 10;
  constexpr unsigned kG = 3u | 0u << 2 | 0u << 4 | 2u << 6 | 1u << 8 | 1u << 10;
  constexpr unsigned kR = 0u | 2u << 2 | 1u << 4 | 1u << 6 | 3u << 8 | 0u << 10;
  const int k = 2 * ((int)sec % 6);                           // H < 180: sec in [0, 5]
  b = hsv_out(pick((kB >> k) & 3), tail);
  g = hsv_out(pick((kG >> k) & 3), tail);
  r = hsv_out(pick((kR >> k) & 3), tail);
}

__global__ void __launch_bounds__(kAugThreads) augment_colour_kernel(const raft_augment_sample* __restrict__ samples,
                                                                     uint8_t* __restrict__ ws) {
  __shared__ int sdiv[256], hdiv[256];
  __shared__ uint8_t lut[2][4][256];
  const raft_augment_sample& s = samples[blockIdx.y];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    sdiv[i] = i ? rint_div(255 << 12, i) : 0;
    hdiv[i] = i ? rint_div(180 << 12, 6 * i) : 0;
  }
  for (int i = threadIdx.x; i < 2 * 4 * 256; i += blockDim.x) (&lut[0][0][0])[i] = (&s.lut[0][0][0])[i];
  __syncthreads();
  const size_t hw = (size_t)s.H * s.W;
  const AugLayout L = aug_layout(s.H, s.W, 0, 0, false);
  uint8_t* base = ws + s.ws_offset;
  unsigned long long sum[3] = {0ull, 0ull, 0ull};
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < 2 * hw; i += (size_t)gridDim.x * blockDim.x) {
    const int k = i >= hw;
    const size_t p = 3 * (k ? i - hw : i);
    const uint8_t* src = (k ? s.img2 : s.img1) + p;
    int r = lut[k][0][src[0]], g = lut[k][0][src[1]], b = lut[k][0][src[2]];
    if (s.hsv[k]) {
      int h, sa, v;
      rgb2hsv_u8(r, g, b, sdiv, hdiv, h, sa, v);
      const bool tail = (int)((p / 3) % s.W) >= s.W - s.W % kHsvBlock;      // cv2's scalar row tail
      hsv2rgb_u8(lut[k][1][h], lut[k][2][sa], lut[k][3][v], tail, r, g, b);
    }
    uint8_t* dst = base + (k ? L.img2 : L.img1) + p;
    dst[0] = (uint8_t)r;
    dst[1] = (uint8_t)g;
    dst[2] = (uint8_t)b;
    if (k) {
      sum[0] += r;
      sum[1] += g;
      sum[2] += b;
    }
  }
  if (s.n_rects == 0) return;                                      // uniform per block
  unsigned long long* sums = reinterpret_cast<unsigned long long*>(base + L.sums);
  for (int c = 0; c < 3; ++c) {
    unsigned long long v = sum[c];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(sums + c, v);     // integer sums: the order does not matter
  }
}

// resize_sparse_flow_map (augmentor.py:183-215): source (x, y) with valid >= 1 lands at (rint(x*fx), rint(y*fy)), fp64,
// half to even; kept iff 0 < xx < rw and 0 < yy < rh.  NumPy's fancy assignment keeps the last source in index order.
__global__ void __launch_bounds__(kAugThreads) augment_scatter_kernel(const raft_augment_sample* __restrict__ samples,
                                                                      uint8_t* __restrict__ ws) {
  const raft_augment_sample& s = samples[blockIdx.y];
  if (!s.spatial) return;
  const int rh = aug_resized(s.H, s.scale_y), rw = aug_resized(s.W, s.scale_x);
  int* m = reinterpret_cast<int*>(ws + s.ws_offset + aug_layout(s.H, s.W, rh, rw, true).map);
  const int n = s.H * s.W;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (!(s.valid[i] >= 1.0f)) continue;
    const int xx = __double2int_rn(__dmul_rn((double)(i % s.W), s.scale_x));
    const int yy = __double2int_rn(__dmul_rn((double)(i / s.W), s.scale_y));
    if (xx > 0 && xx < rw && yy > 0 && yy < rh) atomicMax(m + (size_t)yy * rw + xx, i);
  }
}

// ------------------------------------------------------------------------------------------------
// Gather.  cv2.resize INTER_LINEAR at output (X, Y) of an (H, W) source scaled by (fx, fy):
//   f = float((d + 0.5) * (1/scale) - 0.5) (fp64, rounded once each), s = floor(f), f -= s;
//   x: outside [0, W-1) the tap is the edge pixel with f = 0 (and a left tap at the last column reads S alone);
//   y: rows clamp(s), clamp(s + 1) with the unclamped weights (1 - f, f).
// uint8: weights rint(w*2048), exact horizontal sum, vertical ((S0>>4)*b0 >> 16) + ((S1>>4)*b1 >> 16) + 2 >> 2.
// float32: S0*a0 + S1*a1 per row, then R0*b0 + R1*b1, each operation rounded.
// ------------------------------------------------------------------------------------------------
struct Taps {
  int x0, x1, y0, y1;
  bool two;
  float a0, a1, b0, b1;
};

__device__ __forceinline__ float src_coord(int d, double inv) {
  return __double2float_rn(__dsub_rn(__dmul_rn((double)d + 0.5, inv), 0.5));
}

__device__ __forceinline__ Taps resize_taps(int X, int Y, int H, int W, double inv_x, double inv_y) {
  Taps t;
  float fx = src_coord(X, inv_x);
  const float sx = floorf(fx);
  fx = __fsub_rn(fx, sx);
  int ix = (int)sx;
  t.two = ix < W - 1;
  if (ix < 0 || ix >= W - 1) {
    fx = 0.0f;
    ix = min(max(ix, 0), W - 1);
  }
  t.x0 = ix;
  t.x1 = min(ix + 1, W - 1);
  t.a0 = __fsub_rn(1.0f, fx);
  t.a1 = fx;
  float fy = src_coord(Y, inv_y);
  const float sy = floorf(fy);
  fy = __fsub_rn(fy, sy);
  const int iy = (int)sy;
  t.y0 = min(max(iy, 0), H - 1);
  t.y1 = min(max(iy + 1, 0), H - 1);
  t.b0 = __fsub_rn(1.0f, fy);
  t.b1 = fy;
  return t;
}

struct Eraser {
  int n;
  const int (*rect)[4];
  uint8_t mean[3];
  __device__ __forceinline__ bool covers(int x, int y) const {
    bool in = false;
    for (int r = 0; r < n; ++r)
      in |= x >= rect[r][0] && x - rect[r][0] < rect[r][2] && y >= rect[r][1] && y - rect[r][1] < rect[r][3];
    return in;
  }
};

__device__ __forceinline__ void texel(const uint8_t* img, int W, int x, int y, const Eraser* er, int out[3]) {
  if (er && er->covers(x, y)) {
    out[0] = er->mean[0], out[1] = er->mean[1], out[2] = er->mean[2];
    return;
  }
  const uint8_t* p = img + 3 * ((size_t)y * W + x);
  out[0] = p[0], out[1] = p[1], out[2] = p[2];
}

__device__ __forceinline__ void resize_u8(const uint8_t* img, int W, const Taps& t, const Eraser* er, uint8_t* out) {
  const int a0 = __float2int_rn(__fmul_rn(t.a0, 2048.0f)), a1 = __float2int_rn(__fmul_rn(t.a1, 2048.0f));
  const int b0 = __float2int_rn(__fmul_rn(t.b0, 2048.0f)), b1 = __float2int_rn(__fmul_rn(t.b1, 2048.0f));
  int p00[3], p01[3], p10[3], p11[3];
  texel(img, W, t.x0, t.y0, er, p00);
  texel(img, W, t.x1, t.y0, er, p01);
  texel(img, W, t.x0, t.y1, er, p10);
  texel(img, W, t.x1, t.y1, er, p11);
  for (int c = 0; c < 3; ++c) {
    const int d0 = p00[c] * a0 + p01[c] * a1, d1 = p10[c] * a0 + p11[c] * a1;
    const int v = ((((d0 >> 4) * b0) >> 16) + (((d1 >> 4) * b1) >> 16) + 2) >> 2;
    out[c] = (uint8_t)min(max(v, 0), 255);
  }
}

__device__ __forceinline__ float resize_row_f32(const float* row, const Taps& t, int c) {
  const float s0 = row[2 * t.x0 + c];
  return t.two ? __fadd_rn(__fmul_rn(s0, t.a0), __fmul_rn(row[2 * t.x1 + c], t.a1)) : __fmul_rn(s0, 1.0f);
}

__global__ void __launch_bounds__(kAugThreads) augment_gather_kernel(const raft_augment_sample* __restrict__ samples,
                                                                     const uint8_t* __restrict__ ws, int sparse) {
  const raft_augment_sample& s = samples[blockIdx.y];
  const int rh = s.spatial ? aug_resized(s.H, s.scale_y) : s.H, rw = s.spatial ? aug_resized(s.W, s.scale_x) : s.W;
  const AugLayout L = aug_layout(s.H, s.W, rh, rw, sparse && s.spatial);
  const uint8_t* base = ws + s.ws_offset;
  const uint8_t* c1 = base + L.img1;
  const uint8_t* c2 = base + L.img2;
  const int* map = reinterpret_cast<const int*>(base + L.map);
  Eraser er;
  er.n = s.n_rects;
  er.rect = s.rect;
  if (er.n) {
    const unsigned long long* sums = reinterpret_cast<const unsigned long long*>(base + L.sums);
    const double n = (double)s.H * s.W;
    for (int c = 0; c < 3; ++c) er.mean[c] = (uint8_t)(int)__ddiv_rn((double)sums[c], n);   // np.mean, truncated
  }
  const double inv_x = __drcp_rn(s.scale_x), inv_y = __drcp_rn(s.scale_y);
  const int n_out = s.crop_h * s.crop_w;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < n_out; p += gridDim.x * blockDim.x) {
    int Y = s.y0 + p / s.crop_w, X = s.x0 + p % s.crop_w;   // in the flipped, resized image
    if (s.vflip) Y = rh - 1 - Y;
    if (s.hflip) X = rw - 1 - X;
    uint8_t o1[3], o2[3];
    double fx, fy;
    float valid;
    if (s.spatial) {
      const Taps t = resize_taps(X, Y, s.H, s.W, inv_x, inv_y);
      resize_u8(c1, s.W, t, nullptr, o1);
      resize_u8(c2, s.W, t, er.n ? &er : nullptr, o2);
      if (!sparse) {
        const float* r0 = s.flow + (size_t)t.y0 * s.W * 2;
        const float* r1 = s.flow + (size_t)t.y1 * s.W * 2;
        const float vx = __fadd_rn(__fmul_rn(resize_row_f32(r0, t, 0), t.b0), __fmul_rn(resize_row_f32(r1, t, 0), t.b1));
        const float vy = __fadd_rn(__fmul_rn(resize_row_f32(r0, t, 1), t.b0), __fmul_rn(resize_row_f32(r1, t, 1), t.b1));
        fx = __dmul_rn((double)vx, s.scale_x);
        fy = __dmul_rn((double)vy, s.scale_y);
      } else {
        const int i = map[(size_t)Y * rw + X];
        fx = i >= 0 ? (double)__double2float_rn(__dmul_rn((double)s.flow[2 * (size_t)i], s.scale_x)) : 0.0;
        fy = i >= 0 ? (double)__double2float_rn(__dmul_rn((double)s.flow[2 * (size_t)i + 1], s.scale_y)) : 0.0;
        valid = i >= 0 ? 1.0f : 0.0f;
      }
    } else {
      int t1[3], t2[3];
      texel(c1, s.W, X, Y, nullptr, t1);
      texel(c2, s.W, X, Y, er.n ? &er : nullptr, t2);
      for (int c = 0; c < 3; ++c) o1[c] = (uint8_t)t1[c], o2[c] = (uint8_t)t2[c];
      const size_t q = (size_t)Y * s.W + X;
      fx = (double)s.flow[2 * q];
      fy = (double)s.flow[2 * q + 1];
      if (sparse) valid = s.valid[q];
    }
    if (s.hflip) fx = -fx;                                    // flow * [-1.0, 1.0]
    if (s.vflip) fy = -fy;
    if (!sparse) valid = (fabs(fx) < 1000.0 && fabs(fy) < 1000.0) ? 1.0f : 0.0f;   // dataset.py:102, on the fp64 flow
    for (int c = 0; c < 3; ++c) {
      s.out_img1[3 * (size_t)p + c] = o1[c];
      s.out_img2[3 * (size_t)p + c] = o2[c];
    }
    s.out_flow[2 * (size_t)p] = __double2float_rn(fx);
    s.out_flow[2 * (size_t)p + 1] = __double2float_rn(fy);
    s.out_valid[p] = valid;
  }
}

}  // namespace raft
