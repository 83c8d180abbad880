// Flow warping and flow composition (additions beyond tf-raft): backward warping of an image, feature map or label map
// by a flow, and the chaining step of long-range tracking.  Both use fb_occlusion_kernel's landing, frame test and
// bilinear rule (video.cuh), restated here so that kernel's code stays as it is.
#pragma once
#include "kernels.cuh"

namespace raft {

// Landing p = (x + fx, y + fy) of pixel (x, y) and the closed-frame test on a (Hs, Ws) grid; NaN is never inside.
struct Landing {
  float px, py;
  bool inside;
};

__device__ __forceinline__ Landing land(float2 f, int x, int y, int Hs, int Ws) {
  Landing l;
  l.px = __fadd_rn((float)x, f.x);
  l.py = __fadd_rn((float)y, f.y);
  l.inside = l.px >= 0.0f && l.px <= (float)(Ws - 1) && l.py >= 0.0f && l.py <= (float)(Hs - 1);
  return l;
}

// Corners and weights of the bilinear sample at an inside landing: x0 = floor(px), x1 = min(x0 + 1, Ws - 1),
// ax = px - x0, bx = 1 - ax (y likewise); offsets are texel indices (y * Ws + x) within the image.
struct Bilinear {
  size_t o00, o01, o10, o11;
  float ax, bx, ay, by;
};

__device__ __forceinline__ Bilinear bilinear_at(const Landing& l, int Hs, int Ws) {
  const float fx0 = floorf(l.px), fy0 = floorf(l.py);
  const int x0 = (int)fx0, y0 = (int)fy0;
  const int x1 = min(x0 + 1, Ws - 1), y1 = min(y0 + 1, Hs - 1);
  Bilinear s;
  s.ax = __fsub_rn(l.px, fx0);
  s.bx = __fsub_rn(1.0f, s.ax);
  s.ay = __fsub_rn(l.py, fy0);
  s.by = __fsub_rn(1.0f, s.ay);
  s.o00 = (size_t)y0 * Ws + x0;
  s.o01 = (size_t)y0 * Ws + x1;
  s.o10 = (size_t)y1 * Ws + x0;
  s.o11 = (size_t)y1 * Ws + x1;
  return s;
}

// by*(bx*t00 + ax*t01) + ay*(bx*t10 + ax*t11), each operation one rounded fp32 operation (no FMA); a non-finite texel
// makes the result non-finite even at weight 0.
__device__ __forceinline__ float blend(const Bilinear& s, float t00, float t01, float t10, float t11) {
  return __fadd_rn(__fmul_rn(s.by, __fadd_rn(__fmul_rn(s.bx, t00), __fmul_rn(s.ax, t01))),
                   __fmul_rn(s.ay, __fadd_rn(__fmul_rn(s.bx, t10), __fmul_rn(s.ax, t11))));
}

// Nearest texel of an inside landing: floor(p + 0.5) (one fp32 addition), clamped to the last row / column.
__device__ __forceinline__ size_t nearest_at(const Landing& l, int Hs, int Ws) {
  const int xi = min((int)floorf(__fadd_rn(l.px, 0.5f)), Ws - 1);
  const int yi = min((int)floorf(__fadd_rn(l.py, 0.5f)), Hs - 1);
  return (size_t)yi * Ws + xi;
}

// ------------------------------------------------------------------------------------------------
// warp: out[b, y, x, c] = sample of src[b] (Hs, Ws, C) at the landing of flow[b, y, x] (an (H, W) grid), `fill` where
// the landing is outside src's closed frame or not finite, and occ[b, y, x] = 1 there (0 elsewhere; occ may be NULL).
// One thread per output element (pixel, channel), grid-stride; the channel-0 thread writes occ.
// ------------------------------------------------------------------------------------------------
template <class T>
struct WarpParams {
  const T* src;
  const float2* flow;
  T* out;
  uint8_t* occ;
  int B, Hs, Ws, C, H, W;
  T fill;
};

template <class T, bool kBilinear>
__global__ void warp_kernel(const WarpParams<T> p) {
  const size_t hw = (size_t)p.H * p.W, n = (size_t)p.B * hw * p.C, src_img = (size_t)p.Hs * p.Ws * p.C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const size_t pix = i / p.C;
    const int c = (int)(i - pix * p.C);
    const size_t b = pix / hw, q = pix - b * hw;
    const Landing l = land(p.flow[pix], (int)(q % p.W), (int)(q / p.W), p.Hs, p.Ws);
    T v = p.fill;
    if (l.inside) {
      const T* s = p.src + b * src_img + c;
      if constexpr (kBilinear) {
        const Bilinear w = bilinear_at(l, p.Hs, p.Ws);
        v = blend(w, s[w.o00 * p.C], s[w.o01 * p.C], s[w.o10 * p.C], s[w.o11 * p.C]);
      } else {
        v = s[nearest_at(l, p.Hs, p.Ws) * p.C];
      }
    }
    p.out[i] = v;
    if (p.occ && c == 0) p.occ[pix] = l.inside ? 0 : 1;
  }
}

// ------------------------------------------------------------------------------------------------
// compose_flow: with p the landing of f1 at pixel (x, y) of image b,
//   out(x) = f1(x) + bilinear(f2[b], p),
//   occ_out(x) = occ1(x) || !inside(p) || occ2[b](nearest(p)) || !finite(out(x)),
// and out(x) = f1(x) wherever occ_out(x) is set.  occ1 / occ2 may be NULL (no mask).  Each thread reads f1 and occ1 at
// its own pixel only, so out may be f1 and occ_out may be occ1; f2 is read at other pixels and must not be out.
// ------------------------------------------------------------------------------------------------
__global__ void compose_flow_kernel(const float2* f1, const float2* __restrict__ f2, const uint8_t* occ1,
                                    const uint8_t* __restrict__ occ2, int B, int H, int W, float2* out,
                                    uint8_t* occ_out) {
  const size_t hw = (size_t)H * W, n = (size_t)B * hw;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const size_t b = i / hw, q = i - b * hw;
    const float2 f = f1[i];
    bool lost = occ1 && occ1[i];
    float2 o = f;
    const Landing l = land(f, (int)(q % W), (int)(q / W), H, W);
    if (!l.inside) lost = true;
    if (!lost) {
      const float2* g = f2 + b * hw;
      const Bilinear w = bilinear_at(l, H, W);
      const float2 g00 = g[w.o00], g01 = g[w.o01], g10 = g[w.o10], g11 = g[w.o11];
      const float sx = __fadd_rn(f.x, blend(w, g00.x, g01.x, g10.x, g11.x));
      const float sy = __fadd_rn(f.y, blend(w, g00.y, g01.y, g10.y, g11.y));
      if (occ2 && occ2[b * hw + nearest_at(l, H, W)]) lost = true;
      if (!isfinite(sx) || !isfinite(sy)) lost = true;
      if (!lost) o = make_float2(sx, sy);
    }
    out[i] = o;
    occ_out[i] = lost ? 1 : 0;
  }
}

}  // namespace raft
