// Evaluation padding (DESIGN.md section 3.5):
//   pad_planes_kernel  grid (row blocks, planes): every (H, W, c) destination plane of a batch -- image1, image2, flow
//                      and valid of each item -- written in one launch from its (h, w, c) source placed at (top, left):
//                      dst(y, x) = src(clamp(y - top), clamp(x - left)) (replicate: RAFT's InputPadder) or src(y - top,
//                      x - left) inside the source and 0 outside it (zero: CropOrPadder).  Pure copies, bit-exact.
#pragma once
#include "kernels.cuh"

namespace raft {

constexpr int kPadThreads = 256;
constexpr int kPadMaxRowBlocks = 2048;         // grid.x: rows of a plane are strided over at most this many CTAs

template <typename T>
__device__ __forceinline__ void pad_plane_rows(const raft_pad_plane& p) {
  const T* __restrict__ src = static_cast<const T*>(p.src);
  T* __restrict__ dst = static_cast<T*>(p.dst);
  const int c = p.c, row = p.W * c, src_row = p.w * c;
  const bool rep = p.mode == RAFT_PAD_REPLICATE;
  for (int y = blockIdx.x; y < p.H; y += gridDim.x) {
    int sy = y - p.top;
    bool in_y = sy >= 0 && sy < p.h;
    if (rep) {
      sy = min(max(sy, 0), p.h - 1);
      in_y = true;
    }
    const T* s = src + (in_y ? (size_t)sy * src_row : 0);
    T* d = dst + (size_t)y * row;
    for (int i = threadIdx.x; i < row; i += kPadThreads) {
      const int x = i / c, ch = i - x * c;
      int sx = x - p.left;
      bool in = in_y && sx >= 0 && sx < p.w;
      if (rep) {
        sx = min(max(sx, 0), p.w - 1);
        in = true;
      }
      d[i] = in ? s[sx * c + ch] : T(0);
    }
  }
}

__global__ void __launch_bounds__(kPadThreads) pad_planes_kernel(const raft_pad_plane* __restrict__ planes) {
  const raft_pad_plane p = planes[blockIdx.y];
  if (p.dtype == RAFT_PAD_U8) pad_plane_rows<uint8_t>(p);
  else pad_plane_rows<float>(p);
}

}  // namespace raft
