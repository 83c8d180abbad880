// Host-side TMA tensor-map construction.  cuTensorMapEncodeTiled is resolved at run time through
// cudaGetDriverEntryPoint so the library links against cudart only (no libcuda at build time).
#pragma once
#include <mutex>

#include "common.cuh"

namespace raft {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

// fp16 tensor, innermost dim contiguous, 128-byte swizzle, zero fill out of bounds.
// dims/box innermost-first; strides_bytes has rank-1 entries (dims 1..rank-1).
inline int make_tmap_f16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                         const uint64_t* strides_bytes, const uint32_t* box, const uint32_t* elem_strides = nullptr) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn) return RAFT_ERR_DRIVER;
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = elem_strides ? elem_strides[i] : 1;
    if (i > 0) gstr[i - 1] = strides_bytes[i - 1];
  }
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx,
                  es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : RAFT_ERR_DRIVER;
}

// The hi and lo planes of every operand are fetched by ONE box (TMA cost is per box more than per byte): the plane index
// is an extra tensor dimension whose stride is (lo - hi) bytes.
// Activation planes: rank-5 map (C, W, H, B, plane), box {64, tw*s, th*s, 1, 2} -> smem [hi 128 rows | lo 128 rows].
inline int make_tmap_act2(CUtensorMap* out, const __half* hi, const __half* lo, int B, int H, int W, int cstride, int tw,
                          int th, int stride = 1) {
  const ptrdiff_t pstride = reinterpret_cast<const char*>(lo) - reinterpret_cast<const char*>(hi);
  if (pstride <= 0 || (pstride & 15)) return RAFT_ERR_BAD_ARG;
  if (tw * stride > 256 || th * stride > 256) return RAFT_ERR_BAD_SHAPE;
  // dims (C, W, H, B, plane): strides stay monotonic; the box takes one image and both planes
  uint64_t dims[5] = {(uint64_t)cstride, (uint64_t)W, (uint64_t)H, (uint64_t)B, 2};
  uint64_t str[4] = {(uint64_t)cstride * 2, (uint64_t)W * cstride * 2, (uint64_t)H * W * cstride * 2, (uint64_t)pstride};
  uint32_t box[5] = {64, (uint32_t)(tw * stride), (uint32_t)(th * stride), 1, 2};
  uint32_t es[5] = {1, (uint32_t)stride, (uint32_t)stride, 1, 1};
  return make_tmap_f16(out, hi, 5, dims, str, box, es);
}
// Weight planes: rank-4 map (cin_pad, cout_pad, taps, plane), box {64, bn, 1, 2} -> smem [hi bn rows | lo bn rows].
inline int make_tmap_wgt2(CUtensorMap* out, const __half* hi, const __half* lo, int taps, int cout_pad, int cin_pad,
                          int bn) {
  const ptrdiff_t pstride = reinterpret_cast<const char*>(lo) - reinterpret_cast<const char*>(hi);
  if (pstride <= 0 || (pstride & 15)) return RAFT_ERR_BAD_ARG;
  uint64_t dims[4] = {(uint64_t)cin_pad, (uint64_t)cout_pad, (uint64_t)taps, 2};
  uint64_t str[3] = {(uint64_t)cin_pad * 2, (uint64_t)cout_pad * cin_pad * 2, (uint64_t)pstride};
  uint32_t box[4] = {64, (uint32_t)bn, 1, 2};
  return make_tmap_f16(out, hi, 4, dims, str, box);
}

}  // namespace raft
