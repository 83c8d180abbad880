// wgmma implicit-GEMM kernel: one kernel serves every convolution of the encoders and the update blocks.
//
//   D[128 px, bn cout] = sum over (tap, 64-channel chunk) of  A_tap[128 px, 64] * W_tap[bn, 64]^T
//
// * A operand: a TH x TW pixel patch of an NHWC fp16 activation plane, fetched by ONE TMA box per (tap, chunk) at
//   coordinates shifted by the tap offset; out-of-image rows/cols are zero-filled by the TMA unit, which *is* Keras
//   'same' padding -- no im2col buffer, no halo logic.
// * B operand: packed weights [tap][cout][cin] fp16, one TMA box per (tap, chunk).
// * Both operands land in shared memory K-major with the 128-byte swizzle and are consumed in place by
//   wgmma.mma_async (m64nNk16, fp16 x fp16 -> fp32 registers).
// * fp32-grade arithmetic from fp16 tensor cores: each operand is a (hi, lo) fp16 pair and every K step issues hi*hi,
//   hi*lo, lo*hi into the same accumulator (DESIGN.md "Precision").
// * Tensor-core fp32 accumulation is not IEEE round-to-nearest, so a 1920-deep GRU contraction issued as one 360-step
//   chain drifts far more than an FFMA chain.  The K loop is therefore cut into groups of `group_chunks` 64-channel
//   chunks; each group accumulates into a fresh register tile that is then promoted -- added in IEEE fp32 -- into a
//   second register tile.  Two register copies of a 64 x N accumulator per warpgroup bound N to kMaxTileN = 128; the
//   host splits wider layers into column tiles.
// * Warp roles: warps 0..7 = two consumer warpgroups (rows [0, 64) and [64, 128) of the tile: MMAs, promotion and the
//   fused epilogue -- bias / activation / GRU gating / hi-lo re-split -> global, through a 64-column shared-memory
//   staging tile so that each thread owns one pixel row); warp 8 = TMA producer (one elected lane; its warpgroup hands
//   its registers to the consumers with setmaxnreg, so the two accumulator copies fit without spills).  mbarrier ring:
//   full (producer -> consumers) / empty (consumers -> producer).  The producer runs up to nstages ahead, so the loads of
//   tile i+1 overlap the epilogue of tile i.
#pragma once
#include "common.cuh"
#include "kernels.cuh"
#include "tmap.cuh"

namespace raft {

enum TcEpilogue : int {
  EPI_LINEAR = 0,  // v = act(acc*inv_scale + bias) * out_scale  -> optional fp32 and/or fp16 hi/lo planes
  EPI_GRU_ZR = 1,  // cols [0,hid): z = sigmoid(v) -> z plane; cols [hid,2hid): r = sigmoid(v), r*h -> hi/lo planes
  EPI_GRU_Q = 2,   // q = tanh(v); h = (1-z)*h + z*q -> h fp32 (in place) + hi/lo planes
};
enum TcAct : int { ACT_NONE = 0, ACT_RELU = 1 };

constexpr int kTileM = 128;
constexpr int kChunkK = 64;                       // fp16 elements per 128-byte swizzled row
constexpr int kABytes = kTileM * kChunkK * 2;     // 16 KiB per A plane per stage
constexpr int kMaxTileN = 128;                    // accumulator columns per tile (two register copies per thread, see above)
constexpr int kConsumerWGs = 2;                   // MMA + epilogue warpgroups: rows [0, 64) and [64, 128) of the tile
constexpr int kConsumerWarps = 4 * kConsumerWGs;
constexpr int kTcThreads = 128 * kConsumerWGs + 128;  // + a producer warpgroup: its first warp issues the TMA loads
constexpr int kStageCols = 64;                    // epilogue staging: 64 rows x 64 fp32 columns per warpgroup
constexpr int kStagingBytes = kConsumerWGs * 64 * kStageCols * 4;
constexpr int kSmemMax = 227 * 1024;              // dynamic shared memory per block on sm_90
constexpr int kSmemFixed = 1024 /*align slack*/ + kStagingBytes + 512 /*barriers, item queue*/;

struct alignas(64) TcConvParams {
  CUtensorMap a_map[2];           // (hi, lo) plane pair of up to two channel-concatenated sources (K segments)
  CUtensorMap b_map;              // (hi, lo) plane pair of the packed weights
  int nseg, seg_chunks[2], seg_c0[2];
  int kh, kw, ph, pw;             // taps and 'same' padding (pad before)
  int stride;                     // 1 or 2: input pixel = output pixel * stride + tap - pad (TMA elementStrides)
  int B, H, W, TH, TW, tiles_x, tiles_y;
  int bn, n_total;                // N per CTA (multiple of 16, <= kMaxTileN); total valid output columns
  int n_tiles_n;                  // column tiles (tile id = n_tile * pixel_tiles + pixel_tile)
  int nstages, stage_bytes;
  int group_chunks;               // K chunks per promotion group (accumulation chain = 12 * group_chunks MMAs)
  int mode, act;
  const float* bias;              // [n_total padded to bn multiple]; may be null
  const float* inv_scale;         // device scalar: 1 / (2^k weight scale); may be null (=1)
  float out_scale;                // applied after the activation (0.25 for the mask head)
  float* out_f32; int f32_stride, f32_c0;
  __half* out_hi; __half* out_lo; int h_stride, h_c0;
  const float* post_scale;        // EPI_LINEAR: optional per-column affine after the bias (folded BatchNorm):
  const float* post_shift;        //   v = v * post_scale[col] + post_shift[col]
  const float* residual; int res_stride, res_c0;   // EPI_LINEAR: optional skip input: v = relu(act(v) + residual)
  const float* concat_src; int concat_n;   // EPI_LINEAR: fp32 (px, concat_n) appended at columns [n_total, n_total+concat_n)
  float* z; int hid;                       // GRU: z plane (px, hid) fp32
  float* h;                                // GRU: hidden state (px, hid) fp32, updated in place by EPI_GRU_Q
  // EPI_LINEAR with n_total == 2 (flow_head.conv2) inside the iteration loop: coords1 += delta_flow and
  // flow = coords1 - coords0 (model.py:102, :97) are applied by the thread that holds the pixel's two output columns.
  float* adv_coords;                       // (px, 2) coords1, updated in place; null = no fused advance
  float* adv_flow;                         // (px, 2) coords1 - pixel grid
};

#if defined(__CUDA_ARCH__)
// 16-byte global accesses and the fast activation forms used by every epilogue.
__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
// 32 bytes per lane as two 16-byte accesses (sm_90 has no 32-byte global load / store).  `p` must be 32-byte aligned.
__device__ __forceinline__ void st8u(void* p, const uint32_t (&r)[8]) {
  reinterpret_cast<uint4*>(p)[0] = make_uint4(r[0], r[1], r[2], r[3]);
  reinterpret_cast<uint4*>(p)[1] = make_uint4(r[4], r[5], r[6], r[7]);
}
// L2-coherent (tensors another CTA of the same grid may have written) and read-only forms.
__device__ __forceinline__ void ldcg8(const float* p, float (&r)[8]) {
  const float4 a = __ldcg(reinterpret_cast<const float4*>(p)), b = __ldcg(reinterpret_cast<const float4*>(p) + 1);
  r[0] = a.x; r[1] = a.y; r[2] = a.z; r[3] = a.w; r[4] = b.x; r[5] = b.y; r[6] = b.z; r[7] = b.w;
}
__device__ __forceinline__ void ldnc8(const float* p, float (&r)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  r[0] = a.x; r[1] = a.y; r[2] = a.z; r[3] = a.w; r[4] = b.x; r[5] = b.y; r[6] = b.z; r[7] = b.w;
}
__device__ __forceinline__ void st8f(float* p, float a, float b, float c, float d, float e, float f, float g, float h) {
  const uint32_t r[8] = {__float_as_uint(a), __float_as_uint(b), __float_as_uint(c), __float_as_uint(d),
                         __float_as_uint(e), __float_as_uint(f), __float_as_uint(g), __float_as_uint(h)};
  st8u(p, r);
}
// L2-coherent 16-byte load (ld.global.cg): z and h may have been written by another CTA of the SAME grid (update_mega_kernel),
// so they must not be served from this SM's L1 nor through the non-coherent path.
__device__ __forceinline__ float4 ldcg4(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }

__device__ __forceinline__ float fast_sigmoid(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
__device__ __forceinline__ float fast_tanh(float x) { return 1.0f - __fdividef(2.0f, 1.0f + __expf(2.0f * x)); }

// ------------------------------------------------------------------------------------------------
// Register-resident epilogue of one 32-column chunk of one pixel row (thread == row).
//
// With 227 KB of the unified L1/shared array configured as shared memory, per-thread local memory does not stay in L1,
// so nothing here leaves registers: the routine is inlined and specialised on the epilogue mode at compile time, loops
// are fully unrolled so the independent 16-byte global loads (bias, h, z, residual) are all in flight together, and the
// activation math uses the fast exp / reciprocal units (|error| ~1e-7, far inside the parity budget).
// ------------------------------------------------------------------------------------------------
template <int MODE>
__device__ __forceinline__ void tc_epilogue_regs(const TcConvParams& p, float (&v)[32], size_t pix, int col, int ncol,
                                                 float inv_scale) {
  // bias + folded BatchNorm affine (arrays are zero-padded past the last column)
  if (p.bias) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float4 bq = ldg4(p.bias + col + 4 * q);
      v[4 * q] = v[4 * q] * inv_scale + bq.x; v[4 * q + 1] = v[4 * q + 1] * inv_scale + bq.y;
      v[4 * q + 2] = v[4 * q + 2] * inv_scale + bq.z; v[4 * q + 3] = v[4 * q + 3] * inv_scale + bq.w;
    }
  } else {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] *= inv_scale;
  }
  if (MODE == EPI_LINEAR && p.post_scale) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float4 sc = ldg4(p.post_scale + col + 4 * q), sh = ldg4(p.post_shift + col + 4 * q);
      v[4 * q] = v[4 * q] * sc.x + sh.x; v[4 * q + 1] = v[4 * q + 1] * sc.y + sh.y;
      v[4 * q + 2] = v[4 * q + 2] * sc.z + sh.z; v[4 * q + 3] = v[4 * q + 3] * sc.w + sh.w;
    }
  }

  __half* dhi = nullptr;
  __half* dlo = nullptr;
  if (MODE == EPI_LINEAR) {
    const bool full = col + 32 <= p.n_total;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      if (p.act == ACT_RELU) v[j] = relu_nan(v[j]);
      v[j] *= p.out_scale;
    }
    if (full) {
      if (p.residual) {
        const float* rp = p.residual + pix * (size_t)p.res_stride + p.res_c0 + col;
        if (((p.res_stride | p.res_c0) & 7) == 0) {
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            float r8[8];
            ldnc8(rp + 8 * q, r8);
#pragma unroll
            for (int e = 0; e < 8; ++e) v[8 * q + e] = relu_nan(v[8 * q + e] + r8[e]);
          }
        } else if (((p.res_stride | p.res_c0) & 3) == 0) {
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            const float4 r4 = ldg4(rp + 4 * q);
            v[4 * q] = relu_nan(v[4 * q] + r4.x); v[4 * q + 1] = relu_nan(v[4 * q + 1] + r4.y);
            v[4 * q + 2] = relu_nan(v[4 * q + 2] + r4.z); v[4 * q + 3] = relu_nan(v[4 * q + 3] + r4.w);
          }
        } else {
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = relu_nan(v[j] + __ldg(rp + j));
        }
      }
    } else {                                           // ragged tail: concat columns / zeros / residual per column
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int cj = col + j - p.n_total;
        if (cj >= 0) v[j] = (p.concat_src && cj < p.concat_n) ? __ldg(p.concat_src + pix * p.concat_n + cj) : 0.0f;
        else if (p.residual) v[j] = relu_nan(v[j] + __ldg(p.residual + pix * (size_t)p.res_stride + p.res_c0 + col + j));
      }
    }
    if (p.out_f32) {
      const int nvalid = min(ncol, p.n_total - col);
      float* dst = p.out_f32 + pix * (size_t)p.f32_stride + p.f32_c0 + col;
      if (nvalid == 32 && ((p.f32_stride | p.f32_c0) & 7) == 0) {
#pragma unroll
        for (int q = 0; q < 4; ++q)
          st8f(dst + 8 * q, v[8 * q], v[8 * q + 1], v[8 * q + 2], v[8 * q + 3], v[8 * q + 4], v[8 * q + 5], v[8 * q + 6], v[8 * q + 7]);
      } else if (nvalid == 32 && ((p.f32_stride | p.f32_c0) & 3) == 0) {
#pragma unroll
        for (int q = 0; q < 8; ++q) st4(dst + 4 * q, make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]));
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (j < nvalid) dst[j] = v[j];
      }
    }
    if (p.out_hi && ncol == 32) {
      const size_t o = pix * (size_t)p.h_stride + p.h_c0 + col;
      dhi = p.out_hi + o;
      dlo = p.out_lo + o;
    }
    if (p.adv_coords && col == 0) {                    // model.py:102: coords1 += delta; flow = coords1 - coords0 (pixel grid)
      float2 c1 = __ldcg(reinterpret_cast<const float2*>(p.adv_coords) + pix);
      c1.x = __fadd_rn(c1.x, v[0]);
      c1.y = __fadd_rn(c1.y, v[1]);
      reinterpret_cast<float2*>(p.adv_coords)[pix] = c1;
      const float gx = (float)(pix % p.W), gy = (float)((pix / p.W) % p.H);
      reinterpret_cast<float2*>(p.adv_flow)[pix] = make_float2(__fsub_rn(c1.x, gx), __fsub_rn(c1.y, gy));
    }
  } else if (MODE == EPI_GRU_ZR) {
    if (col < p.hid) {                                 // z gate -> fp32 plane
      float* dst = p.z + pix * (size_t)p.hid + col;
      if ((p.hid & 7) == 0) {
#pragma unroll
        for (int q = 0; q < 4; ++q)
          st8f(dst + 8 * q, fast_sigmoid(v[8 * q]), fast_sigmoid(v[8 * q + 1]), fast_sigmoid(v[8 * q + 2]), fast_sigmoid(v[8 * q + 3]),
               fast_sigmoid(v[8 * q + 4]), fast_sigmoid(v[8 * q + 5]), fast_sigmoid(v[8 * q + 6]), fast_sigmoid(v[8 * q + 7]));
      } else {
#pragma unroll
        for (int q = 0; q < 8; ++q)
          st4(dst + 4 * q, make_float4(fast_sigmoid(v[4 * q]), fast_sigmoid(v[4 * q + 1]), fast_sigmoid(v[4 * q + 2]),
                                       fast_sigmoid(v[4 * q + 3])));
      }
    } else {                                           // r gate -> r*h, re-split for the q convolution
      const int hc = col - p.hid;
      const float* hp = p.h + pix * (size_t)p.hid + hc;
      if ((p.hid & 7) == 0) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          float h8[8];
          ldcg8(hp + 8 * q, h8);
#pragma unroll
          for (int e = 0; e < 8; ++e) v[8 * q + e] = fast_sigmoid(v[8 * q + e]) * h8[e];
        }
      } else {
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const float4 hv = ldcg4(hp + 4 * q);
          v[4 * q] = fast_sigmoid(v[4 * q]) * hv.x; v[4 * q + 1] = fast_sigmoid(v[4 * q + 1]) * hv.y;
          v[4 * q + 2] = fast_sigmoid(v[4 * q + 2]) * hv.z; v[4 * q + 3] = fast_sigmoid(v[4 * q + 3]) * hv.w;
        }
      }
      const size_t o = pix * (size_t)p.h_stride + p.h_c0 + hc;
      dhi = p.out_hi + o;
      dlo = p.out_lo + o;
    }
  } else if (MODE == EPI_GRU_Q) {                      // h = (1-z)*h + z*tanh(v), in place
    float* hrow = p.h + pix * (size_t)p.hid + col;
    const float* zp = p.z + pix * (size_t)p.hid + col;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float4 zv = ldcg4(zp + 4 * q), hv = ldcg4(hrow + 4 * q);
      v[4 * q] = (1.0f - zv.x) * hv.x + zv.x * fast_tanh(v[4 * q]);
      v[4 * q + 1] = (1.0f - zv.y) * hv.y + zv.y * fast_tanh(v[4 * q + 1]);
      v[4 * q + 2] = (1.0f - zv.z) * hv.z + zv.z * fast_tanh(v[4 * q + 2]);
      v[4 * q + 3] = (1.0f - zv.w) * hv.w + zv.w * fast_tanh(v[4 * q + 3]);
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) st4(hrow + 4 * q, make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]));
    const size_t o = pix * (size_t)p.h_stride + p.h_c0 + col;
    dhi = p.out_hi + o;
    dlo = p.out_lo + o;
  }

  if (dhi) {                                           // fp16 hi/lo re-split, 16 channels (32 bytes) per store
    // (operand planes: channel strides are multiples of 64 and slices start at multiples of 32 channels -> 32-byte aligned;
    //  a slice that starts elsewhere takes the 16-byte form)
    const bool wide = ((reinterpret_cast<uintptr_t>(dhi) | reinterpret_cast<uintptr_t>(dlo)) & 31) == 0;
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      uint32_t ph[8], pl[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) split_f16x2(v[16 * q + 2 * e], v[16 * q + 2 * e + 1], ph[e], pl[e]);
      if (wide) {
        st8u(dhi + 16 * q, ph);
        st8u(dlo + 16 * q, pl);
      } else {
        reinterpret_cast<uint4*>(dhi)[2 * q] = make_uint4(ph[0], ph[1], ph[2], ph[3]);
        reinterpret_cast<uint4*>(dhi)[2 * q + 1] = make_uint4(ph[4], ph[5], ph[6], ph[7]);
        reinterpret_cast<uint4*>(dlo)[2 * q] = make_uint4(pl[0], pl[1], pl[2], pl[3]);
        reinterpret_cast<uint4*>(dlo)[2 * q + 1] = make_uint4(pl[4], pl[5], pl[6], pl[7]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// The shared-memory ring of all three tensor-core kernels (conv_tc_kernel, update_mega_kernel, corr_tc_kernel).  A slot
// holds one 64-channel chunk of both operands, [A_hi | A_lo | B_hi | B_lo]; full[s] completes on the slot's TMA bytes,
// empty[s] on one arrival per consumer warp.
// The geometry arguments (slot_bytes, nst, tx, group_chunks) are taken by reference: update_mega_kernel passes fields of
// its parameter block at a run-time layer index, and a reference lets them be re-read after each barrier wait instead of
// held in registers across the loop (its producer warpgroup runs in 40 registers; held, they add spills).
// ------------------------------------------------------------------------------------------------
struct RingPos {            // next ring slot and the parity of every slot's use count (producer and consumers each keep one)
  int slot;
  uint32_t par;
};

__device__ __forceinline__ int ring_next(RingPos& r, int nst) {
  const int s = r.slot;
  r.slot = s + 1 == nst ? 0 : s + 1;
  return s;
}

// Thread 0, before the CTA-wide barrier that precedes the first use; the caller then issues fence_mbar_init().
__device__ __forceinline__ void ring_init(uint64_t* full_bar, uint64_t* empty_bar, int nst) {
  for (int s = 0; s < nst; ++s) {
    mbar_init(&full_bar[s], 1);
    mbar_init(&empty_bar[s], kConsumerWarps);
  }
}

struct RingSlot {
  uint8_t* data;
  uint64_t* full;           // the barrier the slot's TMA loads complete on
};

// Producer: waits for the next slot to be free and arms its full barrier for `tx` bytes of TMA loads.
__device__ __forceinline__ RingSlot ring_acquire(uint8_t* stages, const int& slot_bytes, const int& nst, uint64_t* full_bar,
                                                 uint64_t* empty_bar, RingPos& rp, const int& tx) {
  const int s = ring_next(rp, nst);
  mbar_wait(&empty_bar[s], ((rp.par >> s) & 1u) ^ 1u);
  rp.par ^= 1u << s;
  mbar_arrive_expect_tx(&full_bar[s], (uint32_t)tx);
  return RingSlot{stages + (size_t)s * slot_bytes, &full_bar[s]};
}

// Consumer, all 128 threads of warpgroup `wg` (rows [64 wg, 64 wg + 64) of the A tile): the MMAs of `total` consecutive
// slots, promoted -- added in IEEE fp32 into racc -- every `group_chunks` chunks, each group accumulating into a fresh
// register tile.  N is the instantiated MMA width; b_lo_off is the byte offset of B_lo behind B_hi.
template <int N>
__device__ __forceinline__ void ring_mma(float (&racc)[N / 2], uint8_t* stages, const int& slot_bytes, const int& nst,
                                         uint64_t* full_bar, uint64_t* empty_bar, RingPos& rp, int wg, uint32_t b_lo_off,
                                         int total, const int& group_chunks) {
  const int lane = threadIdx.x & 31;
  float acc[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] = racc[i] = 0.0f;
  for (int done = 0; done < total;) {
    const int gend = min(total, done + group_chunks);
    for (int first = 1; done < gend; ++done, first = 0) {
      const int s = ring_next(rp, nst);
      mbar_wait(&full_bar[s], (rp.par >> s) & 1u);
      rp.par ^= 1u << s;
      const uint32_t sa = smem_u32(stages + (size_t)s * slot_bytes);
      const uint32_t arow = (uint32_t)wg * 64 * 128;
      wgmma_fence_regs(acc);
      wgmma_fence();
      wgmma_chunk3<N>(acc, make_desc_sw128(sa + arow), make_desc_sw128(sa + kABytes + arow), make_desc_sw128(sa + 2 * kABytes),
                      make_desc_sw128(sa + 2 * kABytes + b_lo_off), first != 0);
      wgmma_commit();
      wgmma_wait_all();
      wgmma_fence_regs(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[s]);       // this warp's reads of the slot are complete
    }
#pragma unroll
    for (int i = 0; i < N / 2; ++i) racc[i] += acc[i];   // IEEE fp32 promotion
  }
}

// ------------------------------------------------------------------------------------------------
// Shared by conv_tc_kernel and update_mega_kernel: the ring walk of one convolution tile, producer and consumer side.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int tc_total_chunks(const TcConvParams& c) {
  return c.kh * c.kw * (c.seg_chunks[0] + (c.nseg > 1 ? c.seg_chunks[1] : 0));
}

// Producer: streams the (tap, chunk) stages of one tile.  claim != null: *claim = atomicAdd(next_item) just before the last
// stage (late enough that the CTA is about to be free, early enough that the atomic hides behind the slot wait).
__device__ __forceinline__ void tc_produce_tile(const TcConvParams& c, uint8_t* stages, uint64_t* full_bar, uint64_t* empty_bar,
                                                RingPos& rp, int nt, int b, int ty, int tx, unsigned int* next_item = nullptr,
                                                int* claim = nullptr) {
  const int ntaps = c.kh * c.kw;
  const int x0 = tx * c.TW * c.stride, y0 = ty * c.TH * c.stride, n0 = nt * c.bn;
  int left = tc_total_chunks(c);
  for (int tap = 0; tap < ntaps; ++tap) {
    const int dy = tap / c.kw - c.ph, dx = tap % c.kw - c.pw;
    int kc = 0;
    for (int seg = 0; seg < c.nseg; ++seg) {
      for (int ch = 0; ch < c.seg_chunks[seg]; ++ch, ++kc) {
        if (--left == 0 && claim) *claim = (int)atomicAdd(next_item, 1u);
        const RingSlot st = ring_acquire(stages, c.stage_bytes, c.nstages, full_bar, empty_bar, rp, c.stage_bytes);
        // two boxes per stage: [A_hi | A_lo] and [B_hi | B_lo]
        tma_load_5d(st.data, &c.a_map[seg], st.full, c.seg_c0[seg] + ch * kChunkK, x0 + dx, y0 + dy, b, 0);
        tma_load_4d(st.data + 2 * kABytes, &c.b_map, st.full, kc * kChunkK, n0, tap, 0);
      }
    }
  }
}

// Staging tile of one warpgroup: 64 rows x 64 fp32, 16-byte groups XOR-swizzled by row (conflict-free row reads).
__device__ __forceinline__ int stg_idx(int r, int c) { return r * kStageCols + ((((c >> 2) ^ (r & 7))) << 2) + (c & 3); }

// Consumer side of one tile, all 128 threads of warpgroup `wg` (tid = thread index inside it): the ring's MMAs with
// IEEE-fp32 promotion every group_chunks chunks, then the epilogue of the warpgroup's 64 rows.  N >= c.bn is the
// instantiated MMA width (columns past bn read other shared memory and are discarded).
template <int N>
__device__ __forceinline__ void tc_consume_tile(const TcConvParams& c, uint8_t* stages, float* staging, uint64_t* full_bar,
                                                uint64_t* empty_bar, RingPos& rp, int wg, int tid, int nt, int b, int ty,
                                                int tx) {
  const int lane = tid & 31, w = tid >> 5;
  float racc[N / 2];
  ring_mma<N>(racc, stages, c.stage_bytes, c.nstages, full_bar, empty_bar, rp, wg, (uint32_t)(c.bn * kChunkK * 2),
              tc_total_chunks(c), c.group_chunks);

  // ---- epilogue: 64-column blocks through the staging tile; thread (row, half) then owns 32 columns of one pixel row ----
  float* stg = staging + wg * 64 * kStageCols;
  const int row = tid & 63, half = tid >> 6;
  const int m = wg * 64 + row;
  const int x = tx * c.TW + m % c.TW, y = ty * c.TH + m / c.TW;
  const bool inside = x < c.W && y < c.H;
  const size_t pix = ((size_t)b * c.H + y) * c.W + x;
  const float inv_scale = c.inv_scale ? __ldg(c.inv_scale) : 1.0f;
#pragma unroll
  for (int cb = 0; cb < (N + kStageCols - 1) / kStageCols; ++cb) {
    if (cb * kStageCols >= c.bn) break;
    wg_sync(wg);                                       // the previous block's readers are done with the tile
#pragma unroll
    for (int i = cb * 8; i < min(cb * 8 + 8, N / 8); ++i) {
      const int col = 8 * (i - cb * 8) + 2 * (lane & 3), r0 = 16 * w + (lane >> 2);
      *reinterpret_cast<float2*>(stg + stg_idx(r0, col)) = make_float2(racc[4 * i], racc[4 * i + 1]);
      *reinterpret_cast<float2*>(stg + stg_idx(r0 + 8, col)) = make_float2(racc[4 * i + 2], racc[4 * i + 3]);
    }
    wg_sync(wg);
    const int c0 = cb * kStageCols + half * 32;
    if (inside && c0 < c.bn) {
      const int ncol = min(32, c.bn - c0);
      float v[32];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float4 t4 = *reinterpret_cast<const float4*>(stg + stg_idx(row, half * 32 + 4 * q));
        v[4 * q] = t4.x; v[4 * q + 1] = t4.y; v[4 * q + 2] = t4.z; v[4 * q + 3] = t4.w;
      }
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (j >= ncol) v[j] = 0.0f;
      if (c.mode == EPI_LINEAR) tc_epilogue_regs<EPI_LINEAR>(c, v, pix, nt * c.bn + c0, ncol, inv_scale);
      else if (c.mode == EPI_GRU_ZR) tc_epilogue_regs<EPI_GRU_ZR>(c, v, pix, nt * c.bn + c0, ncol, inv_scale);
      else tc_epilogue_regs<EPI_GRU_Q>(c, v, pix, nt * c.bn + c0, ncol, inv_scale);
    }
  }
}

// Instantiated MMA widths: bn (a multiple of 16, <= 128) rounds up to the next of these.
template <class F>
__device__ __forceinline__ void with_mma_n(int bn, F&& f) {
  if (bn <= 16) f(std::integral_constant<int, 16>{});
  else if (bn <= 32) f(std::integral_constant<int, 32>{});
  else if (bn <= 64) f(std::integral_constant<int, 64>{});
  else if (bn <= 96) f(std::integral_constant<int, 96>{});
  else f(std::integral_constant<int, 128>{});
}

// Register split between the producer warpgroup and the two consumer warpgroups: 128 * 40 + 256 * 232 <= 64 K.
__device__ __forceinline__ void regs_producer() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory"); }
__device__ __forceinline__ void regs_consumer() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory"); }

__device__ __forceinline__ void tc_decode_tile(const TcConvParams& c, int t, int& nt, int& b, int& ty, int& tx) {
  const int mtiles = c.B * c.tiles_y * c.tiles_x;
  nt = t / mtiles;
  int mt = t - nt * mtiles;
  tx = mt % c.tiles_x;
  mt /= c.tiles_x;
  ty = mt % c.tiles_y;
  b = mt / c.tiles_y;
}
#endif

__global__ void __launch_bounds__(kTcThreads, 1) conv_tc_kernel(const __grid_constant__ TcConvParams p) {
#if defined(__CUDA_ARCH__)
  // Persistent: CTA c processes output tiles c, c + gridDim.x, ...  A tile is (pixel tile, column tile).  Producer and
  // consumers walk the same tile sequence; the ring carries straight across tile boundaries.
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int nst = p.nstages;
  uint8_t* stages = smem;
  float* staging = reinterpret_cast<float*>(stages + (size_t)nst * p.stage_bytes);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(staging) + kStagingBytes);
  uint64_t* empty_bar = full_bar + nst;

  const int warp = threadIdx.x >> 5;
  const int mtiles = p.B * p.tiles_y * p.tiles_x;
  const int ntiles = mtiles * p.n_tiles_n;

  if (threadIdx.x == 0) {
    ring_init(full_bar, empty_bar, nst);
    fence_mbar_init();
  }
  if (warp == kConsumerWarps && (threadIdx.x & 31) == 0) {
    prefetch_tmap(&p.a_map[0]);
    prefetch_tmap(&p.b_map);
    if (p.nseg > 1) prefetch_tmap(&p.a_map[1]);
  }
  __syncthreads();
  // Launched with programmatic dependent launch (tc_launch): the barriers and tensor-map prefetch above touch no global
  // data and overlap the previous kernel's tail; from here on its results are read (and its inputs overwritten), so wait
  // for it, then let the next grid in the stream start its own prologue.
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  RingPos rp{0, 0u};
  if (warp >= kConsumerWarps) {
    // ===================== TMA producer =====================
    regs_producer();
    if (warp == kConsumerWarps && elect_one()) {
      for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        int nt, b, ty, tx;
        tc_decode_tile(p, t, nt, b, ty, tx);
        tc_produce_tile(p, stages, full_bar, empty_bar, rp, nt, b, ty, tx);
      }
    }
  } else {
    // ===================== MMA + epilogue (warpgroups 0, 1) =====================
    regs_consumer();
    const int wg = warp >> 2, tid = threadIdx.x & 127;
    with_mma_n(p.bn, [&](auto n) {
      for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        int nt, b, ty, tx;
        tc_decode_tile(p, t, nt, b, ty, tx);
        tc_consume_tile<decltype(n)::value>(p, stages, staging, full_bar, empty_bar, rp, wg, tid, nt, b, ty, tx);
      }
    });
  }
#endif
}

// ------------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------------
inline void tc_pick_tile(int W, int H, int* tw, int* th) {
  // TW*TH = 128 with TW a power of two; minimise padded area, prefer wide tiles on ties.
  long best = -1;
  for (int t = 128; t >= 8; t >>= 1) {
    const int hh = 128 / t;
    const long area = (long)round_up(W, t) * round_up(H, hh);
    if (best < 0 || area < best) {
      best = area;
      *tw = t;
      *th = hh;
    }
  }
}

// Column tiling of a layer whose N per CTA exceeds kMaxTileN: the CTA's N is divided by the returned factor and the
// number of column tiles multiplied by it (0: no such split keeps N a multiple of 16).
inline int tc_n_split(int bn) {
  const int f = ceil_div(bn, kMaxTileN);
  return bn % (16 * f) == 0 ? f : 0;
}

// Fills the derived launch fields (tile grid, stages) of `p`; returns bytes of dynamic shared memory.  Caller has set
// bn, B, H, W, TH, TW.
inline int tc_finalize(TcConvParams& p) {
  p.tiles_x = ceil_div(p.W, p.TW);
  p.tiles_y = ceil_div(p.H, p.TH);
  p.stage_bytes = 2 * kABytes + 2 * p.bn * kChunkK * 2;
  int nst = (kSmemMax - kSmemFixed) / p.stage_bytes;
  if (nst > 8) nst = 8;
  p.nstages = nst;
  return nst * p.stage_bytes + kSmemFixed;
}

// group_chunks has no default: every caller states its promotion group (a precision decision, DESIGN.md section 4).
inline int tc_check(const TcConvParams& p) {
  if (p.bn % 16 != 0 || p.bn < 16 || p.bn > kMaxTileN || p.TW * p.TH != kTileM) return RAFT_ERR_BAD_SHAPE;
  if (p.mode != EPI_LINEAR && p.mode != EPI_GRU_ZR && p.mode != EPI_GRU_Q) return RAFT_ERR_UNSUPPORTED;
  if (p.group_chunks < 1) return RAFT_ERR_BAD_ARG;
  return RAFT_OK;
}

// Grid of a persistent tensor-core kernel: one CTA per SM, never more CTAs than work items.  The first call for a kernel
// on a device raises the kernel's dynamic shared-memory limit to `smem` and caches the device's SM count (one entry per
// kernel and device ordinal; benign race: the calls are idempotent).
template <auto Kernel>
inline int persistent_grid(int smem, long items, unsigned* grid) {
  static int num_sms[64] = {0};
  int dev = 0;
  RAFT_CUDA_TRY(cudaGetDevice(&dev));
  int& sms = num_sms[dev & 63];
  if (!sms) {
    RAFT_CUDA_TRY(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    RAFT_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  }
  *grid = (unsigned)(items < sms ? items : sms);
  return RAFT_OK;
}

inline int tc_launch(TcConvParams& p, int n_tiles_n, cudaStream_t stream) {
  RAFT_TRY(tc_check(p));
  if (p.stride < 1) p.stride = 1;
  const int smem = tc_finalize(p);
  if (p.nstages < 2) return RAFT_ERR_UNSUPPORTED;
  p.n_tiles_n = n_tiles_n;
  unsigned grid = 0;
  RAFT_TRY(persistent_grid<conv_tc_kernel>(kSmemMax, (long)p.B * p.tiles_y * p.tiles_x * n_tiles_n, &grid));
  cudaLaunchConfig_t cfg;                              // programmatic-serialization attribute: see the kernel prologue
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3((unsigned)kTcThreads);
  cfg.dynamicSmemBytes = (size_t)smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  ++g_launches;
  RAFT_CUDA_TRY(cudaLaunchKernelEx(&cfg, conv_tc_kernel, p));
  return raft_launch_status();
}

// ------------------------------------------------------------------------------------------------
// Packed weights of one tensor-core convolution, the format conv_tc_kernel and update_mega_kernel read.  A slot in a
// prepared-weights blob (update blocks and encoders alike) holds, each part 256-byte aligned and in this order:
//   hi, lo   [tap][cout_pad][cin_pad] fp16 planes of w * 2^k (2^k puts max|w| in [2^12, 2^13), see weight_scale_kernel)
//   bias     cout_pad + 64 floats (the epilogue reads whole 32-column chunks past the last column)
//   scale    (2^k, 2^-k)
//   absmax   the bits of max|w|, reduced while packing
// ------------------------------------------------------------------------------------------------
struct TcWeightSlot {
  size_t hi, lo, bias, scale, absmax;    // byte offsets inside the blob
  int kh, kw, cin_pad, cout_pad;
};

// Reserves a slot at byte offset `off` of a blob and advances `off` past it.
inline TcWeightSlot tc_weight_slot(size_t& off, int kh, int kw, int cin_pad, int cout_pad) {
  auto take = [&](size_t bytes) { const size_t o = off; off = align_up(off + bytes, 256); return o; };
  TcWeightSlot s;
  s.kh = kh; s.kw = kw; s.cin_pad = cin_pad; s.cout_pad = cout_pad;
  const size_t plane = (size_t)kh * kw * cout_pad * cin_pad * sizeof(__half);
  s.hi = take(plane);
  s.lo = take(plane);
  s.bias = take(sizeof(float) * (cout_pad + 64));
  s.scale = take(2 * sizeof(float));
  s.absmax = take(sizeof(unsigned int));
  return s;
}

// Where the input channels of a packed convolution land: source channels [src0[r], src0[r] + n[r]) go to packed
// channels [dst0[r], dst0[r] + n[r]), r < nrange.
struct TcCinMap { int nrange, src0[2], n[2], dst0[2]; };

// Writes slot `s` of the zeroed blob at `base` from nsrc (1 or 2) HWIO convolutions, concatenated along cout.
// cin_map == null keeps the channels where they are.  flatten: each source runs as a 1x1 convolution over its
// kh * kw * cin window channels (HWIO is already [tap * cin + c][cout]), for layers fed by im2col planes.  The scale is
// shared by the sources: it comes from the absmax over all of them.
inline int tc_pack_weights(uint8_t* base, const TcWeightSlot& s, const raft_conv* const src[], int nsrc,
                           const TcCinMap* cin_map, bool flatten, cudaStream_t st) {
  unsigned int* amax = reinterpret_cast<unsigned int*>(base + s.absmax);
  float* scale = reinterpret_cast<float*>(base + s.scale);
  for (int i = 0; i < nsrc; ++i) {
    const size_t nw = (size_t)src[i]->kh * src[i]->kw * src[i]->cin * src[i]->cout;
    RAFT_TRY(launch(absmax_kernel, grid_for(nw), 256, 0, st, src[i]->kernel, nw, amax));
  }
  RAFT_TRY(launch(weight_scale_kernel, 1, 1, 0, st, amax, scale));
  int cout_off = 0;
  for (int i = 0; i < nsrc; ++i) {
    const raft_conv& cv = *src[i];
    PackParams pp;
    memset(&pp, 0, sizeof(pp));
    pp.w = cv.kernel;
    pp.kh = cv.kh; pp.kw = cv.kw; pp.cin = cv.cin; pp.cout = cv.cout;
    if (flatten) { pp.cin = pp.kh * pp.kw * pp.cin; pp.kh = pp.kw = 1; }
    pp.hi = reinterpret_cast<__half*>(base + s.hi);
    pp.lo = reinterpret_cast<__half*>(base + s.lo);
    pp.cout_pad = s.cout_pad; pp.cin_pad = s.cin_pad; pp.cout_off = cout_off;
    const TcCinMap m = cin_map ? *cin_map : TcCinMap{1, {0, 0}, {pp.cin, 0}, {0, 0}};
    pp.nrange = m.nrange;
    for (int r = 0; r < m.nrange; ++r) {
      pp.r_src0[r] = m.src0[r];
      pp.r_n[r] = m.n[r];
      pp.r_dst0[r] = m.dst0[r];
    }
    pp.scale = scale;
    RAFT_TRY(launch(pack_weights_kernel, grid_for((size_t)cv.kh * cv.kw * cv.cin * cv.cout), 256, 0, st, pp));
    RAFT_CUDA_TRY(cudaMemcpyAsync(base + s.bias + cout_off * sizeof(float), cv.bias, cv.cout * sizeof(float),
                                  cudaMemcpyDeviceToDevice, st));
    cout_off += cv.cout;
  }
  return RAFT_OK;
}

// Points `p` at the packed weights of slot `s` of the blob at `base`, read in column tiles of bn: weight tensor map,
// taps, bias and 2^-k.
inline int tc_use_weights(TcConvParams& p, const uint8_t* base, const TcWeightSlot& s, int bn) {
  RAFT_TRY(make_tmap_wgt2(&p.b_map, reinterpret_cast<const __half*>(base + s.hi),
                          reinterpret_cast<const __half*>(base + s.lo), s.kh * s.kw, s.cout_pad, s.cin_pad, bn));
  p.kh = s.kh; p.kw = s.kw;
  p.bn = bn;
  p.bias = reinterpret_cast<const float*>(base + s.bias);
  p.inv_scale = reinterpret_cast<const float*>(base + s.scale) + 1;
  return RAFT_OK;
}

}  // namespace raft
