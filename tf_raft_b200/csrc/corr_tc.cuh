// All-pairs correlation pyramid (tf_raft/layers/corr.py:100-114, 154-162) on the tensor cores: ONE persistent
// warp-specialised wgmma kernel writes every level of the pyramid,
//
//   pyr[l][b, q, n] = < fmap1[b, q, :], avgpool^l(fmap2)[b, n, :] > / sqrt(C)          (pooling is linear: the 256-channel
//                                                                                       features are pooled, not the volume)
// plus one preparation kernel that pools fmap2 and splits both feature maps into the fp16 (hi, lo) operand planes.
//
// Tile = 128 queries x bn <= 128 targets, K = C in 64-channel chunks of a 3-stage ring (64 KB stages), three fp16 passes
// per chunk (hi*hi, hi*lo, lo*hi; fp32-grade, DESIGN.md section 4).  The ring and its MMA loop are the convolutions'
// (ring_acquire / ring_mma, conv_tc.cuh) with a promotion group of one chunk: every chunk accumulates into a fresh register
// tile (a 12-MMA chain) and the chunk results are added in IEEE fp32 ((0 + c0) + c1 + ...).  The pyramid feeds the sampler,
// which is discontinuous at integer coordinates (DESIGN.md section 4), so the correlation takes the shortest chains:
// with 24-MMA chains a query of the benchmark pair (448x512, seed 0/1) crosses a discontinuity at iteration 5 on the H100,
// with 12 it stays within 3e-4 of the oracle.
// Warps 0..7 = two consumer warpgroups (queries [0, 64) and [64, 128) of the tile): MMAs, then the scaled store straight
// from the accumulator registers -- each lane writes 8-byte column pairs, a warp covers 8 rows x 32 contiguous bytes per
// store, whole 32-byte sectors.  Warp 8 = TMA producer.  The tile list runs over all levels (level 0 first), consecutive
// CTAs take consecutive query tiles of the same target tile, so the target features are shared through L2.
#pragma once
#include "conv_tc.cuh"
#include "kernels.cuh"

namespace raft {

constexpr int kCorrBn = 128;                                              // target columns per tile
constexpr int kCorrStageBytes = 2 * kABytes + 2 * kCorrBn * kChunkK * 2;  // 64 KB: A (hi|lo) 32 KB + B (hi|lo) up to 32 KB
constexpr int kCorrStages = 3;
constexpr int kCorrSmemBytes = 1024 /*align slack*/ + kCorrStages * kCorrStageBytes + 2048 /*MMA over-read, barriers*/;
static_assert(kCorrSmemBytes <= kSmemMax, "correlation kernel shared memory");

struct alignas(64) CorrTcParams {
  CUtensorMap a_map;                        // fmap1 (hi, lo): (C, N, 1, B, plane), box {64, 128, 1, 1, 2}
  CUtensorMap b_map[RAFT_MAX_LEVELS];       // level-l target features (hi, lo): (C, N2_l, B, plane), box {64, bn_l, 1, 2}
  float* out[RAFT_MAX_LEVELS];              // pyr[l]: (B * N, N2_l) fp32
  int n2[RAFT_MAX_LEVELS], bn[RAFT_MAX_LEVELS];
  int tile0[RAFT_MAX_LEVELS + 1];           // first tile index of each level; tile0[levels] = total
  int levels, B, N, chunks;                 // chunks = C / 64
  int mtiles_img;                           // query tiles per image = ceil(N / 128)
  float corr_mul, corr_div;                 // 1/sqrt(C) when that is an exact power of two, else 0 and the divisor is used
};

#if defined(__CUDA_ARCH__)
// tile t -> (level, target tile, query tile): levels in order, query tile fastest
__device__ __forceinline__ void corr_decode(const CorrTcParams& p, int t, int& l, int& nt, int& mt) {
  l = 0;
  while (l + 1 < p.levels && t >= p.tile0[l + 1]) ++l;
  const int r = t - p.tile0[l];
  const int mtiles = p.B * p.mtiles_img;
  nt = r / mtiles;
  mt = r - nt * mtiles;
}

template <int N>
__device__ __forceinline__ void corr_consume_tile(const CorrTcParams& p, uint8_t* stages, uint64_t* full_bar, uint64_t* empty_bar,
                                                  RingPos& rp, int wg, int tid, int l, int nt, int mt) {
  const int lane = tid & 31, w = tid >> 5;
  const int bn = p.bn[l], n2 = p.n2[l];
  float racc[N / 2];                                   // promotion group 1: IEEE fp32 sum of the 12-MMA chunk chains
  ring_mma<N>(racc, stages, int{kCorrStageBytes}, int{kCorrStages}, full_bar, empty_bar, rp, wg, (uint32_t)(bn * kChunkK * 2),
              p.chunks, 1);
  // ---- store ----
  const int b = mt / p.mtiles_img, m0 = (mt - b * p.mtiles_img) * kTileM, n0 = nt * bn;
  const int col_end = min(n2, n0 + bn);
  const bool vec = (n2 & 1) == 0;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = m0 + wg * 64 + 16 * w + (lane >> 2) + 8 * h;
    if (row >= p.N) continue;
    float* dst = p.out[l] + ((size_t)b * p.N + row) * n2;
#pragma unroll
    for (int i = 0; i < N / 8; ++i) {
      const int col = n0 + 8 * i + 2 * (lane & 3);
      float v0 = racc[4 * i + 2 * h], v1 = racc[4 * i + 2 * h + 1];
      if (p.corr_mul != 0.0f) {
        v0 *= p.corr_mul; v1 *= p.corr_mul;
      } else {
        v0 = __fdiv_rn(v0, p.corr_div); v1 = __fdiv_rn(v1, p.corr_div);
      }
      if (vec && col + 1 < col_end) {
        *reinterpret_cast<float2*>(dst + col) = make_float2(v0, v1);
      } else {
        if (col < col_end) dst[col] = v0;
        if (col + 1 < col_end) dst[col + 1] = v1;
      }
    }
  }
}
#endif

__global__ void __launch_bounds__(kTcThreads, 1) corr_tc_kernel(const __grid_constant__ CorrTcParams p) {
#if defined(__CUDA_ARCH__)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* stages = smem;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kCorrStages * kCorrStageBytes + 1024);   // (past the MMA over-read)
  uint64_t* empty_bar = full_bar + kCorrStages;

  const int warp = threadIdx.x >> 5;
  const int ntiles = p.tile0[p.levels];

  if (threadIdx.x == 0) {
    ring_init(full_bar, empty_bar, kCorrStages);
    fence_mbar_init();
    prefetch_tmap(&p.a_map);
    for (int l = 0; l < p.levels; ++l) prefetch_tmap(&p.b_map[l]);
  }
  __syncthreads();

  RingPos rp{0, 0u};
  if (warp >= kConsumerWarps) {
    // ===================== TMA producer =====================
    regs_producer();
    if (warp == kConsumerWarps && elect_one()) {
      for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        int l, nt, mt;
        corr_decode(p, t, l, nt, mt);
        const int b = mt / p.mtiles_img, m0 = (mt - b * p.mtiles_img) * kTileM, n0 = nt * p.bn[l];
        const int bytes = 2 * kABytes + p.bn[l] * kChunkK * 4;     // slots are a fixed 64 KB; B fills bn rows of them
        for (int kc = 0; kc < p.chunks; ++kc) {
          const RingSlot st = ring_acquire(stages, int{kCorrStageBytes}, int{kCorrStages}, full_bar, empty_bar, rp, bytes);
          tma_load_5d(st.data, &p.a_map, st.full, kc * kChunkK, m0, 0, b, 0);
          tma_load_4d(st.data + 2 * kABytes, &p.b_map[l], st.full, kc * kChunkK, n0, b, 0);
        }
      }
    }
  } else {
    // ===================== MMA + store (warpgroups 0, 1) =====================
    regs_consumer();
    const int wg = warp >> 2, tid = threadIdx.x & 127;
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
      int l, nt, mt;
      corr_decode(p, t, l, nt, mt);
      with_mma_n(p.bn[l], [&](auto n) { corr_consume_tile<decltype(n)::value>(p, stages, full_bar, empty_bar, rp, wg, tid, l, nt, mt); });
    }
  }
#endif
}

// ------------------------------------------------------------------------------------------------
// Preparation: fmap1 -> (hi, lo) planes; fmap2 -> pooled levels 1..levels-1 (2x2 mean, VALID, successively, the same
// fp32 arithmetic as avgpool2x2_kernel) and the (hi, lo) planes of every level.  One launch:
//   blocks [0, npatch): one 8 x 8 patch of fmap2 pixels (a complete pooling tree down to level 3), thread = channel pair;
//   blocks [npatch, ...): elementwise split of fmap1, 4 channels per thread.
// levels <= 4 here (deeper pyramids take the generic kernels).
// ------------------------------------------------------------------------------------------------
struct CorrPrepParams {
  const float* f1; const float* f2;
  __half *f1_hi, *f1_lo;
  __half *f2_hi[4], *f2_lo[4];
  int B, h, w, C, levels;
  int patches_x, patches_y, npatch;
};

__device__ __forceinline__ void store_split2(__half* hi, __half* lo, size_t o, float x, float y) {
  uint32_t h2, l2;
  split_f16x2(x, y, h2, l2);
  *reinterpret_cast<uint32_t*>(hi + o) = h2;
  *reinterpret_cast<uint32_t*>(lo + o) = l2;
}
__device__ __forceinline__ float pool4(float a, float b, float c, float d) {
  return __fmul_rn(__fadd_rn(__fadd_rn(a, b), __fadd_rn(c, d)), 0.25f);
}

__global__ void __launch_bounds__(128) corr_prep_kernel(const CorrPrepParams p) {
  if ((int)blockIdx.x >= p.npatch) {                 // ---- fmap1: elementwise split ----
    const size_t n4 = (size_t)p.B * p.h * p.w * p.C / 4;
    const size_t nb = gridDim.x - p.npatch;
    for (size_t i = (size_t)(blockIdx.x - p.npatch) * blockDim.x + threadIdx.x; i < n4; i += nb * blockDim.x) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(p.f1) + i);
      uint32_t h01, l01, h23, l23;
      split_f16x2(v.x, v.y, h01, l01);
      split_f16x2(v.z, v.w, h23, l23);
      reinterpret_cast<uint2*>(p.f1_hi)[i] = make_uint2(h01, h23);
      reinterpret_cast<uint2*>(p.f1_lo)[i] = make_uint2(l01, l23);
    }
    return;
  }
  int t = blockIdx.x;
  const int px = t % p.patches_x; t /= p.patches_x;
  const int py = t % p.patches_y;
  const int b = t / p.patches_y;
  const int C = p.C;
  int hl[4], wl[4];
  hl[0] = p.h; wl[0] = p.w;
#pragma unroll
  for (int l = 1; l < 4; ++l) { hl[l] = hl[l - 1] / 2; wl[l] = wl[l - 1] / 2; }
  for (int c = 2 * threadIdx.x; c < C; c += 2 * blockDim.x) {
    float2 l1p[4], l2p[2];                            // level-1 row / level-2 row waiting for their partner
#pragma unroll 1
    for (int rp = 0; rp < 4; ++rp) {                  // row pairs of the patch (rolled: 16 loads in flight at a time)
      const int y0 = py * 8 + rp * 2;
      float2 v[2][8];
#pragma unroll
      for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int x = 0; x < 8; ++x) {
          const int yy = y0 + dy, xx = px * 8 + x;
          v[dy][x] = (yy < hl[0] && xx < wl[0])
                         ? __ldg(reinterpret_cast<const float2*>(p.f2 + (((size_t)b * hl[0] + yy) * wl[0] + xx) * C + c))
                         : make_float2(0.f, 0.f);
        }
#pragma unroll
      for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int x = 0; x < 8; ++x) {
          const int yy = y0 + dy, xx = px * 8 + x;
          if (yy < hl[0] && xx < wl[0])
            store_split2(p.f2_hi[0], p.f2_lo[0], (((size_t)b * hl[0] + yy) * wl[0] + xx) * C + c, v[dy][x].x, v[dy][x].y);
        }
      float2 l1[4];
#pragma unroll
      for (int x = 0; x < 4; ++x) {
        l1[x].x = pool4(v[0][2 * x].x, v[0][2 * x + 1].x, v[1][2 * x].x, v[1][2 * x + 1].x);
        l1[x].y = pool4(v[0][2 * x].y, v[0][2 * x + 1].y, v[1][2 * x].y, v[1][2 * x + 1].y);
        const int y1 = py * 4 + rp, x1 = px * 4 + x;
        if (p.levels > 1 && y1 < hl[1] && x1 < wl[1])
          store_split2(p.f2_hi[1], p.f2_lo[1], (((size_t)b * hl[1] + y1) * wl[1] + x1) * C + c, l1[x].x, l1[x].y);
      }
      if (rp & 1) {
        float2 l2[2];
#pragma unroll
        for (int x = 0; x < 2; ++x) {
          l2[x].x = pool4(l1p[2 * x].x, l1p[2 * x + 1].x, l1[2 * x].x, l1[2 * x + 1].x);
          l2[x].y = pool4(l1p[2 * x].y, l1p[2 * x + 1].y, l1[2 * x].y, l1[2 * x + 1].y);
          const int y2 = py * 2 + (rp >> 1), x2 = px * 2 + x;
          if (p.levels > 2 && y2 < hl[2] && x2 < wl[2])
            store_split2(p.f2_hi[2], p.f2_lo[2], (((size_t)b * hl[2] + y2) * wl[2] + x2) * C + c, l2[x].x, l2[x].y);
        }
        if (rp == 3) {
          if (p.levels > 3 && py < hl[3] && px < wl[3])
            store_split2(p.f2_hi[3], p.f2_lo[3], (((size_t)b * hl[3] + py) * wl[3] + px) * C + c,
                         pool4(l2p[0].x, l2p[1].x, l2[0].x, l2[1].x), pool4(l2p[0].y, l2p[1].y, l2[0].y, l2[1].y));
        } else {
          l2p[0] = l2[0]; l2p[1] = l2[1];
        }
      } else {
#pragma unroll
        for (int x = 0; x < 4; ++x) l1p[x] = l1[x];
      }
    }
  }
}

}  // namespace raft
