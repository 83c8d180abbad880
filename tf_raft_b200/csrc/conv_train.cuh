// Tensor-core convolutions of the training step (train_precision='f16x2'): forward, input gradient and weight gradient of a
// stride-1 convolution with odd, symmetric 'same' padding (a 1x1 'valid' convolution is the 1x1 case of it), NHWC fp32
// activations, HWIO fp32 kernels.
//
// * Forward: the kernel is packed into a slot of the workspace (tc_pack_weights, w * 2^k_w), x is split into hi/lo planes
//   that the caller keeps for the backward, and conv_tc_kernel runs it (EPI_LINEAR, bias, fp32 out).
// * Input gradient: a 'same' convolution of the gradient with the kernel rotated 180 degrees and cin / cout swapped, on
//   conv_tc_kernel.  The gradient is scaled by 2^k_g before it is split (operand_scale_kernel), the kernel by 2^k_w; the
//   epilogue multiplies by 2^-(k_w + k_g).  x is scaled the same way (2^k_x) in the forward.
// * Weight gradient: conv_wgrad_tc_kernel, below, over the x planes and the scaled gradient planes, split-K over pixel
//   slices into fp32 partial tiles, then wgrad_reduce_kernel adds the slices in order and multiplies by 2^-k_g.
#pragma once
#include <float.h>
#include <limits.h>

#include <algorithm>

#include "conv_tc.cuh"

namespace raft {

constexpr int kWgradGroupChunks = 2;      // pixel tiles (128 px) per promotion group: a chain of 2 * 24 = 48 MMAs
constexpr int kWgradStages = 2;
constexpr int kWgradSlotBytes = 6 * kABytes;  // [g chunk 0 hi | lo][g chunk 1 hi | lo][x hi | lo], 128 px x 64 ch each
constexpr int kWgradSmem = 1024 + kWgradStages * kWgradSlotBytes + 256;
constexpr int kWgradItemTarget = 256;     // work items the slice count aims at; a constant, not the device's SM count
constexpr int kConvTrainMaxC = 1024;      // channel counts the plan covers
constexpr int kConvTrainMaxK = 7;         // taps per side

inline int train_pad64(int c) { return round_up(c, 64); }
// Packed output columns of a conv_tc_kernel layer: a multiple of 16, split into column tiles of at most kMaxTileN.
inline int train_cout_pad(int cout) {
  const int f = ceil_div(cout, kMaxTileN);
  return round_up(cout, 16 * f);
}

// Work decomposition of the weight gradient.  Item i = ((slice * taps + tap) * co_blocks + cb) * ci_blocks + ib covers
// output rows (cout) [128 cb, 128 cb + 128) -- 64 per consumer warpgroup -- columns (cin) [64 ib, 64 ib + 64) of tap
// `tap`, over the pixel tiles [slice * tiles_per_slice, min(ptiles, (slice + 1) * tiles_per_slice)).  It writes the fp32
// partial tile partial[slice][tap][co][ci] once; nothing else writes it.
struct WgradPlan {
  int taps, co_chunks, co_blocks, ci_blocks;
  int tw, th, tiles_x, tiles_y, ptiles;
  int slices, tiles_per_slice, items;
  int cin_pad, cout_pad;      // 64-padded channel strides of the x and gradient planes
};

inline int wgrad_plan(int B, int H, int W, int cin, int kh, int kw, int cout, WgradPlan& pl) {
  pl.taps = kh * kw;
  pl.cin_pad = train_pad64(cin);
  pl.cout_pad = train_pad64(cout);
  pl.co_chunks = pl.cout_pad / 64;
  pl.co_blocks = ceil_div(pl.co_chunks, 2);
  pl.ci_blocks = pl.cin_pad / 64;
  tc_pick_tile(W, H, &pl.tw, &pl.th);
  pl.tiles_x = ceil_div(W, pl.tw);
  pl.tiles_y = ceil_div(H, pl.th);
  const long ptiles = (long)B * pl.tiles_x * pl.tiles_y;
  if (ptiles > INT_MAX / 2) return RAFT_ERR_BAD_SHAPE;
  pl.ptiles = (int)ptiles;
  const int base = pl.taps * pl.co_blocks * pl.ci_blocks;
  int slices = std::min(std::max(ceil_div(kWgradItemTarget, base), 1), pl.ptiles);
  pl.tiles_per_slice = ceil_div(pl.ptiles, slices);
  pl.slices = ceil_div(pl.ptiles, pl.tiles_per_slice);         // no empty slice
  pl.items = pl.slices * base;
  return RAFT_OK;
}

// Item -> (slice, tap, cout block, cin block): the kernel's decode, also called by the host-side plan checks.
__host__ __device__ __forceinline__ void wgrad_decode(const WgradPlan& pl, int item, int& slice, int& tap, int& cb,
                                                      int& ib) {
  ib = item % pl.ci_blocks;
  item /= pl.ci_blocks;
  cb = item % pl.co_blocks;
  item /= pl.co_blocks;
  tap = item % pl.taps;
  slice = item / pl.taps;
}

struct alignas(64) WgradParams {
  CUtensorMap g_map;          // gradient planes (hi, lo), channel stride cout_pad
  CUtensorMap x_map;          // input planes (hi, lo), channel stride cin_pad
  WgradPlan pl;
  int H, W, kw, ph, pw;
  float* partial;             // [slices][taps][cout_pad][cin_pad]
};

// Workspace of one training convolution, every part 256-byte aligned: forward slot, rotated slot, gradient planes,
// weight-gradient partials, scalars.
struct ConvTrainLayout {
  TcWeightSlot fwd, rot;
  size_t g_hi, g_lo, partial, gmax, gscale, dscale, fscale, total;
  WgradPlan pl;
};

inline int conv_train_layout(int B, int H, int W, int cin, int kh, int kw, int cout, ConvTrainLayout& L) {
  RAFT_TRY(wgrad_plan(B, H, W, cin, kh, kw, cout, L.pl));
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off = align_up(off + bytes, 256); return o; };
  L.fwd = tc_weight_slot(off, kh, kw, train_pad64(cin), train_cout_pad(cout));
  L.rot = tc_weight_slot(off, kh, kw, train_pad64(cout), train_cout_pad(cin));
  const size_t npix = (size_t)B * H * W;
  L.g_hi = take(npix * L.pl.cout_pad * sizeof(__half));
  L.g_lo = take(npix * L.pl.cout_pad * sizeof(__half));
  L.partial = take((size_t)L.pl.slices * L.pl.taps * L.pl.cout_pad * L.pl.cin_pad * sizeof(float));
  L.gmax = take(sizeof(unsigned int));
  L.gscale = take(2 * sizeof(float));
  L.dscale = take(sizeof(float));
  L.fscale = take(sizeof(float));
  L.total = off;
  return RAFT_OK;
}

// The x planes a forward writes and its backward reads: fp16 hi plane, lo plane (npix x round_up(cin, 64) each), then
// 256 bytes holding the absmax bits of x (offset 0) and its scale (2^k_x, 2^-k_x) (offset 16).  The scale travels with the
// planes, not in the workspace, because layers of one shape share a workspace between their forward and backward.
inline size_t conv_train_planes_bytes(size_t npix, int cin) { return 2 * npix * train_pad64(cin) * sizeof(__half) + 256; }
inline size_t conv_train_planes_tail(size_t npix, int cin) { return 2 * npix * train_pad64(cin) * sizeof(__half); }

// Shapes the training convolutions take.  Every box is at most 128 x 64 (tc_pick_tile), channel strides are multiples of
// 64 (so every plane base and stride the maps see is 16-byte aligned when the planes are), and the TMA coordinates --
// channel, x, y, image -- stay far inside int32 when B * H * W does.
inline int conv_train_check(int B, int H, int W, int cin, int kh, int kw, int cout) {
  if (B < 1 || H < 1 || W < 1 || (size_t)B * H * W > (size_t)INT_MAX) return RAFT_ERR_BAD_SHAPE;
  if (cin < 16 || cin > kConvTrainMaxC || cout < 1 || cout > kConvTrainMaxC) return RAFT_ERR_BAD_SHAPE;
  if (kh < 1 || kw < 1 || kh > kConvTrainMaxK || kw > kConvTrainMaxK || !(kh & 1) || !(kw & 1)) return RAFT_ERR_BAD_SHAPE;
  return RAFT_OK;
}

// fp32 NHWC (npix, nch) -> fp16 hi / lo planes (npix, nch_pad) of v * scale (scale: device scalar, null = 1); channels
// [nch, nch_pad) are zeros.  A non-finite entry becomes NaN in both planes (the inference split saturates +-inf to
// +-65504, which would hide an overflowed gradient), so it reaches every output whose sum includes it.
__global__ void train_split_kernel(const float* __restrict__ src, int nch, int nch_pad, __half* __restrict__ hi,
                                   __half* __restrict__ lo, size_t npix, const float* __restrict__ scale) {
  const float s = scale ? *scale : 1.0f;
  const size_t total = npix * (size_t)nch_pad;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t px = i / nch_pad;
    const int c = (int)(i - px * nch_pad);
    __half h = __float2half_rn(0.f), l = h;
    if (c < nch) {
      const float v = src[px * nch + c];
      if (isfinite(v)) split_f16(v * s, h, l);
      else h = l = __float2half_rn(__int_as_float(0x7fc00000));
    }
    hi[i] = h;
    lo[i] = l;
  }
}

// max |g| over the FINITE entries (NaN and +-inf are left out, so they cannot set the scale), as float bits.
__global__ void absmax_finite_kernel(const float* __restrict__ g, size_t n, unsigned int* __restrict__ out_bits) {
  float m = 0.f;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float a = fabsf(g[i]);
    if (a <= FLT_MAX) m = fmaxf(m, a);
  }
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(out_bits, __float_as_uint(m));
}

// Operand scale 2^k of an activation or gradient tensor: max finite |v| * 2^k in [2^12, 2^13), the weights' rule, with k
// clamped to [-100, 100] so that 2^-(k_w + k) (|k_w| <= 24) stays a normal float; k = 0 when no entry is finite and
// non-zero.  scale = (2^k, 2^-k); with wscale (the packed kernel's (2^k_w, 2^-k_w)), epi = 2^-(k_w + k), the factor of
// the conv_tc_kernel epilogue that consumes the scaled operand.
__global__ void operand_scale_kernel(const unsigned int* __restrict__ amax_bits, const float* __restrict__ wscale,
                                     float* __restrict__ scale, float* __restrict__ epi) {
  const float m = __uint_as_float(*amax_bits);
  int k = 0;
  if (m > 0.f) {
    int e;
    frexpf(m, &e);
    k = max(-100, min(100, 13 - e));
  }
  scale[0] = ldexpf(1.0f, k);
  scale[1] = ldexpf(1.0f, -k);
  if (wscale) *epi = ldexpf(wscale[1], -k);
}

// dW[tap][ci][co] = 2^-k_g 2^-k_x * sum over slices, in slice order, of partial[slice][tap][co][ci].  The two powers of
// two are applied one after the other: their product alone could underflow where the result does not.
__global__ void wgrad_reduce_kernel(const float* __restrict__ partial, int slices, int taps, int cout_pad, int cin_pad,
                                    int cin, int cout, const float* __restrict__ gscale, const float* __restrict__ xscale,
                                    float* __restrict__ dw) {
  const float inv_g = gscale[1], inv_x = xscale[1];
  const size_t total = (size_t)taps * cin * cout, slice = (size_t)taps * cout_pad * cin_pad;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int co = (int)(i % cout);
    const int ci = (int)((i / cout) % cin);
    const int tap = (int)(i / ((size_t)cout * cin));
    const float* p = partial + ((size_t)tap * cout_pad + co) * cin_pad + ci;
    float s = p[0];
    for (int sl = 1; sl < slices; ++sl) s += p[sl * slice];
    dw[i] = (s * inv_g) * inv_x;
  }
}

#if defined(__CUDA_ARCH__)
// wgmma with both operands MN-major (transpose bits set; fp16 allows it): D[64 x 64] (+)= A[64 x 16] * B[16 x 64] where
// A's 64 rows and B's 64 columns are contiguous in each 128-byte shared-memory row and the 16 K rows are 128 bytes apart.
__device__ __forceinline__ void wgmma_mn_64x64(float (&d)[32], uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(scale_d));
}

// MN-major, 128-byte-swizzled operand descriptor: a 64-wide MN block (one 128-byte row per K index, the layout a TMA box
// of 64 channels writes pixel by pixel), 8-row K groups 1024 bytes apart.  With a single 64-wide MN block the MN-block
// stride is never used; it is set to the K-group stride too, so every field addresses inside the operand.
__device__ __forceinline__ uint64_t make_desc_mn_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)(1024 >> 4) << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// One 128-pixel tile of the three-pass product g_hi x_hi + g_hi x_lo + g_lo x_hi, 8 K steps of 16 pixels (2048 bytes,
// 128 descriptor units, apart), in wgmma_chunk3's order: per step hi*hi then hi*lo, then the lo*hi steps.
__device__ __forceinline__ void wgrad_tile3(float (&d)[32], uint32_t g_hi, uint32_t g_lo, uint32_t x_hi, uint32_t x_lo,
                                            bool first) {
  const uint64_t gh = make_desc_mn_sw128(g_hi), gl = make_desc_mn_sw128(g_lo);
  const uint64_t xh = make_desc_mn_sw128(x_hi), xl = make_desc_mn_sw128(x_lo);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    wgmma_mn_64x64(d, gh + 128 * k, xh + 128 * k, (!first || k > 0) ? 1u : 0u);
    wgmma_mn_64x64(d, gh + 128 * k, xl + 128 * k, 1u);
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) wgmma_mn_64x64(d, gl + 128 * k, xh + 128 * k, 1u);
}

#endif

__global__ void __launch_bounds__(kTcThreads, 1) conv_wgrad_tc_kernel(const __grid_constant__ WgradParams p) {
#if defined(__CUDA_ARCH__)
  // Persistent: CTA c processes items c, c + gridDim.x, ...  Producer and consumers walk the same sequence of (item,
  // pixel tile) stages through the ring; a warpgroup whose 64 couts lie past cout_pad waits and releases its stages
  // without MMAs.  A tile that overhangs the image has zero-filled gradient rows there; the x rows they meet are zeroed
  // too, so that a non-finite x entry near the edge cannot enter a sum through 0 * NaN.
  extern __shared__ uint8_t smem_raw[];
  uint8_t* stages = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(stages + (size_t)kWgradStages * kWgradSlotBytes);
  uint64_t* empty_bar = full_bar + kWgradStages;
  const WgradPlan& pl = p.pl;
  const int warp = threadIdx.x >> 5;
  const int slot_bytes = kWgradSlotBytes, nst = kWgradStages;

  if (threadIdx.x == 0) {
    ring_init(full_bar, empty_bar, nst);
    fence_mbar_init();
  }
  if (warp == kConsumerWarps && (threadIdx.x & 31) == 0) {
    prefetch_tmap(&p.g_map);
    prefetch_tmap(&p.x_map);
  }
  __syncthreads();

  RingPos rp{0, 0u};
  if (warp >= kConsumerWarps) {
    // ===================== TMA producer =====================
    if (warp == kConsumerWarps && elect_one()) {
      for (int item = blockIdx.x; item < pl.items; item += gridDim.x) {
        int slice, tap, cb, ib;
        wgrad_decode(pl, item, slice, tap, cb, ib);
        const int nco = min(2, pl.co_chunks - 2 * cb);
        const int tx_bytes = (nco + 1) * 2 * kABytes;
        const int dy = tap / p.kw - p.ph, dx = tap % p.kw - p.pw;
        const int t1 = min(pl.ptiles, (slice + 1) * pl.tiles_per_slice);
        for (int t = slice * pl.tiles_per_slice; t < t1; ++t) {
          const int tx = t % pl.tiles_x, ty = (t / pl.tiles_x) % pl.tiles_y, b = t / (pl.tiles_x * pl.tiles_y);
          const int x0 = tx * pl.tw, y0 = ty * pl.th;
          const RingSlot st = ring_acquire(stages, slot_bytes, nst, full_bar, empty_bar, rp, tx_bytes);
          for (int j = 0; j < nco; ++j)
            tma_load_5d(st.data + j * 2 * kABytes, &p.g_map, st.full, (2 * cb + j) * kChunkK, x0, y0, b, 0);
          tma_load_5d(st.data + 4 * kABytes, &p.x_map, st.full, ib * kChunkK, x0 + dx, y0 + dy, b, 0);
        }
      }
    }
  } else {
    // ===================== MMA + partial-tile store (warpgroups 0, 1) =====================
    const int wg = warp >> 2, tid = threadIdx.x & 127, lane = tid & 31, w = tid >> 5;
    float racc[32], acc[32];
    for (int item = blockIdx.x; item < pl.items; item += gridDim.x) {
      int slice, tap, cb, ib;
      wgrad_decode(pl, item, slice, tap, cb, ib);
      const bool mine = 2 * cb + wg < pl.co_chunks;
      const int n = min(pl.ptiles, (slice + 1) * pl.tiles_per_slice) - slice * pl.tiles_per_slice;
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[i] = racc[i] = 0.0f;
      for (int done = 0; done < n;) {
        const int gend = min(n, done + kWgradGroupChunks);
        for (int first = 1; done < gend; ++done, first = 0) {
          const int s = ring_next(rp, nst);
          mbar_wait(&full_bar[s], (rp.par >> s) & 1u);
          rp.par ^= 1u << s;
          const int t = slice * pl.tiles_per_slice + done;
          const int x0 = (t % pl.tiles_x) * pl.tw, y0 = ((t / pl.tiles_x) % pl.tiles_y) * pl.th;
          if (x0 + pl.tw > p.W || y0 + pl.th > p.H) {       // both consumer warpgroups, uniformly
            uint4* xs = reinterpret_cast<uint4*>(stages + (size_t)s * slot_bytes + 4 * kABytes);
            for (int i = threadIdx.x; i < 2 * kTileM * 8; i += 128 * kConsumerWGs) {   // [plane][pixel row][16 B]
              const int m = (i >> 3) & (kTileM - 1);
              if (x0 + m % pl.tw >= p.W || y0 + m / pl.tw >= p.H) xs[i] = make_uint4(0u, 0u, 0u, 0u);
            }
            fence_proxy_async();                           // generic writes -> the MMAs' async-proxy reads
            asm volatile("bar.sync 3, %0;" ::"n"(128 * kConsumerWGs) : "memory");
          }
          if (mine) {
            const uint32_t sa = smem_u32(stages + (size_t)s * slot_bytes);
            const uint32_t ga = sa + wg * 2 * kABytes, xa = sa + 4 * kABytes;
            wgmma_fence_regs(acc);
            wgmma_fence();
            wgrad_tile3(acc, ga, ga + kABytes, xa, xa + kABytes, first != 0);
            wgmma_commit();
            wgmma_wait_all();
            wgmma_fence_regs(acc);
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[s]);
        }
#pragma unroll
        for (int i = 0; i < 32; ++i) racc[i] += acc[i];   // IEEE fp32 promotion
      }
      if (mine) {
        const int co = (2 * cb + wg) * 64 + 16 * w + (lane >> 2);
        float* dst = p.partial + (((size_t)slice * pl.taps + tap) * pl.cout_pad + co) * pl.cin_pad + ib * 64 + 2 * (lane & 3);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          *reinterpret_cast<float2*>(dst + 8 * i) = make_float2(racc[4 * i], racc[4 * i + 1]);
          *reinterpret_cast<float2*>(dst + 8 * (size_t)pl.cin_pad + 8 * i) = make_float2(racc[4 * i + 2], racc[4 * i + 3]);
        }
      }
    }
  }
#endif
}

// ------------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------------
inline int conv_train_fwd_params(TcConvParams& p, const __half* hi, const __half* lo, int cstride, int B, int H, int W,
                                 int kh, int kw, int n_total, int cout_pad, int* nsplit) {
  memset(&p, 0, sizeof(p));
  int tw, th;
  tc_pick_tile(W, H, &tw, &th);
  *nsplit = tc_n_split(cout_pad);
  if (!*nsplit) return RAFT_ERR_BAD_SHAPE;
  RAFT_TRY(make_tmap_act2(&p.a_map[0], hi, lo, B, H, W, cstride, tw, th));
  p.nseg = 1; p.seg_chunks[0] = cstride / kChunkK; p.seg_c0[0] = 0;
  p.stride = 1;
  p.ph = (kh - 1) / 2; p.pw = (kw - 1) / 2;
  p.B = B; p.H = H; p.W = W; p.TH = th; p.TW = tw;
  p.n_total = n_total;
  p.mode = EPI_LINEAR; p.act = ACT_NONE; p.out_scale = 1.0f;
  // Promotion group of the training convolutions: the update block's (2 chunks, 24 MMA steps), whose gradients, like its
  // forward, feed a 12-iteration recurrence.
  p.group_chunks = 2;
  return RAFT_OK;
}

inline int conv_train_forward(const float* x, const float* kernel, const float* bias, int B, int H, int W, int cin, int kh,
                              int kw, int cout, float* out, __half* x_planes, uint8_t* ws, const ConvTrainLayout& L,
                              cudaStream_t st) {
  const size_t npix = (size_t)B * H * W;
  const int cin_pad = L.pl.cin_pad;
  __half* xh = x_planes;
  __half* xl = x_planes + npix * cin_pad;
  uint8_t* tail = reinterpret_cast<uint8_t*>(x_planes) + conv_train_planes_tail(npix, cin);
  unsigned int* xmax = reinterpret_cast<unsigned int*>(tail);
  float* xscale = reinterpret_cast<float*>(tail + 16);
  float* fscale = reinterpret_cast<float*>(ws + L.fscale);
  // the slot is packed afresh every call (weights change every step): its absmax and padding start from zero
  RAFT_CUDA_TRY(cudaMemsetAsync(ws + L.fwd.hi, 0, L.rot.hi - L.fwd.hi, st));
  raft_conv cv{kernel, bias, kh, kw, cin, cout};
  const raft_conv* src[1] = {&cv};
  RAFT_TRY(tc_pack_weights(ws, L.fwd, src, 1, nullptr, false, st));
  // x is scaled like the gradient (max finite |x| 2^k_x in [2^12, 2^13)): small activations stay inside the split's window
  RAFT_CUDA_TRY(cudaMemsetAsync(xmax, 0, sizeof(unsigned int), st));
  RAFT_TRY(launch(absmax_finite_kernel, grid_for(npix * cin), 256, 0, st, x, npix * cin, xmax));
  RAFT_TRY(launch(operand_scale_kernel, 1, 1, 0, st, (const unsigned int*)xmax,
                  reinterpret_cast<const float*>(ws + L.fwd.scale), xscale, fscale));
  RAFT_TRY(launch(train_split_kernel, grid_for(npix * cin_pad), 256, 0, st, x, cin, cin_pad, xh, xl, npix,
                  (const float*)xscale));
  TcConvParams p;
  int nsplit;
  RAFT_TRY(conv_train_fwd_params(p, xh, xl, cin_pad, B, H, W, kh, kw, cout, L.fwd.cout_pad, &nsplit));
  RAFT_TRY(tc_use_weights(p, ws, L.fwd, L.fwd.cout_pad / nsplit));
  p.inv_scale = fscale;
  p.out_f32 = out; p.f32_stride = cout; p.f32_c0 = 0;
  return tc_launch(p, nsplit, st);
}

inline int conv_train_backward(const __half* x_planes, const float* kernel, const float* grad_out, int B, int H, int W,
                               int cin, int kh, int kw, int cout, float* grad_x, float* grad_kernel, uint8_t* ws,
                               const ConvTrainLayout& L, cudaStream_t st) {
  const size_t npix = (size_t)B * H * W;
  const WgradPlan& pl = L.pl;
  __half* gh = reinterpret_cast<__half*>(ws + L.g_hi);
  __half* gl = reinterpret_cast<__half*>(ws + L.g_lo);
  unsigned int* gmax = reinterpret_cast<unsigned int*>(ws + L.gmax);
  float* gscale = reinterpret_cast<float*>(ws + L.gscale);
  float* dscale = reinterpret_cast<float*>(ws + L.dscale);
  const float* xscale = reinterpret_cast<const float*>(reinterpret_cast<const uint8_t*>(x_planes) +
                                                      conv_train_planes_tail(npix, cin) + 16);
  // 1. with an input gradient, the rotated kernel (its 2^k_w enters dscale); the gradient scale, then the scaled gradient
  //    planes
  if (grad_x) {
    RAFT_CUDA_TRY(cudaMemsetAsync(ws + L.rot.hi, 0, L.g_hi - L.rot.hi, st));
    raft_conv cv{kernel, nullptr, kh, kw, cin, cout};
    const raft_conv* src[1] = {&cv};
    RAFT_TRY(tc_pack_weights(ws, L.rot, src, 1, nullptr, false, st, true));
  }
  RAFT_CUDA_TRY(cudaMemsetAsync(gmax, 0, sizeof(unsigned int), st));
  const size_t ng = npix * cout;
  RAFT_TRY(launch(absmax_finite_kernel, grid_for(ng), 256, 0, st, grad_out, ng, gmax));
  RAFT_TRY(launch(operand_scale_kernel, 1, 1, 0, st, (const unsigned int*)gmax,
                  grad_x ? reinterpret_cast<const float*>(ws + L.rot.scale) : (const float*)nullptr, gscale, dscale));
  RAFT_TRY(launch(train_split_kernel, grid_for(npix * pl.cout_pad), 256, 0, st, grad_out, cout, pl.cout_pad, gh, gl, npix,
                  (const float*)gscale));
  // 2. input gradient on conv_tc_kernel
  if (grad_x) {
    TcConvParams p;
    int nsplit;
    RAFT_TRY(conv_train_fwd_params(p, gh, gl, pl.cout_pad, B, H, W, kh, kw, cin, L.rot.cout_pad, &nsplit));
    RAFT_TRY(tc_use_weights(p, ws, L.rot, L.rot.cout_pad / nsplit));
    p.bias = nullptr;
    p.inv_scale = dscale;
    p.out_f32 = grad_x; p.f32_stride = cin; p.f32_c0 = 0;
    RAFT_TRY(tc_launch(p, nsplit, st));
  }
  // 3. weight gradient: partial tiles, then the ordered slice sum
  WgradParams wp;
  memset(&wp, 0, sizeof(wp));
  wp.pl = pl;
  wp.H = H; wp.W = W; wp.kw = kw; wp.ph = (kh - 1) / 2; wp.pw = (kw - 1) / 2;
  wp.partial = reinterpret_cast<float*>(ws + L.partial);
  RAFT_TRY(make_tmap_act2(&wp.g_map, gh, gl, B, H, W, pl.cout_pad, pl.tw, pl.th));
  RAFT_TRY(make_tmap_act2(&wp.x_map, x_planes, x_planes + npix * pl.cin_pad, B, H, W, pl.cin_pad, pl.tw, pl.th));
  unsigned grid = 0;
  RAFT_TRY(persistent_grid<conv_wgrad_tc_kernel>(kWgradSmem, pl.items, &grid));
  RAFT_TRY(launch(conv_wgrad_tc_kernel, grid, kTcThreads, kWgradSmem, st, wp));
  return launch(wgrad_reduce_kernel, grid_for((size_t)pl.taps * cin * cout), 256, 0, st, (const float*)wp.partial,
                pl.slices, pl.taps, pl.cout_pad, pl.cin_pad, cin, cout, (const float*)gscale, xscale, grad_kernel);
}

}  // namespace raft
