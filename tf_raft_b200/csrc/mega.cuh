// update_mega_kernel: every tensor-core layer of one update-block application (tf_raft/layers/update.py:143-153 -- motion
// encoder, SepConvGRU / ConvGRU, flow head, mask head) in ONE persistent warp-specialised wgmma kernel.
//
// The per-layer kernel (conv_tc.cuh) is launched 11 times per iteration; each launch pays its prologue and exposes its
// epilogue with no next tile to hide behind.  Here the work list is (layer, tile) for all layers of the block, in layer
// order; the CTAs (one per SM) claim items in list order with the same roles as conv_tc_kernel:
//   warp 8  TMA producer: claims the items; before the first load of an item it waits for the tiles of the SOURCE
//           layer(s) that cover the item's halo -- a per-(layer, tile) counter in global memory that the 8 consumer warps
//           of the producing CTA increment (release) after their stores -- then streams (tap, 64-channel chunk) stages;
//   warps 0..7  two consumer warpgroups: wgmma MMAs with IEEE-fp32 promotion groups, the fused epilogue of the layer's
//           mode (bias / ReLU / GRU gates / hi-lo re-split), then the item's completion counter.
// The shared-memory ring runs straight across items, so the epilogue of one item overlaps the loads of the next (of
// another layer).  Dependencies always point to earlier items of the list and every CTA consumes its items in list
// order, so with all CTAs co-resident (1 per SM) the wait graph is acyclic.  Activations written by generic-proxy stores
// and read back by TMA (async proxy) are ordered by fence.proxy.async on both sides of the release / acquire pair; z and
// h, which epilogues re-read with ordinary loads, are read through L2 (ld.global.cg).
#pragma once
#include "conv_tc.cuh"

namespace raft {

constexpr int kMegaMaxLayers = 14;
constexpr int kMegaMaxStages = 8;

struct alignas(64) MegaLayer {
  TcConvParams c;                 // the layer exactly as the per-layer kernel would run it (tensor maps, epilogue, tiling)
  int item0;                      // first item of this layer in the work list
  int flag0;                      // first completion counter of this layer (n_tiles_n * pixel tiles of them)
  int ndep;
  int dep_layer[2];               // source layers (positions in MegaParams::layer)
  int dep_nlo[2], dep_nhi[2];     // column tiles of the source that are read
  int dep_ry, dep_rx;             // halo of the dependency in tiles (>= 1: also covers the write-after-read hazards)
};

struct alignas(64) MegaParams {
  MegaLayer layer[kMegaMaxLayers];
  int nlayers, nitems;
  unsigned int* flags;            // zeroed before the launch
  unsigned int* next_item;        // work-list cursor (zeroed with the flags): CTAs claim items with atomicAdd
};
constexpr int kMegaQueue = 16;    // per-CTA ring of claimed item numbers (producer -> consumers)

#if defined(__CUDA_ARCH__)
__device__ __forceinline__ unsigned int ld_acquire_gpu(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_gpu_add(unsigned int* p, unsigned int v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }

__device__ __forceinline__ int mega_layer_of(const MegaParams& P, int item) {
  int L = 0;
  while (L + 1 < P.nlayers && item >= P.layer[L + 1].item0) ++L;
  return L;
}
#endif

__global__ void __launch_bounds__(kTcThreads, 1) update_mega_kernel(const __grid_constant__ MegaParams P) {
#if defined(__CUDA_ARCH__)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int kRingBytes = kSmemMax - kSmemFixed;                         // stages of the current layer live here
  uint8_t* stages = smem;
  float* staging = reinterpret_cast<float*>(smem + kRingBytes);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kRingBytes + kStagingBytes);
  uint64_t* empty_bar = full_bar + kMegaMaxStages;
  uint64_t* q_bar = empty_bar + kMegaMaxStages;         // [kMegaQueue] producer -> consumers: item number published
  int* item_q = reinterpret_cast<int*>(q_bar + kMegaQueue);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    ring_init(full_bar, empty_bar, kMegaMaxStages);
    for (int i = 0; i < kMegaQueue; ++i) mbar_init(&q_bar[i], 1);
    fence_mbar_init();
  }
  if (warp == 0 && lane < P.nlayers) {                   // descriptor fetches off the first stage of every layer
    const TcConvParams& c = P.layer[lane].c;
    prefetch_tmap(&c.a_map[0]);
    if (c.nseg > 1) prefetch_tmap(&c.a_map[1]);
    prefetch_tmap(&c.b_map);
  }
  __syncthreads();

  if (warp >= kConsumerWarps) {
    // ===================== TMA producer =====================
    regs_producer();
    if (warp == kConsumerWarps && elect_one()) {
      RingPos rp{0, 0u};
      int cur_nst = 0, cur_bytes = 0;
      // Items are CLAIMED, not pre-assigned: a CTA that becomes free takes the lowest unclaimed item of the list (layer
      // order = priority order), so no CTA sits on a blocked item while a runnable one waits behind it in a fixed
      // per-CTA sequence.  Every dependency points to a lower item number, which some co-resident CTA has already claimed,
      // so the wait graph stays acyclic.  The claimed number is handed to the consumers through item_q / q_bar.
      int item = (int)atomicAdd(P.next_item, 1u);
      for (int k = 0;; ++k) {
        const int qs = k & (kMegaQueue - 1);
        item_q[qs] = item < P.nitems ? item : -1;
        mbar_arrive(&q_bar[qs]);                         // (release: the slot's item number is visible to the waiters)
        if (item >= P.nitems) break;
        const int L = mega_layer_of(P, item);
        const MegaLayer& ML = P.layer[L];
        const TcConvParams& c = ML.c;
        int nt, b, ty, tx;
        tc_decode_tile(c, item - ML.item0, nt, b, ty, tx);
        // ---- dependencies: tiles of the source layers that cover this tile's halo ----
        if (ML.ndep > 0) {
          const int mtiles = c.B * c.tiles_y * c.tiles_x;
          for (int d = 0; d < ML.ndep; ++d) {
            const MegaLayer& SL = P.layer[ML.dep_layer[d]];
            for (int n = ML.dep_nlo[d]; n <= ML.dep_nhi[d]; ++n)
              for (int yy = max(0, ty - ML.dep_ry); yy <= min(c.tiles_y - 1, ty + ML.dep_ry); ++yy)
                for (int xx = max(0, tx - ML.dep_rx); xx <= min(c.tiles_x - 1, tx + ML.dep_rx); ++xx) {
                  const unsigned int* f = P.flags + SL.flag0 + n * mtiles + (b * c.tiles_y + yy) * c.tiles_x + xx;
                  if (ld_acquire_gpu(f) < (unsigned)kConsumerWarps) {
                    const long long t0 = clock64();
                    while (ld_acquire_gpu(f) < (unsigned)kConsumerWarps) {
                      __nanosleep(64);
                      if (clock64() - t0 > 8000000000LL) __trap();        // protocol bug -> trapped kernel, never a hang
                    }
                  }
                }
          }
          fence_proxy_async_all();          // acquired generic-proxy writes -> visible to the TMA loads issued below
        }
        // ---- ring geometry: a layer with another stage size re-carves the ring once it has drained ----
        if (c.nstages != cur_nst || c.stage_bytes != cur_bytes) {
          for (int s = 0; s < kMegaMaxStages; ++s)        // the last use of every slot has been consumed (an unused slot
            mbar_wait(&empty_bar[s], ((rp.par >> s) & 1u) ^ 1u);   // passes at once: its parity wait names a past phase)
          rp.slot = 0;
          cur_nst = c.nstages;
          cur_bytes = c.stage_bytes;
        }
        int nxt = P.nitems;
        tc_produce_tile(c, stages, full_bar, empty_bar, rp, nt, b, ty, tx, P.next_item, &nxt);
        item = nxt;
      }
    }
  } else {
    // ===================== MMA + epilogue (warpgroups 0, 1) =====================
    regs_consumer();
    const int wg = warp >> 2, tid = threadIdx.x & 127;
    RingPos rp{0, 0u};
    int cur_nst = 0, cur_bytes = 0;
    for (int k = 0;; ++k) {
      mbar_wait(&q_bar[k & (kMegaQueue - 1)], (uint32_t)(k / kMegaQueue) & 1u);
      const int item = item_q[k & (kMegaQueue - 1)];
      if (item < 0) break;
      const MegaLayer& ML = P.layer[mega_layer_of(P, item)];
      const TcConvParams& c = ML.c;
      if (c.nstages != cur_nst || c.stage_bytes != cur_bytes) {
        rp.slot = 0;
        cur_nst = c.nstages;
        cur_bytes = c.stage_bytes;
      }
      int nt, b, ty, tx;
      tc_decode_tile(c, item - ML.item0, nt, b, ty, tx);
      with_mma_n(c.bn, [&](auto n) {
        tc_consume_tile<decltype(n)::value>(c, stages, staging, full_bar, empty_bar, rp, wg, tid, nt, b, ty, tx);
      });
      // ---- publish: this warp's stores of the item are visible gpu-wide, to generic loads and to TMA ----
      __syncwarp();
      if (lane == 0) {
        fence_proxy_async_all();
        const int mtiles = c.B * c.tiles_y * c.tiles_x;
        red_release_gpu_add(P.flags + ML.flag0 + nt * mtiles + (b * c.tiles_y + ty) * c.tiles_x + tx, 1u);
      }
    }
  }
#endif
}

// ------------------------------------------------------------------------------------------------
// Host side: the plan of one update-block application.
// ------------------------------------------------------------------------------------------------
// A layer reads output columns [col0, col1) of an earlier layer of the plan (col1 == 0: all of them).
struct MegaDep { int layer, col0, col1; };

struct MegaPlan {
  MegaParams P;
  int nflags;
  MegaPlan() {
    memset(&P, 0, sizeof(P));
    nflags = 0;
  }
};

inline int mega_flag_words(int B, int tiles) { return kMegaMaxLayers * 6 * B * tiles + 1; }   // upper bound used by the workspace layout

// Appends a planned layer (p complete except for the launch fields).  Mirrors the checks of tc_launch().  A dependency
// waits on the source's column tiles that hold the columns it reads.
inline int mega_add(MegaPlan& M, TcConvParams& p, int n_tiles_n, int ndep, const MegaDep deps[]) {
  if (M.P.nlayers >= kMegaMaxLayers || ndep < 0 || ndep > 2) return RAFT_ERR_UNSUPPORTED;
  RAFT_TRY(tc_check(p));
  if (p.stride < 1) p.stride = 1;
  tc_finalize(p);
  if (p.nstages < 2) return RAFT_ERR_UNSUPPORTED;
  if (p.nstages > kMegaMaxStages) p.nstages = kMegaMaxStages;
  p.n_tiles_n = n_tiles_n;
  MegaLayer& ML = M.P.layer[M.P.nlayers];
  ML.c = p;
  const int mtiles = p.B * p.tiles_y * p.tiles_x;
  ML.item0 = M.P.nitems;
  ML.flag0 = M.nflags;
  ML.ndep = ndep;
  for (int d = 0; d < ndep; ++d) {
    const MegaDep& D = deps[d];
    if (D.layer < 0 || D.layer >= M.P.nlayers) return RAFT_ERR_BAD_ARG;   // a source layer is planned before its consumer
    const TcConvParams& s = M.P.layer[D.layer].c;
    ML.dep_layer[d] = D.layer;
    ML.dep_nlo[d] = D.col0 / s.bn;
    ML.dep_nhi[d] = D.col1 > 0 ? (D.col1 - 1) / s.bn : s.n_tiles_n - 1;
    if (ML.dep_nlo[d] > ML.dep_nhi[d] || ML.dep_nhi[d] >= s.n_tiles_n) return RAFT_ERR_BAD_ARG;
  }
  ML.dep_ry = ceil_div(p.ph > 0 ? p.ph : 1, p.TH);
  ML.dep_rx = ceil_div(p.pw > 0 ? p.pw : 1, p.TW);
  if (ML.dep_ry < 1) ML.dep_ry = 1;
  if (ML.dep_rx < 1) ML.dep_rx = 1;
  M.P.nitems += mtiles * n_tiles_n;
  M.nflags += mtiles * n_tiles_n;
  ++M.P.nlayers;
  return RAFT_OK;
}

inline int mega_launch(MegaPlan& M, unsigned int* flags, size_t flag_words, bool zero_flags, cudaStream_t stream) {
  if (M.P.nlayers == 0) return RAFT_OK;
  if ((size_t)M.nflags + 1 > flag_words) return RAFT_ERR_WORKSPACE;
  M.P.flags = flags;
  M.P.next_item = flags + M.nflags;
  // Items wait on items claimed by other CTAs: every claimed item is held by a RUNNING CTA, so the wait graph is acyclic
  // whatever the number of co-resident CTAs; one CTA per SM (shared memory), never more CTAs than SMs.
  unsigned grid = 0;
  RAFT_TRY(persistent_grid<update_mega_kernel>(kSmemMax, M.P.nitems, &grid));
  if (zero_flags) RAFT_CUDA_TRY(cudaMemsetAsync(flags, 0, ((size_t)M.nflags + 1) * sizeof(unsigned int), stream));
  return launch(update_mega_kernel, grid, kTcThreads, kSmemMax, stream, M.P);
}

}  // namespace raft
