// Test-only program (not part of the library): runs the shared wgmma mainloop -- conv_tc_kernel, or a plan of layers in
// one update_mega_kernel launch -- on operands written by tests/test_gpu_mainloop.py, with the ring depth, the promotion
// group and the grid chosen by the case instead of derived, and writes back every operand the MMAs read and every output.
//
//   conv_tc_probe describe <case dir>   finalized geometry of every layer as JSON (host code only, no device call)
//   conv_tc_probe run <case dir> ...    runs each case; the same JSON per case on stdout, results into the case dir
//
// A case dir holds `case.txt` (one `key values...` per line) and raw little-endian fp32 files named there:
//   mode conv|mega             conv: one conv_tc_kernel launch per layer, in order; mega: one update_mega_kernel launch
//   grid G                     CTAs per launch (0: min(items, SMs), what the library launches)
//   plane B H W C cstride F    fp16 hi/lo operand plane (planes are numbered in order): F = fp32 (B, H, W, C) file split
//                              with split_plane_kernel (channels [C, cstride) zero), or `-` = output plane (canary)
//   buf N F                    fp32 buffer of N floats (numbered in order): F = file, or `-` = canary
//   layer                      starts a layer; the lines below it belong to it
//   wsrc kh kw cin cout W B    one HWIO convolution (files W, B) of the layer's packed weights; 1 or 2, along cout
//   pack cin_pad cout_pad flatten
//   cinmap n src0 n0 dst0 src1 n1 dst1   TcCinMap of the packing (absent: channels stay where they are)
//   seg plane c0 chunks        one K segment (1 or 2)
//   geom B H W stride ph pw TW TH        output grid, TMA element stride, 'same' pads; TW = 0: tc_pick_tile
//   tile bn ntn n_total
//   epi mode act out_scale
//   out32 buf stride c0 / out16 plane c0 / post scalebuf shiftbuf / residual buf stride c0 / concat buf n /
//   gru zbuf hbuf hid / adv coordsbuf flowbuf / dep layer col0 col1
//   group G                    promotion group (required: the library has no default either)
//   nstages S                  ring depth (absent: what tc_finalize derives)
// Results: P<i>_hi.bin / P<i>_lo.bin (uint16 planes), B<i>.bin (fp32 buffers), L<i>_whi.bin / L<i>_wlo.bin (packed weights,
// [tap][cout_pad][cin_pad]) and L<i>_scale.bin (2^k, 2^-k).  Output planes and buffers start as canary NaNs (fp16 0x7e5a,
// fp32 0x7fc0cafe).  On any error the program prints it and exits non-zero; it never retries.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "../tf_raft_b200/csrc/mega.cuh"

namespace raft {
thread_local long long g_launches = 0;
}
using namespace raft;

static const char* g_case = "";
#define CK(expr)                                                                                          \
  do {                                                                                                    \
    const int _s = (int)(expr);                                                                           \
    if (_s != 0) {                                                                                        \
      fprintf(stderr, "%s: %s failed: status %d (%s)\n", g_case, #expr, _s,                              \
              _s > 0 ? cudaGetErrorString((cudaError_t)_s) : "library status");                           \
      exit(1);                                                                                            \
    }                                                                                                     \
  } while (0)
#define REQUIRE(cond, ...)                                                                                \
  do {                                                                                                    \
    if (!(cond)) {                                                                                        \
      fprintf(stderr, "%s: ", g_case);                                                                    \
      fprintf(stderr, __VA_ARGS__);                                                                       \
      fprintf(stderr, "\n");                                                                              \
      exit(1);                                                                                            \
    }                                                                                                     \
  } while (0)

struct Plane { int B, H, W, C, cs; std::string file; __half *hi = nullptr, *lo = nullptr; size_t n = 0; };
struct Buf { size_t n; std::string file; float* d = nullptr; };
struct Layer {
  int nw = 0, wk[2][4] = {}; std::string wfile[2], bfile[2];
  int cin_pad = 0, cout_pad = 0, flatten = 0; bool has_map = false; TcCinMap map = {};
  int nseg = 0, seg_plane[2] = {}, seg_c0[2] = {}, seg_chunks[2] = {};
  int B = 0, H = 0, W = 0, stride = 1, ph = 0, pw = 0, TW = 0, TH = 0;
  int bn = 0, ntn = 1, n_total = 0, mode = 0, act = 0; float out_scale = 1.0f;
  int out32 = -1, f32_stride = 0, f32_c0 = 0, out16 = -1, h_c0 = 0;
  int post_s = -1, post_t = -1, res = -1, res_stride = 0, res_c0 = 0, concat = -1, concat_n = 0;
  int zb = -1, hb = -1, hid = 0, advc = -1, advf = -1;
  int group = 0, nstages = 0, ndep = 0; MegaDep dep[2] = {};
  TcWeightSlot slot = {}; uint8_t* blob = nullptr; TcConvParams p = {};
};
struct Case { std::string dir; bool mega = false; int grid = 0; std::vector<Plane> planes; std::vector<Buf> bufs; std::vector<Layer> layers; };

static Case parse(const std::string& dir) {
  Case c;
  c.dir = dir;
  const std::string path = dir + "/case.txt";
  FILE* f = fopen(path.c_str(), "r");
  REQUIRE(f, "cannot open %s", path.c_str());
  char line[512];
  Layer* L = nullptr;
  while (fgets(line, sizeof(line), f)) {
    char key[32] = {}, s1[256] = {}, s2[256] = {};
    if (sscanf(line, "%31s", key) != 1 || key[0] == '#') continue;
    const char* r = line + strlen(key);
    const std::string k = key;
    auto need = [&](int got, int want) { REQUIRE(got == want, "bad line: %s", line); };
    auto lay = [&]() { REQUIRE(L, "`%s` outside a layer", key); return L; };
    if (k == "mode") { need(sscanf(r, "%255s", s1), 1); c.mega = strcmp(s1, "mega") == 0; }
    else if (k == "grid") need(sscanf(r, "%d", &c.grid), 1);
    else if (k == "plane") {
      Plane p; need(sscanf(r, "%d %d %d %d %d %255s", &p.B, &p.H, &p.W, &p.C, &p.cs, s1), 6);
      p.file = s1; c.planes.push_back(p);
    } else if (k == "buf") {
      Buf b; long long n; need(sscanf(r, "%lld %255s", &n, s1), 2);
      b.n = (size_t)n; b.file = s1; c.bufs.push_back(b);
    } else if (k == "layer") { c.layers.emplace_back(); L = &c.layers.back(); }
    else if (k == "wsrc") {
      REQUIRE(lay()->nw < 2, "more than two weight sources");
      int* w = L->wk[L->nw];
      need(sscanf(r, "%d %d %d %d %255s %255s", &w[0], &w[1], &w[2], &w[3], s1, s2), 6);
      L->wfile[L->nw] = s1; L->bfile[L->nw] = s2; ++L->nw;
    } else if (k == "pack") need(sscanf(r, "%d %d %d", &lay()->cin_pad, &L->cout_pad, &L->flatten), 3);
    else if (k == "cinmap") {
      TcCinMap& m = lay()->map; L->has_map = true;
      need(sscanf(r, "%d %d %d %d %d %d %d", &m.nrange, &m.src0[0], &m.n[0], &m.dst0[0], &m.src0[1], &m.n[1], &m.dst0[1]), 7);
    } else if (k == "seg") {
      REQUIRE(lay()->nseg < 2, "more than two segments");
      need(sscanf(r, "%d %d %d", &L->seg_plane[L->nseg], &L->seg_c0[L->nseg], &L->seg_chunks[L->nseg]), 3); ++L->nseg;
    } else if (k == "geom") need(sscanf(r, "%d %d %d %d %d %d %d %d", &lay()->B, &L->H, &L->W, &L->stride, &L->ph, &L->pw, &L->TW, &L->TH), 8);
    else if (k == "tile") need(sscanf(r, "%d %d %d", &lay()->bn, &L->ntn, &L->n_total), 3);
    else if (k == "epi") need(sscanf(r, "%d %d %f", &lay()->mode, &L->act, &L->out_scale), 3);
    else if (k == "out32") need(sscanf(r, "%d %d %d", &lay()->out32, &L->f32_stride, &L->f32_c0), 3);
    else if (k == "out16") need(sscanf(r, "%d %d", &lay()->out16, &L->h_c0), 2);
    else if (k == "post") need(sscanf(r, "%d %d", &lay()->post_s, &L->post_t), 2);
    else if (k == "residual") need(sscanf(r, "%d %d %d", &lay()->res, &L->res_stride, &L->res_c0), 3);
    else if (k == "concat") need(sscanf(r, "%d %d", &lay()->concat, &L->concat_n), 2);
    else if (k == "gru") need(sscanf(r, "%d %d %d", &lay()->zb, &L->hb, &L->hid), 3);
    else if (k == "adv") need(sscanf(r, "%d %d", &lay()->advc, &L->advf), 2);
    else if (k == "dep") {
      REQUIRE(lay()->ndep < 2, "more than two dependencies");
      MegaDep& d = L->dep[L->ndep++];
      need(sscanf(r, "%d %d %d", &d.layer, &d.col0, &d.col1), 3);
    } else if (k == "group") need(sscanf(r, "%d", &lay()->group), 1);
    else if (k == "nstages") need(sscanf(r, "%d", &lay()->nstages), 1);
    else REQUIRE(false, "unknown key `%s`", key);
  }
  fclose(f);
  for (const Layer& l : c.layers) {
    REQUIRE(l.nw >= 1 && l.nseg >= 1 && l.group >= 1 && l.bn > 0, "layer needs wsrc, seg, tile and group");
    for (int s = 0; s < l.nseg; ++s) REQUIRE(l.seg_plane[s] >= 0 && l.seg_plane[s] < (int)c.planes.size(), "bad plane");
  }
  return c;
}

// Host-only part of the parameter block: everything tc_finalize and the ring walk depend on.
static void fill_geometry(Layer& L) {
  TcConvParams& p = L.p;
  memset(&p, 0, sizeof(p));
  int tw = L.TW, th = L.TH;
  if (!tw) tc_pick_tile(L.W, L.H, &tw, &th);
  p.nseg = L.nseg;
  for (int s = 0; s < L.nseg; ++s) { p.seg_chunks[s] = L.seg_chunks[s]; p.seg_c0[s] = L.seg_c0[s]; }
  p.kh = L.flatten ? 1 : L.wk[0][0];
  p.kw = L.flatten ? 1 : L.wk[0][1];
  p.ph = L.ph; p.pw = L.pw; p.stride = L.stride;
  p.B = L.B; p.H = L.H; p.W = L.W; p.TW = tw; p.TH = th;
  p.bn = L.bn; p.n_total = L.n_total;
  p.group_chunks = L.group;
  p.mode = L.mode; p.act = L.act; p.out_scale = L.out_scale;
  p.hid = L.hid;
}

// Finalizes like tc_launch (conv) or mega_add (mega), then applies the ring-depth override.  Returns dynamic smem bytes.
static int finalize(Layer& L, bool mega) {
  TcConvParams& p = L.p;
  CK(tc_check(p));
  int smem = tc_finalize(p);
  const int max_st = mega && p.nstages > kMegaMaxStages ? kMegaMaxStages : p.nstages;
  p.nstages = max_st;
  if (L.nstages) {
    REQUIRE(L.nstages >= 2 && L.nstages <= max_st, "nstages %d outside [2, %d]", L.nstages, max_st);
    p.nstages = L.nstages;
  }
  p.n_tiles_n = L.ntn;
  smem = p.nstages * p.stage_bytes + kSmemFixed;
  return smem;
}

static void describe(const Case& c, const Layer& L, int i, int smem, int grid, int sms) {
  const TcConvParams& p = L.p;
  const int total = p.kh * p.kw * (p.seg_chunks[0] + (p.nseg > 1 ? p.seg_chunks[1] : 0));
  const long items = (long)p.B * p.tiles_y * p.tiles_x * p.n_tiles_n;
  const int mma_n = p.bn <= 16 ? 16 : p.bn <= 32 ? 32 : p.bn <= 64 ? 64 : p.bn <= 96 ? 96 : 128;
  printf("%s{\"layer\": %d, \"mode\": \"%s\", \"stage_bytes\": %d, \"nstages\": %d, \"smem\": %d, \"tiles_x\": %d, "
         "\"tiles_y\": %d, \"TW\": %d, \"TH\": %d, \"n_tiles_n\": %d, \"items\": %ld, \"bn\": %d, \"mma_n\": %d, "
         "\"kh\": %d, \"kw\": %d, \"stride\": %d, \"nseg\": %d, \"chunks_per_tap\": %d, \"total_chunks\": %d, "
         "\"group_chunks\": %d, \"groups_per_tile\": %d, \"total_mod_nstages\": %d, \"grid\": %d, \"sms\": %d}",
         i ? ",\n  " : "  ", i, c.mega ? "mega" : "conv", p.stage_bytes, p.nstages, smem, p.tiles_x, p.tiles_y, p.TW,
         p.TH, p.n_tiles_n, items, p.bn, mma_n, p.kh, p.kw, p.stride, p.nseg, total / (p.kh * p.kw), total,
         p.group_chunks, ceil_div(total, p.group_chunks), total % p.nstages, grid, sms);
}

static std::vector<char> read_file(const std::string& path, size_t bytes) {
  FILE* f = fopen(path.c_str(), "rb");
  REQUIRE(f, "cannot open %s", path.c_str());
  std::vector<char> v(bytes);
  const size_t got = fread(v.data(), 1, bytes, f);
  const bool extra = fgetc(f) != EOF;
  fclose(f);
  REQUIRE(got == bytes && !extra, "%s: expected %zu bytes", path.c_str(), bytes);
  return v;
}
static void write_file(const std::string& path, const void* d, size_t bytes) {
  std::vector<char> h(bytes);
  CK(cudaMemcpy(h.data(), d, bytes, cudaMemcpyDeviceToHost));
  FILE* f = fopen(path.c_str(), "wb");
  REQUIRE(f && fwrite(h.data(), 1, bytes, f) == bytes, "cannot write %s", path.c_str());
  fclose(f);
}
static float* upload(const std::string& path, size_t n) {
  std::vector<char> h = read_file(path, n * sizeof(float));
  float* d;
  CK(cudaMalloc(&d, n * sizeof(float)));
  CK(cudaMemcpy(d, h.data(), n * sizeof(float), cudaMemcpyHostToDevice));
  return d;
}

__global__ void fill16(uint16_t* p, size_t n, uint16_t v) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}
__global__ void fill32(uint32_t* p, size_t n, uint32_t v) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}
constexpr uint16_t kCanary16 = 0x7e5a;
constexpr uint32_t kCanary32 = 0x7fc0cafeu;

static void run(Case& c, int sms) {
  std::vector<void*> allocs;
  // ---- operands and buffers ----
  for (Plane& P : c.planes) {
    P.n = (size_t)P.B * P.H * P.W * P.cs;
    const size_t lo_off = align_up(P.n, 512);
    __half* base;
    CK(cudaMalloc(&base, 2 * lo_off * sizeof(__half)));
    allocs.push_back(base);
    P.hi = base; P.lo = base + lo_off;
    if (P.file == "-") {
      CK(launch(fill16, 256, 256, 0, nullptr, reinterpret_cast<uint16_t*>(base), 2 * lo_off, kCanary16));
    } else {
      const size_t npix = (size_t)P.B * P.H * P.W;
      float* src = upload(c.dir + "/" + P.file, npix * P.C);
      CK(launch(split_plane_kernel, grid_for(npix * P.cs), 256, 0, nullptr, (const float*)src, P.C, 0, P.C, P.cs, P.hi,
                P.lo, P.cs, 0, npix, 1.0f));
      CK(cudaDeviceSynchronize());
      CK(cudaFree(src));
    }
  }
  for (Buf& b : c.bufs) {
    if (b.file == "-") {
      CK(cudaMalloc(&b.d, b.n * sizeof(float)));
      CK(launch(fill32, 256, 256, 0, nullptr, reinterpret_cast<uint32_t*>(b.d), b.n, kCanary32));
    } else {
      b.d = upload(c.dir + "/" + b.file, b.n);
    }
    allocs.push_back(b.d);
  }
  auto buf = [&](int i) -> float* { return i < 0 ? nullptr : c.bufs.at(i).d; };

  // ---- weights: packed by the library, parameters filled the way enc_conv_tc / update_core_tc fill them ----
  MegaPlan plan;
  std::vector<int> smem(c.layers.size());
  for (size_t i = 0; i < c.layers.size(); ++i) {
    Layer& L = c.layers[i];
    size_t off = 0;
    L.slot = tc_weight_slot(off, L.flatten ? 1 : L.wk[0][0], L.flatten ? 1 : L.wk[0][1], L.cin_pad, L.cout_pad);
    CK(cudaMalloc(&L.blob, off));
    CK(cudaMemset(L.blob, 0, off));
    allocs.push_back(L.blob);
    raft_conv cv[2];
    const raft_conv* src[2];
    for (int s = 0; s < L.nw; ++s) {
      const int* w = L.wk[s];
      cv[s].kh = w[0]; cv[s].kw = w[1]; cv[s].cin = w[2]; cv[s].cout = w[3];
      float* kd = upload(c.dir + "/" + L.wfile[s], (size_t)w[0] * w[1] * w[2] * w[3]);
      float* bd = upload(c.dir + "/" + L.bfile[s], (size_t)w[3]);
      allocs.push_back(kd); allocs.push_back(bd);
      cv[s].kernel = kd; cv[s].bias = bd;
      src[s] = &cv[s];
    }
    CK(tc_pack_weights(L.blob, L.slot, src, L.nw, L.has_map ? &L.map : nullptr, L.flatten != 0, nullptr));
    fill_geometry(L);
    TcConvParams& p = L.p;
    for (int s = 0; s < L.nseg; ++s) {
      const Plane& P = c.planes[L.seg_plane[s]];
      CK(make_tmap_act2(&p.a_map[s], P.hi, P.lo, P.B, P.H, P.W, P.cs, p.TW, p.TH, L.stride));
    }
    const int kh = p.kh, kw = p.kw;
    CK(tc_use_weights(p, L.blob, L.slot, L.bn));
    REQUIRE(p.kh == kh && p.kw == kw, "packed taps differ");
    if (L.out32 >= 0) { p.out_f32 = buf(L.out32); p.f32_stride = L.f32_stride; p.f32_c0 = L.f32_c0; }
    if (L.out16 >= 0) {
      const Plane& P = c.planes.at(L.out16);
      p.out_hi = P.hi; p.out_lo = P.lo; p.h_stride = P.cs; p.h_c0 = L.h_c0;
    }
    p.post_scale = buf(L.post_s); p.post_shift = buf(L.post_t);
    p.residual = buf(L.res); p.res_stride = L.res_stride; p.res_c0 = L.res_c0;
    p.concat_src = buf(L.concat); p.concat_n = L.concat_n;
    p.z = buf(L.zb); p.h = buf(L.hb);
    p.adv_coords = buf(L.advc); p.adv_flow = buf(L.advf);
    if (c.mega) {
      TcConvParams q = p;
      CK(mega_add(plan, q, L.ntn, L.ndep, L.dep));
      MegaLayer& ML = plan.P.layer[plan.P.nlayers - 1];
      smem[i] = finalize(L, true);
      REQUIRE(ML.c.stage_bytes == p.stage_bytes && ML.c.tiles_x == p.tiles_x && ML.c.tiles_y == p.tiles_y,
              "mega_add finalized differently");
      ML.c.nstages = p.nstages;
    } else {
      smem[i] = finalize(L, false);
    }
  }
  CK(cudaDeviceSynchronize());

  // ---- launch ----
  printf("{\"case\": \"%s\", \"layers\": [\n", c.dir.c_str());
  if (c.mega) {
    CK(cudaFuncSetAttribute(update_mega_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax));
    unsigned int* flags;
    CK(cudaMalloc(&flags, ((size_t)plan.nflags + 1) * sizeof(unsigned int)));
    allocs.push_back(flags);
    CK(cudaMemset(flags, 0, ((size_t)plan.nflags + 1) * sizeof(unsigned int)));
    plan.P.flags = flags;
    plan.P.next_item = flags + plan.nflags;
    const int grid = c.grid ? c.grid : (plan.P.nitems < sms ? plan.P.nitems : sms);
    REQUIRE(grid >= 1 && grid <= sms, "mega grid %d outside [1, %d]: all CTAs must be co-resident", grid, sms);
    for (size_t i = 0; i < c.layers.size(); ++i) describe(c, c.layers[i], (int)i, kSmemMax, grid, sms);
    CK(launch(update_mega_kernel, grid, kTcThreads, kSmemMax, nullptr, plan.P));
    CK(cudaDeviceSynchronize());
  } else {
    CK(cudaFuncSetAttribute(conv_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax));
    for (size_t i = 0; i < c.layers.size(); ++i) {
      const TcConvParams& p = c.layers[i].p;
      const long items = (long)p.B * p.tiles_y * p.tiles_x * p.n_tiles_n;
      const int grid = c.grid ? c.grid : (int)(items < sms ? items : sms);
      REQUIRE(grid >= 1, "empty grid");
      describe(c, c.layers[i], (int)i, smem[i], grid, sms);
      cudaLaunchConfig_t cfg;
      memset(&cfg, 0, sizeof(cfg));
      cfg.gridDim = dim3((unsigned)grid);
      cfg.blockDim = dim3((unsigned)kTcThreads);
      cfg.dynamicSmemBytes = (size_t)smem[i];
      CK(cudaLaunchKernelEx(&cfg, conv_tc_kernel, p));
      CK(cudaDeviceSynchronize());
    }
  }
  printf("\n]}\n");

  // ---- results ----
  for (size_t i = 0; i < c.planes.size(); ++i) {
    const Plane& P = c.planes[i];
    write_file(c.dir + "/P" + std::to_string(i) + "_hi.bin", P.hi, P.n * sizeof(__half));
    write_file(c.dir + "/P" + std::to_string(i) + "_lo.bin", P.lo, P.n * sizeof(__half));
  }
  for (size_t i = 0; i < c.bufs.size(); ++i)
    write_file(c.dir + "/B" + std::to_string(i) + ".bin", c.bufs[i].d, c.bufs[i].n * sizeof(float));
  for (size_t i = 0; i < c.layers.size(); ++i) {
    const Layer& L = c.layers[i];
    const size_t plane = (size_t)L.slot.kh * L.slot.kw * L.slot.cout_pad * L.slot.cin_pad * sizeof(__half);
    const std::string pre = c.dir + "/L" + std::to_string(i);
    write_file(pre + "_whi.bin", L.blob + L.slot.hi, plane);
    write_file(pre + "_wlo.bin", L.blob + L.slot.lo, plane);
    write_file(pre + "_scale.bin", L.blob + L.slot.scale, 2 * sizeof(float));
  }
  for (void* a : allocs) CK(cudaFree(a));
}

int main(int argc, char** argv) {
  if (argc < 3 || (strcmp(argv[1], "describe") && strcmp(argv[1], "run"))) {
    fprintf(stderr, "usage: %s describe <case dir> | run <case dir>...\n", argv[0]);
    return 2;
  }
  if (strcmp(argv[1], "describe") == 0) {
    g_case = argv[2];
    Case c = parse(argv[2]);
    printf("{\"case\": \"%s\", \"layers\": [\n", argv[2]);
    for (size_t i = 0; i < c.layers.size(); ++i) {
      Layer& L = c.layers[i];
      fill_geometry(L);
      const int smem = finalize(L, c.mega);
      describe(c, L, (int)i, c.mega ? kSmemMax : smem, c.grid, 0);
    }
    printf("\n]}\n");
    return 0;
  }
  int dev = 0, sms = 0;
  CK(cudaGetDevice(&dev));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  for (int a = 2; a < argc; ++a) {
    g_case = argv[a];
    Case c = parse(argv[a]);
    run(c, sms);
  }
  fflush(stdout);
  return 0;
}
