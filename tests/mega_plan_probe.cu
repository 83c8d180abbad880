// Test-only host program (not part of the library): prints, as JSON, the update_mega_kernel plan that update_core_tc
// builds for one update-block application, so that tests/test_mega_plan.py can check its waits on a machine without a GPU.
//
//   mega_plan_probe <basic|small> B h w <mask 0|1> <advance 0|1>
//
// Nothing touches a device: the workspace, prepared-weights blob, hidden state and coords1 sit at fake 1 KB-aligned
// addresses, fim_ready keeps the im2col kernel from being launched, and with a plan every layer is appended to it instead
// of launched.  Tensor maps are built through cuTensorMapEncodeTiled, which update_core_tc resolves with
// cudaGetDriverEntryPoint: this program defines that function itself (linked against the shared cudart, the executable's
// definition is the one its calls bind to) and hands out an encoder that records the global address, dimensions, strides
// and box of each map in the map's own bytes, so the checker also sees which planes the TMA loads address.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../tf_raft_b200/csrc/update.cuh"

namespace raft {
thread_local long long g_launches = 0;
}

// Layout of the recorded map (CUtensorMap is 128 opaque bytes = 16 x 64-bit words).
enum { TM_ADDR = 0, TM_RANK = 1, TM_DIMS = 2, TM_STRIDES = 7, TM_BOX = 11 };

static CUresult stub_encode_tiled(CUtensorMap* m, CUtensorMapDataType, cuuint32_t rank, void* addr, const cuuint64_t* dims,
                                  const cuuint64_t* strides, const cuuint32_t* box, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill) {
  if (rank < 1 || rank > 5) return CUDA_ERROR_INVALID_VALUE;
  uint64_t* o = reinterpret_cast<uint64_t*>(m);
  memset(m, 0, sizeof(*m));
  o[TM_ADDR] = reinterpret_cast<uint64_t>(addr);
  o[TM_RANK] = rank;
  for (cuuint32_t i = 0; i < rank; ++i) {
    o[TM_DIMS + i] = dims[i];
    if (i > 0) o[TM_STRIDES + i - 1] = strides[i - 1];
    reinterpret_cast<uint32_t*>(o + TM_BOX)[i] = box[i];
  }
  return CUDA_SUCCESS;
}

cudaError_t CUDARTAPI cudaGetDriverEntryPoint(const char* symbol, void** fn, unsigned long long,
                                              cudaDriverEntryPointQueryResult* status) {
  const bool ok = strcmp(symbol, "cuTensorMapEncodeTiled") == 0;
  *fn = ok ? reinterpret_cast<void*>(&stub_encode_tiled) : nullptr;
  if (status) *status = ok ? cudaDriverEntryPointSuccess : cudaDriverEntryPointSymbolNotFound;
  return ok ? cudaSuccess : cudaErrorSymbolNotFound;
}

static unsigned long long u(const void* p) { return (unsigned long long)reinterpret_cast<uintptr_t>(p); }

static void print_map(const CUtensorMap& m) {
  const uint64_t* o = reinterpret_cast<const uint64_t*>(&m);
  const int rank = (int)o[TM_RANK];
  printf("{\"addr\": %llu, \"dims\": [", (unsigned long long)o[TM_ADDR]);
  for (int i = 0; i < rank; ++i) printf("%s%llu", i ? ", " : "", (unsigned long long)o[TM_DIMS + i]);
  printf("], \"strides\": [");
  for (int i = 1; i < rank; ++i) printf("%s%llu", i > 1 ? ", " : "", (unsigned long long)o[TM_STRIDES + i - 1]);
  printf("], \"box\": [");
  for (int i = 0; i < rank; ++i) printf("%s%u", i ? ", " : "", reinterpret_cast<const uint32_t*>(o + TM_BOX)[i]);
  printf("]}");
}

int main(int argc, char** argv) {
  using namespace raft;
  if (argc != 7) {
    fprintf(stderr, "usage: %s <basic|small> B h w <mask 0|1> <advance 0|1>\n", argv[0]);
    return 2;
  }
  const int variant = strcmp(argv[1], "basic") == 0 ? RAFT_VARIANT_BASIC : RAFT_VARIANT_SMALL;
  const int B = atoi(argv[2]), h = atoi(argv[3]), w = atoi(argv[4]);
  const bool with_mask = atoi(argv[5]) != 0, advance = atoi(argv[6]) != 0;

  // Fake device addresses, each region far from the others (1 TB apart) and 1 KB aligned.
  uint8_t* const ws = reinterpret_cast<uint8_t*>(uintptr_t(1) << 40);
  const uint8_t* const prepared = reinterpret_cast<const uint8_t*>(uintptr_t(2) << 40);
  float* const hidden = reinterpret_cast<float*>(uintptr_t(3) << 40);
  float* const coords1 = reinterpret_cast<float*>(uintptr_t(4) << 40);

  UpdateCtx c;
  memset(&c, 0, sizeof(c));
  c.variant = variant;
  c.precision = RAFT_PREC_F16X2;
  c.B = B; c.h = h; c.w = w;
  c.prepared = prepared;
  c.PL = prepared_layout(variant, RAFT_PREC_F16X2);
  c.W = workspace_layout(ws, variant, B, h, w, RAFT_PREC_F16X2);
  c.stream = nullptr;
  c.fim_ready = true;
  MegaPlan plan;
  c.plan = &plan;
  const Workspace& W = c.W;
  const int st = update_core_tc(c, hidden, W.delta, with_mask ? W.mask : nullptr, advance ? coords1 : nullptr);
  if (st != 0 || g_launches != 0) {
    fprintf(stderr, "update_core_tc: status %d, %lld launches\n", st, g_launches);
    return 1;
  }

  const VariantDims d = variant_dims(variant);
  printf("{\"variant\": \"%s\", \"B\": %d, \"h\": %d, \"w\": %d, \"mask\": %d, \"advance\": %d,\n", argv[1], B, h, w,
         (int)with_mask, (int)advance);
  printf(" \"hid\": %d, \"nitems\": %d, \"nlayers\": %d, \"nflags\": %d, \"mega_flag_words\": %llu,\n", d.hid,
         plan.P.nitems, plan.P.nlayers, plan.nflags, (unsigned long long)W.mega_flag_words);
  // fp16 operand planes (hi, lo, channel stride) in TcPlane order, then the fp32 buffers
  printf(" \"planes\": [[%llu, %llu, %d], [%llu, %llu, %d], [%llu, %llu, %d], [%llu, %llu, %d], [%llu, %llu, %d], "
         "[%llu, %llu, %d], [%llu, %llu, %d], [%llu, %llu, %d], [%llu, %llu, %d]],\n",
         u(W.corr_hi), u(W.corr_lo), d.s_corr, u(W.cor1_hi), u(W.cor1_lo), d.s_cor1, u(W.cf_hi), u(W.cf_lo), d.s_cf,
         u(W.flo1_hi), u(W.flo1_lo), d.s_flo1, u(W.x_hi), u(W.x_lo), d.s_x, u(W.h_hi), u(W.h_lo), d.s_h, u(W.rh_hi),
         u(W.rh_lo), d.s_h, u(W.fm_hi), u(W.fm_lo), d.s_fm, u(W.fim_hi), u(W.fim_lo), 128);
  printf(" \"f32\": {\"h\": %llu, \"z\": %llu, \"flow\": %llu, \"coords1\": %llu, \"delta\": %llu, \"mask\": %llu},\n",
         u(hidden), u(W.z), u(W.flow), u(coords1), u(W.delta), u(W.mask));
  printf(" \"layers\": [\n");
  const TcLayer* rows = tc_layers(variant);
  for (int i = 0; i < plan.P.nlayers; ++i) {
    const MegaLayer& ML = plan.P.layer[i];
    const TcConvParams& p = ML.c;
    const TcLayer& R = rows[i];            // update_core_tc plans row i at position i (it refuses otherwise)
    printf("  {\"row\": %d, \"table\": {\"segs\": [", i);
    for (int s = 0; s < 2 && R.seg[s].chunks; ++s)
      printf("%s[%d, %d, %d]", s ? ", " : "", R.seg[s].plane, R.seg[s].c0, R.seg[s].chunks);
    printf("], \"out\": %d, \"out_c0\": %d, \"mode\": %d, \"flags\": %d, \"bn\": %d, \"ntn\": %d, \"n_total\": %d, "
           "\"kh\": %d, \"kw\": %d, \"ndep\": %d, \"dep\": [",
           R.out, R.out_c0, R.mode, R.flags, R.bn, R.ntn, R.n_total, R.kh, R.kw, R.ndep);
    for (int k = 0; k < R.ndep; ++k) printf("%s[%d, %d, %d]", k ? ", " : "", R.dep[k].layer, R.dep[k].col0, R.dep[k].col1);
    printf("]},\n   \"nseg\": %d, \"seg_c0\": [%d, %d], \"seg_chunks\": [%d, %d], \"a_map\": [", p.nseg, p.seg_c0[0],
           p.seg_c0[1], p.seg_chunks[0], p.seg_chunks[1]);
    for (int s = 0; s < p.nseg; ++s) {
      if (s) printf(", ");
      print_map(p.a_map[s]);
    }
    printf("],\n   \"kh\": %d, \"kw\": %d, \"ph\": %d, \"pw\": %d, \"stride\": %d, \"B\": %d, \"H\": %d, \"W\": %d, "
           "\"TH\": %d, \"TW\": %d, \"tiles_y\": %d, \"tiles_x\": %d, \"bn\": %d, \"n_total\": %d, \"n_tiles_n\": %d, "
           "\"mode\": %d, \"hid\": %d,\n",
           p.kh, p.kw, p.ph, p.pw, p.stride, p.B, p.H, p.W, p.TH, p.TW, p.tiles_y, p.tiles_x, p.bn, p.n_total,
           p.n_tiles_n, p.mode, p.hid);
    printf("   \"out_hi\": %llu, \"out_lo\": %llu, \"h_stride\": %d, \"h_c0\": %d, \"out_f32\": %llu, \"f32_stride\": %d, "
           "\"f32_c0\": %d, \"residual\": %llu, \"concat_src\": %llu, \"concat_n\": %d, \"z\": %llu, \"h\": %llu, "
           "\"adv_coords\": %llu, \"adv_flow\": %llu,\n",
           u(p.out_hi), u(p.out_lo), p.h_stride, p.h_c0, u(p.out_f32), p.f32_stride, p.f32_c0, u(p.residual),
           u(p.concat_src), p.concat_n, u(p.z), u(p.h), u(p.adv_coords), u(p.adv_flow));
    printf("   \"item0\": %d, \"flag0\": %d, \"ndep\": %d, \"dep_layer\": [%d, %d], \"dep_nlo\": [%d, %d], "
           "\"dep_nhi\": [%d, %d], \"dep_ry\": %d, \"dep_rx\": %d}%s\n",
           ML.item0, ML.flag0, ML.ndep, ML.dep_layer[0], ML.dep_layer[1], ML.dep_nlo[0], ML.dep_nlo[1], ML.dep_nhi[0],
           ML.dep_nhi[1], ML.dep_ry, ML.dep_rx, i + 1 < plan.P.nlayers ? "," : "");
  }
  printf(" ]}\n");
  return 0;
}
