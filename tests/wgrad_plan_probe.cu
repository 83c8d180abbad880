// Test-only host program (not part of the library): prints, as JSON, the weight-gradient work decomposition that
// conv_train.cuh plans for one shape, so that tests/test_conv_train_cases.py can check it on a machine without a GPU.
//
//   wgrad_plan_probe B H W cin kh kw cout
//
// Nothing touches a device: wgrad_plan is a function of the shape alone.
#include <stdio.h>
#include <stdlib.h>

#include "../tf_raft_b200/csrc/conv_train.cuh"

namespace raft {
thread_local long long g_launches = 0;
}

int main(int argc, char** argv) {
  if (argc != 8) {
    fprintf(stderr, "usage: wgrad_plan_probe B H W cin kh kw cout\n");
    return 2;
  }
  int a[7];
  for (int i = 0; i < 7; ++i) a[i] = atoi(argv[i + 1]);
  const int st = raft::conv_train_check(a[0], a[1], a[2], a[3], a[4], a[5], a[6]);
  raft::ConvTrainLayout L;
  const int sl = st ? st : raft::conv_train_layout(a[0], a[1], a[2], a[3], a[4], a[5], a[6], L);
  if (sl) {
    printf("{\"status\": %d}\n", sl);
    return 0;
  }
  const raft::WgradPlan& p = L.pl;
  printf("{\"status\": 0, \"taps\": %d, \"co_chunks\": %d, \"co_blocks\": %d, \"ci_blocks\": %d, \"tw\": %d, \"th\": %d, "
         "\"tiles_x\": %d, \"tiles_y\": %d, \"ptiles\": %d, \"slices\": %d, \"tiles_per_slice\": %d, \"items\": %d, "
         "\"cin_pad\": %d, \"cout_pad\": %d, \"partial_bytes\": %zu, \"workspace_bytes\": %zu, \"group_chunks\": %d, "
         "\"items_list\": [",
         p.taps, p.co_chunks, p.co_blocks, p.ci_blocks, p.tw, p.th, p.tiles_x, p.tiles_y, p.ptiles, p.slices,
         p.tiles_per_slice, p.items, p.cin_pad, p.cout_pad, L.gmax - L.partial, L.total, raft::kWgradGroupChunks);
  // item -> (slice, tap, cb, ib) through the kernel's own decode, and the slice's pixel tiles [t0, t1)
  for (int item = 0; item < p.items; ++item) {
    int slice, tap, cb, ib;
    raft::wgrad_decode(p, item, slice, tap, cb, ib);
    const int t0 = slice * p.tiles_per_slice, t1 = std::min(p.ptiles, t0 + p.tiles_per_slice);
    printf("%s[%d, %d, %d, %d, %d, %d]", item ? ", " : "", slice, tap, cb, ib, t0, t1);
  }
  printf("]}\n");
  return 0;
}
