// Test-only program (not part of the library): applies the library's ReLU and fp16 hi/lo split routines (csrc/common.cuh)
// to a list of float32 bit patterns on the GPU and prints, per input, the bits of
//   relu_nan(v)  fmaxf(v, 0)  split_f16(v).hi  split_f16(v).lo  split_f16x2(v, -v).hi[0] .lo[0] .hi[1] .lo[1]
// one line of hexadecimal words each, so that tests/test_gpu_values.py can compare them bit for bit with fmaxf and with
// a NumPy emulation of the split.
//
//   values_probe <hex bits> ...
#include <stdio.h>
#include <stdlib.h>

#include "../tf_raft_b200/csrc/common.cuh"

namespace raft {
thread_local long long g_launches = 0;
}

__global__ void probe_kernel(const float* in, int n, uint32_t* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = in[i];
  uint32_t* o = out + 8 * (size_t)i;
  o[0] = __float_as_uint(raft::relu_nan(v));
  o[1] = __float_as_uint(fmaxf(v, 0.f));
  __half hi, lo;
  raft::split_f16(v, hi, lo);
  o[2] = __half_as_ushort(hi);
  o[3] = __half_as_ushort(lo);
  uint32_t h2, l2;
  raft::split_f16x2(v, -v, h2, l2);
  o[4] = h2 & 0xffffu;
  o[5] = l2 & 0xffffu;
  o[6] = h2 >> 16;
  o[7] = l2 >> 16;
}

int main(int argc, char** argv) {
  const int n = argc - 1;
  if (n < 1) return 2;
  float* h_in = (float*)malloc(sizeof(float) * n);
  uint32_t* h_out = (uint32_t*)malloc(sizeof(uint32_t) * 8 * n);
  for (int i = 0; i < n; ++i) {
    const uint32_t b = (uint32_t)strtoul(argv[i + 1], nullptr, 16);
    memcpy(&h_in[i], &b, 4);
  }
  float* d_in;
  uint32_t* d_out;
  if (cudaMalloc(&d_in, sizeof(float) * n) != cudaSuccess || cudaMalloc(&d_out, sizeof(uint32_t) * 8 * n) != cudaSuccess)
    return 3;
  cudaMemcpy(d_in, h_in, sizeof(float) * n, cudaMemcpyHostToDevice);
  probe_kernel<<<(n + 127) / 128, 128>>>(d_in, n, d_out);
  const cudaError_t e = cudaMemcpy(h_out, d_out, sizeof(uint32_t) * 8 * n, cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) {
    fprintf(stderr, "%s\n", cudaGetErrorString(e));
    return 4;
  }
  for (int i = 0; i < n; ++i) {
    for (int k = 0; k < 8; ++k) printf(k ? " %08x" : "%08x", h_out[8 * i + k]);
    printf("\n");
  }
  cudaFree(d_in);
  cudaFree(d_out);
  free(h_in);
  free(h_out);
  return 0;
}
