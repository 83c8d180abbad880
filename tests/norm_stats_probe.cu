// Test-only program (not part of the library): runs the encoders' normalisation statistics (norm_stats_kernel, then
// norm_final_kernel, csrc/kernels.cuh) on a float32 array read from a file and writes what they produce, so that
// tests/test_gpu_encoders.py can compare the mean and variance of each channel with float64.
//
//   norm_stats_probe <in> <out> G P C
//
// <in> holds G x P x C float32 values (G groups of P pixels with C channels, the layout of a raw convolution output).
// <out> receives G x C means, then G x C multipliers rsqrt(var), float32 (gamma = 1 and eps = 0, so var = mult^-2).
#include <stdio.h>
#include <stdlib.h>

#include <vector>

#include "../tf_raft_b200/csrc/kernels.cuh"

namespace raft {
thread_local long long g_launches = 0;
}

int main(int argc, char** argv) {
  if (argc != 6) return 2;
  const int G = atoi(argv[3]), P = atoi(argv[4]), C = atoi(argv[5]);
  if (G < 1 || P < 1 || C < 8 || C > 256 || C % 8) return 2;
  const size_t n = (size_t)G * P * C;
  std::vector<float> y(n), res(2 * (size_t)G * C), gamma(C, 1.f);
  FILE* f = fopen(argv[1], "rb");
  if (!f || fread(y.data(), sizeof(float), n, f) != n) return 3;
  fclose(f);
  const int nsplit = 64;                                         // kNormSplit of encoder.cuh
  float *d_y, *d_part, *d_gamma, *d_mean, *d_mult;
  if (cudaMalloc(&d_y, n * sizeof(float)) != cudaSuccess ||
      cudaMalloc(&d_part, (size_t)G * nsplit * 3 * C * sizeof(float)) != cudaSuccess ||
      cudaMalloc(&d_gamma, C * sizeof(float)) != cudaSuccess || cudaMalloc(&d_mean, G * C * sizeof(float)) != cudaSuccess ||
      cudaMalloc(&d_mult, G * C * sizeof(float)) != cudaSuccess)
    return 4;
  cudaMemcpy(d_y, y.data(), n * sizeof(float), cudaMemcpyHostToDevice);
  cudaMemcpy(d_gamma, gamma.data(), C * sizeof(float), cudaMemcpyHostToDevice);
  raft::norm_stats_kernel<<<dim3(G, nsplit), 256>>>(d_y, P, C, nsplit, d_part);
  raft::norm_final_kernel<<<(G * C * 32 + 255) / 256, 256>>>(d_part, G, C, nsplit, d_gamma, 0.f, d_mean, d_mult);
  cudaMemcpy(res.data(), d_mean, G * C * sizeof(float), cudaMemcpyDeviceToHost);
  const cudaError_t e = cudaMemcpy(res.data() + G * C, d_mult, G * C * sizeof(float), cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) {
    fprintf(stderr, "%s\n", cudaGetErrorString(e));
    return 5;
  }
  f = fopen(argv[2], "wb");
  if (!f || fwrite(res.data(), sizeof(float), res.size(), f) != res.size()) return 6;
  fclose(f);
  cudaFree(d_y); cudaFree(d_part); cudaFree(d_gamma); cudaFree(d_mean); cudaFree(d_mult);
  return 0;
}
