// diag8_bench.cu — what bounds the 8x8 pivot block of the tile Cholesky (csrc/chol_tiles.cuh)?
//   * issue rate of independent FP64 FMAs from ONE warp (the pivot block is one warp's work)
//   * the pivot block in the DMMA fragment layout (ct_diag8_frag), in the form chol_tiles.cuh ships
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o diag8_bench diag8_bench.cu
#include "../../open_vins_b200/csrc/chol_tiles.cuh"
#include <cstdio>
#include <vector>
#include <random>
#include <cmath>

template <int NACC> __global__ void k_dfma_tp(double *out, int iters, long long *cyc) {
  double c[NACC];
  for (int i = 0; i < NACC; i++)
    c[i] = threadIdx.x * 1e-3 + i;
  const double a = 1.0000001, b = 1e-9;
  __syncthreads();
  long long t0 = clock64();
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < NACC; i++)
      c[i] = fma(c[i], a, b);
  }
  long long t1 = clock64();
  double s = 0;
  for (int i = 0; i < NACC; i++)
    s += c[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0 && blockIdx.x == 0)
    *cyc = t1 - t0;
}

__global__ void k_diag8(double *tiles, int reps, long long *cyc, int variant) {
  __shared__ __align__(16) double tile[64], Linv[64], invd[8], xp[8 * CT_XP];
  __shared__ int flag;
  long long tot = 0;
  for (int r = 0; r < reps; r++) {
    for (int e = threadIdx.x; e < 64; e += 32)
      tile[e] = tiles[e];
    __syncwarp();
    long long t0 = clock64();
    {
      double2 c = *reinterpret_cast<const double2 *>(tile + 2 * threadIdx.x);
      if (variant == 0)
        ct_diag8_frag(c.x, c.y, 8, invd, true, 0.0, &flag);
      else
        ct_diag8_frag(c.x, c.y, 8, invd, false, 1e-30, &flag);
      *reinterpret_cast<double2 *>(tile + 2 * threadIdx.x) = c;
    }
    __syncwarp();
    tot += clock64() - t0;
  }
  for (int e = threadIdx.x; e < 64; e += 32)
    tiles[64 * (1 + variant) + e] = tile[e];
  if (threadIdx.x < 8)
    tiles[64 * 3 + 8 * variant + threadIdx.x] = invd[threadIdx.x];
  if (threadIdx.x == 0)
    *cyc = tot / reps;
  (void)xp;
}

int main() {
  double *out;
  long long *cyc, hc;
  cudaMalloc(&out, sizeof(double) * 148 * 1024);
  cudaMalloc(&cyc, 8);
  const int it = 4000;
  for (int warps : {1, 2, 4, 8, 12}) {
    k_dfma_tp<8><<<1, warps * 32>>>(out, it, cyc);
    cudaMemcpy(&hc, cyc, 8, cudaMemcpyDeviceToHost);
    printf("independent DFMA, %2d warps on one SM, 8 accumulators each: %.2f cycles per DFMA per warp\n", warps, hc / (8.0 * it));
  }
  std::vector<double> h(64 * 4, 0.0), B(64);
  std::mt19937_64 rng(3);
  std::normal_distribution<double> nd;
  for (auto &v : B) v = nd(rng);
  for (int i = 0; i < 8; i++)
    for (int j = 0; j <= i; j++) {
      double s = (i == j) ? 0.5 : 0.0;
      for (int k = 0; k < 8; k++) s += B[i * 8 + k] * B[j * 8 + k];
      h[i * 8 + j] = s;
      h[j * 8 + i] = s;
    }
  double *d;
  cudaMalloc(&d, sizeof(double) * 64 * 4);
  for (int variant = 0; variant < 2; variant++) {
    cudaMemcpy(d, h.data(), sizeof(double) * 64, cudaMemcpyHostToDevice);
    k_diag8<<<1, 32>>>(d, 200, cyc, variant);
    cudaMemcpy(&hc, cyc, 8, cudaMemcpyDeviceToHost);
    printf("diag8 variant %d (%s): %lld cycles\n", variant, variant ? "fragment layout, floored pivots" : "fragment layout, strict", hc);
  }
  std::vector<double> r(64 * 4);
  cudaMemcpy(r.data(), d, sizeof(double) * 64 * 4, cudaMemcpyDeviceToHost);
  double md = 0, mi = 0;
  for (int i = 0; i < 8; i++)
    for (int j = 0; j <= i; j++)
      md = fmax(md, fabs(r[64 + i * 8 + j] - r[128 + i * 8 + j]));
  for (int i = 0; i < 8; i++)
    mi = fmax(mi, fabs(r[192 + i] - r[200 + i]));
  printf("max |L0 - L1| = %.3e, max |inv0 - inv1| = %.3e (L[7][7] = %.6f)\n", md, mi, r[64 + 63]);
  cudaError_t e = cudaDeviceSynchronize();
  printf("%s\n", cudaGetErrorString(e));
  return 0;
}
