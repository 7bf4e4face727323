// Micro-benchmark: single-CTA blocked Cholesky variants (cycles by clock64), n = 154 (EKF) and n = 81 (chi2 gate).
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -I open_vins_b200/csrc -o tools/ubench/chol_bench tools/ubench/chol_bench.cu
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cmath>
#include <cuda_runtime.h>
#include "chol.cuh"
#include "chol_old.cuh"

template <int THREADS, int VAR>
__global__ void __launch_bounds__(THREADS) k_bench(const double *Sin, int n, long long *cyc, double *chk) {
  extern __shared__ __align__(16) double W[];
  __shared__ int flag;
  __shared__ double invd[16];
  const int ld = n | 1;
  for (int e = threadIdx.x; e < (n + 1) * n; e += THREADS) {
    int i = e / n, j = e % n;
    W[i * ld + j] = Sin[i * n + j];
  }
  if (threadIdx.x == 0)
    flag = 0;
  __syncthreads();
  long long t0 = clock64();
  if (VAR == 0)
    chol_lower_block_old<THREADS>(W, ld, n, 1, &flag, invd);
  else if (VAR == 1)
    chol_lower_block<THREADS, 1>(W, ld, n, 1, &flag, invd);
  else if (VAR == 2)
    chol_lower_block<THREADS, 2>(W, ld, n, 1, &flag, invd);
  else if (VAR == 3)
    chol_lower_block<THREADS, 4>(W, ld, n, 1, &flag, invd);
  __syncthreads();
  long long t1 = clock64();
  if (threadIdx.x == 0) {
    *cyc = t1 - t0;
    double s = 0;
    for (int i = 0; i <= n; i++)
      for (int j = 0; j <= (i < n ? i : n - 1); j++)
        s += W[i * ld + j] * (1 + 0.001 * ((i * 7 + j * 3) % 11));
    *chk = s + flag * 1e9;
  }
}

template <int THREADS, int VAR>
void run(const double *dS, int n, const char *name) {
  long long *dc;
  double *dk;
  cudaMalloc(&dc, 8);
  cudaMalloc(&dk, 8);
  size_t smem = sizeof(double) * (size_t)(n + 1) * (n | 1);
  cudaFuncSetAttribute(k_bench<THREADS, VAR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  long long best = 1LL << 60, c;
  double k = 0;
  for (int it = 0; it < 5; it++) {
    k_bench<THREADS, VAR><<<1, THREADS, smem>>>(dS, n, dc, dk);
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
      printf("%s: %s\n", name, cudaGetErrorString(e));
      return;
    }
    cudaMemcpy(&c, dc, 8, cudaMemcpyDeviceToHost);
    cudaMemcpy(&k, dk, 8, cudaMemcpyDeviceToHost);
    if (c < best)
      best = c;
  }
  printf("n=%3d threads=%4d %-28s cycles=%8lld  chk=%.12e\n", n, THREADS, name, best, k);
  cudaFree(dc);
  cudaFree(dk);
}

int main() {
  for (int n : {154, 81}) {
    std::vector<double> A((size_t)n * n), S((size_t)(n + 1) * n);
    srand(1);
    for (auto &v : A)
      v = rand() / (double)RAND_MAX - 0.5;
    for (int i = 0; i < n; i++)
      for (int j = 0; j < n; j++) {
        double s = (i == j) ? 0.5 : 0.0;
        for (int k = 0; k < n; k++)
          s += A[(size_t)i * n + k] * A[(size_t)j * n + k];
        S[(size_t)i * n + j] = s;
      }
    for (int j = 0; j < n; j++)
      S[(size_t)n * n + j] = rand() / (double)RAND_MAX;
    double *dS;
    cudaMalloc(&dS, sizeof(double) * S.size());
    cudaMemcpy(dS, S.data(), sizeof(double) * S.size(), cudaMemcpyHostToDevice);
    if (n == 154) {
      run<1024, 0>(dS, n, "r01 first version");
      run<1024, 1>(dS, n, "rb1");
      run<1024, 2>(dS, n, "rb2");
      run<512, 2>(dS, n, "rb2");
      run<512, 3>(dS, n, "rb4");
      run<256, 3>(dS, n, "rb4");
    } else {
      run<256, 0>(dS, n, "r01 first version");
      run<256, 1>(dS, n, "rb1");
      run<256, 2>(dS, n, "rb2");
      run<256, 3>(dS, n, "rb4");
    }
    cudaFree(dS);
  }
  return 0;
}
