// cholqr_bench.cu — stand-alone timing of the CholeskyQR2 kernels (csrc/k_cholqr.cu) and of the DMMA latency/throughput
// they are built on. Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 [-DCQ_PROBE] -o cholqr_bench cholqr_bench.cu
#include "../../open_vins_b200/csrc/k_cholqr.cu"
#include <cstdio>
#include <cstring>
#include <vector>
#include <random>

__global__ void k_dmma_chain(double *out, int iters, long long *cyc) {
  double c0 = 0, c1 = 0;
  double a = threadIdx.x * 1e-3, b = 1.0 + threadIdx.x * 1e-6;
  long long t0 = clock64();
  for (int it = 0; it < iters; it++) {
    dmma(c0, c1, a, b);
    dmma(c0, c1, a, b);
    dmma(c0, c1, a, b);
    dmma(c0, c1, a, b);
  }
  long long t1 = clock64();
  out[threadIdx.x] = c0 + c1;
  if (threadIdx.x == 0)
    *cyc = t1 - t0;
}
template <int NACC> __global__ void k_dmma_tp(double *out, int iters, long long *cyc) {
  double c[NACC][2];
  for (int i = 0; i < NACC; i++)
    c[i][0] = c[i][1] = 0;
  double a = threadIdx.x * 1e-3, b = 1.0 + threadIdx.x * 1e-6;
  __syncthreads();
  long long t0 = clock64();
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < NACC; i++)
      dmma(c[i][0], c[i][1], a, b);
  }
  __syncthreads();
  long long t1 = clock64();
  double s = 0;
  for (int i = 0; i < NACC; i++)
    s += c[i][0] + c[i][1];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0 && blockIdx.x == 0)
    *cyc = t1 - t0;
}
__global__ void k_dfma_chain(double *out, int iters, long long *cyc) {
  double x = threadIdx.x * 1e-3, b = 1.0000001, c = 1e-9;
  long long t0 = clock64();
  for (int it = 0; it < iters; it++) {
    x = x * b + c; x = x * b + c; x = x * b + c; x = x * b + c;
  }
  long long t1 = clock64();
  out[threadIdx.x] = x;
  if (threadIdx.x == 0) *cyc = t1 - t0;
}
__global__ void k_rsqrt_chain(double *out, int iters, long long *cyc) {
  double x = 2.0 + threadIdx.x * 1e-3;
  long long t0 = clock64();
  for (int it = 0; it < iters; it++) {
    x = fast_rsqrt(x) + 1.5; x = fast_rsqrt(x) + 1.5; x = fast_rsqrt(x) + 1.5; x = fast_rsqrt(x) + 1.5;
  }
  long long t1 = clock64();
  out[threadIdx.x] = x;
  if (threadIdx.x == 0) *cyc = t1 - t0;
}
__global__ void k_shfl_chain(double *out, int iters, long long *cyc) {
  double x = 2.0 + threadIdx.x * 1e-3;
  long long t0 = clock64();
  for (int it = 0; it < iters; it++) {
    x = __shfl_sync(0xffffffffu, x, (threadIdx.x + 1) & 31); x = __shfl_sync(0xffffffffu, x, (threadIdx.x + 1) & 31);
    x = __shfl_sync(0xffffffffu, x, (threadIdx.x + 1) & 31); x = __shfl_sync(0xffffffffu, x, (threadIdx.x + 1) & 31);
  }
  long long t1 = clock64();
  out[threadIdx.x] = x;
  if (threadIdx.x == 0) *cyc = t1 - t0;
}

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); return 1; } } while (0)

int main() {
  cudaDeviceProp p;
  cudaGetDeviceProperties(&p, 0);
  const int sms = p.multiProcessorCount;
  double *out;
  long long *cyc, hc;
  CK(cudaMalloc(&out, sizeof(double) * sms * 1024));
  CK(cudaMalloc(&cyc, 8));
  const int it = 2000;
  k_dmma_chain<<<1, 32>>>(out, it, cyc); cudaMemcpy(&hc, cyc, 8, cudaMemcpyDeviceToHost); printf("DMMA dependent latency: %.1f cycles\n", hc / (4.0 * it));
  k_dfma_chain<<<1, 32>>>(out, it, cyc); cudaMemcpy(&hc, cyc, 8, cudaMemcpyDeviceToHost); printf("DFMA dependent latency: %.1f cycles\n", hc / (4.0 * it));
  k_rsqrt_chain<<<1, 32>>>(out, it, cyc); cudaMemcpy(&hc, cyc, 8, cudaMemcpyDeviceToHost); printf("fast_rsqrt+add chain: %.1f cycles\n", hc / (4.0 * it));
  k_shfl_chain<<<1, 32>>>(out, it, cyc); cudaMemcpy(&hc, cyc, 8, cudaMemcpyDeviceToHost); printf("shfl f64 chain: %.1f cycles\n", hc / (4.0 * it));
  for (int warps : {1, 2, 4, 8, 16}) {
    k_dmma_tp<8><<<sms, warps * 32>>>(out, it, cyc); cudaMemcpy(&hc, cyc, 8, cudaMemcpyDeviceToHost);
    printf("DMMA throughput, %2d warps/SM x 8 independent accumulators: %.2f cycles per DMMA per SM (%.1f FMA/clk/SM)\n", warps, hc / (8.0 * it * warps),
           256.0 * 8 * it * warps / hc);
  }
  // ---- kernels on the config-2 shape (12 008 stacked rows, 155 columns with the residual)
  const int m = 12008, n = 154, nt = n + 1, ld = 156;
  std::vector<double> hA((size_t)m * ld);
  std::mt19937_64 rng(1);
  std::normal_distribution<double> nd;
  for (auto &v : hA) v = nd(rng);
  double *A, *A0, *Gpart, *Gpart2, *G, *R1, *R2, *Rout;
  const int ldW = CQ_MAXN + 8;
  const size_t part_doubles = (size_t)sms * 16 * 1024;
  CK(cudaMalloc(&A, sizeof(double) * hA.size()));
  CK(cudaMalloc(&A0, sizeof(double) * hA.size()));
  CK(cudaMemcpy(A0, hA.data(), sizeof(double) * hA.size(), cudaMemcpyHostToDevice));
  CK(cudaMalloc(&Gpart, sizeof(double) * part_doubles));
  CK(cudaMalloc(&Gpart2, sizeof(double) * part_doubles));
  CK(cudaMalloc(&G, sizeof(double) * ldW * ldW * 4));
  R1 = G + ldW * ldW; R2 = R1 + ldW * ldW; Rout = R2 + ldW * ldW;
  double *Rpk; CK(cudaMalloc(&Rpk, sizeof(double) * CQ_PK_DOUBLES));
  const int nT = (nt + 31) / 32, BW = nT;
  int nslab = sms, slab_rows = (((m + nslab - 1) / nslab) + 3) & ~3;
  nslab = (m + slab_rows - 1) / slab_rows;
  const size_t gram_smem = sizeof(double) * 2 * CQ_KB * (size_t)(BW * 32 + 4);
  const size_t trsm_smem = CQ_TRSM_SMEM;
  CK(cudaFuncSetAttribute(k_cq_gram, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
  CK(cudaFuncSetAttribute(k_cq_chol_gram, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CqCholSmem)));
  CK(cudaFuncSetAttribute(k_cq_trsm<10, 10>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CQ_TRSM_SMEM));
  ovb_ctx ctx{}; // default stream, no PDL, no profiling: only what the solve + Gram launcher reads
  ctx.sm_count = sms;
  cq_attrs(&ctx);
  double *Qtail;
  CK(cudaMalloc(&Qtail, sizeof(double) * (cq_solve_gram_scratch(nslab, nt, BW, slab_rows) + 1)));
  std::vector<double> p1(part_doubles), p2(part_doubles);
  cudaEvent_t e[10];
  for (auto &x : e) cudaEventCreate(&x);
  for (int rep = 0; rep < 4; rep++) {
    CK(cudaMemcpy(A, A0, sizeof(double) * hA.size(), cudaMemcpyDeviceToDevice));
    cudaDeviceSynchronize();
    cudaEventRecord(e[0]);
    k_cq_gram<<<dim3(1, nslab), CQ_GRAM_T, gram_smem>>>(A, ld, m, nt, slab_rows, BW, 1, Gpart, 1);
    cudaEventRecord(e[1]);
    k_cq_reduce<<<dim3(CQ_RED_GX, 1), CQ_RED_T>>>(Gpart, nslab, 1, BW, 1, nt, G, ldW, 1);
    cudaEventRecord(e[2]);
    k_cq_chol_gram<<<1, CQ_CHOL_T, sizeof(CqCholSmem)>>>(G, ldW, nt, 1e-11, Rpk, 1);
    cudaEventRecord(e[3]);
    // pass 2 fused (A untouched) ...
    cq_launch_solve_gram(&ctx, nslab, A, ld, m, nt, Rpk, slab_rows, BW, Gpart2, Qtail);
    cudaEventRecord(e[4]);
    // ... and unfused: Q1 written over A, then its Gram
    k_cq_trsm<10, 10><<<sms, CQ_TRSM_T, trsm_smem>>>(A, ld, m, nt, Rpk);
    cudaEventRecord(e[5]);
    k_cq_gram<<<dim3(1, nslab), CQ_GRAM_T, gram_smem>>>(A, ld, m, nt, slab_rows, BW, 1, Gpart, 1);
    cudaEventRecord(e[6]);
    k_cq_trmm<<<dim3((nt + 15) / 16, (nt + 15) / 16), 256>>>(Rpk, Rpk, nt, Rout, ld);
    cudaEventRecord(e[7]);
    k_cq_trsm<10, 10><<<7, CQ_TRSM_T, trsm_smem>>>(A, ld, 194, nt, Rpk);
    cudaEventRecord(e[8]);
    k_cq_trsm<10, 10><<<1, CQ_TRSM_T, trsm_smem>>>(A, ld, 8, nt, Rpk);
    cudaEventRecord(e[9]);
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(p1.data(), Gpart, sizeof(double) * part_doubles, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(p2.data(), Gpart2, sizeof(double) * part_doubles, cudaMemcpyDeviceToHost));
    size_t ndiff = 0; // the tile warps' partials (BW(BW+1)/2 of 16 per slab) of both pass-2 routes
    for (int s = 0; s < nslab; s++)
      for (int w = 0; w < BW * (BW + 1) / 2; w++)
        for (int i = 0; i < 1024; i++) {
          const size_t k = ((size_t)s * 16 + w) * 1024 + i;
          ndiff += memcmp(&p1[k], &p2[k], sizeof(double)) != 0;
        }
    float t[9];
    for (int i = 0; i < 9; i++) cudaEventElapsedTime(&t[i], e[i], e[i + 1]);
    printf("rep %d: gram %.1f us  reduce %.1f us  chol %.1f us  solve+gram %.1f us (trsm %.1f + gram %.1f unfused; partials differing in %zu doubles)  trmm %.1f us  "
           "trsm(194 rows) %.1f us  trsm(8 rows) %.1f us\n",
           rep, 1e3 * t[0], 1e3 * t[1], 1e3 * t[2], 1e3 * t[3], 1e3 * t[4], 1e3 * t[5], ndiff, 1e3 * t[6], 1e3 * t[7], 1e3 * t[8]);
  }
  return 0;
}
