// fp64_rate.cu — microbenchmark of the FP64 paths of the current GPU: DFMA, and the FP64 tensor-core mma.sync shapes
// m8n8k4 (SASS DMMA.8x8x4) and sm_90's m16n8k4 / m16n8k8 / m16n8k16 (DMMA.16x8x4 / .16x8x8 / .16x8x16).
//   * throughput per SM at 1-16 warps per SM (one CTA per SM, 8 independent accumulators per warp)
//   * dependent-issue latency of each shape (one warp, one accumulator chain)
//   * bit identity on random inputs, with and without cancellation: one m16n8k4 against its two m8n8k4 halves, one
//     m16n8k8 against two chained m16n8k4 (k 0-3, then 4-7), one m16n8k16 against four chained m16n8k4; and the tensor
//     core against scalar DFMA: m8n8k4 and m16n8k4 against four chained fma.rn.f64 in ascending k starting from C, four
//     chained m16n8k4 against sixteen
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp64_rate fp64_rate.cu
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>
#include <cuda_runtime.h>

// Fragments (g = lane >> 2, q = lane & 3): A row-major, B column-major, C/D row-major.
//   m8n8k4    a = A[g][q]                     b = B[q][g]            c = {C[g][2q], C[g][2q+1]}
//   m16n8kK   a[i] = A[g + 8*(i&1)][q + 4*(i>>1)]   b[j] = B[q + 4j][g]   c = {C[g][2q], C[g][2q+1], C[g+8][2q], C[g+8][2q+1]}
__device__ __forceinline__ void mma884(double *c, const double *a, const double *b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c[0]), "+d"(c[1]) : "d"(a[0]), "d"(b[0]));
}
__device__ __forceinline__ void mma1684(double *c, const double *a, const double *b) {
  asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
               : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(b[0]));
}
__device__ __forceinline__ void mma1688(double *c, const double *a, const double *b) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
}
__device__ __forceinline__ void mma16816(double *c, const double *a, const double *b) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, "
               "{%0,%1,%2,%3};"
               : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
               : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
                 "d"(b[2]), "d"(b[3]));
}

// Shape S: M x 8 x K per instruction; NC accumulator doubles, NA / NB operand doubles per lane.
struct S884 { static constexpr int M = 8, K = 4, NC = 2, NA = 1, NB = 1; static __device__ void mma(double *c, const double *a, const double *b) { mma884(c, a, b); } };
struct S1684 { static constexpr int M = 16, K = 4, NC = 4, NA = 2, NB = 1; static __device__ void mma(double *c, const double *a, const double *b) { mma1684(c, a, b); } };
struct S1688 { static constexpr int M = 16, K = 8, NC = 4, NA = 4, NB = 2; static __device__ void mma(double *c, const double *a, const double *b) { mma1688(c, a, b); } };
struct S16816 { static constexpr int M = 16, K = 16, NC = 4, NA = 8, NB = 4; static __device__ void mma(double *c, const double *a, const double *b) { mma16816(c, a, b); } };

__global__ void k_dfma(double *out, int iters) {
  double a[8];
  for (int i = 0; i < 8; i++) a[i] = threadIdx.x * 1e-3 + i;
  double b = 1.0000001, c = 1e-9;
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < 8; i++) a[i] = a[i] * b + c;
  }
  double s = 0; for (int i = 0; i < 8; i++) s += a[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// NACC independent accumulators per warp; block 0 reports the cycles of its timed loop
template <class S, int NACC> __global__ void __launch_bounds__(512) k_mma_tp(double *out, int iters, long long *cyc) {
  double c[NACC][S::NC], a[S::NA], b[S::NB];
  for (int i = 0; i < NACC; i++)
    for (int j = 0; j < S::NC; j++) c[i][j] = 0;
  for (int j = 0; j < S::NA; j++) a[j] = threadIdx.x * 1e-3 + j;
  for (int j = 0; j < S::NB; j++) b[j] = 1.0 + threadIdx.x * 1e-6 + j * 1e-3;
  __syncthreads();
  long long t0 = clock64();
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < NACC; i++) S::mma(c[i], a, b);
  }
  __syncthreads();
  long long t1 = clock64();
  double s = 0;
  for (int i = 0; i < NACC; i++)
    for (int j = 0; j < S::NC; j++) s += c[i][j];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}

// one warp, one dependent chain
template <class S> __global__ void k_mma_chain(double *out, int iters, long long *cyc) {
  double c[S::NC], a[S::NA], b[S::NB];
  for (int j = 0; j < S::NC; j++) c[j] = 0;
  for (int j = 0; j < S::NA; j++) a[j] = threadIdx.x * 1e-3 + j;
  for (int j = 0; j < S::NB; j++) b[j] = 1.0 + threadIdx.x * 1e-6 + j * 1e-3;
  long long t0 = clock64();
  for (int it = 0; it < iters; it++) {
    S::mma(c, a, b); S::mma(c, a, b); S::mma(c, a, b); S::mma(c, a, b);
  }
  long long t1 = clock64();
  double s = 0;
  for (int j = 0; j < S::NC; j++) s += c[j];
  out[threadIdx.x] = s;
  if (threadIdx.x == 0) *cyc = t1 - t0;
}

// Bit identity. Each warp w takes A[16 x 16], B[16 x 8] (B[k][n] at B[k*8+n]) and C[16 x 8] from the inputs and writes
// D = C + A B four ways into out[w][way][16*8]:
//   way 0  k 0-3 : two m8n8k4 (rows 0-7, rows 8-15)          way 1  k 0-3 : one m16n8k4
//   way 2  k 0-7 : two chained m16n8k4                       way 3  k 0-7 : one m16n8k8
//   way 4  k 0-15: four chained m16n8k4                      way 5  k 0-15: one m16n8k16
//   way 6  k 0-3 : d = fma(a3, b3, fma(a2, b2, fma(a1, b1, fma(a0, b0, c))))      way 7  k 0-15: the same chain, 16 long
#define NWAYS 8
__global__ void k_bits(const double *A, const double *B, const double *C, double *out) {
  const int w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const double *Aw = A + (size_t)w * 256, *Bw = B + (size_t)w * 128, *Cw = C + (size_t)w * 128;
  double *ow = out + (size_t)w * NWAYS * 128;
  auto ldc = [&](double *c) { c[0] = Cw[g * 8 + 2 * q]; c[1] = Cw[g * 8 + 2 * q + 1]; c[2] = Cw[(g + 8) * 8 + 2 * q]; c[3] = Cw[(g + 8) * 8 + 2 * q + 1]; };
  auto stc = [&](int way, const double *c) {
    double *o = ow + way * 128;
    o[g * 8 + 2 * q] = c[0]; o[g * 8 + 2 * q + 1] = c[1]; o[(g + 8) * 8 + 2 * q] = c[2]; o[(g + 8) * 8 + 2 * q + 1] = c[3];
  };
  auto lda = [&](int i, int kb) { return Aw[(g + 8 * (i & 1)) * 16 + kb + q + 4 * (i >> 1)]; };
  auto ldb = [&](int j, int kb) { return Bw[(kb + q + 4 * j) * 8 + g]; };
  double c[4], a[8], b[4];
  { // way 0
    ldc(c);
    double a0 = lda(0, 0), a1 = lda(1, 0), b0 = ldb(0, 0);
    mma884(c, &a0, &b0);
    mma884(c + 2, &a1, &b0);
    stc(0, c);
  }
  { ldc(c); a[0] = lda(0, 0); a[1] = lda(1, 0); b[0] = ldb(0, 0); mma1684(c, a, b); stc(1, c); }
  {
    ldc(c);
    for (int kb = 0; kb < 8; kb += 4) { a[0] = lda(0, kb); a[1] = lda(1, kb); b[0] = ldb(0, kb); mma1684(c, a, b); }
    stc(2, c);
  }
  { ldc(c); for (int i = 0; i < 4; i++) a[i] = lda(i, 0); for (int j = 0; j < 2; j++) b[j] = ldb(j, 0); mma1688(c, a, b); stc(3, c); }
  {
    ldc(c);
    for (int kb = 0; kb < 16; kb += 4) { a[0] = lda(0, kb); a[1] = lda(1, kb); b[0] = ldb(0, kb); mma1684(c, a, b); }
    stc(4, c);
  }
  { ldc(c); for (int i = 0; i < 8; i++) a[i] = lda(i, 0); for (int j = 0; j < 4; j++) b[j] = ldb(j, 0); mma16816(c, a, b); stc(5, c); }
  for (int way = 6; way < 8; way++) { // this lane's four outputs C[g + 8h][2q + e], h = u >> 1, e = u & 1
    const int kmax = way == 6 ? 4 : 16;
    ldc(c);
    for (int u = 0; u < 4; u++) {
      const int r = g + 8 * (u >> 1), n = 2 * q + (u & 1);
      for (int k = 0; k < kmax; k++)
        c[u] = __fma_rn(Aw[r * 16 + k], Bw[k * 8 + n], c[u]);
    }
    stc(way, c);
  }
}

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); return 1; } } while (0)

template <class S> int run_shape(const char *name, int sms, double ghz, double *out, long long *cyc, cudaEvent_t e0, cudaEvent_t e1) {
  const int it = 4000, NACC = 8;
  long long hc;
  k_mma_chain<S><<<1, 32>>>(out, 100, cyc);
  k_mma_chain<S><<<1, 32>>>(out, it, cyc);
  CK(cudaGetLastError());
  CK(cudaMemcpy(&hc, cyc, 8, cudaMemcpyDeviceToHost));
  printf("%-8s dependent-issue latency: %.1f cycles\n", name, hc / (4.0 * it));
  const double flop = 2.0 * S::M * 8 * S::K;
  for (int warps : {1, 2, 4, 8, 16}) {
    float ms;
    k_mma_tp<S, NACC><<<sms, warps * 32>>>(out, 100, cyc);
    CK(cudaDeviceSynchronize());
    CK(cudaEventRecord(e0));
    k_mma_tp<S, NACC><<<sms, warps * 32>>>(out, it, cyc);
    CK(cudaGetLastError());
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    CK(cudaEventElapsedTime(&ms, e0, e1));
    CK(cudaMemcpy(&hc, cyc, 8, cudaMemcpyDeviceToHost));
    const double n = (double)NACC * it * warps; // instructions per SM
    printf("%-8s warps/SM=%2d : %6.2f cycles/instr/SM  %6.1f FLOP/clk/SM  %6.2f TFLOP/s (events)\n", name, warps, hc / n, flop * n / hc,
           flop * n * sms / (ms * 1e-3) / 1e12);
  }
  (void)ghz;
  return 0;
}

int main() {
  cudaDeviceProp p;
  CK(cudaGetDeviceProperties(&p, 0));
  const int sms = p.multiProcessorCount;
  int clk_khz = 0;
  cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
  const double ghz = clk_khz * 1e-6;
  printf("device %s, %d SMs, %.2f GHz max SM clock\n", p.name, sms, ghz);
  double *out;
  long long *cyc;
  CK(cudaMalloc(&out, sizeof(double) * sms * 8 * 1024));
  CK(cudaMalloc(&cyc, 8));
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  for (int warps = 2; warps <= 32; warps *= 2) {
    int threads = warps * 32, iters = 20000; float ms;
    k_dfma<<<sms, threads>>>(out, 100); CK(cudaDeviceSynchronize());
    CK(cudaEventRecord(e0)); k_dfma<<<sms, threads>>>(out, iters); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
    CK(cudaEventElapsedTime(&ms, e0, e1));
    double fma = (double)sms * threads * iters * 8;
    printf("DFMA     warps/SM=%2d : %.2f TFLOP/s  (%.1f FMA/clk/SM at %.2f GHz)\n", warps, 2 * fma / ms / 1e9, fma / (ms * 1e-3) / (ghz * 1e9) / sms, ghz);
  }
  if (run_shape<S884>("m8n8k4", sms, ghz, out, cyc, e0, e1) || run_shape<S1684>("m16n8k4", sms, ghz, out, cyc, e0, e1) ||
      run_shape<S1688>("m16n8k8", sms, ghz, out, cyc, e0, e1) || run_shape<S16816>("m16n8k16", sms, ghz, out, cyc, e0, e1))
    return 1;

  // ---- bit identity: 3 input families x NW warps each
  const int NW = 8192;
  std::vector<double> hA((size_t)NW * 256), hB((size_t)NW * 128), hC((size_t)NW * 128), hD((size_t)NW * NWAYS * 128);
  double *dA, *dB, *dC, *dD;
  CK(cudaMalloc(&dA, hA.size() * 8)); CK(cudaMalloc(&dB, hB.size() * 8)); CK(cudaMalloc(&dC, hC.size() * 8)); CK(cudaMalloc(&dD, hD.size() * 8));
  std::mt19937_64 rng(20261018);
  std::uniform_real_distribution<double> U(-1.0, 1.0);
  std::uniform_int_distribution<int> E(-30, 30);
  const char *fam[3] = {"uniform [-1,1]", "wide exponents 2^+-30", "cancellation"};
  long total_bad = 0, total_dfma_bad = 0;
  for (int f = 0; f < 3; f++) {
    for (int w = 0; w < NW; w++) {
      double *A = &hA[(size_t)w * 256], *B = &hB[(size_t)w * 128], *C = &hC[(size_t)w * 128];
      for (int i = 0; i < 256; i++) A[i] = f == 0 ? U(rng) : std::ldexp(U(rng), E(rng));
      for (int i = 0; i < 128; i++) B[i] = f == 0 ? U(rng) : std::ldexp(U(rng), E(rng));
      for (int i = 0; i < 128; i++) C[i] = f == 0 ? U(rng) : std::ldexp(U(rng), E(rng));
      if (f == 2) {
        // products that cancel in pairs up to a small perturbation, and C that cancels the sum of the rest
        for (int r = 0; r < 16; r++)
          for (int k = 1; k < 16; k += 2) A[r * 16 + k] = -A[r * 16 + k - 1] * (1.0 + std::ldexp(U(rng), -40));
        for (int k = 1; k < 16; k += 2)
          for (int n = 0; n < 8; n++) B[k * 8 + n] = B[(k - 1) * 8 + n];
        for (int r = 0; r < 16; r++)
          for (int n = 0; n < 8; n++) {
            double s = 0;
            for (int k = 0; k < 4; k++) s += A[r * 16 + k] * B[k * 8 + n];
            C[r * 8 + n] = -s * (1.0 + std::ldexp(U(rng), -45));
          }
      }
    }
    CK(cudaMemcpy(dA, hA.data(), hA.size() * 8, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dB, hB.data(), hB.size() * 8, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dC, hC.data(), hC.size() * 8, cudaMemcpyHostToDevice));
    k_bits<<<NW / 4, 128>>>(dA, dB, dC, dD);
    CK(cudaGetLastError());
    CK(cudaMemcpy(hD.data(), dD, hD.size() * 8, cudaMemcpyDeviceToHost));
    // pairs of ways that must agree; the last three compare the tensor core with the scalar FMA chain, element by element
    const int pairs[6][2] = {{0, 1}, {2, 3}, {4, 5}, {0, 6}, {1, 6}, {4, 7}};
    long bad[6] = {0, 0, 0, 0, 0, 0};
    for (int w = 0; w < NW; w++) {
      const double *o = &hD[(size_t)w * NWAYS * 128];
      for (int pr = 0; pr < 3; pr++)
        if (memcmp(o + pairs[pr][0] * 128, o + pairs[pr][1] * 128, 128 * 8) != 0) bad[pr]++;
      for (int pr = 3; pr < 6; pr++)
        for (int e = 0; e < 128; e++)
          if (memcmp(o + pairs[pr][0] * 128 + e, o + pairs[pr][1] * 128 + e, 8) != 0) bad[pr]++;
    }
    printf("bits [%s], %d warps: m16n8k4 != 2x m8n8k4: %ld   m16n8k8 != 2x m16n8k4: %ld   m16n8k16 != 4x m16n8k4: %ld\n", fam[f], NW,
           bad[0], bad[1], bad[2]);
    printf("bits [%s], %d outputs: m8n8k4 != 4 chained DFMA: %ld   m16n8k4 != 4 chained DFMA: %ld   4x m16n8k4 != 16 chained DFMA: %ld\n",
           fam[f], NW * 128, bad[3], bad[4], bad[5]);
    total_bad += bad[0] + bad[1] + bad[2];
    total_dfma_bad += bad[3] + bad[4] + bad[5];
  }
  printf("bit identity: %s\n", total_bad ? "DIFFERS" : "all identical");
  printf("DMMA against chained DFMA: %s\n", total_dfma_bad ? "DIFFERS" : "all identical");
  return 0;
}
