// k_ekf.cu — dense covariance algebra on the device-resident P.
// Replaces StateHelper::EKFUpdate (ov_msckf/src/state/StateHelper.cpp:116-197), StateHelper::EKFPropagation (:36-114),
// StateHelper::clone / augment_clone's time-offset term (:341-391, :604-615), StateHelper::marginalize (:271-339) and
// get_marginal_covariance (:226-254).
//
// EKFUpdate on the device:   M = P[:,cols] H'   S = H M[cols,:] + R   S = L L'   Y = M L^-T   w = L^-1 res
//                            P <- sym_U(P - Y Y')      dx = Y w
// (K M' = M S^-1 M' = Y Y' and K res = Y w, so neither S^-1 nor K is formed; the reference forms both.)
// P is row-major with a fixed leading dimension so clone() grows it in place.
#include "chol_tiles.cuh"
#include "ovb_internal.cuh"

#define EK_T 32

// C[x][y] = sum_j Aop(x,j) * Bop(j,y), 32x32 tile per CTA, 256 threads (4 outputs each), K tiles of 32.
//  mode 0 (M = P[:,cols] H'):  Aop(a,j) = P[cs[j]*ldP + a]      Bop(j,i) = H[i*ldH + j]      C = M [N x r]
//  mode 1 (S = H M[cols,:]+R): Aop(i,j) = H[i*ldH + j]          Bop(j,k) = M[cs[j]*ldM + k]  C = S [r x r], lower tiles only
__global__ void __launch_bounds__(256) k_ekf_gemm(int mode, const double *__restrict__ P, int ldP, const double *__restrict__ H, int ldH,
                                                  const double *__restrict__ Min, int ldM, const DevUpdateInfo *__restrict__ info, int X, int Y,
                                                  int K, double *__restrict__ Cout, int ldC, double sigma2, const double *__restrict__ Rdiag) {
  OVB_PDL_ENTER();
  __shared__ double As[EK_T][EK_T + 1]; // [j][x]
  __shared__ double Bs[EK_T][EK_T + 1]; // [j][y]
  const int x0 = blockIdx.x * EK_T, y0 = blockIdx.y * EK_T;
  if (mode == 1 && y0 > x0 + EK_T - 1)
    return; // strictly upper tile of S
  const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5; // ty 0..7
  double acc[4] = {0, 0, 0, 0};
  const int *cs = info->col_state;
  for (int j0 = 0; j0 < K; j0 += EK_T) {
    // load tiles
    for (int e = tid; e < EK_T * EK_T; e += 256) {
      int jj = e >> 5, q = e & 31; // jj = k index in tile, q = x or y
      int j = j0 + jj;
      double av = 0.0, bv = 0.0;
      if (j < K) {
        if (mode == 0) {
          int a = x0 + q;
          if (a < X)
            av = P[(size_t)cs[j] * ldP + a];
        } else {
          // Aop(i,j) = H[i][j]: transpose load (lanes over q=i → strided); small matrices, acceptable
          int i = x0 + q;
          if (i < X)
            av = H[(size_t)i * ldH + j];
        }
        if (mode == 0) {
          int i = y0 + q;
          if (i < Y)
            bv = H[(size_t)i * ldH + j];
        } else {
          int k = y0 + q;
          if (k < Y)
            bv = Min[(size_t)cs[j] * ldM + k];
        }
      }
      As[jj][q] = av;
      Bs[jj][q] = bv;
    }
    __syncthreads();
#pragma unroll 8
    for (int jj = 0; jj < EK_T; jj++) {
      double b = Bs[jj][tx];
#pragma unroll
      for (int u = 0; u < 4; u++)
        acc[u] += As[jj][ty + 8 * u] * b;
    }
    __syncthreads();
  }
#pragma unroll
  for (int u = 0; u < 4; u++) {
    int x = x0 + ty + 8 * u, y = y0 + tx;
    if (x < X && y < Y) {
      double v = acc[u];
      if (mode == 1 && x == y)
        v += Rdiag ? Rdiag[x] : sigma2;
      Cout[(size_t)x * ldC + y] = v;
    }
  }
}

// single CTA: S (r x r, lower) plus the residual as row r  ->  L and w = L^-1 res in row r. Works in shared memory when
// it fits, else in place in global memory (L2).
__global__ void __launch_bounds__(EKC_THREADS) k_ekf_chol(double *__restrict__ S, int ldS, int r, const double *__restrict__ res, double *__restrict__ w,
                                                   double *__restrict__ invdiag, DevUpdateInfo *__restrict__ info, int use_smem) {
  OVB_PDL_ENTER();
  extern __shared__ __align__(16) double chol_sm[];
  __shared__ int flag;
  __shared__ double invd_sh[16];
  const int tid = threadIdx.x;
  if (tid == 0)
    flag = 0;
  for (int j = tid; j < r; j += EKC_THREADS)
    S[(size_t)r * ldS + j] = res[j];
  __syncthreads();
  double *W = S;
  int ld = ldS;
  const int lane = tid & 31, wid = tid >> 5;
  if (use_smem) {
    ld = r | 1;
    W = chol_sm;
    stage_lower_async<EKC_THREADS>(W, ld, S, (size_t)ldS, r + 1, r);
  }
  chol_lower_block<EKC_THREADS, 4>(W, ld, r, 1, &flag, invd_sh, nullptr, 0.0, invdiag);
  __syncthreads();
  if (use_smem) {
    for (int i = wid; i < r; i += EKC_THREADS / 32) {
      for (int j = lane; j <= i; j += 32)
        S[(size_t)i * ldS + j] = W[i * ld + j];
    }
  }
  for (int j = tid; j < r; j += EKC_THREADS)
    w[j] = W[(size_t)r * ld + j];
  if (tid == 0 && flag)
    info->not_spd = 1;
}

// Y = M L^-T : one WARP per row of M (independent forward substitutions y = L^-1 m), blocked by 8 columns. L is staged
// once per CTA in shared memory (the substitution is a serial chain: an L2 round trip per step would dominate); the eight
// dot products against the solved part run as independent chains, one butterfly reduces them, then every lane solves
// the 8x8 triangle redundantly with the reciprocal pivots written by the Cholesky kernel.
#define TR_ROWS 8 // rows of M (warps) per CTA
__global__ void __launch_bounds__(32 * TR_ROWS) k_ekf_trsm(const double *__restrict__ M, int ldM, const double *__restrict__ L, int ldL,
                                                           const double *__restrict__ invdiag, int N, int r, double *__restrict__ Yout, int ldY,
                                                           int L_in_smem, const DevUpdateInfo *__restrict__ info) {
  OVB_PDL_ENTER();
  extern __shared__ __align__(16) double tsm[]; // [TR_ROWS][r] y rows, then r reciprocal pivots, then L (r x ldl) when it fits
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (info->not_spd)
    return; // failed factor: leave P untouched (the status code is then recoverable, include/ovb200.h)
  const int ldl = r | 1;
  double *inv_s = tsm + (size_t)TR_ROWS * r;
  double *Ls = inv_s + r;
  for (int e = threadIdx.x; e < r; e += 32 * TR_ROWS)
    inv_s[e] = invdiag[e];
  if (L_in_smem)
    stage_lower_async<32 * TR_ROWS>(Ls, ldl, L, (size_t)ldL, r, r);
  else
    __syncthreads();
  const double *Lp = L_in_smem ? Ls : L;
  const int lp = L_in_smem ? ldl : ldL;
  const int a = blockIdx.x * TR_ROWS + wid;
  if (a >= N)
    return;
  double *y = tsm + (size_t)wid * r;
  for (int t = lane; t < r; t += 32)
    y[t] = M[(size_t)a * ldM + t];
  __syncwarp();
  for (int kb = 0; kb < r; kb += 8) {
    const int nbk = min(8, r - kb);
    double s[8];
#pragma unroll
    for (int c = 0; c < 8; c++)
      s[c] = 0.0;
    for (int t = lane; t < kb; t += 32) {
      const double yt = y[t];
#pragma unroll
      for (int c = 0; c < 8; c++)
        if (c < nbk)
          s[c] += Lp[(size_t)(kb + c) * lp + t] * yt;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int c = 0; c < 8; c++)
        s[c] += __shfl_xor_sync(0xffffffffu, s[c], o);
    }
    double yn[8];
#pragma unroll
    for (int c = 0; c < 8; c++) {
      if (c < nbk) {
        const double *Lr = Lp + (size_t)(kb + c) * lp + kb;
        // everything that does not depend on yn[c-1] first: the serial chain is one FMA + one multiply per column
        double v = y[kb + c] - s[c];
#pragma unroll
        for (int t = 0; t < 8; t++)
          if (t + 1 < c)
            v -= Lr[t] * yn[t];
        if (c > 0)
          v -= Lr[c - 1] * yn[c - 1];
        yn[c] = v * inv_s[kb + c];
      }
    }
    __syncwarp();
    if (lane < nbk) {
      double v = yn[0];
#pragma unroll
      for (int c = 1; c < 8; c++)
        v = (lane == c) ? yn[c] : v;
      y[kb + lane] = v;
    }
    __syncwarp();
  }
  for (int t = lane; t < r; t += 32)
    Yout[(size_t)a * ldY + t] = y[t];
}

// P <- sym_U(P - Y Y'): upper tiles only, mirrored on write; negative-diagonal check; dx = Y w on the diagonal tiles' rows
__global__ void __launch_bounds__(256) k_ekf_downdate(double *__restrict__ P, int ldP, const double *__restrict__ Yin, int ldY, int N, int r,
                                                      const double *__restrict__ w, double *__restrict__ dx, DevUpdateInfo *__restrict__ info) {
  OVB_PDL_ENTER();
  __shared__ double As[EK_T][EK_T + 1]; // [k][a]
  __shared__ double Bs[EK_T][EK_T + 1]; // [k][b]
  const int a0 = blockIdx.x * EK_T, b0 = blockIdx.y * EK_T;
  if (b0 < a0)
    return;
  const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
  if (info->not_spd) { // failed factor: P stays as it was, no correction
    if (a0 == b0 && tid < EK_T && a0 + tid < N)
      dx[a0 + tid] = 0.0;
    return;
  }
  double acc[4] = {0, 0, 0, 0};
  double dxa = 0.0; // dx partial for row a0 + tid (diagonal tiles, tid < 32)
  for (int k0 = 0; k0 < r; k0 += EK_T) {
    for (int e = tid; e < EK_T * EK_T; e += 256) {
      int q = e >> 5, kk = e & 31; // lanes over k: coalesced rows of Y
      int k = k0 + kk;
      As[kk][q] = (k < r && a0 + q < N) ? Yin[(size_t)(a0 + q) * ldY + k] : 0.0;
      Bs[kk][q] = (k < r && b0 + q < N) ? Yin[(size_t)(b0 + q) * ldY + k] : 0.0;
    }
    __syncthreads();
#pragma unroll 8
    for (int kk = 0; kk < EK_T; kk++) {
      double b = Bs[kk][tx];
#pragma unroll
      for (int u = 0; u < 4; u++)
        acc[u] += As[kk][ty + 8 * u] * b;
    }
    if (a0 == b0 && tid < EK_T) {
      for (int kk = 0; kk < EK_T; kk++)
        if (k0 + kk < r)
          dxa += As[kk][tid] * w[k0 + kk];
    }
    __syncthreads();
  }
#pragma unroll
  for (int u = 0; u < 4; u++) {
    int a = a0 + ty + 8 * u, b = b0 + tx;
    if (a < N && b < N && b >= a) {
      double v = P[(size_t)a * ldP + b] - acc[u];
      P[(size_t)a * ldP + b] = v;
      P[(size_t)b * ldP + a] = v;
      if (a == b && v < 0.0)
        atomicMin(&info->neg_diag_index, a);
      if (!isfinite(v))
        info->nonfinite = 1;
    }
  }
  if (a0 == b0 && tid < EK_T && a0 + tid < N)
    dx[a0 + tid] = dxa;
}

// ---- one-shot variants for K <= EK1_KMAX (the whole inner dimension staged at once: a CTA pays ONE L2 round trip instead
// of one per 32-wide K tile; at config-2 sizes these products are latency-, not flop-bound). Same contract as k_ekf_gemm.
// Each CTA computes a 16 x 8 output tile on the FP64 tensor cores, m16n8k16 per 16 k (ct_dmma2k16): each output is the
// chain acc = fma(a_k, b_k, acc) over ascending k from zero, the bits of the scalar loops before (the instruction gives the
// chained DFMA's bits, tools/ubench/fp64_rate.cu). K is padded to a multiple of 16 with zeros, which leave a chain that
// starts at +0 unchanged. Small tiles give the grid enough CTAs to cover the SMs (config 2: 260, 110, 169). The DMMA chain
// is one warp's; the CTA's four warps share the issue of the staging copies, which one warp alone spends longer on.
#define EK1_KMAX 160
#define EK1_M 16 // output rows per CTA
#define EK1_N 8  // output columns per CTA
#define EK1_T 128
__device__ __forceinline__ void ek_cpa8(double *dst_smem, const double *src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((unsigned)__cvta_generic_to_shared(dst_smem)), "l"(src) : "memory");
}
__host__ __device__ __forceinline__ int ek1_kpad(int K) { return (K + 15) & ~15; }
// An operand of R rows (A: 16, B: 8) over Kp = ek1_kpad(K) k, staged in one of two layouts, both read without bank conflicts
// by the fragment loads:  row-major  X[x][k] at x (Kp + 4) + k  (source rows contiguous in k; warp w copies rows w, w+4, ..)
//                         k-major    X[x][k] at k (R + 4) + x   (source columns contiguous in x: the rows gathered by cs)
// Outside [0, xmax) x [0, K) the operand is zero.
template <int R> __device__ __forceinline__ void ek1_stage_rows(double *dst, int Kp, const double *src, size_t ld, int x0, int xmax, int K) {
  const int lane = threadIdx.x & 31;
  for (int x = threadIdx.x >> 5; x < R; x += EK1_T / 32)
    for (int k = lane; k < Kp; k += 32) {
      if (x0 + x < xmax && k < K)
        ek_cpa8(&dst[x * (Kp + 4) + k], &src[(size_t)(x0 + x) * ld + k]);
      else
        dst[x * (Kp + 4) + k] = 0.0;
    }
}
template <int R> __device__ __forceinline__ void ek1_stage_cols(double *dst, int Kp, const double *src, size_t ld, const int *cs_s, int x0, int xmax, int K) {
  const int x = threadIdx.x % R;
  for (int k = threadIdx.x / R; k < Kp; k += EK1_T / R) {
    if (x0 + x < xmax && k < K)
      ek_cpa8(&dst[k * (R + 4) + x], &src[(size_t)cs_s[k] * ld + x0 + x]);
    else
      dst[k * (R + 4) + x] = 0.0;
  }
}
__device__ __forceinline__ void ek1_stage_wait() {
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();
}
// c = A B over k < Kp for the warp's 16 x 8 tile; A_KMAJOR / B_KMAJOR: the operands' layouts. Lane (g, q) = (lane>>2,
// lane&3) ends with c[0], c[1] = C[g][2q], C[g][2q+1] and c[2], c[3] = C[g+8][2q], C[g+8][2q+1].
template <bool A_KMAJOR, bool B_KMAJOR> __device__ __forceinline__ void ek1_mma_tile(const double *As, const double *Bs, int Kp, double (&c)[4]) {
  const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const int asx = A_KMAJOR ? 1 : Kp + 4, ask = A_KMAJOR ? EK1_M + 4 : 1;
  const int bsx = B_KMAJOR ? 1 : Kp + 4, bsk = B_KMAJOR ? EK1_N + 4 : 1;
  const double *ap = As + g * asx + q * ask, *bp = Bs + g * bsx + q * bsk;
  c[0] = c[1] = c[2] = c[3] = 0.0;
#pragma unroll 2
  for (int kb = 0; kb < Kp; kb += 16) {
    double a[8], b[4];
#pragma unroll
    for (int i = 0; i < 8; i++)
      a[i] = ap[8 * (i & 1) * asx + (kb + 4 * (i >> 1)) * ask];
#pragma unroll
    for (int j = 0; j < 4; j++)
      b[j] = bp[(kb + 4 * j) * bsk];
    ct_dmma2k16(c[0], c[1], c[2], c[3], a, b);
  }
}

__global__ void __launch_bounds__(EK1_T) k_ekf_gemm1(int mode, const double *__restrict__ P, int ldP, const double *__restrict__ H, int ldH,
                                                     const double *__restrict__ Min, int ldM, const DevUpdateInfo *__restrict__ info, int X, int Y,
                                                     int K, double *__restrict__ Cout, int ldC, double sigma2, const double *__restrict__ Rdiag) {
  // Programmatic dependent launch, in the order that lets mode 1 read H and the column map before its wait: mode 0 waits
  // BEFORE it lets its dependant (mode 1) launch, so when mode 1 runs, k_ekf_prep and every kernel before it (k_cq_trmm,
  // which writes H; k_init_prep, which writes the column map on the landmark-initialisation paths) have completed. Only M,
  // mode 0's output, is read after mode 1's wait. Mode 0 itself reads nothing before its wait.
  if (mode == 0)
    asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  extern __shared__ __align__(16) double g1[];
  __shared__ int cs_s[EK1_KMAX];
  const int x0 = blockIdx.x * EK1_M, y0 = blockIdx.y * EK1_N;
  if (mode == 1 && y0 > x0 + EK1_M - 1)
    return; // strictly upper tile of S
  const int tid = threadIdx.x, lane = tid & 31, g = lane >> 2, q = lane & 3;
  const int Kp = ek1_kpad(K);
  // A: Kp x 20 doubles (either layout fits), then B: Kp x 12
  double *As = g1, *Bs = g1 + (size_t)Kp * (EK1_M + 4);
  // H's rows first: their copies are in flight while the column map, which the gathered operand's addresses need, arrives
  // (mode 1: both before the wait)
  if (mode == 0)
    ek1_stage_rows<EK1_N>(Bs, Kp, H, (size_t)ldH, y0, Y, K);
  else
    ek1_stage_rows<EK1_M>(As, Kp, H, (size_t)ldH, x0, X, K);
  const int *cs = info->col_state;
  for (int j = tid; j < K; j += EK1_T)
    cs_s[j] = cs[j];
  if (mode == 1)
    asm volatile("griddepcontrol.wait;" ::: "memory");
  __syncthreads();
  // M[a][i] = sum_j P[cs[j]][a] H[i][j]: A = P's gathered rows (k-major), B = H's rows (row-major)
  // S[i][k] = sum_j H[i][j] M[cs[j]][k]: A = H's rows (row-major), B = M's gathered rows (k-major)
  if (mode == 0)
    ek1_stage_cols<EK1_M>(As, Kp, P, (size_t)ldP, cs_s, x0, X, K);
  else
    ek1_stage_cols<EK1_N>(Bs, Kp, Min, (size_t)ldM, cs_s, y0, Y, K);
  ek1_stage_wait();
  if (tid >= 32)
    return;
  double c[4];
  if (mode == 0)
    ek1_mma_tile<true, false>(As, Bs, Kp, c);
  else
    ek1_mma_tile<false, true>(As, Bs, Kp, c);
#pragma unroll
  for (int u = 0; u < 4; u++) {
    const int x = x0 + g + 8 * (u >> 1), y = y0 + 2 * q + (u & 1);
    if (x < X && y < Y) {
      double v = c[u];
      if (mode == 1 && x == y)
        v += Rdiag ? Rdiag[x] : sigma2;
      Cout[(size_t)x * ldC + y] = v;
    }
  }
}

// P <- sym_U(P - Y Y'), dx = Y w, r <= EK1_KMAX (same contract as k_ekf_downdate): the 16 x 8 tile of P at rows a0.., columns
// b0.. from rows a0.. and b0.. of Y; tiles wholly below the diagonal exit. Warp 0 runs the DMMA chain and writes P; on the
// tile with b0 == a0, warp 1 computes dx[a0..a0+16) beside it. Smem: Y's rows a0.. (16 x (Kp + 4)), rows b0..
// (8 x (Kp + 4)), then w (r).
__global__ void __launch_bounds__(EK1_T, 1) k_ekf_downdate1(double *__restrict__ P, int ldP, const double *__restrict__ Yin, int ldY, int N, int r,
                                                         const double *__restrict__ w, double *__restrict__ dx, DevUpdateInfo *__restrict__ info) {
  OVB_PDL_ENTER();
  extern __shared__ __align__(16) double d1[];
  const int a0 = blockIdx.x * EK1_M, b0 = blockIdx.y * EK1_N;
  if (b0 + EK1_N - 1 < a0)
    return;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, g = lane >> 2, q = lane & 3;
  const bool dx_tile = b0 == a0;
  const int Kp = ek1_kpad(r);
  double *As = d1, *Bs = As + (size_t)EK1_M * (Kp + 4), *ws = Bs + (size_t)EK1_N * (Kp + 4);
  // the copies, warp 0's entries of P and the factor's verdict all in flight at once (Y is staged before the verdict is
  // known, and used only when the factor succeeded)
  ek1_stage_rows<EK1_M>(As, Kp, Yin, (size_t)ldY, a0, N, r);
  ek1_stage_rows<EK1_N>(Bs, Kp, Yin, (size_t)ldY, b0, N, r);
  if (dx_tile)
    for (int k = tid; k < r; k += EK1_T)
      ek_cpa8(&ws[k], &w[k]);
  double pv[4];
#pragma unroll
  for (int u = 0; u < 4; u++) {
    const int a = a0 + g + 8 * (u >> 1), b = b0 + 2 * q + (u & 1);
    pv[u] = (wid == 0 && a < N && b < N && b >= a) ? P[(size_t)a * ldP + b] : 0.0;
  }
  const int not_spd = info->not_spd;
  ek1_stage_wait();
  if (not_spd) { // failed factor: P stays as it was, no correction
    if (dx_tile && tid < EK1_M && a0 + tid < N)
      dx[a0 + tid] = 0.0;
    return;
  }
  if (wid == 0) {
    double c[4];
    ek1_mma_tile<false, false>(As, Bs, Kp, c);
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const int a = a0 + g + 8 * (u >> 1), b = b0 + 2 * q + (u & 1);
      if (a < N && b < N && b >= a) {
        const double v = pv[u] - c[u];
        P[(size_t)a * ldP + b] = v;
        P[(size_t)b * ldP + a] = v;
        if (a == b && v < 0.0)
          atomicMin(&info->neg_diag_index, a);
        if (!isfinite(v))
          info->nonfinite = 1;
      }
    }
  } else if (wid == 1 && dx_tile) {
    // dx[a] = s0 + s1, s0 over the even k and s1 over the odd k (ascending): lanes 0-15 carry s0 of rows a0 + lane, lanes
    // 16-31 s1 of the same rows
    const double *Ar = As + (lane & 15) * (Kp + 4);
    double s = 0.0;
    for (int k = lane >> 4; k < r; k += 2)
      s = fma(Ar[k], ws[k], s);
    const double s1 = __shfl_down_sync(0xffffffffu, s, 16);
    if (lane < EK1_M && a0 + lane < N)
      dx[a0 + lane] = s + s1;
  }
}

// resets the failure flags and stages the residual, column n of H's first r rows, in w for the Cholesky kernels
__global__ void k_ekf_prep(DevUpdateInfo *info, const int *skip, const double *__restrict__ H, int ldH, int r, int n, double *__restrict__ w) {
  OVB_PDL_ENTER();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < r)
    w[i] = H[(size_t)i * ldH + n];
  if (i == 0) {
    info->neg_diag_index = OVB_NO_NEG_DIAG;
    info->not_spd = (skip && *skip) ? 1 : 0; // a skipped update takes the failed-factor exits of the kernels below
    info->nonfinite = 0;
  }
}

// H: r x (n+1) (row-major, ldHm), r <= n <= N (callers compress first when r > n); column j < n of H is state column
// d_info->col_state[j], column n the residual. Everything is enqueued on the context stream; flags land in d_info.
// gate_only: stop after the Cholesky — d_w then holds w = L^-1 res (|w|^2 = res' S^-1 res) and P is untouched
// (the Mahalanobis test of StateHelper::initialize, StateHelper.cpp:458-470).
void launch_ekf_update(ovb_ctx *ctx, const double *H, int ldHm, int r, int n, bool gate_only, double sigma2, const double *Rdiag_dev,
                       const int *skip_dev) {
  const int N = ctx->N;
  const int ld = ctx->ldP;
  double *P = ctx->P[ctx->cur];
  ovb_launch(ctx, k_ekf_prep, dim3(r > 128 ? (r + 127) / 128 : 1), dim3(128), (size_t)(0), ctx->d_info, skip_dev, H, ldHm, r, n, ctx->d_w);
  if (r <= 0 || n <= 0)
    return;
  if (!ctx->attr_done[2]) { // function attributes are per device: one flag per context
    cudaFuncSetAttribute(k_ekf_chol, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(k_ekf_trsm, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(k_ekf_gemm1, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    cudaFuncSetAttribute(k_ekf_downdate1, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    ctx->attr_done[2] = 1;
  }
  // small inner dimensions (config 2: n = r = 154): one-shot staged products, DMMA Cholesky + register solve of k_cholqr.cu
  const bool one_shot = ctx->ekf_chol_dmma && n <= EK1_KMAX && r <= EK1_KMAX;
  if (one_shot) {
    const size_t sm01 = sizeof(double) * (size_t)ek1_kpad(n) * (EK1_M + 4 + EK1_N + 4);
    const dim3 t0((N + EK1_M - 1) / EK1_M, (r + EK1_N - 1) / EK1_N), t1((r + EK1_M - 1) / EK1_M, (r + EK1_N - 1) / EK1_N);
    ovb_launch(ctx, k_ekf_gemm1, t0, dim3(EK1_T), sm01, 0, P, ld, H, ldHm, nullptr, 0, ctx->d_info, N, r, n, ctx->d_M, ld, 0.0, nullptr);
    ovb_launch(ctx, k_ekf_gemm1, t1, dim3(EK1_T), sm01, 1, P, ld, H, ldHm, ctx->d_M, ld, ctx->d_info, r, r, n, ctx->d_S, ld, sigma2, Rdiag_dev);
  } else {
    dim3 g0((N + EK_T - 1) / EK_T, (r + EK_T - 1) / EK_T);
    dim3 g1((r + EK_T - 1) / EK_T, (r + EK_T - 1) / EK_T);
    ovb_launch(ctx, k_ekf_gemm, dim3(g0), dim3(256), (size_t)(0), 0, P, ld, H, ldHm, nullptr, 0, ctx->d_info, N, r, n, ctx->d_M, ld, 0.0, nullptr);
    ovb_launch(ctx, k_ekf_gemm, dim3(g1), dim3(256), (size_t)(0), 1, P, ld, H, ldHm, ctx->d_M, ld, ctx->d_info, r, r, n, ctx->d_S, ld, sigma2, Rdiag_dev);
  }
  size_t chol_bytes = sizeof(double) * (size_t)(r + 1) * (size_t)(r | 1);
  int use_smem = chol_bytes <= 200 * 1024;
  double *invdiag = ctx->d_w + ctx->cfg.max_state; // d_w holds 4 x max_state doubles: [w | 1/diag(L) | ...]
  double *Lpk = nullptr; // packed factor for the register solve (only written by the DMMA Cholesky)
  unsigned long long epoch = 0; // nonzero: the factor streams into that solve
  const bool dmma_chol = ctx->ekf_chol_dmma && launch_chol_ekf_dmma(ctx, ctx->d_S, ld, r, ctx->d_w, ctx->d_w, invdiag, &Lpk, gate_only ? nullptr : &epoch);
  // wider than one CTA's Cholesky: blocked DMMA factorisation + blocked solve (Y = M L^-T in place over M)
  const bool wide = !dmma_chol && ctx->ekf_chol_dmma && r < ld && launch_chol_solve_wide(ctx, ctx->d_S, ld, r, ctx->d_w, invdiag, ctx->d_M, ld, N, gate_only);
  if (wide) {
    if (gate_only)
      return;
    dim3 g2w((N + EK_T - 1) / EK_T, (N + EK_T - 1) / EK_T);
    ovb_launch(ctx, k_ekf_downdate, dim3(g2w), dim3(256), (size_t)(0), P, ld, (const double *)ctx->d_M, ld, N, r, ctx->d_w, ctx->d_dx, ctx->d_info);
    return;
  }
  if (!dmma_chol)
    ovb_launch(ctx, k_ekf_chol, dim3(1), dim3(EKC_THREADS), (size_t)(use_smem ? chol_bytes : 0), ctx->d_S, ld, r, ctx->d_w, ctx->d_w, invdiag, ctx->d_info, use_smem);
  if (gate_only)
    return;
  const double *Yd = ctx->d_Y;
  if (dmma_chol && Lpk != nullptr && launch_trsm_rows(ctx, ctx->d_M, ld, N, r, Lpk, epoch)) {
    Yd = ctx->d_M; // Y = M L^-T in place
  } else {
    size_t trsm_small = sizeof(double) * ((size_t)TR_ROWS * r + r);
    size_t trsm_full = trsm_small + sizeof(double) * (size_t)r * (size_t)(r | 1);
    int L_in_smem = trsm_full <= 200 * 1024;
    ovb_launch(ctx, k_ekf_trsm, dim3((N + TR_ROWS - 1) / TR_ROWS), dim3(32 * TR_ROWS), (size_t)(L_in_smem ? trsm_full : trsm_small), ctx->d_M, ld, ctx->d_S, ld, invdiag, N,
               r, ctx->d_Y, ld, L_in_smem, ctx->d_info);
  }
  if (one_shot) {
    const size_t smd = sizeof(double) * ((size_t)(EK1_M + EK1_N) * (ek1_kpad(r) + 4) + r);
    const dim3 t2((N + EK1_M - 1) / EK1_M, (N + EK1_N - 1) / EK1_N);
    ovb_launch(ctx, k_ekf_downdate1, t2, dim3(EK1_T), smd, P, ld, Yd, ld, N, r, ctx->d_w, ctx->d_dx, ctx->d_info);
  } else {
    dim3 g2((N + EK_T - 1) / EK_T, (N + EK_T - 1) / EK_T);
    ovb_launch(ctx, k_ekf_downdate, dim3(g2), dim3(256), (size_t)(0), P, ld, Yd, ld, N, r, ctx->d_w, ctx->d_dx, ctx->d_info);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// covariance structure operations

// StateHelper::initialize_invertible (StateHelper.cpp:484-577): grow P by the k-wide new variable.
//   m = P[:, cols] Hx'            (N x k)     Hx = invertible part's state Jacobian (k x n), cols from info->col_state
//   M = Hx P[cols, cols] Hx' + s2 I (k x k, upper triangle mirrored like selfadjointView<Upper>)
//   P[0:N, N:N+k] = -m Hinv',  P[N:N+k, 0:N] = its transpose,  P[N:N+k, N:N+k] = Hinv M Hinv'
// Single CTA (N <= a few hundred rows, k <= 3): the step is a serial point in the reference as well.
// N_dev (optional): N is read there (ovb_slam_delayed_init_batch: the size the gates before have left); N_max sizes m
__global__ void k_cov_init_augment(double *__restrict__ P, int ld, int N_max, int k, int n, const DevUpdateInfo *__restrict__ info,
                                   const double *__restrict__ Hx, const double *__restrict__ Hinv, double sigma2, const int *__restrict__ skip,
                                   const int *__restrict__ N_dev) {
  extern __shared__ double ism[]; // m[N][k], then M[k][k]
  double *m = ism, *M = ism + (size_t)N_max * k;
  OVB_PDL_ENTER();
  const int tid = threadIdx.x;
  if (skip && *skip)
    return;
  const int N = N_dev ? *N_dev : N_max;
  for (int a = tid; a < N; a += blockDim.x) {
    for (int i = 0; i < k; i++) {
      double acc = 0.0;
      for (int j = 0; j < n; j++)
        acc += P[(size_t)a * ld + info->col_state[j]] * Hx[i * n + j];
      m[a * k + i] = acc;
    }
  }
  __syncthreads();
  if (tid < k * k) {
    const int i = tid / k, i2 = tid % k;
    double acc = 0.0;
    for (int j = 0; j < n; j++)
      acc += Hx[i * n + j] * m[info->col_state[j] * k + i2];
    M[i * k + i2] = acc + (i == i2 ? sigma2 : 0.0);
  }
  __syncthreads();
  if (tid < k * k) {
    const int i = tid / k, i2 = tid % k;
    if (i2 < i)
      M[i * k + i2] = M[i2 * k + i]; // selfadjointView<Upper>
  }
  __syncthreads();
  for (int a = tid; a < N; a += blockDim.x) {
    for (int q = 0; q < k; q++) {
      double acc = 0.0;
      for (int i = 0; i < k; i++)
        acc += m[a * k + i] * Hinv[q * k + i];
      P[(size_t)a * ld + N + q] = -acc;
      P[(size_t)(N + q) * ld + a] = -acc;
    }
  }
  if (tid < k * k) {
    const int q = tid / k, q2 = tid % k;
    double acc = 0.0;
    for (int i = 0; i < k; i++)
      for (int i2 = 0; i2 < k; i2++)
        acc += Hinv[q * k + i] * M[i * k + i2] * Hinv[q2 * k + i2];
    // the reference's dense product leaves P_LL symmetric only to rounding; write the upper entry to both places so the
    // resident covariance stays exactly symmetric
    if (q <= q2) {
      P[(size_t)(N + q) * ld + N + q2] = acc;
      P[(size_t)(N + q2) * ld + N + q] = acc;
    }
  }
}

bool launch_cov_init_augment(ovb_ctx *ctx, int k, int n, const double *Hx_dev, const double *Hinv_dev, double sigma2, const int *skip_dev,
                             const int *N_dev) {
  const int N = ctx->N;
  size_t smem = sizeof(double) * ((size_t)N * k + (size_t)k * k);
  if (smem > 200 * 1024)
    return false; // N*k doubles must fit one CTA's shared memory (N <= ~8500 for a 3-wide landmark)
  if (!ctx->attr_done[5]) {
    cudaFuncSetAttribute(k_cov_init_augment, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    ctx->attr_done[5] = 1;
  }
  return ovb_launch(ctx, k_cov_init_augment, dim3(1), dim3(256), smem, ctx->P[ctx->cur], ctx->ldP, N, k, n, ctx->d_info, Hx_dev, Hinv_dev, sigma2,
                    skip_dev, N_dev) == cudaSuccess;
}

// ovb_slam_delayed_init, after the per-feature kernel: the head of the init system (status, chi2, skip flag), H_L^-1 of the
// k x k invertible block by Gauss-Jordan with partial pivoting (the host's order in ovb_cov_initialize), dx_new = H_L^-1 r,
// and the column map for the augmentation and the EKF update. H_L is rows/columns 3-k..2 of the kernel's 3 x 3 block.
__global__ void k_init_prep(const DevFeat *__restrict__ feat, DevInitSys *__restrict__ sys, DevUpdateInfo *__restrict__ info, int k, int n) {
  OVB_PDL_ENTER();
  const int tid = threadIdx.x;
  const bool ok = feat->status == OVB_FEAT_OK;
  if (ok)
    for (int j = tid; j < n; j += blockDim.x)
      info->col_state[j] = sys->col_state[j];
  if (tid != 0)
    return;
  sys->status = feat->status;
  sys->chi2 = feat->chi2;
  int fail = sys->n != n ? 2 : 0;
  const int o = 3 - k;
  double A[9], Inv[9];
  for (int i = 0; i < k; i++)
    for (int j = 0; j < k; j++) {
      A[i * k + j] = sys->HL[(o + i) * 3 + o + j];
      Inv[i * k + j] = (i == j) ? 1.0 : 0.0;
    }
  for (int c0 = 0; c0 < k && !fail; c0++) {
    int piv = c0;
    for (int i = c0 + 1; i < k; i++)
      if (fabs(A[i * k + c0]) > fabs(A[piv * k + c0]))
        piv = i;
    if (!(fabs(A[piv * k + c0]) > 0.0)) {
      fail = 1;
      break;
    }
    if (piv != c0)
      for (int j = 0; j < k; j++) {
        double t = A[c0 * k + j];
        A[c0 * k + j] = A[piv * k + j];
        A[piv * k + j] = t;
        t = Inv[c0 * k + j];
        Inv[c0 * k + j] = Inv[piv * k + j];
        Inv[piv * k + j] = t;
      }
    const double d = A[c0 * k + c0];
    for (int j = 0; j < k; j++) {
      A[c0 * k + j] /= d;
      Inv[c0 * k + j] /= d;
    }
    for (int i = 0; i < k; i++) {
      if (i == c0)
        continue;
      const double f = A[i * k + c0];
      for (int j = 0; j < k; j++) {
        A[i * k + j] -= f * A[c0 * k + j];
        Inv[i * k + j] -= f * Inv[c0 * k + j];
      }
    }
  }
  for (int q = 0; q < 3; q++) {
    double acc = 0.0;
    if (q < k)
      for (int i = 0; i < k; i++)
        acc += Inv[q * k + i] * sys->res[o + i];
    sys->dx_new[q] = acc;
  }
  for (int i = 0; i < k * k; i++)
    sys->Hinv[i] = Inv[i];
  sys->fail = ok ? fail : 0;
  sys->skip = (!ok || fail) ? 1 : 0;
}

void launch_init_prep(ovb_ctx *ctx, int feat, int k, int n) {
  ovb_launch(ctx, k_init_prep, dim3(1), dim3(256), (size_t)0, ctx->d_feat + feat, ctx->d_init, ctx->d_info, k, n);
}

// StateHelper::clone: append a copy of the `size`-wide variable at old_off (StateHelper.cpp:371-373)
// neg_diag (optional): the flag of a propagation enqueued before; a negative diagonal there cancels the clone
__global__ void k_cov_clone(double *P, int ld, int N, int old_off, int size, const int *neg_diag) {
  OVB_PDL_ENTER();
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  int N2 = N + size;
  if (idx >= N2 * size || (neg_diag && *neg_diag != OVB_NO_NEG_DIAG))
    return;
  int i = idx / size, j = idx % size; // element (i, N+j) and its mirror (N+j, i)
  double v;
  if (i < N)
    v = P[(size_t)i * ld + old_off + j];
  else
    v = P[(size_t)(old_off + (i - N)) * ld + old_off + j];
  double vr = (i < N) ? P[(size_t)(old_off + j) * ld + i] : v;
  P[(size_t)i * ld + N + j] = v;
  if (i < N)
    P[(size_t)(N + j) * ld + i] = vr;
}
// augment_clone time-offset term, step 1: P[:, N..N+size) += P[:, dt] dnc'   (StateHelper.cpp:611-612)
__global__ void k_cov_dt_cols(double *P, int ld, int N2, int new_off, int size, int dt_off, const double *dnc, const int *neg_diag) {
  OVB_PDL_ENTER();
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N2 * size || (neg_diag && *neg_diag != OVB_NO_NEG_DIAG))
    return;
  int i = idx / size, j = idx % size;
  P[(size_t)i * ld + new_off + j] += P[(size_t)i * ld + dt_off] * dnc[j];
}
// step 2: P[N..N+size, :] += dnc P[dt, :]   (StateHelper.cpp:613-614) — reads the row written by step 1
__global__ void k_cov_dt_rows(double *P, int ld, int N2, int new_off, int size, int dt_off, const double *dnc, const int *neg_diag) {
  OVB_PDL_ENTER();
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N2 * size || (neg_diag && *neg_diag != OVB_NO_NEG_DIAG))
    return;
  int i = idx / N2, j = idx % N2;
  P[(size_t)(new_off + i) * ld + j] += dnc[i] * P[(size_t)dt_off * ld + j];
}

void launch_cov_clone(ovb_ctx *ctx, int old_off, int size, const double *dnc_dt_dev, int dt_off, const int *neg_diag_dev) {
  double *P = ctx->P[ctx->cur];
  int N = ctx->N, N2 = N + size;
  int tot = N2 * size;
  const dim3 grid((tot + 255) / 256), block(256);
  ovb_launch(ctx, k_cov_clone, grid, block, (size_t)0, P, ctx->ldP, N, old_off, size, neg_diag_dev);
  if (dnc_dt_dev) {
    ovb_launch(ctx, k_cov_dt_cols, grid, block, (size_t)0, P, ctx->ldP, N2, N, size, dt_off, dnc_dt_dev, neg_diag_dev);
    ovb_launch(ctx, k_cov_dt_rows, grid, block, (size_t)0, P, ctx->ldP, N2, N, size, dt_off, dnc_dt_dev, neg_diag_dev);
  }
}

// StateHelper::marginalize (StateHelper.cpp:293-313): out of place into the other buffer; the x2-x1 block is the
// transpose of the copied x1-x2 block exactly as the reference builds it.
__global__ void k_cov_marg(const double *Pin, double *Pout, int ld, int N, int off, int size) {
  OVB_PDL_ENTER();
  int N2 = N - size;
  int i = blockIdx.y * blockDim.y + threadIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N2 || j >= N2)
    return;
  int si = i < off ? i : i + size, sj = j < off ? j : j + size;
  double v = (i >= off && j < off) ? Pin[(size_t)sj * ld + si] : Pin[(size_t)si * ld + sj];
  Pout[(size_t)i * ld + j] = v;
}

void launch_cov_marginalize(ovb_ctx *ctx, int off, int size) {
  int N2 = ctx->N - size;
  dim3 b(32, 8), g((N2 + 31) / 32, (N2 + 7) / 8);
  ovb_launch(ctx, k_cov_marg, g, b, (size_t)0, ctx->P[ctx->cur], ctx->P[ctx->cur ^ 1], ctx->ldP, ctx->N, off, size);
}

// EKFPropagation (StateHelper.cpp:80-100). old_idx[k] = covariance index of Phi's column k (q of them).
//  C[a][j]   = sum_k P[a][old_idx[k]] Phi[j][k]                       (Cov_PhiT, N x p)  -> Cbuf
//  PCP[i][j] = Qsym[i][j] + sum_k Phi[i][k] C[old_idx[k]][j]          (p x p)            -> Sbuf
// The two per-entry expressions are shared with ovb_marginalize_window's kernels below, which must give the same bits.
__device__ __forceinline__ double prop_C_entry(const double *P, int ld, int a, int j, int q, const int *old_idx, const double *Phi) {
  double acc = 0.0;
  for (int k = 0; k < q; k++)
    acc += P[(size_t)a * ld + old_idx[k]] * Phi[(size_t)j * q + k];
  return acc;
}
// C[x][j] at C[x * sx + j * sj]
__device__ __forceinline__ double prop_PCP_entry(double acc, int i, int j, int q, const int *old_idx, const double *Phi, const double *C, size_t sx,
                                                 size_t sj) {
  for (int k = 0; k < q; k++)
    acc += Phi[(size_t)i * q + k] * C[(size_t)old_idx[k] * sx + (size_t)j * sj];
  return acc;
}
__global__ void k_prop_C(const double *P, int ld, int N, int p, int q, const int *old_idx, const double *Phi, double *Cbuf, int ldC) {
  OVB_PDL_ENTER();
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * p)
    return;
  int a = idx / p, j = idx % p;
  Cbuf[(size_t)a * ldC + j] = prop_C_entry(P, ld, a, j, q, old_idx, Phi);
}
__global__ void k_prop_PCP(const double *Cbuf, int ldC, int p, int q, const int *old_idx, const double *Phi, const double *Q, double *Sbuf,
                           int ldS) {
  OVB_PDL_ENTER();
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= p * p)
    return;
  int i = idx / p, j = idx % p;
  double acc = (i <= j) ? Q[(size_t)i * p + j] : Q[(size_t)j * p + i];
  Sbuf[(size_t)i * ldS + j] = prop_PCP_entry(acc, i, j, q, old_idx, Phi, Cbuf, ldC, 1);
}
__global__ void k_prop_write(double *P, int ld, int N, int new_off, int p, const double *Cbuf, int ldC, const double *Sbuf, int ldS,
                             DevUpdateInfo *info) {
  OVB_PDL_ENTER();
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * p)
    return;
  int a = idx / p, j = idx % p;
  if (a >= new_off && a < new_off + p) {
    double v = Sbuf[(size_t)(a - new_off) * ldS + j];
    P[(size_t)a * ld + new_off + j] = v;
    if (a - new_off == j && v < 0.0)
      atomicMin(&info->neg_diag_index, a);
  } else {
    double v = Cbuf[(size_t)a * ldC + j];
    P[(size_t)a * ld + new_off + j] = v;
    P[(size_t)(new_off + j) * ld + a] = v;
  }
}

void launch_cov_propagate(ovb_ctx *ctx, int new_off, int p, int q, const int *old_idx_dev, const double *Phi_dev, const double *Q_dev) {
  double *P = ctx->P[ctx->cur];
  int N = ctx->N, ld = ctx->ldP;
  ovb_launch(ctx, k_ekf_prep, dim3(1), dim3(1), (size_t)(0), ctx->d_info, (const int *)nullptr, (const double *)nullptr, 0, 0, 0, (double *)nullptr);
  ovb_launch(ctx, k_prop_C, dim3((N * p + 255) / 256), dim3(256), (size_t)0, P, ld, N, p, q, old_idx_dev, Phi_dev, ctx->d_M, ld);
  ovb_launch(ctx, k_prop_PCP, dim3((p * p + 255) / 256), dim3(256), (size_t)0, ctx->d_M, ld, p, q, old_idx_dev, Phi_dev, Q_dev, ctx->d_S, ld);
  ovb_launch(ctx, k_prop_write, dim3((N * p + 255) / 256), dim3(256), (size_t)0, P, ld, N, new_off, p, ctx->d_M, ld, ctx->d_S, ld, ctx->d_info);
}

// ovb_marginalize_window: the anchor changes of landmarks l = 0..n-1 (in call order) as one T P T', then the marginalized
// ranges dropped, with the bits of the sequence  for l: EKFPropagation(l, Phi_l, Q = 0);  marginalize each range, highest
// first. Writing P' for P after the propagations and u for a moved row (landmark l, row j < p_l), the sequence gives
//   P'[u][a] = P'[a][u] = C_l[a][j]       for a outside every moved landmark (C_l as k_prop_C computes it on the prior P:
//                                           a's row and the columns Phi_l reads are untouched by the landmarks before l)
//   P'[u][v]             = S_l[j][r]       for v = (l, r): k_prop_PCP with Q = 0, from the same C_l
//   P'[u][v] = P'[v][u]  = C_L[e][jL]      for landmarks E < L, e the row of E, jL the row of L: k_prop_C at L's step reads
//                                           E's already-moved row, which is C_E over the columns Phi_L reads (L's own
//                                           columns included: at E's step L's rows were the prior's)
// Phase 1 (k_win_rows) writes R[u][a] = C_l[a][j] for every a; phase 2 (k_win_blocks) the K x K blocks from R.
__global__ void k_win_rows(int K, int N, const DevWinLM *__restrict__ lms, const int *__restrict__ row_lm, const double *__restrict__ phi,
                           const int *__restrict__ idx, const int *__restrict__ q, const double *__restrict__ P, int ld, double *__restrict__ R,
                           int ldR, const int *flags) {
  OVB_PDL_ENTER();
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= K * N || flags[1] != 0) // a singular H_f left this landmark without Phi
    return;
  const int u = t / N, a = t % N, l = row_lm[u];
  R[(size_t)u * ldR + a] = prop_C_entry(P, ld, a, u - lms[l].row0, q[l], idx + OVB_WIN_Q * l, phi + (size_t)OVB_WIN_PHI * l);
}
__global__ void k_win_blocks(int K, const DevWinLM *__restrict__ lms, const int *__restrict__ row_lm, const double *__restrict__ phi,
                             const int *__restrict__ idx, const int *__restrict__ q, const double *__restrict__ R, int ldR, double *__restrict__ B,
                             int *flags) {
  OVB_PDL_ENTER();
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= K * K || flags[1] != 0)
    return;
  const int u = t / K, v = t % K, lu = row_lm[u], lv = row_lm[v];
  double val;
  if (lu == lv) {
    const DevWinLM &lm = lms[lu];
    const int i = u - lm.row0, j = v - lm.row0;
    val = prop_PCP_entry(0.0, i, j, q[lu], idx + OVB_WIN_Q * lu, phi + (size_t)OVB_WIN_PHI * lu, R + (size_t)lm.row0 * ldR, 1, ldR);
    if (i == j && val < 0.0)
      atomicMin(&flags[0], lm.lm_off + i);
  } else {
    const int L = lu > lv ? lu : lv, ue = lu > lv ? v : u, uL = lu > lv ? u : v;
    val = prop_C_entry(R, ldR, ue, uL - lms[L].row0, q[L], idx + OVB_WIN_Q * L, phi + (size_t)OVB_WIN_PHI * L);
  }
  B[(size_t)u * K + v] = val;
}
// StateHelper::marginalize of every range at once (k_cov_marg composed from the highest range down): output (i, j) comes
// from prior indices (src[i], src[j]); it is read transposed when it lies below the diagonal with at least one removed
// range between its row and its column (exactly one of the sequential steps transposes it then). mv[x] = the moved row
// of prior index x, or -1. flags set: nothing is written.
__global__ void k_win_compact(const double *__restrict__ Pin, double *__restrict__ Pout, int ld, int N2, const int *__restrict__ src,
                              const int *__restrict__ mv, const double *__restrict__ R, int ldR, const double *__restrict__ B, int K,
                              const int *__restrict__ flags) {
  OVB_PDL_ENTER();
  const int i = blockIdx.y * blockDim.y + threadIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N2 || j >= N2 || flags[0] != OVB_NO_NEG_DIAG || flags[1] != 0)
    return;
  const int si = src[i], sj = src[j];
  const bool tr = i > j && si - sj != i - j;
  const int x = tr ? sj : si, y = tr ? si : sj;
  const int ux = mv[x], uy = mv[y];
  double v;
  if (ux >= 0 && uy >= 0)
    v = B[(size_t)ux * K + uy];
  else if (ux >= 0)
    v = R[(size_t)ux * ldR + y];
  else if (uy >= 0)
    v = R[(size_t)uy * ldR + x];
  else
    v = Pin[(size_t)x * ld + y];
  Pout[(size_t)i * ld + j] = v;
}

void launch_window_shift(ovb_ctx *ctx, int n, int K, int N2, const DevWinLM *lms, const int *row_lm, const double *phi, const int *idx,
                         const int *q, const int *src, const int *mv, int *flags, double *R, int ldR, double *B) {
  const double *P = ctx->P[ctx->cur];
  const int N = ctx->N, ld = ctx->ldP;
  if (n > 0) {
    ovb_launch(ctx, k_win_rows, dim3((K * N + 255) / 256), dim3(256), (size_t)0, K, N, lms, row_lm, phi, idx, q, P, ld, R, ldR, flags);
    ovb_launch(ctx, k_win_blocks, dim3((K * K + 255) / 256), dim3(256), (size_t)0, K, lms, row_lm, phi, idx, q, R, ldR, B, flags);
  }
  dim3 b(32, 8), g((N2 + 31) / 32, (N2 + 7) / 8);
  ovb_launch(ctx, k_win_compact, g, b, (size_t)0, P, ctx->P[ctx->cur ^ 1], ld, N2, src, mv, R, ldR, B, K, flags);
}

// Propagator::propagate_and_clone's accumulation over the IMU steps (Propagator.cpp:83-99, Qd of each step :453-464), in
// one CTA with Phi, Q and the temporaries in shared memory. For s = 0..steps-1:
//   Qd  = sym(G_s diag(qc_s[k/3]) G_s')       Phi = F_s Phi       Q = sym(F_s Q F_s' + Qd)        (sym(X) = 0.5 (X + X'))
// Bit-identical to the host loop of include/ovb200_vio.hpp: every entry is one dot product over ascending k from 0.0 with
// separate multiply and add, as the host computes it (__dmul_rn / __dadd_rn keep -fmad out of it), and the dense F keeps
// its zero terms so signed zeros agree too. The symmetrisations are computed by the owner of each pair (i <= j), which
// writes both halves: 0.5 (x + y) does not depend on the order of x and y.
// Step s+1's F / G / qc are staged with cp.async while step s computes. Phi and Q go to Phi_out / Q_out (n x n).
#define PA_THREADS 1024

__device__ __forceinline__ void pa_stage(double *dst, const double *src, int count, int tid) {
  for (int e = tid; e < count; e += PA_THREADS) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(dst + e);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(d), "l"(src + e) : "memory");
  }
}

__global__ void __launch_bounds__(PA_THREADS) k_prop_accumulate(int n, int steps, const double *__restrict__ F, const double *__restrict__ G,
                                                                const double *__restrict__ qc, double *__restrict__ Phi_out,
                                                                double *__restrict__ Q_out) {
  extern __shared__ double pa_sm[];
  const int tid = threadIdx.x, nn = n * n, rec = nn + 12 * n + 4, npairs = n * (n + 1) / 2;
  double *Phi = pa_sm, *Phi2 = Phi + nn, *Q = Phi2 + nn, *T = Q + nn, *stg = T + nn; // stg: two records [F nn | G 12n | qc 4]
  unsigned char *pi = (unsigned char *)(stg + 2 * rec), *pj = pi + npairs;         // the pairs i <= j, row by row
  OVB_PDL_ENTER();
  for (int e = tid; e < nn; e += PA_THREADS) {
    Phi[e] = (e / n == e % n) ? 1.0 : 0.0;
    Q[e] = 0.0;
  }
  if (tid < n)
    for (int j = tid, t = tid * n - tid * (tid - 1) / 2; j < n; j++, t++)
      pi[t] = (unsigned char)tid, pj[t] = (unsigned char)j;
  auto stage = [&](int s) {
    double *r = stg + (s & 1) * rec;
    pa_stage(r, F + (size_t)s * nn, nn, tid);
    pa_stage(r + nn, G + (size_t)s * 12 * n, 12 * n, tid);
    pa_stage(r + nn + 12 * n, qc + (size_t)s * 4, 4, tid);
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  if (steps > 0)
    stage(0);
  for (int s = 0; s < steps; s++) {
    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncthreads(); // step s's record has landed; step s-1 is done with Phi, Q and the other record
    if (s + 1 < steps)
      stage(s + 1);
    const double *f = stg + (s & 1) * rec, *g = f + nn, *w = g + 12 * n;
    // T = F Q, Phi2 = F Phi
    for (int e = tid; e < 2 * nn; e += PA_THREADS) {
      const bool phi = e >= nn;
      const int ee = phi ? e - nn : e, i = ee / n, j = ee % n;
      const double *B = phi ? Phi : Q;
      double acc = 0.0;
      for (int k = 0; k < n; k++)
        acc = __dadd_rn(acc, __dmul_rn(f[i * n + k], B[k * n + j]));
      (phi ? Phi2 : T)[ee] = acc;
    }
    __syncthreads();
    // Q = sym(T F' + Qd), Qd = sym(Qt), Qt = G diag(qc) G'
    for (int t = tid; t < npairs; t += PA_THREADS) {
      const int i = pi[t], j = pj[t];
      double qij = 0.0, qji = 0.0, tij = 0.0, tji = 0.0;
      for (int k = 0; k < 12; k++) {
        qij = __dadd_rn(qij, __dmul_rn(__dmul_rn(g[i * 12 + k], w[k / 3]), g[j * 12 + k]));
        qji = __dadd_rn(qji, __dmul_rn(__dmul_rn(g[j * 12 + k], w[k / 3]), g[i * 12 + k]));
      }
      for (int k = 0; k < n; k++) {
        tij = __dadd_rn(tij, __dmul_rn(T[i * n + k], f[j * n + k]));
        tji = __dadd_rn(tji, __dmul_rn(T[j * n + k], f[i * n + k]));
      }
      const double qd = __dmul_rn(0.5, __dadd_rn(qij, qji));
      const double v = __dmul_rn(0.5, __dadd_rn(__dadd_rn(tij, qd), __dadd_rn(tji, qd)));
      Q[i * n + j] = v;
      Q[j * n + i] = v;
    }
    double *x = Phi;
    Phi = Phi2, Phi2 = x;
  }
  __syncthreads();
  for (int e = tid; e < nn; e += PA_THREADS) {
    Phi_out[e] = Phi[e];
    Q_out[e] = Q[e];
  }
}

static size_t prop_accumulate_smem(int n) {
  const size_t nn = (size_t)n * n;
  return sizeof(double) * (4 * nn + 2 * (nn + 12 * (size_t)n + 4)) + (size_t)n * (n + 1);
}

bool launch_prop_accumulate(ovb_ctx *ctx, int n, int steps, const double *F_dev, const double *G_dev, const double *qc_dev, double *Phi_dev,
                            double *Q_dev) {
  const size_t smem = prop_accumulate_smem(n);
  if (!ctx->attr_done[7]) {
    if (cudaFuncSetAttribute(k_prop_accumulate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)prop_accumulate_smem(OVB_PROP_MAX_N)) != cudaSuccess)
      return false;
    ctx->attr_done[7] = 1;
  }
  return ovb_launch(ctx, k_prop_accumulate, dim3(1), dim3(PA_THREADS), smem, n, steps, F_dev, G_dev, qc_dev, Phi_dev, Q_dev) == cudaSuccess;
}
