// k_gram.cu — measurement compression through the normal equations ("Cholesky-QR"):  [R z] = chol([H r]'[H r]).
// Alternative to the Householder TSQR of k_tsqr.cu for UpdaterHelper::measurement_compress_inplace
// (ov_msckf/src/update/UpdaterHelper.cpp:456-487).
//
// Why it is admissible: StateHelper::EKFUpdate (state/StateHelper.cpp:116-197) depends on the compressed system only
// through R'R = H'H and R'z = H'r (any orthogonal transform of the rows of [R z] gives the same K H, K res, P+), and a
// Cholesky factor of the Gram matrix is backward stable in exactly that sense: R'R = H'H + O(eps |H|'|H|), the same order
// as the backward error a Householder QR commits on H. What is lost is row-wise accuracy of R for ill-conditioned H
// (error ~ cond(H)^2 eps instead of cond(H) eps) — the filter never looks at individual rows. The stacked MSCKF Jacobian
// is rank deficient (global position/yaw gauge, SURVEY.md App. A.6): pivots at round-off level are zeroed (semidefinite
// Cholesky) instead of failing; the reference's Givens sweep leaves O(eps |H|) noise rows in their place.
//
// Why it is the GPU shape of the problem: one streaming pass over [H r] (L2/HBM), all flops in register-tiled FP64 FMA
// GEMM tiles spread over every SM, deterministic two-stage reduction, then ONE small factorisation — instead of
// 154 x 3 sequential Householder steps. Multi-GPU needs no second-stage QR: Gram matrices add.
#include "chol.cuh"
#include "ovb_internal.cuh"

#define GR_T 64   // output tile
#define GR_K 32   // rows per shared-memory chunk
#define GR_THREADS 256

// partial Gram of a row slab: tile (ti, tj), ti <= tj, of A[r0:r1, :]' A[r0:r1, :]
__global__ void __launch_bounds__(GR_THREADS) k_gram_partial(const double *__restrict__ A, int ldA, int m, int nt, int slab_rows, int ntile,
                                                             double *__restrict__ Gpart) {
  __shared__ __align__(16) double As[GR_K][GR_T];
  __shared__ __align__(16) double Bs[GR_K][GR_T];
  OVB_PDL_ENTER();
  // upper tile index -> (ti, tj)
  int t = blockIdx.x, ti = 0;
  while (t >= ntile - ti) {
    t -= ntile - ti;
    ti++;
  }
  const int tj = ti + t;
  const int slab = blockIdx.y;
  const int r0 = slab * slab_rows, r1 = min(m, r0 + slab_rows);
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int ci0 = ti * GR_T, cj0 = tj * GR_T;
  double acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; a++)
#pragma unroll
    for (int b = 0; b < 4; b++)
      acc[a][b] = 0.0;
  for (int rc = r0; rc < r1; rc += GR_K) {
    // coalesced loads: 64 consecutive doubles per row per tile
    for (int e = tid; e < GR_K * GR_T; e += GR_THREADS) {
      const int k = e >> 6, c = e & 63;
      const int r = rc + k;
      double va = 0.0, vb = 0.0;
      if (r < r1) {
        if (ci0 + c < nt)
          va = A[(size_t)r * ldA + ci0 + c];
        if (cj0 + c < nt)
          vb = A[(size_t)r * ldA + cj0 + c];
      }
      As[k][c] = va;
      Bs[k][c] = vb;
    }
    __syncthreads();
#pragma unroll 8
    for (int k = 0; k < GR_K; k++) {
      const double2 a01 = *reinterpret_cast<const double2 *>(&As[k][4 * ty]);
      const double2 a23 = *reinterpret_cast<const double2 *>(&As[k][4 * ty + 2]);
      const double2 b01 = *reinterpret_cast<const double2 *>(&Bs[k][4 * tx]);
      const double2 b23 = *reinterpret_cast<const double2 *>(&Bs[k][4 * tx + 2]);
      const double av[4] = {a01.x, a01.y, a23.x, a23.y};
      const double bv[4] = {b01.x, b01.y, b23.x, b23.y};
#pragma unroll
      for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = 0; b < 4; b++)
          acc[a][b] += av[a] * bv[b];
    }
    __syncthreads();
  }
  double *dst = Gpart + ((size_t)slab * gridDim.x + blockIdx.x) * (GR_T * GR_T);
#pragma unroll
  for (int a = 0; a < 4; a++)
#pragma unroll
    for (int b = 0; b < 4; b++)
      dst[(4 * ty + a) * GR_T + 4 * tx + b] = acc[a][b];
}

// G[i][j] = sum over slabs (fixed order: bitwise reproducible), written for i <= j and mirrored
__global__ void k_gram_reduce(const double *__restrict__ Gpart, int nslab, int ntile, int ntp, int nt, double *__restrict__ G, int ldG) {
  OVB_PDL_ENTER();
  const int i = blockIdx.y * 16 + (threadIdx.x >> 4), j = blockIdx.x * 16 + (threadIdx.x & 15);
  if (i >= nt || j >= nt || i > j)
    return;
  const int ti = i / GR_T, tj = j / GR_T;
  // linear index of upper tile (ti, tj)
  int tidx = 0;
  for (int a = 0; a < ti; a++)
    tidx += ntile - a;
  tidx += tj - ti;
  const double *src = Gpart + (size_t)tidx * (GR_T * GR_T) + (i - ti * GR_T) * GR_T + (j - tj * GR_T);
  double s = 0.0;
  for (int sl = 0; sl < nslab; sl++)
    s += src[(size_t)sl * ntp * (GR_T * GR_T)];
  G[(size_t)i * ldG + j] = s;
  G[(size_t)j * ldG + i] = s;
}

// single CTA: semidefinite Cholesky of G[0:n,0:n] with row n (= H'r) carried as right-hand side; writes the
// upper-triangular R = L' and z = L^-1 H'r into Rout (n x (n+1), row-major)
__global__ void __launch_bounds__(EKC_THREADS) k_gram_chol(const double *__restrict__ G, int ldG, int n, double *__restrict__ Rout, int ldR,
                                                    double *__restrict__ work, int use_smem) {
  extern __shared__ __align__(16) double gsm[];
  __shared__ int flag;
  __shared__ double invd_sh[16];
  OVB_PDL_ENTER();
  const int tid = threadIdx.x;
  if (tid == 0)
    flag = 0;
  const int ld = use_smem ? (n | 1) : ldG;
  double *W = use_smem ? gsm : work;                 // (n+1) x ld
  double *d0 = use_smem ? (gsm + (size_t)(n + 1) * ld) : (work + (size_t)(n + 1) * ld); // original diagonal
  for (int e = tid; e < (n + 1) * n; e += EKC_THREADS) {
    const int i = e / n, j = e % n;
    if (j <= i)
      W[(size_t)i * ld + j] = G[(size_t)i * ldG + j];
  }
  for (int j = tid; j < n; j += EKC_THREADS)
    d0[j] = G[(size_t)j * ldG + j];
  __syncthreads();
  // pivots below ~n*eps of the column's own squared norm carry no information (gauge directions, unused variables)
  chol_lower_block<EKC_THREADS, 4>(W, ld, n, 1, &flag, invd_sh, d0, 1e-13);
  __syncthreads();
  for (int e = tid; e < n * (n + 1); e += EKC_THREADS) {
    const int i = e / (n + 1), j = e % (n + 1);
    double v = 0.0;
    if (j == n)
      v = W[(size_t)n * ld + i]; // z_i
    else if (j >= i)
      v = W[(size_t)j * ld + i]; // R[i][j] = L[j][i]
    Rout[(size_t)i * ldR + j] = v;
  }
}

// [R | z] (n x (n+1)) <- chol of the Gram of A (m x (n+1), last column = residual). A is not modified.
bool launch_compress_gram(ovb_ctx *ctx, const double *A, int m, int n, int ldA, double *Rout, int ldR) {
  const int nt = n + 1;
  const int ntile = (nt + GR_T - 1) / GR_T;
  const int ntp = ntile * (ntile + 1) / 2;
  int slab_rows = 256;
  while ((m + slab_rows - 1) / slab_rows > 128)
    slab_rows *= 2;
  const int nslab = (m + slab_rows - 1) / slab_rows;
  const size_t need_part = (size_t)nslab * ntp * GR_T * GR_T;
  const int ldG = (nt + 3) & ~3;
  const size_t need_G = (size_t)(nt + 2) * ldG * 2; // G plus the global-memory Cholesky workspace
  if (need_part > ctx->Gpart_cap) {
    if (ctx->d_Gpart)
      cudaFree(ctx->d_Gpart);
    ctx->d_Gpart = nullptr;
    if (cudaMalloc(&ctx->d_Gpart, sizeof(double) * need_part) != cudaSuccess)
      return false;
    ctx->Gpart_cap = need_part;
  }
  if (need_G > ctx->G_cap) {
    if (ctx->d_G)
      cudaFree(ctx->d_G);
    ctx->d_G = nullptr;
    if (cudaMalloc(&ctx->d_G, sizeof(double) * need_G) != cudaSuccess)
      return false;
    ctx->G_cap = need_G;
  }
  ovb_launch(ctx, k_gram_partial, dim3(ntp, nslab), dim3(GR_THREADS), (size_t)0, A, ldA, m, nt, slab_rows, ntile, ctx->d_Gpart);
  ovb_launch(ctx, k_gram_reduce, dim3((nt + 15) / 16, (nt + 15) / 16), dim3(256), (size_t)0, ctx->d_Gpart, nslab, ntile, ntp, nt,
             ctx->d_G, ldG);
  const size_t smem = sizeof(double) * ((size_t)(n + 1) * (n | 1) + n + 8);
  const int use_smem = smem <= 220 * 1024;
  if (!ctx->attr_done[3]) { // function attributes are per device: one flag per context
    cudaFuncSetAttribute(k_gram_chol, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
    ctx->attr_done[3] = 1;
  }
  double *work = ctx->d_G + (size_t)(nt + 2) * ldG;
  ovb_launch(ctx, k_gram_chol, dim3(1), dim3(EKC_THREADS), use_smem ? smem : 0, ctx->d_G, ldG, n, Rout, ldR, work, use_smem);
  return true;
}
