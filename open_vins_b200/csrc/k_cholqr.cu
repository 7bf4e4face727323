// k_cholqr.cu — measurement compression as a shifted CholeskyQR2 on the FP64 tensor-core path (DMMA), plus the
// single-CTA DMMA Cholesky shared with the EKF update.
// Replaces UpdaterHelper::measurement_compress_inplace (ov_msckf/src/update/UpdaterHelper.cpp:456-487: a Givens sweep of
// 3mn² flops with stride-m accesses) for stacked systems of up to CQ_MAXN columns (residual included).
//
//   pass 1   G1 = [H r]'[H r]                      k_cq_gram (DMMA, row slabs over all SMs) + k_cq_reduce (fixed order)
//            R1'R1 = G1 + s1 I                      k_cq_chol_gram (one CTA, tile-packed in shared memory: chol_tiles.cuh)
//   pass 2   G2 = Q1'Q1,  Q1 = [H r] R1^-1          k_cq_solve_gram: each slab's rows solved in shared memory (k_cq_trsm's
//                                                   row solve) and fed straight to k_cq_gram's k-steps; only a slab's last
//                                                   rows past the buffer pass through a small scratch, the rest of Q1 never
//                                                   reaches global memory, and [H r] is left as it was. Then k_cq_reduce.
//            R2'R2 = G2 + s2 I                      k_cq_chol_gram
//            [R z] = rows 0..n-1 of R2 R1           k_cq_trmm
// Systems wider than CQ_MAXN take the blocked path (cq_compress_wide), which overwrites [H r] with Q1.
//
// Why two passes are enough for the filter (DESIGN.md §4): StateHelper::EKFUpdate (state/StateHelper.cpp:116-197) sees
// the compressed system only through R'R = H'H and R'z = H'r. With Q1 = A R1^-1 computed by row-wise backward-stable
// substitution (A + dA = Q1 R1, |dA| <= c u |Q1||R1|, the same column-wise backward error a Householder QR commits),
//   R'R = R1'(Q1'Q1 + E) R1 = (A+dA)'(A+dA) + R1' E R1,     -eps I <= E <= eps I  (Gram rounding + s2, |Q1 e_j| <= 1)
// and R1'E R1 is bounded IN THE POSITIVE-SEMIDEFINITE ORDER by eps (G1 + s1 I): a relative perturbation eps of the
// information the measurements carry plus an absolute eps*s1 ~ 1e-24 |A|² — no condition-number factor, whatever R1
// was (R1 only has to keep |Q1| <= ~1, which the shift s1 guarantees). A single pass (k_gram.cu) has the kappa² loss
// that failed the 1e-9 bar with weakly observable calibration columns; the second pass removes it. The shifts make the
// factorisations total on the rank-deficient MSCKF system (gauge nullspace, SURVEY.md App. A.6).
//
// Everything is deterministic (no atomics, fixed reduction order): replicas on different GPUs stay bitwise equal.
#include "chol.cuh"
#include "chol_tiles.cuh"
#include "ovb_internal.cuh"
#include <math.h>
#include <cstdio>

#define CQ_MAXN 160      // columns incl. the residual that the single-CTA Cholesky / register TRSM take
#define CQ_MAXB 20       // CQ_MAXN / 8
#define CQ_MAXRB 22      // row blocks of the Cholesky (n + extra right-hand-side rows <= 176)
#define CQ_GRAM_T 512    // threads of k_cq_gram (16 warps, one 32x32 output tile each)
#define CQ_KB 32         // rows per staged chunk in k_cq_gram
#ifndef CQ_CHOL_T
#define CQ_CHOL_T 384
#endif
#define CQ_XP CT_XP     // pitch of the panel buffer (chol_tiles.cuh)
#define CQ_TRSM_T 640

namespace {

// D(8x8) += A(8x4) B(4x8), FP64 tensor-core path. a = A[lane>>2][lane&3], b = B[lane&3][lane>>2], d0/d1 = D[lane>>2][2*(lane&3)+{0,1}]
__device__ __forceinline__ void dmma(double &d0, double &d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}
__device__ __forceinline__ unsigned s_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cpa16(unsigned dst, const void *src, unsigned bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cpa8(unsigned dst, const void *src, unsigned bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cpa_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cpa_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void bar_group(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }
__device__ __forceinline__ int tri(int b) { return (b * (b + 1)) >> 1; }

// ---- factor streaming: a factor kernel (k_cq_chol_gram of pass 1, k_cq_chol_ekf) hands its packed factor to the next
// kernel of the stream (k_cq_solve_gram, k_cq_trsm), which PDL has made resident early, block column by block column.
// The producer publishes on a 64-bit counter in global memory, (epoch << 6) | s:
//   s = 1       its griddepcontrol.wait has returned: every kernel before it has completed, so the consumer may read and
//               write its own inputs and outputs
//   s = 2 + k   block column k of the packed factor (tiles (i, k) and reciprocal pivots 8k..8k+7) is in global memory
// The host draws a fresh epoch for every publishing launch, so the counter only grows and is never reset. One counter
// per context serves both producers: a producer publishes only after its griddepcontrol.wait, when the consumer of the
// one before it has completed. The epoch is drawn on the host; an update captured into a CUDA graph would have to draw
// it on the device instead.
__device__ __forceinline__ void cq_pub_store(unsigned long long *ctr, unsigned long long v) {
  asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(ctr), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long cq_pub_load(const unsigned long long *ctr) {
  unsigned long long v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(ctr) : "memory");
  return v;
}
// the consumer reads the factor with the bulk-copy engine (async proxy), the producer writes it with ordinary stores
__device__ __forceinline__ void cq_fence_proxy() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
__device__ __forceinline__ void cq_mbar_init(unsigned bar) { asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void cq_mbar_arrive(unsigned bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
// wait for phase 0 of an mbarrier; returns at once ever after (the loop stays inside the asm block: no branch for the
// compiler to guard with convergence code in the unrolled solve)
__device__ __forceinline__ void cq_mbar_wait(unsigned bar) {
  asm volatile("{\n\t.reg .pred p;\n\tCQ_MWAIT:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n\t@!p bra CQ_MWAIT;\n\t}" ::"r"(bar) : "memory");
}

// Output tile owned by warp w of Gram block blk. The Gram matrix is cut into blocks of BW x BW warp tiles (32 x 32 each);
// only blocks bI <= bJ exist; a diagonal block keeps its upper warp tiles only. Returns false for an idle warp.
__device__ __forceinline__ bool cq_tile_origin(int blk, int w, int BW, int nblk_side, int &ci, int &cj, int &offI, int &offJ, bool &diag) {
  int bI = 0, t = blk;
  while (t >= nblk_side - bI) {
    t -= nblk_side - bI;
    bI++;
  }
  const int bJ = bI + t;
  diag = (bI == bJ);
  int a, b;
  if (diag) {
    a = 0;
    int u = w;
    while (a < BW && u >= BW - a) {
      u -= BW - a;
      a++;
    }
    if (a >= BW)
      return false;
    b = a + u;
  } else {
    if (w >= BW * BW)
      return false;
    a = w / BW;
    b = w % BW;
  }
  offI = a * 32;
  offJ = (diag ? 0 : BW * 32) + b * 32;
  ci = (bI * BW + a) * 32;
  cj = (bJ * BW + b) * 32;
  return true;
}

// Rows rc..rc+nrows-1 of A into buf (row-major, `pitch` doubles): columns [cI0, cI0+WI) and, nrng == 2, [cJ0, cJ0+WI)
// after them, by 16-byte cp.async (NT threads, one commit group) with zero fill for rows >= r1 and columns >= nt.
template <int NT>
__device__ __forceinline__ void cq_issue_rows(double *buf, int pitch, const double *__restrict__ A, int ldA, int rc, int nrows, int r1, int nt, int cI0, int cJ0,
                                              int WI, int nrng) {
  const int units_per_row = nrng * WI / 2;
  for (int e = threadIdx.x; e < nrows * units_per_row; e += NT) {
    const int k = e / units_per_row, u = e - k * units_per_row;
    const int r = rc + k;
    const int dcol = 2 * u, col = (dcol < WI) ? cI0 + dcol : cJ0 + (dcol - WI);
    unsigned bytes = 0;
    if (r < r1)
      bytes = (col + 1 < nt) ? 16u : (col < nt ? 8u : 0u);
    const double *src = bytes ? (A + (size_t)r * ldA + col) : A;
    cpa16(s_u32(buf + (size_t)k * pitch + dcol), src, bytes);
  }
  cpa_commit();
}

// acc += one k-step (4 staged rows at `row0`) of one warp tile. Both Gram kernels accumulate through this, k-step by k-step
// in row order, so their partials over the same rows agree bit for bit. Both DMMA operands are the fragment
// X[lane&3][c0 + (lane>>2)] of the staged rows, at c0 = offI (row side) and offJ (column side); same: offI == offJ.
__device__ __forceinline__ void cq_gram_kstep(double (&acc)[4][4][2], const double *row0, int pitch, int offI, int offJ, bool same, int g, int q) {
  const double *row = row0 + (size_t)q * pitch + g;
  double fa[4], fb[4];
#pragma unroll
  for (int b = 0; b < 4; b++)
    fa[b] = row[offI + 8 * b];
  if (same) {
#pragma unroll
    for (int b = 0; b < 4; b++)
      fb[b] = fa[b];
  } else {
#pragma unroll
    for (int b = 0; b < 4; b++)
      fb[b] = row[offJ + 8 * b];
  }
  // output blocks a and a+1 share fb[b]: one m16n8k4 each pair
#pragma unroll
  for (int a = 0; a < 4; a += 2)
#pragma unroll
    for (int b = 0; b < 4; b++)
      ct_dmma2(acc[a][b][0], acc[a][b][1], acc[a + 1][b][0], acc[a + 1][b][1], fa[a], fa[a + 1], fb[b]);
}

} // namespace

// ------------------------------------------------------------------------------------------------------------ Gram
// Partial Gram matrix of one row slab: Gpart[slab][blk][warp][32x32] = A[slab rows, I cols]' A[slab rows, J cols].
// The slab streams through shared memory in chunks of CQ_KB rows (cp.async, double buffered, zero fill past the edges);
// both DMMA operands are the SAME fragment pattern X[k0 + (lane&3)][c0 + (lane>>2)] of the staged rows, so one staged
// chunk feeds the row- and the column-side of every tile. grid = (upper blocks, slabs).
__global__ void __launch_bounds__(CQ_GRAM_T) k_cq_gram(const double *__restrict__ A, int ldA, int m, int nt, int slab_rows, int BW, int nblk_side,
                                                      double *__restrict__ Gpart, int cs) {
  OVB_PDL_ENTER();
  extern __shared__ __align__(16) double gsm[];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, g = lane >> 2, q = lane & 3;
  int ci, cj, offI, offJ;
  bool diag;
  const bool active = cq_tile_origin(blockIdx.x, wid, BW, nblk_side, ci, cj, offI, offJ, diag);
  // column ranges staged per row: [I range (BW*32)] then, for off-diagonal blocks, [J range (BW*32)]
  int bI = 0, tt = blockIdx.x;
  while (tt >= nblk_side - bI) {
    tt -= nblk_side - bI;
    bI++;
  }
  const int bJ = bI + tt;
  const int WI = BW * 32;
  const int nrng = (bI == bJ) ? 1 : 2;
  const int pitch = nrng * WI + 4; // = 4 mod 16: conflict-free fragment loads
  const int cI0 = bI * WI, cJ0 = bJ * WI;
  const int r0 = blockIdx.y * slab_rows, r1 = min(m, r0 + slab_rows);
  const int nchunks = (r1 > r0) ? (r1 - r0 + CQ_KB - 1) / CQ_KB : 0;
  double acc[4][4][2];
#pragma unroll
  for (int a = 0; a < 4; a++)
#pragma unroll
    for (int b = 0; b < 4; b++)
      acc[a][b][0] = acc[a][b][1] = 0.0;

  auto issue = [&](int c) { cq_issue_rows<CQ_GRAM_T>(gsm + (size_t)(c & 1) * CQ_KB * pitch, pitch, A, ldA, r0 + c * CQ_KB, CQ_KB, r1, nt, cI0, cJ0, WI, nrng); };
  if (nchunks > 0)
    issue(0);
  for (int c = 0; c < nchunks; c++) {
    if (c + 1 < nchunks) {
      issue(c + 1);
      cpa_wait<1>();
    } else {
      cpa_wait<0>();
    }
    __syncthreads();
    if (active) {
      const double *buf = gsm + (size_t)(c & 1) * CQ_KB * pitch;
#pragma unroll
      for (int ks = 0; ks < CQ_KB / 4; ks++)
        cq_gram_kstep(acc, buf + (size_t)4 * ks * pitch, pitch, offI, offJ, diag && offI == offJ, g, q);
    }
    __syncthreads();
  }
  if (cs <= 1) {
    if (active) {
      double *dst = Gpart + (((size_t)blockIdx.y * gridDim.x + blockIdx.x) * 16 + wid) * 1024;
#pragma unroll
      for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = 0; b < 4; b++)
          *reinterpret_cast<double2 *>(dst + (8 * a + g) * 32 + 8 * b + 2 * q) = make_double2(acc[a][b][0], acc[a][b][1]);
    }
    return;
  }
  // ---- cluster of `cs` slabs (cluster dims (1, cs, 1)): the partial tiles meet in distributed shared memory, each CTA sums
  // 1/cs of every tile in rank order (fixed order: bitwise reproducible) and only the cluster's sum goes to global memory —
  // cs times less partial traffic for the reduction kernel to read back
  double *stage = gsm; // the pipeline buffers are free now (the loop ended with a barrier): [16 warps][1024]
  if (active) {
    double *dst = stage + (size_t)wid * 1024;
#pragma unroll
    for (int a = 0; a < 4; a++)
#pragma unroll
      for (int b = 0; b < 4; b++)
        *reinterpret_cast<double2 *>(dst + (8 * a + g) * 32 + 8 * b + 2 * q) = make_double2(acc[a][b][0], acc[a][b][1]);
  }
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
  unsigned rank;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
  if (active) {
    const int per = 1024 / cs; // elements of each tile this CTA sums
    double *dst = Gpart + ((((size_t)blockIdx.y / cs) * gridDim.x + blockIdx.x) * 16 + wid) * 1024 + (size_t)rank * per;
    const unsigned base = s_u32(stage + (size_t)wid * 1024 + (size_t)rank * per);
    for (int e = lane; e < per; e += 32) {
      double sum = 0.0;
      for (int r = 0; r < cs; r++) {
        unsigned ra;
        double v;
        asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(base + 8u * (unsigned)e), "r"((unsigned)r));
        asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(ra) : "memory");
        sum += v;
      }
      dst[e] = sum;
    }
  }
  // nobody leaves while a peer may still read its shared memory
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// G[i][j] = sum over slabs in a FIXED order (bitwise reproducible), for i <= j, mirrored. grid = (16 warp tiles x 8 chunks
// of 128 elements, blocks); the 1024 threads of a CTA are 128 elements x 8 slab groups (group g sums slabs g, g+8, ...),
// the eight partial sums meet in shared memory and are added as a balanced tree.
#define CQ_RED_T 1024
#define CQ_RED_CH 8
#define CQ_RED_GX (16 * CQ_RED_CH)
// tiled != 0: G receives the lower triangle in the tile-packed layout of chol_tiles.cuh (diagonal tiles whole), which the
// Cholesky kernel then takes in with one bulk copy; else row-major, both triangles.
__global__ void __launch_bounds__(CQ_RED_T) k_cq_reduce(const double *__restrict__ Gpart, int nslab, int nblk, int BW, int nblk_side, int nt,
                                                       double *__restrict__ G, int ldG, int tiled) {
  OVB_PDL_ENTER();
  __shared__ double red[8][128];
  int ci, cj, offI, offJ;
  bool diag;
  const int w = blockIdx.x / CQ_RED_CH, ch = blockIdx.x % CQ_RED_CH, blk = blockIdx.y;
  if (!cq_tile_origin(blk, w, BW, nblk_side, ci, cj, offI, offJ, diag))
    return;
  if (ci >= nt || cj >= nt)
    return;
  const int el = threadIdx.x & 127, sg = threadIdx.x >> 7;
  const int e = ch * 128 + el;
  const double *src = Gpart + ((size_t)blk * 16 + w) * 1024 + e;
  const size_t stride = (size_t)nblk * 16 * 1024;
  double s0 = 0.0, s1 = 0.0;
  int sl = sg;
  for (; sl + 8 < nslab; sl += 16) {
    s0 += src[(size_t)sl * stride];
    s1 += src[(size_t)(sl + 8) * stride];
  }
  if (sl < nslab)
    s0 += src[(size_t)sl * stride];
  red[sg][el] = s0 + s1;
  __syncthreads();
  if (sg == 0) {
    const int i = ci + (e >> 5), j = cj + (e & 31);
    if (i < nt && j < nt && i <= j) {
      const double s = ((red[0][el] + red[1][el]) + (red[2][el] + red[3][el])) + ((red[4][el] + red[5][el]) + (red[6][el] + red[7][el]));
      if (tiled) {
        G[ct_idx(j, i)] = s;
        if ((i >> 3) == (j >> 3))
          G[(size_t)(tri(j >> 3) + (j >> 3)) * 64 + (i & 7) * 8 + (j & 7)] = s; // upper half of a diagonal tile
      } else {
        G[(size_t)i * ldG + j] = s;
        G[(size_t)j * ldG + i] = s;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------ Cholesky
// Single-CTA Cholesky of an n x n SPD matrix (n <= CQ_MAXN) with `extra` right-hand-side rows appended as rows n.. .
// The lower triangle lives in shared memory as packed 8x8 tiles (tile (bi,bj), bj <= bi, at (bi(bi+1)/2 + bj)*64,
// row-major inside): a tile IS the DMMA accumulator fragment (lane reads its two doubles at 2*lane: conflict free), and
// the whole 160 x 160 triangle is 107 KB. The factorisation itself — warp 0 on the pivot chain, helper warps on the
// panels and the trailing update — is ct_chol_tiles (chol_tiles.cuh).
struct CqCholSmem {
  double T[(CQ_MAXRB * (CQ_MAXRB + 1) / 2) * 64];
  double Xp[2][CQ_MAXRB * 8 * CQ_XP];
  double invd[CQ_MAXRB * 8];
  double Linv[2][64];       // inverse of the current / next diagonal block
  double red[32];
  double dummyT[64];        // target of the masked-out tile of a pair (operands zero: it stays zero)
  double dummyX[2 * CQ_XP]; // zero operand rows for it
  int flag;
};

// The factor as the other kernels consume it (written by the Cholesky kernel as a straight copy of its shared memory):
//   [tile-packed lower triangle of L = R', tile (bi,bj) at (bi(bi+1)/2 + bj)*64, row-major 8x8] [reciprocal pivots 1/L_jj]
// Entries past n are zero (the solve treats the padded diagonal as 1).
#define CQ_PK_INV ((CQ_MAXB * (CQ_MAXB + 1) / 2) * 64)
#define CQ_PK_DOUBLES (CQ_PK_INV + CQ_MAXB * 8)

namespace {

// Publication of the packed factor of an n-column factorisation (ctr == nullptr: nobody streams). column() is
// ct_chol_tiles' hook (warp 8); it stores tiles (i, k) and pivots 8k..8k+7 at the addresses and with the values the
// epilogue's copy writes, then the count. Each lane's stores, a fence, then one lane's release of the count.
struct CqPublish {
  double *Lpk;
  unsigned long long *ctr, epoch;
  int n;
  __device__ __forceinline__ void column(const CtView &sm, int k) const {
    if (ctr == nullptr)
      return;
    const int lane = threadIdx.x & 31, NB = (n + 7) >> 3;
    for (int i = k; i < NB; i++) {
      const size_t o = (size_t)(ct_tri(i) + k) * 64 + 2 * lane;
      *reinterpret_cast<double2 *>(Lpk + o) = *reinterpret_cast<const double2 *>(sm.T + o);
    }
    if (lane < 8)
      Lpk[CQ_PK_INV + 8 * k + lane] = (8 * k + lane < n) ? sm.invd[8 * k + lane] : 1.0;
    cq_fence_proxy();
    __threadfence();
    __syncwarp();
    if (lane == 0)
      cq_pub_store(ctr, (epoch << 6) | (unsigned long long)(k + 2));
  }
  // the epilogue's copy starts past what column() has published: the last block column (its diagonal tile) and the pivots
  __device__ __forceinline__ int first_tile_el() const { return ctr ? (tri((n + 7) >> 3) - 1) * 64 : 0; }
  __device__ __forceinline__ int first_pivot() const { return ctr ? 8 * (((n + 7) >> 3) - 1) : 0; }
  // the whole CTA, after its share of the epilogue's copy: the last column's count
  __device__ __forceinline__ void finish() const {
    if (ctr == nullptr)
      return;
    cq_fence_proxy();
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0)
      cq_pub_store(ctr, (epoch << 6) | (unsigned long long)(((n + 7) >> 3) + 1));
  }
};

// The factorisation proper lives in chol_tiles.cuh (shared with the per-feature gate); this kernel family runs it with
// CQ_CHOL_T threads (256 / 512 / 640 were measured: 40.9 / 37.7 / 38.9 us against 36.8 us at 384, n = 155).
__device__ __forceinline__ void cq_chol_tiles(CqCholSmem &sm, int n, int nrows, bool strict, double floor_d, const CqPublish &pub) {
  CtView v;
  v.T = sm.T;
  v.Xp0 = sm.Xp[0];
  v.Xp1 = sm.Xp[1];
  v.invd = sm.invd;
  v.Linv0 = sm.Linv[0];
  v.Linv1 = sm.Linv[1];
  v.dummyT = sm.dummyT;
  v.dummyX = sm.dummyX;
  v.flag = &sm.flag;
  ct_chol_tiles<CQ_CHOL_T>(v, n, nrows, strict, floor_d, pub);
}

// stage the lower triangle of a row-major global matrix (rows < nrows, cols < n; rows >= n come from `rhs` when given)
// into the tile-packed layout with 16-byte cp.async (one warp per row, every load of the CTA in flight at once); whole
// diagonal tiles are fetched, everything past the edges is zero-filled. ldG must be even (16-byte aligned row starts).
__device__ void cq_load_tiles(CqCholSmem &sm, const double *__restrict__ G, size_t ldG, int n, int nrows, const double *__restrict__ rhs, int ld_rhs) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int NB = (n + 7) >> 3, NRB = (nrows + 7) >> 3;
  for (int i = wid; i < 8 * NRB; i += CQ_CHOL_T / 32) {
    const double *row = (i >= n && rhs != nullptr) ? rhs + (size_t)(i - n) * ld_rhs : G + (size_t)i * ldG;
    const int jmax = min(i | 7, 8 * NB - 1);
    double *dst = sm.T + (size_t)tri(i >> 3) * 64 + (i & 7) * 8;
    for (int j = 2 * lane; j <= jmax; j += 64) {
      unsigned bytes = 0;
      if (i < nrows)
        bytes = (j + 1 < n) ? 16u : (j < n ? 8u : 0u);
      cpa16(s_u32(dst + (size_t)(j >> 3) * 64 + (j & 7)), bytes ? (const void *)(row + j) : (const void *)G, bytes);
    }
  }
  cpa_commit();
  for (int e = tid; e < 2 * CQ_MAXRB * 8 * CQ_XP; e += CQ_CHOL_T)
    (&sm.Xp[0][0])[e] = 0.0;
  if (tid < 64)
    sm.dummyT[tid] = 0.0;
  if (tid < 2 * CQ_XP)
    sm.dummyX[tid] = 0.0;
  if (tid == 0)
    sm.flag = 0;
  cpa_wait<0>();
}

__device__ __forceinline__ double cq_el(const double *T, int i, int j) { return T[(size_t)(tri(i >> 3) + (j >> 3)) * 64 + (i & 7) * 8 + (j & 7)]; }

} // namespace

// Gram mode: L L' = G + shift_rel * max(diag G) * I; writes L (= R') in the packed layout above to Lpk. ldG even.
// pub_ctr != nullptr: streams L to the next kernel on that counter (see cq_pub_store).
__global__ void __launch_bounds__(CQ_CHOL_T) k_cq_chol_gram(const double *__restrict__ G, int ldG, int n, double shift_rel, double *__restrict__ Lpk, int tiled,
                                                           unsigned long long *pub_ctr, unsigned long long epoch) {
  OVB_PDL_ENTER();
  if (pub_ctr != nullptr && threadIdx.x == 0)
    cq_pub_store(pub_ctr, (epoch << 6) | 1ull);
  const CqPublish pub{Lpk, pub_ctr, epoch, n};
  extern __shared__ __align__(16) unsigned char cq_raw[];
  CqCholSmem &sm = *reinterpret_cast<CqCholSmem *>(cq_raw);
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
#ifdef CQ_PROBE
  const long long q0 = clock64();
#endif
  if (tiled) {
    // G is already tile-packed (k_cq_reduce): one bulk copy (TMA engine) on an mbarrier instead of a scatter of 16-byte cp.asyncs
    __shared__ __align__(8) unsigned long long g_bar;
    const unsigned bar = s_u32(&g_bar);
    const int NB = (n + 7) >> 3;
    if (tid == 0) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar) : "memory");
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0) {
      const unsigned bytes = (unsigned)(tri(NB) * 64 * sizeof(double));
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(s_u32(sm.T)), "l"(G), "r"(bytes), "r"(bar)
                   : "memory");
    }
    for (int e = tid; e < 2 * CQ_MAXRB * 8 * CQ_XP; e += CQ_CHOL_T)
      (&sm.Xp[0][0])[e] = 0.0;
    if (tid < 64)
      sm.dummyT[tid] = 0.0;
    if (tid < 2 * CQ_XP)
      sm.dummyX[tid] = 0.0;
    if (tid == 0)
      sm.flag = 0;
    asm volatile("{\n\t.reg .pred p;\n\tCQ_GWAIT:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n\t@p bra CQ_GDONE;\n\tbra CQ_GWAIT;\n\tCQ_GDONE:\n\t}" ::"r"(bar)
                 : "memory");
    // rows past n of the last block row are whatever an earlier, wider system left in G: the factorisation multiplies the
    // padding by zeros, so it has to BE zero
    const int r0 = n - 8 * (NB - 1);
    if (r0 < 8) {
      double *last = sm.T + (size_t)tri(NB - 1) * 64;
      for (int e = tid; e < NB * 64; e += CQ_CHOL_T)
        if (((e >> 3) & 7) >= r0)
          last[e] = 0.0;
    }
  } else {
    cq_load_tiles(sm, G, (size_t)ldG, n, n, nullptr, 0);
  }
  __syncthreads();
  // largest diagonal entry -> shift
  double mx = 0.0;
  for (int i = tid; i < n; i += CQ_CHOL_T) {
    const double d = sm.T[(size_t)(tri(i >> 3) + (i >> 3)) * 64 + (i & 7) * 9];
    mx = (d > mx) ? d : mx;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double y = __shfl_xor_sync(0xffffffffu, mx, o);
    mx = (y > mx) ? y : mx;
  }
  if (lane == 0)
    sm.red[wid] = mx;
  __syncthreads();
  mx = 0.0;
  for (int w = 0; w < CQ_CHOL_T / 32; w++)
    mx = (sm.red[w] > mx) ? sm.red[w] : mx;
  const double shift = shift_rel * mx;
  for (int i = tid; i < n; i += CQ_CHOL_T)
    sm.T[(size_t)(tri(i >> 3) + (i >> 3)) * 64 + (i & 7) * 9] += shift;
  __syncthreads();
#ifdef CQ_PROBE
  const long long q1 = clock64();
#endif
  cq_chol_tiles(sm, n, n, false, 0.25 * shift, pub);
#ifdef CQ_PROBE
  const long long q2 = clock64();
#endif
  const int NB = (n + 7) >> 3;
  for (int e = pub.first_tile_el() + 2 * tid; e < tri(NB) * 64; e += 2 * CQ_CHOL_T)
    *reinterpret_cast<double2 *>(Lpk + e) = *reinterpret_cast<const double2 *>(sm.T + e);
  for (int e = pub.first_pivot() + tid; e < CQ_MAXB * 8; e += CQ_CHOL_T)
    Lpk[CQ_PK_INV + e] = (e < n) ? sm.invd[e] : 1.0;
  pub.finish();
#ifdef CQ_PROBE
  if (tid == 0)
    printf("chol_gram n=%d: load %lld factor %lld store %lld cycles\n", n, q1 - q0, q2 - q1, clock64() - q2);
#endif
}

// Block mode — EKF (StateHelper::EKFUpdate's LLT, state/StateHelper.cpp:160-161) and the diagonal blocks of the blocked
// factorisation of wide systems: S (r x r, lower triangle in global memory), optionally with the residual as one right-hand-
// side row (res != nullptr) -> L written back over the lower triangle of S, w = L^-1 res, 1/diag(L), the packed factor for
// k_cq_trsm. floor_dev == nullptr: strict, a non-positive pivot raises info->not_spd; else pivots are floored at *floor_dev
// (shifted Gram matrices). ldS even. pub_ctr != nullptr (requires Lpk): streams the packed factor to the next kernel on
// that counter (see cq_pub_store), ahead of the other outputs.
__global__ void __launch_bounds__(CQ_CHOL_T) k_cq_chol_ekf(double *__restrict__ S, int ldS, int r, const double *__restrict__ res, double *__restrict__ w,
                                                          double *__restrict__ invdiag, DevUpdateInfo *__restrict__ info, double *__restrict__ Lpk,
                                                          const double *__restrict__ floor_dev, unsigned long long *pub_ctr, unsigned long long epoch) {
  OVB_PDL_ENTER();
  if (pub_ctr != nullptr && threadIdx.x == 0)
    cq_pub_store(pub_ctr, (epoch << 6) | 1ull);
  const CqPublish pub{Lpk, pub_ctr, epoch, r};
  extern __shared__ __align__(16) unsigned char cq_raw[];
  CqCholSmem &sm = *reinterpret_cast<CqCholSmem *>(cq_raw);
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int nrows = r + (res != nullptr ? 1 : 0);
  cq_load_tiles(sm, S, (size_t)ldS, r, nrows, res, 0);
  __syncthreads();
  if (floor_dev != nullptr)
    cq_chol_tiles(sm, r, nrows, false, *floor_dev, pub);
  else
    cq_chol_tiles(sm, r, nrows, true, 0.0, pub);
  if (Lpk != nullptr) { // the factor as k_cq_trsm consumes it (Y = M L^-T)
    const int NB = (r + 7) >> 3;
    for (int e = pub.first_tile_el() + 2 * tid; e < tri(NB) * 64; e += 2 * CQ_CHOL_T)
      *reinterpret_cast<double2 *>(Lpk + e) = *reinterpret_cast<const double2 *>(sm.T + e);
    for (int e = pub.first_pivot() + tid; e < CQ_MAXB * 8; e += CQ_CHOL_T)
      Lpk[CQ_PK_INV + e] = (e < r) ? sm.invd[e] : 1.0;
    pub.finish();
  }
  for (int i = wid; i < r; i += CQ_CHOL_T / 32)
    for (int j = lane; j <= i; j += 32)
      S[(size_t)i * ldS + j] = cq_el(sm.T, i, j);
  if (res != nullptr)
    for (int j = tid; j < r; j += CQ_CHOL_T)
      w[j] = cq_el(sm.T, r, j);
  if (invdiag != nullptr)
    for (int j = tid; j < r; j += CQ_CHOL_T)
      invdiag[j] = sm.invd[j];
  if (tid == 0 && sm.flag && info != nullptr)
    info->not_spd = 1;
}

// ------------------------------------------------------------------------------------------------------------ TRSM
// A <- A R^-1 in place, R = L' upper triangular nt x nt (nt <= CQ_MAXN). One warp owns 8 rows, whose column blocks live
// in registers as DMMA accumulator fragments. The columns are taken in two halves of NH blocks so that a row group
// needs 2*NH accumulator doubles per lane: 20 warps (row groups) are resident per SM and the FP64 tensor pipe always has
// somebody's DMMAs to run while the others sit in their substitution chains. Within a half, right-looking:
//   gather   the four lanes of a quad exchange their column pairs, so every lane holds its row's 8 entries of the block
//   solve    x R_jj = v by substitution in registers, redundantly in the four lanes (backward stable row by row; the
//            dependent chain is one multiply + one FMA per column, no shuffle on it)
//   push     the solved block IS then the A-operand (register select): -X_j R[j][j+1..] goes into the later blocks of
//            the half with independent DMMAs; the fragments are also parked in shared memory for the second half,
//            which starts with the plain product  A[:, half 2] -= X[:, half 1] R[half 1, half 2].
// L sits in shared memory in the Cholesky kernel's tile layout: tile (j, jb) read at g*8 + 4ks + q is exactly the
// B-operand fragment of R[8jb.., 8j..] (conflict free).
#define CQ_TRSM_NH 10 // column blocks per half (at most)
#define CQ_TRSM_SMEM (sizeof(double) * ((size_t)CQ_PK_DOUBLES + (size_t)(CQ_TRSM_T / 32) * CQ_TRSM_NH * 2 * 32))
// All control flow around the DMMAs is compile-time (NH blocks, padded with zero tiles): a run-time bound inside the
// unrolled loops makes the compiler guard every mma.sync / shfl.sync with convergence code and several code versions.
// WAIT: the factor is streaming in (cq_stream_fetch); block B reads block column B only, so it waits for mbarrier
// cbar + 8B first.
template <int NH, bool WAIT = false>
__device__ __forceinline__ void cq_trsm_half(double (&acc)[NH][2], int b0, const double *Lt, const double *Ri, double *xs, int lane, unsigned cbar = 0) {
  const int g = lane >> 2, q = lane & 3;
#pragma unroll
  for (int jb = 0; jb < NH; jb++) {
    const int B = b0 + jb;
    if constexpr (WAIT)
      cq_mbar_wait(cbar + 8 * B);
    const double *Ld = Lt + (size_t)(tri(B) + B) * 64; // R[8B+t][8B+c] = Ld[c*8 + t], t <= c
    const double *ri = Ri + B * 8;
    double x[8];
#pragma unroll
    for (int qq = 0; qq < 4; qq++) {
      x[2 * qq] = __shfl_sync(0xffffffffu, acc[jb][0], (lane & ~3) | qq);
      x[2 * qq + 1] = __shfl_sync(0xffffffffu, acc[jb][1], (lane & ~3) | qq);
    }
#pragma unroll
    for (int c = 0; c < 8; c++) {
      x[c] *= ri[c];
#pragma unroll
      for (int c2 = c + 1; c2 < 8; c2++)
        x[c2] -= x[c] * Ld[c2 * 8 + c];
    }
    acc[jb][0] = (q == 0) ? x[0] : (q == 1) ? x[2] : (q == 2) ? x[4] : x[6];
    acc[jb][1] = (q == 0) ? x[1] : (q == 1) ? x[3] : (q == 2) ? x[5] : x[7];
    // A-operand fragments of the two k-steps: element (row g, column 4ks + q), negated
    const double af0 = -((q == 0) ? x[0] : (q == 1) ? x[1] : (q == 2) ? x[2] : x[3]);
    const double af1 = -((q == 0) ? x[4] : (q == 1) ? x[5] : (q == 2) ? x[6] : x[7]);
    if (xs != nullptr) {
      xs[(2 * jb) * 32 + lane] = af0;
      xs[(2 * jb + 1) * 32 + lane] = af1;
    }
#pragma unroll
    for (int j = jb + 1; j < NH; j++) {
      const double *lf = Lt + (size_t)(tri(b0 + j) + B) * 64 + g * 8 + q;
      dmma(acc[j][0], acc[j][1], af0, lf[0]);
      dmma(acc[j][0], acc[j][1], af1, lf[4]);
    }
  }
}

template <int NH>
__device__ __forceinline__ void cq_trsm_load(double (&acc)[NH][2], const double *arow, bool row_ok, int b0, int nt, int q) {
#pragma unroll
  for (int jb = 0; jb < NH; jb++) {
    const int col = 8 * (b0 + jb) + 2 * q;
    acc[jb][0] = acc[jb][1] = 0.0;
    if (row_ok) {
      if (col + 1 < nt) {
        const double2 v = *reinterpret_cast<const double2 *>(arow + col);
        acc[jb][0] = v.x;
        acc[jb][1] = v.y;
      } else if (col < nt) {
        acc[jb][0] = arow[col];
      }
    }
  }
}
template <int NH>
__device__ __forceinline__ void cq_trsm_store(const double (&acc)[NH][2], double *arow, bool row_ok, int b0, int nt, int q) {
  if (!row_ok)
    return;
#pragma unroll
  for (int jb = 0; jb < NH; jb++) {
    const int col = 8 * (b0 + jb) + 2 * q;
    if (col + 1 < nt)
      *reinterpret_cast<double2 *>(arow + col) = make_double2(acc[jb][0], acc[jb][1]);
    else if (col < nt)
      arow[col] = acc[jb][0];
  }
}

// The packed factor into shared memory, padded to NBP blocks (tiles past NB zero, their reciprocal pivots 1). It (up to
// 106 KB, contiguous) arrives as two bulk copies (TMA engine, SASS UBLKCP) signalled on an mbarrier: one instruction issues
// them, nobody spends issue slots or registers on the transfer. Ends with a barrier; NT = threads of the CTA.
template <int NBP, int NT>
__device__ __forceinline__ void cq_fetch_factor(double *Lt, double *Ri, const double *__restrict__ Lpk, int NB) {
  const int tid = threadIdx.x;
  __shared__ __align__(8) unsigned long long l_bar;
  const unsigned bar = s_u32(&l_bar);
  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) {
    const unsigned bytesL = (unsigned)(tri(NB) * 64 * sizeof(double)), bytesR = (unsigned)(NB * 8 * sizeof(double));
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytesL + bytesR) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(s_u32(Lt)), "l"(Lpk), "r"(bytesL), "r"(bar)
                 : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(s_u32(Ri)), "l"(Lpk + CQ_PK_INV), "r"(bytesR),
                 "r"(bar)
                 : "memory");
  }
  for (int e = tri(NB) * 64 + tid; e < tri(NBP) * 64; e += NT)
    Lt[e] = 0.0;
  for (int e = NB * 8 + tid; e < NBP * 8; e += NT)
    Ri[e] = 1.0;
  asm volatile("{\n\t.reg .pred p;\n\tCQ_LWAIT:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n\t@p bra CQ_LDONE;\n\tbra CQ_LWAIT;\n\tCQ_LDONE:\n\t}" ::"r"(bar)
               : "memory");
  __syncthreads();
}

// Consumer side of the factor streaming (see cq_pub_store). bars: NBP + 1 mbarriers in shared memory. bars[0] completes
// once the producer has passed its griddepcontrol.wait (from then on the consumer may touch its inputs and outputs),
// bars[1 + j] once block column j of the factor is in Lt / Ri, at the positions cq_fetch_factor fills. Ends with a
// barrier of all NT threads.
template <int NBP, int NT>
__device__ __forceinline__ void cq_stream_init(unsigned long long *bars, double *Lt, double *Ri, int NB) {
  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int j = 0; j <= NBP; j++)
      cq_mbar_init(s_u32(bars + j));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int e = tri(NB) * 64 + tid; e < tri(NBP) * 64; e += NT)
    Lt[e] = 0.0;
  for (int e = NB * 8 + tid; e < NBP * 8; e += NT)
    Ri[e] = 1.0;
  __syncthreads();
}

// How long the consumer polls before it stops (ns): far beyond a factorisation (tens of us); a time-sliced GPU may
// still get there, so the consumer then waits for the producer grid to complete and takes the rest of the factor at once.
#define CQ_STREAM_POLL_NS 20000000ull

// One thread of a warp that does nothing else: polls the counter (backing off with __nanosleep) and bulk-copies each
// block column of the factor as it is published; the padding columns NB..NBP-1 (cq_stream_init) complete at once.
// Returns once every copy has landed and the producer grid has completed (griddepcontrol.wait): a consumer never
// completes before its producer, so the kernels after it see the producer's other outputs in plain stream order.
__device__ void cq_stream_fetch(unsigned long long *bars, double *Lt, double *Ri, const double *__restrict__ Lpk, int NB, int NBP,
                                const unsigned long long *ctr, unsigned long long epoch) {
  const unsigned long long base = epoch << 6;
  unsigned long long t0, t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  bool poll = true;
  auto reach = [&](int s) {
    while (poll && cq_pub_load(ctr) < (base | (unsigned long long)s)) {
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      if (t - t0 > CQ_STREAM_POLL_NS) {
        asm volatile("griddepcontrol.wait;" ::: "memory");
        poll = false;
      } else {
        __nanosleep(64);
      }
    }
  };
  reach(1);
  cq_mbar_arrive(s_u32(bars));
  for (int j = NB; j < NBP; j++)
    cq_mbar_arrive(s_u32(bars + 1 + j));
  for (int j = 0; j < NB; j++) {
    reach(j + 2);
    cq_fence_proxy();
    const unsigned bar = s_u32(bars + 1 + j);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"((unsigned)((NB - j) * 64 + 8) * 8u) : "memory");
    for (int i = j; i < NB; i++) {
      const size_t o = (size_t)(tri(i) + j) * 64;
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], 512, [%2];" ::"r"(s_u32(Lt + o)), "l"(Lpk + o), "r"(bar)
                   : "memory");
    }
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], 64, [%2];" ::"r"(s_u32(Ri + 8 * j)), "l"(Lpk + CQ_PK_INV + 8 * j),
                 "r"(bar)
                 : "memory");
  }
  asm volatile("griddepcontrol.wait;" ::: "memory");
  for (int j = 0; j < NB; j++)
    cq_mbar_wait(s_u32(bars + 1 + j));
}

// NH1 + NH2 >= ceil(nt / 8); NH2 == 0: single half. STREAM: the factor streams in from the k_cq_chol_ekf launched just
// before on (pub_ctr, epoch), fetched by the last warp (a 21st warp would cut the registers per thread from 96 to 80);
// the other warps take the row groups and read their rows once that producer has passed its own wait.
template <int NH1, int NH2, bool STREAM>
__device__ __forceinline__ void cq_trsm_rows(double *__restrict__ A, int ldA, int m, int nt, const double *__restrict__ Lpk,
                                             const unsigned long long *__restrict__ pub_ctr, unsigned long long epoch) {
  extern __shared__ __align__(16) double tsm[];
  double *Lt = tsm;
  double *Ri = tsm + CQ_PK_INV;
  double *Xs = tsm + CQ_PK_DOUBLES; // per warp: first-half A-operand fragments [NH1][2][32]
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, g = lane >> 2, q = lane & 3;
  unsigned cbar = 0;
  if constexpr (STREAM) {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    __shared__ __align__(8) unsigned long long bars[CQ_MAXB + 1];
    cq_stream_init<NH1 + NH2, CQ_TRSM_T>(bars, Lt, Ri, (nt + 7) >> 3);
    if (wid == CQ_TRSM_T / 32 - 1) {
      if (lane == 0)
        cq_stream_fetch(bars, Lt, Ri, Lpk, (nt + 7) >> 3, NH1 + NH2, pub_ctr, epoch);
      return;
    }
    cq_mbar_wait(s_u32(bars));
    cbar = s_u32(bars + 1);
  } else {
    OVB_PDL_ENTER();
    cq_fetch_factor<NH1 + NH2, CQ_TRSM_T>(Lt, Ri, Lpk, (nt + 7) >> 3);
  }
  double *xs = Xs + (size_t)wid * (CQ_TRSM_NH * 2 * 32);
  const int ngroups = (m + 7) >> 3;
  // row groups are dealt round-robin over the CTAs first (warp w of CTA b takes group b + w * gridDim.x): a short matrix puts
  // one group on each SM instead of twenty on the first
  constexpr int NSW = CQ_TRSM_T / 32 - (STREAM ? 1 : 0); // solving warps
  for (int rg = blockIdx.x + gridDim.x * wid; rg < ngroups; rg += gridDim.x * NSW) {
    const int row = 8 * rg + g;
    const bool row_ok = row < m;
    double *arow = A + (size_t)row * ldA;
#ifdef CQ_PROBE
    long long t0 = clock64(), t1, t2, t3 = 0, t4 = 0;
#endif
    {
      double acc[NH1][2];
      cq_trsm_load<NH1>(acc, arow, row_ok, 0, nt, q);
#ifdef CQ_PROBE
      t1 = clock64();
#endif
      cq_trsm_half<NH1, STREAM>(acc, 0, Lt, Ri, NH2 > 0 ? xs : nullptr, lane, cbar);
#ifdef CQ_PROBE
      t2 = clock64();
#endif
      cq_trsm_store<NH1>(acc, arow, row_ok, 0, nt, q);
    }
    if constexpr (NH2 > 0) {
      double acc[NH2][2];
      cq_trsm_load<NH2>(acc, arow, row_ok, NH1, nt, q);
      __syncwarp();
      // A[:, half 2] -= X[:, half 1] R[half 1, half 2]
#pragma unroll 2
      for (int jb = 0; jb < NH1; jb++) {
        const double af0 = xs[(2 * jb) * 32 + lane], af1 = xs[(2 * jb + 1) * 32 + lane];
#pragma unroll
        for (int j = 0; j < NH2; j++) {
          const double *lf = Lt + (size_t)(tri(NH1 + j) + jb) * 64 + g * 8 + q;
          dmma(acc[j][0], acc[j][1], af0, lf[0]);
          dmma(acc[j][0], acc[j][1], af1, lf[4]);
        }
      }
#ifdef CQ_PROBE
      t3 = clock64();
#endif
      cq_trsm_half<NH2, STREAM>(acc, NH1, Lt, Ri, nullptr, lane, cbar);
#ifdef CQ_PROBE
      t4 = clock64();
#endif
      cq_trsm_store<NH2>(acc, arow, row_ok, NH1, nt, q);
      __syncwarp();
    }
#ifdef CQ_PROBE
    if (blockIdx.x == 0 && (tid == 0 || tid == 32 * 7) && rg < 40)
      printf("trsm rg=%d tid=%d: load %lld half1 %lld gemm+load %lld half2 %lld total %lld\n", rg, tid, t1 - t0, t2 - t1, t3 - t2, t4 - t3, clock64() - t0);
#endif
  }
}
// two overloads of one kernel name: the streaming one takes the counter
template <int NH1, int NH2>
__global__ void __launch_bounds__(CQ_TRSM_T) k_cq_trsm(double *__restrict__ A, int ldA, int m, int nt, const double *__restrict__ Lpk) {
  cq_trsm_rows<NH1, NH2, false>(A, ldA, m, nt, Lpk, nullptr, 0);
}
template <int NH1, int NH2>
__global__ void __launch_bounds__(CQ_TRSM_T) k_cq_trsm(double *__restrict__ A, int ldA, int m, int nt, const double *__restrict__ Lpk,
                                                      const unsigned long long *__restrict__ pub_ctr, unsigned long long epoch) {
  cq_trsm_rows<NH1, NH2, true>(A, ldA, m, nt, Lpk, pub_ctr, epoch);
}
using CqTrsmKernel = void (*)(double *, int, int, int, const double *);
using CqTrsmStreamKernel = void (*)(double *, int, int, int, const double *, const unsigned long long *, unsigned long long);

template <bool STREAM>
static void cq_launch_trsm_t(ovb_ctx *ctx, int ctas, double *A, int ldA, int m, int nt, const double *Lpk, const unsigned long long *pub_ctr,
                             unsigned long long epoch) {
  const int NB = (nt + 7) / 8;
  const size_t smem = CQ_TRSM_SMEM;
  const dim3 grid(ctas), block(CQ_TRSM_T);
  auto go = [&](auto plain, auto streaming) {
    if constexpr (STREAM)
      ovb_launch(ctx, streaming, grid, block, smem, A, ldA, m, nt, Lpk, pub_ctr, epoch);
    else
      ovb_launch(ctx, plain, grid, block, smem, A, ldA, m, nt, Lpk);
  };
  if (NB <= 5)
    go((CqTrsmKernel)k_cq_trsm<5, 0>, (CqTrsmStreamKernel)k_cq_trsm<5, 0>);
  else if (NB <= 10)
    go((CqTrsmKernel)k_cq_trsm<10, 0>, (CqTrsmStreamKernel)k_cq_trsm<10, 0>);
  else if (NB <= 15)
    go((CqTrsmKernel)k_cq_trsm<10, 5>, (CqTrsmStreamKernel)k_cq_trsm<10, 5>);
  else
    go((CqTrsmKernel)k_cq_trsm<10, 10>, (CqTrsmStreamKernel)k_cq_trsm<10, 10>);
}
// pub_ctr != nullptr: the factor streams in from the factor kernel launched just before on (pub_ctr, epoch)
static void cq_launch_trsm(ovb_ctx *ctx, int ctas, double *A, int ldA, int m, int nt, const double *Lpk, const unsigned long long *pub_ctr = nullptr,
                           unsigned long long epoch = 0) {
  if (pub_ctr != nullptr)
    cq_launch_trsm_t<true>(ctx, ctas, A, ldA, m, nt, Lpk, pub_ctr, epoch);
  else
    cq_launch_trsm_t<false>(ctx, ctas, A, ldA, m, nt, Lpk, pub_ctr, epoch);
}

// ------------------------------------------------------------------------------------------------------------ pass 2: solve + Gram
// G2 = Q1'Q1 without Q1 in global memory: the Gram partials of pass 2 straight from A and the packed R1. One CTA per Gram
// slab (pass 1's slabs), CQ_GRAM_T threads, R1 in shared memory as k_cq_trsm holds it. The slab is taken in rounds
// through a shared buffer of `cb` rows, staged as k_cq_gram stages its rows (cp.async, row-major, zero fill past nt and
// past the slab). When the slab's last rows exceed the buffer but not one 8-row group per warp, that last round splits:
// its first rows (a whole number of row groups) go through the buffer, the rest through a per-slab scratch in global
// memory laid out alike, so every row group of the round solves at once:
//   solve   warp w solves rows 8w..8w+7 of the round with k_cq_trsm's row solve (per-row arithmetic unchanged), in place
//           in the buffer or the scratch; the second half takes its A-operands from the solved first half there
//   Gram    the tile warps run k_cq_gram's k-steps over the buffer, then over the scratch rows
// Same slabs, same k-step order, zero rows contributing exact zeros: the partials are bit for bit those k_cq_gram forms
// from a stored Q1, and A is left as it was. Between rounds each tile warp parks its accumulators in its own Gpart slot
// (exact), so neither phase carries the other's registers. A buffer row holds all 8*NBP solved columns (at least the
// BW*32 the Gram reads), pitch = 4 mod 16 for conflict-free fragment loads; the padding columns past nt are solved along
// (zeros against a factor that is zero there) and only reach Gram entries past nt, which k_cq_reduce drops. Next to the
// 107 KB factor the buffer holds 92 rows at 155 columns: config 2's 100-row slabs are one split round (88 + 12 rows)
// instead of a 92-row round followed by a second solve of the last 8 rows.
#define CQ_SG_SMEM (226 * 1024) // dynamic shared memory of k_cq_solve_gram, at most (sm_90 opt-in limit 227 KB, static part included)

__host__ __device__ __forceinline__ int cq_sg_pitch(int BW, int NBP) {
  const int w = (8 * NBP > 32 * BW) ? 8 * NBP : 32 * BW;
  return ((w + 15) & ~15) + 4;
}

// one warp's 8-row group solved in place: xrow = the lane's row (8*NBP columns, zero past nt), k_cq_trsm's row solve; the
// second half takes its A-operands from the solved first half in the row. Lanes with !row_ok (past the rows to solve)
// load zeros and store nothing; their xrow must still be a row of the warp's group.
// The factor may still be streaming in: block B of the solve waits for mbarrier cbar + 8B (the second half's leading
// product reads block columns < NH1 only, which the first half has waited for).
template <int NH1, int NH2>
__device__ __forceinline__ void cq_solve_group(double *xrow, bool row_ok, const double *Lt, const double *Ri, int lane, unsigned cbar) {
  constexpr int NBP = NH1 + NH2;
  const int g = lane >> 2, q = lane & 3;
  {
    double acc[NH1][2];
    cq_trsm_load<NH1>(acc, xrow, row_ok, 0, 8 * NBP, q);
    cq_trsm_half<NH1, true>(acc, 0, Lt, Ri, nullptr, lane, cbar);
    cq_trsm_store<NH1>(acc, xrow, row_ok, 0, 8 * NBP, q);
  }
  if constexpr (NH2 > 0) {
    double acc[NH2][2];
    __syncwarp();
    cq_trsm_load<NH2>(acc, xrow, row_ok, NH1, 8 * NBP, q);
    // A[:, half 2] -= X[:, half 1] R[half 1, half 2]; the A-operand of row g, column 8jb + 4ks + q is the solved X, negated
#pragma unroll 2
    for (int jb = 0; jb < NH1; jb++) {
      const double af0 = -xrow[8 * jb + q], af1 = -xrow[8 * jb + 4 + q];
#pragma unroll
      for (int j = 0; j < NH2; j++) {
        const double *lf = Lt + (size_t)(tri(NH1 + j) + jb) * 64 + g * 8 + q;
        dmma(acc[j][0], acc[j][1], af0, lf[0]);
        dmma(acc[j][0], acc[j][1], af1, lf[4]);
      }
    }
    cq_trsm_half<NH2, true>(acc, NH1, Lt, Ri, nullptr, lane, cbar);
    cq_trsm_store<NH2>(acc, xrow, row_ok, NH1, 8 * NBP, q);
  }
}

// R1 streams in from pass 1's k_cq_chol_gram on (pub_ctr, epoch): the first round's rows are issued as soon as that
// kernel has passed its own wait, so they load while the pivot chain runs, and each row group's solve follows the
// factor block column by block column. Warp 15 fetches the factor (cq_stream_fetch; a 17th warp would cut the registers
// per thread from 128 to 96) and only then joins the first round: it solves its row group there, if the round has
// one, after the last block column has come in. The Gram tiles take warps 0..14 at most.
template <int NH1, int NH2>
__global__ void __launch_bounds__(CQ_GRAM_T) k_cq_solve_gram(const double *__restrict__ A, int ldA, int m, int nt, const double *__restrict__ Lpk, int slab_rows,
                                                          int cb, int ntail_max, int BW, double *__restrict__ Gpart, double *__restrict__ Qtail,
                                                          const unsigned long long *__restrict__ pub_ctr, unsigned long long epoch) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  extern __shared__ __align__(16) double ssm[];
  double *Lt = ssm;
  double *Ri = ssm + CQ_PK_INV;
  double *X = ssm + CQ_PK_DOUBLES; // buffer [cb][pitch]
  constexpr int NBP = NH1 + NH2;
  const int pitch = cq_sg_pitch(BW, NBP);
  const int r0 = blockIdx.x * slab_rows, r1 = min(m, r0 + slab_rows);
  double *tail = Qtail + (size_t)blockIdx.x * ntail_max * pitch;
  // the last round splits when its rows exceed the buffer but not one row group per warp
  auto split_at = [&](int rc) { return r1 - rc > cb && r1 - rc <= 8 * (CQ_GRAM_T / 32); };
  // rows the buffer takes in the round at rc (a partial k-step is padded with zero rows)
  auto nbuf_at = [&](int rc) { return split_at(rc) ? cb & ~7 : min(cb, (r1 - rc + 3) & ~3); };
  constexpr int NF = CQ_GRAM_T - 32; // threads other than the fetching warp
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, g = lane >> 2, q = lane & 3, lr = 8 * wid + g;
  const bool fetcher = threadIdx.x >= NF;
  __shared__ __align__(8) unsigned long long bars[CQ_MAXB + 1];
  cq_stream_init<NBP, CQ_GRAM_T>(bars, Lt, Ri, (nt + 7) >> 3);
  const unsigned cbar = s_u32(bars + 1);
  if (fetcher) {
    if (lane == 0)
      cq_stream_fetch(bars, Lt, Ri, Lpk, (nt + 7) >> 3, NBP, pub_ctr, epoch);
    __syncwarp();
  } else {
    cq_mbar_wait(s_u32(bars)); // A may be read, Gpart and the scratch written (pass 1's k_cq_reduce has completed)
    // the first round's rows are in flight while the factor arrives
    if (r0 < r1)
      cq_issue_rows<NF>(X, pitch, A, ldA, r0, nbuf_at(r0), r1, nt, 0, 0, pitch - 4, 1);
  }
  for (int rc = r0, nbuf = nbuf_at(r0), ntail = 0; rc < r1; rc += nbuf + ntail, nbuf = nbuf_at(rc)) {
    ntail = split_at(rc) ? (r1 - rc - nbuf + 3) & ~3 : 0;
    const int nact = nbuf + ntail;
    const bool first = rc == r0;
    if (!first)
      cq_issue_rows<CQ_GRAM_T>(X, pitch, A, ldA, rc, nbuf, r1, nt, 0, 0, pitch - 4, 1);
    // the rows past the buffer into the scratch, zero-padded like the buffer (the solve then reads every row alike)
    if (!(first && fetcher))
      for (int e = threadIdx.x; e < ntail * (pitch - 4); e += first ? NF : CQ_GRAM_T) {
        const int k = e / (pitch - 4), col = e - k * (pitch - 4), r = rc + nbuf + k;
        tail[(size_t)k * pitch + col] = (r < r1 && col < nt) ? A[(size_t)r * ldA + col] : 0.0;
      }
    cpa_wait<0>();
    if (!first) {
      bar_group(1, CQ_GRAM_T);
    } else if (fetcher) { // the rows the others staged (named barrier 3), once the whole factor is in
      asm volatile("bar.sync 3, %0;" ::"n"(CQ_GRAM_T) : "memory");
    } else {
      asm volatile("bar.arrive 3, %0;" ::"n"(CQ_GRAM_T) : "memory");
      bar_group(2, NF);
    }
    // a row group is all in the buffer or all in the scratch
    if (8 * wid < nbuf)
      cq_solve_group<NH1, NH2>(X + (size_t)min(lr, nbuf - 1) * pitch, lr < nbuf, Lt, Ri, lane, cbar);
    else if (8 * wid < nact)
      cq_solve_group<NH1, NH2>(tail + (size_t)min(lr - nbuf, ntail - 1) * pitch, lr < nact, Lt, Ri, lane, cbar);
    bar_group(1, CQ_GRAM_T);
    int ci, cj, offI, offJ;
    bool diag;
    const bool active = cq_tile_origin(0, wid, BW, 1, ci, cj, offI, offJ, diag);
    double *part = Gpart + ((size_t)blockIdx.x * 16 + wid) * 1024 + g * 32 + 2 * q; // k_cq_gram's cs = 1 layout (one block)
    if (active) {
      double acc[4][4][2];
#pragma unroll
      for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = 0; b < 4; b++) {
          const double2 v = rc > r0 ? *reinterpret_cast<const double2 *>(part + a * 256 + 8 * b) : make_double2(0.0, 0.0);
          acc[a][b][0] = v.x;
          acc[a][b][1] = v.y;
        }
      // the buffer's k-steps, then the scratch rows' where they are (a few k-steps: no second staging and barrier)
#pragma unroll 1 // unrolled, the loads run ahead and the solve phase spills
      for (int k = 0; k < nact; k += 4)
        cq_gram_kstep(acc, k < nbuf ? X + (size_t)k * pitch : tail + (size_t)(k - nbuf) * pitch, pitch, offI, offJ, offI == offJ, g, q);
#pragma unroll
      for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = 0; b < 4; b++)
          *reinterpret_cast<double2 *>(part + a * 256 + 8 * b) = make_double2(acc[a][b][0], acc[a][b][1]);
    }
    bar_group(1, CQ_GRAM_T);
  }
}

// Geometry of k_cq_solve_gram for slabs of slab_rows rows (a multiple of 4) and BW = ceil(nt / 32): buffer pitch, rows
// the buffer takes per round, and rows per round solved into the scratch (ntail * pitch doubles per slab)
struct CqSgShape {
  int pitch, cb, ntail;
};
static CqSgShape cq_sg_shape(int nt, int BW, int slab_rows) {
  const int NB = (nt + 7) / 8, NBP = NB <= 5 ? 5 : NB <= 10 ? 10 : NB <= 15 ? 15 : 20; // NH1 + NH2 of the instance cq_launch_solve_gram picks
  CqSgShape s;
  s.pitch = cq_sg_pitch(BW, NBP);
  const int round = slab_rows < 8 * (CQ_GRAM_T / 32) ? slab_rows : 8 * (CQ_GRAM_T / 32);
  const int fit = (int)((CQ_SG_SMEM - sizeof(double) * CQ_PK_DOUBLES) / (sizeof(double) * s.pitch)) & ~3;
  s.cb = fit < round ? fit : round;
  s.ntail = slab_rows > s.cb ? round - (s.cb & ~7) : 0; // the split last round: buffer rows end on a row-group boundary
  return s;
}
// scratch doubles the launch below needs at Qtail
static size_t cq_solve_gram_scratch(int nslab, int nt, int BW, int slab_rows) {
  const CqSgShape s = cq_sg_shape(nt, BW, slab_rows);
  return (size_t)nslab * s.ntail * s.pitch;
}

template <int NH1, int NH2>
static void cq_launch_solve_gram_t(ovb_ctx *ctx, int nslab, const double *A, int ldA, int m, int nt, const double *Lpk, int slab_rows, int BW, double *Gpart,
                                   double *Qtail, const unsigned long long *pub_ctr, unsigned long long epoch) {
  const CqSgShape s = cq_sg_shape(nt, BW, slab_rows);
  const size_t smem = sizeof(double) * (CQ_PK_DOUBLES + (size_t)s.cb * s.pitch);
  ovb_launch(ctx, k_cq_solve_gram<NH1, NH2>, dim3(nslab), dim3(CQ_GRAM_T), smem, A, ldA, m, nt, Lpk, slab_rows, s.cb, s.ntail, BW, Gpart, Qtail, pub_ctr, epoch);
}
// slabs of slab_rows rows (a multiple of 4), BW = ceil(nt / 32): the Gram geometry of the narrow path; Qtail: scratch of
// cq_solve_gram_scratch() doubles; Lpk streams in from the k_cq_chol_gram launched just before on (pub_ctr, epoch)
static void cq_launch_solve_gram(ovb_ctx *ctx, int nslab, const double *A, int ldA, int m, int nt, const double *Lpk, int slab_rows, int BW, double *Gpart,
                                 double *Qtail, const unsigned long long *pub_ctr, unsigned long long epoch) {
  const int NB = (nt + 7) / 8;
  if (NB <= 5)
    cq_launch_solve_gram_t<5, 0>(ctx, nslab, A, ldA, m, nt, Lpk, slab_rows, BW, Gpart, Qtail, pub_ctr, epoch);
  else if (NB <= 10)
    cq_launch_solve_gram_t<10, 0>(ctx, nslab, A, ldA, m, nt, Lpk, slab_rows, BW, Gpart, Qtail, pub_ctr, epoch);
  else if (NB <= 15)
    cq_launch_solve_gram_t<10, 5>(ctx, nslab, A, ldA, m, nt, Lpk, slab_rows, BW, Gpart, Qtail, pub_ctr, epoch);
  else
    cq_launch_solve_gram_t<10, 10>(ctx, nslab, A, ldA, m, nt, Lpk, slab_rows, BW, Gpart, Qtail, pub_ctr, epoch);
}

// ------------------------------------------------------------------------------------------------------------ R = R2 R1
// Product of two upper-triangular nt x nt factors; rows 0..n-1 (n = nt - 1) go to Rout = [R | z], lower part zeroed.
// both factors arrive as tile-packed L = R'. 16 x 16 output tile per CTA; the tile's whole K range (at most CQ_MAXN deep) is staged in
// one shot, so a CTA pays one L2 round trip.
__global__ void __launch_bounds__(256) k_cq_trmm(const double *__restrict__ L2, const double *__restrict__ L1, int nt, double *__restrict__ Rout, int ldR) {
  OVB_PDL_ENTER();
  __shared__ double As[16][CQ_MAXN + 1]; // R2[16ti + a][k0 + k]
  __shared__ double Bs[CQ_MAXN][17];     // R1[k0 + k][16tj + b]
  const int ti = blockIdx.y, tj = blockIdx.x;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int n = nt - 1;
  const int i = ti * 16 + ty, j = tj * 16 + tx;
  double acc = 0.0;
  if (tj >= ti) {
    const int k0 = ti * 16, k1 = min(nt, tj * 16 + 16); // R2[i][k] = 0 for k < i, R1[k][j] = 0 for k > j
    const int K = k1 - k0;
    for (int e = tid; e < 16 * K; e += 256) {
      const int a = e / K, k = e - a * K;
      const int ii = ti * 16 + a, kk = k0 + k;
      As[a][k] = (ii < nt && kk >= ii) ? L2[(size_t)(tri(kk >> 3) + (ii >> 3)) * 64 + (kk & 7) * 8 + (ii & 7)] : 0.0; // R2[ii][kk] = L2[kk][ii]
    }
    for (int e = tid; e < 16 * K; e += 256) {
      const int k = e >> 4, b = e & 15;
      const int kk = k0 + k, jj = tj * 16 + b;
      Bs[k][b] = (jj < nt && jj >= kk) ? L1[(size_t)(tri(jj >> 3) + (kk >> 3)) * 64 + (jj & 7) * 8 + (kk & 7)] : 0.0; // R1[kk][jj] = L1[jj][kk]
    }
    __syncthreads();
    double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
    int k = 0;
    for (; k + 3 < K; k += 4) {
      a0 += As[ty][k] * Bs[k][tx];
      a1 += As[ty][k + 1] * Bs[k + 1][tx];
      a2 += As[ty][k + 2] * Bs[k + 2][tx];
      a3 += As[ty][k + 3] * Bs[k + 3][tx];
    }
    for (; k < K; k++)
      a0 += As[ty][k] * Bs[k][tx];
    acc = (a0 + a1) + (a2 + a3);
  }
  if (i < n && j < nt)
    Rout[(size_t)i * ldR + j] = (j >= i) ? acc : 0.0;
}

// ------------------------------------------------------------------------------------------------------------ wide systems
// C[M x N] -= A[M x K] B[N x K]'   (all row-major; DMMA). The trailing update of the blocked Cholesky (A = B = the solved
// panel, lower_only) and the panel update of the blocked triangular solve (A = solved columns, B = rows of L).
// CTA tile 64 x 64, 8 warps as 2 x 4 (warp tile 32 x 16), K in chunks of 32 through shared memory (cp.async, zero fill).
#define CQ_GN_T 256
__global__ void __launch_bounds__(CQ_GN_T) k_cq_gemm_nt(double *__restrict__ C, int ldc, const double *__restrict__ A, int lda, const double *__restrict__ B,
                                                       int ldb, int M, int N, int K, int lower_only) {
  OVB_PDL_ENTER();
  __shared__ __align__(16) double As[64][36];
  __shared__ __align__(16) double Bs[64][36];
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  if (lower_only && n0 > m0 + 63)
    return;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, g = lane >> 2, q = lane & 3;
  const int wm = (wid >> 2) * 32, wn = (wid & 3) * 16;
  double acc[4][2][2];
#pragma unroll
  for (int a = 0; a < 4; a++)
#pragma unroll
    for (int b = 0; b < 2; b++)
      acc[a][b][0] = acc[a][b][1] = 0.0;
  for (int k0 = 0; k0 < K; k0 += 32) {
    for (int e = tid; e < 64 * 16; e += CQ_GN_T) {
      const int r = e >> 4, u = e & 15, k = k0 + 2 * u;
      unsigned ba = 0, bb = 0;
      if (m0 + r < M)
        ba = (k + 1 < K) ? 16u : (k < K ? 8u : 0u);
      if (n0 + r < N)
        bb = (k + 1 < K) ? 16u : (k < K ? 8u : 0u);
      cpa16(s_u32(&As[r][2 * u]), ba ? (const void *)(A + (size_t)(m0 + r) * lda + k) : (const void *)A, ba);
      cpa16(s_u32(&Bs[r][2 * u]), bb ? (const void *)(B + (size_t)(n0 + r) * ldb + k) : (const void *)B, bb);
    }
    cpa_commit();
    cpa_wait<0>();
    __syncthreads();
#pragma unroll
    for (int ks = 0; ks < 8; ks++) {
      double fa[4], fb[2];
#pragma unroll
      for (int a = 0; a < 4; a++)
        fa[a] = As[wm + 8 * a + g][4 * ks + q];
#pragma unroll
      for (int b = 0; b < 2; b++)
        fb[b] = Bs[wn + 8 * b + g][4 * ks + q];
#pragma unroll
      for (int a = 0; a < 4; a += 2)
#pragma unroll
        for (int b = 0; b < 2; b++)
          ct_dmma2(acc[a][b][0], acc[a][b][1], acc[a + 1][b][0], acc[a + 1][b][1], fa[a], fa[a + 1], fb[b]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int a = 0; a < 4; a++)
#pragma unroll
    for (int b = 0; b < 2; b++) {
      const int i = m0 + wm + 8 * a + g, j = n0 + wn + 8 * b + 2 * q;
      if (i < M) {
        double *c = C + (size_t)i * ldc + j;
        if (j + 1 < N) {
          double2 v = *reinterpret_cast<double2 *>(c);
          v.x -= acc[a][b][0];
          v.y -= acc[a][b][1];
          *reinterpret_cast<double2 *>(c) = v;
        } else if (j < N) {
          c[0] -= acc[a][b][0];
        }
      }
    }
}

// max diagonal of G -> G += shift_rel * max * I; *floor_out = shift / 4 (the pivot floor of the block factorisations)
__global__ void __launch_bounds__(256) k_cq_shift(double *__restrict__ G, int ldG, int n, double shift_rel, double *__restrict__ floor_out) {
  OVB_PDL_ENTER();
  __shared__ double red[8];
  double mx = 0.0;
  for (int i = threadIdx.x; i < n; i += 256) {
    const double d = G[(size_t)i * ldG + i];
    mx = (d > mx) ? d : mx;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double y = __shfl_xor_sync(0xffffffffu, mx, o);
    mx = (y > mx) ? y : mx;
  }
  if ((threadIdx.x & 31) == 0)
    red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = 0.0;
  for (int w = 0; w < 8; w++)
    mx = (red[w] > mx) ? red[w] : mx;
  const double shift = shift_rel * mx;
  for (int i = threadIdx.x; i < n; i += 256)
    G[(size_t)i * ldG + i] += shift;
  if (threadIdx.x == 0)
    *floor_out = 0.25 * shift;
}

// R = R2 R1 with R1 = L1', R2 = L2' (plain row-major lower factors): Rout[i][j] = sum_{k=i..j} L2[k][i] L1[j][k], rows i < nt-1
__global__ void __launch_bounds__(256) k_cq_trmm_wide(const double *__restrict__ L2, const double *__restrict__ L1, int ldL, int nt, double *__restrict__ Rout,
                                                     int ldR) {
  OVB_PDL_ENTER();
  __shared__ double As[32][33]; // L2[k][i]
  __shared__ double Bs[32][33]; // L1[j][k]
  const int ti = blockIdx.y, tj = blockIdx.x;
  const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
  const int n = nt - 1;
  double acc[4] = {0, 0, 0, 0};
  if (tj >= ti) {
    for (int tk = ti; tk <= tj; tk++) {
      for (int e = tid; e < 1024; e += 256) {
        const int a = e >> 5, b = e & 31;
        const int k = tk * 32 + a, i = ti * 32 + b;
        As[a][b] = (k < nt && i < nt && k >= i) ? L2[(size_t)k * ldL + i] : 0.0;
        const int j = tj * 32 + a, k2 = tk * 32 + b;
        Bs[a][b] = (j < nt && k2 < nt && j >= k2) ? L1[(size_t)j * ldL + k2] : 0.0;
      }
      __syncthreads();
#pragma unroll 8
      for (int kk = 0; kk < 32; kk++) {
        const double b = Bs[tx][kk];
#pragma unroll
        for (int u = 0; u < 4; u++)
          acc[u] += As[kk][ty + 8 * u] * b;
      }
      __syncthreads();
    }
  }
#pragma unroll
  for (int u = 0; u < 4; u++) {
    const int i = ti * 32 + ty + 8 * u, j = tj * 32 + tx;
    if (i < n && j < nt)
      Rout[(size_t)i * ldR + j] = (j >= i) ? acc[u] : 0.0;
  }
}

// ------------------------------------------------------------------------------------------------------------ launchers
#define CQ_GRAM_CS 4 // slabs per cluster in k_cq_gram

static bool cq_attrs(ovb_ctx *ctx) {
  if (!ctx->attr_done[4]) {
    cudaFuncSetAttribute(k_cq_gram, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
    cudaFuncSetAttribute(k_cq_chol_gram, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CqCholSmem));
    cudaFuncSetAttribute(k_cq_chol_ekf, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CqCholSmem));
    cudaFuncSetAttribute((CqTrsmKernel)k_cq_trsm<5, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CQ_TRSM_SMEM);
    cudaFuncSetAttribute((CqTrsmStreamKernel)k_cq_trsm<5, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CQ_TRSM_SMEM);
    cudaFuncSetAttribute((CqTrsmKernel)k_cq_trsm<10, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CQ_TRSM_SMEM);
    cudaFuncSetAttribute((CqTrsmStreamKernel)k_cq_trsm<10, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CQ_TRSM_SMEM);
    cudaFuncSetAttribute((CqTrsmKernel)k_cq_trsm<10, 5>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CQ_TRSM_SMEM);
    cudaFuncSetAttribute((CqTrsmStreamKernel)k_cq_trsm<10, 5>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CQ_TRSM_SMEM);
    cudaFuncSetAttribute((CqTrsmKernel)k_cq_trsm<10, 10>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CQ_TRSM_SMEM);
    cudaFuncSetAttribute((CqTrsmStreamKernel)k_cq_trsm<10, 10>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CQ_TRSM_SMEM);
    cudaFuncSetAttribute(k_cq_solve_gram<5, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, CQ_SG_SMEM);
    cudaFuncSetAttribute(k_cq_solve_gram<10, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, CQ_SG_SMEM);
    cudaFuncSetAttribute(k_cq_solve_gram<10, 5>, cudaFuncAttributeMaxDynamicSharedMemorySize, CQ_SG_SMEM);
    cudaFuncSetAttribute(k_cq_solve_gram<10, 10>, cudaFuncAttributeMaxDynamicSharedMemorySize, CQ_SG_SMEM);
    ctx->attr_done[4] = 1;
  }
  return true;
}

int ovb_cholqr_max_cols(void) { return CQ_MAXN; }

static bool cq_ensure_G(ovb_ctx *ctx) {
  const int ldW = CQ_MAXN + 8;
  const size_t need_G = (size_t)4 * ldW * ldW; // [G (both passes) | L1 | L2 | EKF factor]
  if (need_G > ctx->G_cap) {
    if (ctx->d_G)
      cudaFree(ctx->d_G);
    ctx->d_G = nullptr;
    if (cudaMalloc(&ctx->d_G, sizeof(double) * need_G) != cudaSuccess)
      return false;
    cudaMemsetAsync(ctx->d_G, 0, sizeof(double) * need_G, ctx->stream); // the tile-packed Gram matrix keeps finite padding
    ctx->G_cap = need_G;
  }
  return true;
}

// EKF Cholesky through the DMMA kernel when S (+ the residual row) fits its tile store. With one right-hand-side row the
// last row block may spill past CQ_MAXB blocks; the packed factor (for the register solve) is only offered when it fits.
// epoch_out != nullptr: the packed factor is streamed to the launch_trsm_rows that follows, on the epoch written there
// (0: not streamed).
bool launch_chol_ekf_dmma(ovb_ctx *ctx, double *S, int ldS, int r, const double *res, double *w, double *invdiag, double **Lpk_out,
                          unsigned long long *epoch_out) {
  if (Lpk_out)
    *Lpk_out = nullptr;
  if (epoch_out)
    *epoch_out = 0;
  if (r + 1 > CQ_MAXRB * 8 || r > CQ_MAXN || (ldS & 1))
    return false;
  cq_attrs(ctx);
  double *Lpk = nullptr;
  if (cq_ensure_G(ctx)) {
    const int ldW = CQ_MAXN + 8;
    Lpk = ctx->d_G + (size_t)3 * ldW * ldW;
  }
  const unsigned long long epoch = (epoch_out != nullptr && Lpk != nullptr) ? ++ctx->pub_epoch : 0;
  ovb_launch(ctx, k_cq_chol_ekf, dim3(1), dim3(CQ_CHOL_T), sizeof(CqCholSmem), S, ldS, r, res, w, invdiag, ctx->d_info, Lpk, (const double *)nullptr,
             epoch ? ctx->d_pub : (unsigned long long *)nullptr, epoch);
  if (Lpk_out)
    *Lpk_out = Lpk;
  if (epoch_out)
    *epoch_out = epoch;
  return true;
}

bool launch_trsm_rows(ovb_ctx *ctx, double *A, int ldA, int m, int nt, const double *Lpk, unsigned long long epoch) {
  if (nt > CQ_MAXN || (ldA & 1) || m < 1 || Lpk == nullptr)
    return false;
  cq_attrs(ctx);
  const int ngroups = (m + 7) / 8;
  // short matrices (the EKF's N rows): one row group per CTA while the SMs last — a row group alone on its SM runs its
  // 20-block substitution chain ~3x faster than four groups sharing the SM's FP64 pipe (tools/ubench/cholqr_bench.cu)
  int ctas = ngroups;
  if (ctas > ctx->sm_count)
    ctas = ctx->sm_count;
  cq_launch_trsm(ctx, ctas, A, ldA, m, nt, Lpk, epoch ? ctx->d_pub : nullptr, epoch);
  return true;
}

// ---- wide systems (more columns than one CTA's Cholesky takes): blocked right-looking factorisation in global memory
#define CQ_WB 128                 // diagonal block of the blocked Cholesky / column panel of the blocked solve
#define CQ_WMAX 520               // leading dimension of the wide Gram buffers (nt <= 513)
#define CQ_WBLOCKS ((CQ_WMAX + CQ_WB - 1) / CQ_WB)
static bool cq_ensure_wide(ovb_ctx *ctx) {
  const size_t need = (size_t)2 * CQ_WMAX * CQ_WMAX + (size_t)2 * CQ_WBLOCKS * CQ_PK_DOUBLES + 64;
  if (need > ctx->cqw_cap) {
    if (ctx->d_cqw)
      cudaFree(ctx->d_cqw);
    ctx->d_cqw = nullptr;
    if (cudaMalloc(&ctx->d_cqw, sizeof(double) * need) != cudaSuccess)
      return false;
    ctx->cqw_cap = need;
  }
  return true;
}
static void cq_gemm_nt(ovb_ctx *ctx, double *C, int ldc, const double *A, int lda, const double *B, int ldb, int M, int N, int K, int lower_only) {
  if (M <= 0 || N <= 0 || K <= 0)
    return;
  ovb_launch(ctx, k_cq_gemm_nt, dim3((N + 63) / 64, (M + 63) / 64), dim3(CQ_GN_T), (size_t)0, C, ldc, A, lda, B, ldb, M, N, K, lower_only);
}
static void cq_trsm_any(ovb_ctx *ctx, double *A, int ldA, int m, int nt, const double *Lpk) {
  const int ngroups = (m + 7) / 8;
  int ctas = (ngroups + CQ_TRSM_T / 32 - 1) / (CQ_TRSM_T / 32);
  if (ngroups <= ctx->sm_count)
    ctas = ngroups; // short panels: one row group per CTA (see launch_trsm_rows)
  if (ctas > ctx->sm_count)
    ctas = ctx->sm_count;
  cq_launch_trsm(ctx, ctas, A, ldA, m, nt, Lpk);
}
// L L' = S for the leading n x n block of the (n + extra) x n lower matrix at S (extra right-hand-side rows below it are
// solved along: they end as rhs L^-T). Lpk: CQ_WBLOCKS packed diagonal-block factors. floor_dev: see k_cq_chol_ekf.
static void cq_chol_blocked(ovb_ctx *ctx, double *S, int ld, int n, int extra, double *Lpk, const double *floor_dev, DevUpdateInfo *info) {
  for (int J = 0, b = 0; J < n; J += CQ_WB, b++) {
    const int nb = (n - J < CQ_WB) ? n - J : CQ_WB;
    double *Lb = Lpk + (size_t)b * CQ_PK_DOUBLES;
    ovb_launch(ctx, k_cq_chol_ekf, dim3(1), dim3(CQ_CHOL_T), sizeof(CqCholSmem), S + (size_t)J * ld + J, ld, nb, (const double *)nullptr, (double *)nullptr,
               (double *)nullptr, info, Lb, floor_dev, (unsigned long long *)nullptr, 0ull);
    const int mrem = n + extra - (J + nb);
    if (mrem > 0) {
      double *panel = S + (size_t)(J + nb) * ld + J;
      cq_trsm_any(ctx, panel, ld, mrem, nb, Lb);
      const int ncols = n - (J + nb);
      cq_gemm_nt(ctx, S + (size_t)(J + nb) * ld + (J + nb), ld, panel, ld, panel, ld, mrem, ncols, nb, 1);
    }
  }
}
// X <- X (L')^-1 for the rows of X [m x n] with the blocked factor (plain L in S, packed diagonal blocks in Lpk)
static void cq_trsm_blocked(ovb_ctx *ctx, double *X, int ldx, int m, int n, const double *S, int ld, const double *Lpk) {
  for (int J = 0, b = 0; J < n; J += CQ_WB, b++) {
    const int nb = (n - J < CQ_WB) ? n - J : CQ_WB;
    if (J > 0) // X[:, J..] -= X[:, 0..J) L[J.., 0..J)'
      cq_gemm_nt(ctx, X + J, ldx, X, ldx, S + (size_t)J * ld, ld, m, nb, J, 0);
    cq_trsm_any(ctx, X + J, ldx, m, nb, Lpk + (size_t)b * CQ_PK_DOUBLES);
  }
}

__global__ void k_cq_copy_row(const double *__restrict__ src, double *__restrict__ dst, int n) {
  OVB_PDL_ENTER();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n)
    dst[i] = src[i];
}
__global__ void k_cq_inv_diag(const double *__restrict__ S, int ld, int n, double *__restrict__ inv) {
  OVB_PDL_ENTER();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const double d = S[(size_t)i * ld + i];
    inv[i] = d != 0.0 ? 1.0 / d : 0.0;
  }
}

bool launch_chol_solve_wide(ovb_ctx *ctx, double *S, int ldS, int r, double *w, double *invdiag, double *M, int ldM, int N, bool gate_only) {
  if (r > CQ_WMAX - 8 || (ldS & 1) || (ldM & 1) || r + 1 > ctx->cfg.max_state + 1)
    return false;
  cq_attrs(ctx);
  if (!cq_ensure_wide(ctx))
    return false;
  double *Lpk = ctx->d_cqw + (size_t)2 * CQ_WMAX * CQ_WMAX;
  // the residual rides as row r of S (solved along with the panels): w = L^-1 res
  ovb_launch(ctx, k_cq_copy_row, dim3((r + 127) / 128), dim3(128), (size_t)0, (const double *)w, S + (size_t)r * ldS, r);
  cq_chol_blocked(ctx, S, ldS, r, 1, Lpk, nullptr, ctx->d_info);
  ovb_launch(ctx, k_cq_copy_row, dim3((r + 127) / 128), dim3(128), (size_t)0, (const double *)(S + (size_t)r * ldS), w, r);
  ovb_launch(ctx, k_cq_inv_diag, dim3((r + 127) / 128), dim3(128), (size_t)0, (const double *)S, ldS, r, invdiag);
  if (!gate_only)
    cq_trsm_blocked(ctx, M, ldM, N, r, S, ldS, Lpk);
  return true;
}

// wide CholeskyQR2: same scheme as below with the blocked factorisation / solve
static bool cq_compress_wide(ovb_ctx *ctx, double *A, int m, int n, int ldA, double *Rout, int ldR) {
  const int nt = n + 1;
  if (nt > CQ_WMAX - 7 || !cq_ensure_wide(ctx))
    return false;
  const int nT = (nt + 31) / 32, BW = 4, nblk_side = (nT + BW - 1) / BW, nblk = nblk_side * (nblk_side + 1) / 2;
  int nslab = ctx->sm_count / nblk;
  if (nslab < 1)
    nslab = 1;
  const int max_slabs = (m + CQ_KB - 1) / CQ_KB;
  if (nslab > max_slabs)
    nslab = max_slabs;
  int slab_rows = (((m + nslab - 1) / nslab) + 3) & ~3;
  nslab = (m + slab_rows - 1) / slab_rows;
  const size_t need_part = (size_t)nslab * nblk * 16 * 1024;
  if (need_part > ctx->Gpart_cap) {
    if (ctx->d_Gpart)
      cudaFree(ctx->d_Gpart);
    ctx->d_Gpart = nullptr;
    if (cudaMalloc(&ctx->d_Gpart, sizeof(double) * need_part) != cudaSuccess)
      return false;
    ctx->Gpart_cap = need_part;
  }
  double *G1 = ctx->d_cqw, *G2 = G1 + (size_t)CQ_WMAX * CQ_WMAX, *Lpk1 = G2 + (size_t)CQ_WMAX * CQ_WMAX, *Lpk2 = Lpk1 + (size_t)CQ_WBLOCKS * CQ_PK_DOUBLES;
  double *floor_dev = Lpk2 + (size_t)CQ_WBLOCKS * CQ_PK_DOUBLES;
  const size_t gram_smem = sizeof(double) * 2 * CQ_KB * (size_t)(2 * BW * 32 + 4);
  for (int pass = 0; pass < 2; pass++) {
    double *G = pass == 0 ? G1 : G2;
    ovb_launch(ctx, k_cq_gram, dim3(nblk, nslab), dim3(CQ_GRAM_T), gram_smem, A, ldA, m, nt, slab_rows, BW, nblk_side, ctx->d_Gpart, 1);
    ovb_launch(ctx, k_cq_reduce, dim3(CQ_RED_GX, nblk), dim3(CQ_RED_T), (size_t)0, (const double *)ctx->d_Gpart, nslab, nblk, BW, nblk_side, nt, G, (int)CQ_WMAX, 0);
    ovb_launch(ctx, k_cq_shift, dim3(1), dim3(256), (size_t)0, G, (int)CQ_WMAX, nt, pass == 0 ? 1e-11 : 1e-13, floor_dev + pass);
    cq_chol_blocked(ctx, G, CQ_WMAX, nt, 0, pass == 0 ? Lpk1 : Lpk2, floor_dev + pass, (DevUpdateInfo *)nullptr);
    if (pass == 0)
      cq_trsm_blocked(ctx, A, ldA, m, nt, G1, CQ_WMAX, Lpk1);
  }
  const int nT32 = (nt + 31) / 32;
  ovb_launch(ctx, k_cq_trmm_wide, dim3(nT32, nT32), dim3(256), (size_t)0, (const double *)G2, (const double *)G1, (int)CQ_WMAX, nt, Rout, ldR);
  return true;
}

// [R | z] <- shifted CholeskyQR2 of A [m x (n+1)]: pass 1 k_cq_gram -> k_cq_reduce -> k_cq_chol_gram, pass 2
// k_cq_solve_gram (Q1 = A R1^-1 and its Gram partials in one kernel) -> k_cq_reduce -> k_cq_chol_gram, then k_cq_trmm.
// A is left unchanged here (the wide path overwrites it with Q1). Returns false when the system is too wide for this
// path (the caller falls back to the Householder TSQR).
bool launch_compress_cholqr2(ovb_ctx *ctx, double *A, int m, int n, int ldA, double *Rout, int ldR) {
  const int nt = n + 1;
  if ((ldA & 1) || m < 1)
    return false;
  cq_attrs(ctx);
  if (nt > CQ_MAXN)
    return cq_compress_wide(ctx, A, m, n, ldA, Rout, ldR);
  const int nT = (nt + 31) / 32; // warp tiles per side (<= 5)
  const int BW = nT, nblk_side = 1, nblk = 1;
  int nslab = ctx->sm_count;
  const int max_slabs = (m + CQ_KB - 1) / CQ_KB;
  if (nslab > max_slabs)
    nslab = max_slabs;
  int slab_rows = (m + nslab - 1) / nslab;
  slab_rows = (slab_rows + 3) & ~3;
  nslab = (m + slab_rows - 1) / slab_rows;
  // clusters of CQ_GRAM_CS slabs pre-reduce their partial tiles in distributed shared memory (empty slabs pad the grid)
  const int cs = (ctx->gram_cluster && nslab >= 2 * CQ_GRAM_CS) ? CQ_GRAM_CS : 1;
  const int nslab_pad = (nslab + cs - 1) / cs * cs, npart = nslab_pad / cs;
  const size_t part_doubles = (size_t)nslab_pad * nblk * 16 * 1024;
  const size_t need_part = part_doubles + cq_solve_gram_scratch(nslab, nt, BW, slab_rows); // partials | pass-2 row scratch
  const int ldW = CQ_MAXN + 8;
  if (!cq_ensure_G(ctx))
    return false;
  if (need_part > ctx->Gpart_cap) {
    // the stacked rows grow over a run's first ~30 updates; taking half as much again keeps regrowth to a few early
    // updates (cudaFree waits for the whole device, other contexts' work included: tools/monte_carlo_timing.py)
    const size_t cap = need_part + need_part / 2;
    if (ctx->d_Gpart)
      cudaFree(ctx->d_Gpart);
    ctx->d_Gpart = nullptr;
    ctx->Gpart_cap = 0;
    if (cudaMalloc(&ctx->d_Gpart, sizeof(double) * cap) != cudaSuccess)
      return false;
    ctx->Gpart_cap = cap;
  }
  double *G = ctx->d_G, *L1 = G + (size_t)ldW * ldW, *L2 = L1 + (size_t)ldW * ldW;
  static_assert(CQ_PK_DOUBLES <= (CQ_MAXN + 8) * (CQ_MAXN + 8), "packed factor must fit its slot");
  size_t gram_smem = sizeof(double) * 2 * CQ_KB * (size_t)(BW * 32 + 4);
  if (cs > 1 && gram_smem < sizeof(double) * 16 * 1024)
    gram_smem = sizeof(double) * 16 * 1024; // staging of the 16 warp tiles for the cluster reduction
  // pass 1: G1 = A'A -> R1
  ovb_launch(ctx, k_cq_gram, ovb_grid(dim3(nblk, nslab_pad), dim3(1, cs, 1)), dim3(CQ_GRAM_T), gram_smem, A, ldA, m, nt, slab_rows, BW, nblk_side,
             ctx->d_Gpart, cs);
  ovb_launch(ctx, k_cq_reduce, dim3(CQ_RED_GX, nblk), dim3(CQ_RED_T), (size_t)0, (const double *)ctx->d_Gpart, npart, nblk, BW, nblk_side, nt, G, ldW, 1);
  const unsigned long long epoch = ++ctx->pub_epoch; // R1 streams into k_cq_solve_gram
  ovb_launch(ctx, k_cq_chol_gram, dim3(1), dim3(CQ_CHOL_T), sizeof(CqCholSmem), (const double *)G, ldW, nt, 1e-11, L1, 1, ctx->d_pub, epoch);
  // pass 2: G2 = Q1'Q1 (one partial per slab, no cluster) -> R2
  cq_launch_solve_gram(ctx, nslab, (const double *)A, ldA, m, nt, (const double *)L1, slab_rows, BW, ctx->d_Gpart, ctx->d_Gpart + part_doubles, ctx->d_pub, epoch);
  ovb_launch(ctx, k_cq_reduce, dim3(CQ_RED_GX, nblk), dim3(CQ_RED_T), (size_t)0, (const double *)ctx->d_Gpart, nslab, nblk, BW, nblk_side, nt, G, ldW, 1);
  ovb_launch(ctx, k_cq_chol_gram, dim3(1), dim3(CQ_CHOL_T), sizeof(CqCholSmem), (const double *)G, ldW, nt, 1e-13, L2, 1, (unsigned long long *)nullptr, 0ull);
  const int nT16 = (nt + 15) / 16;
  ovb_launch(ctx, k_cq_trmm, dim3(nT16, nT16), dim3(256), (size_t)0, (const double *)L2, (const double *)L1, nt, Rout, ldR);
  return true;
}
