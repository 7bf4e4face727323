// chol_tiles.cuh — in-CTA Cholesky of a tile-packed lower triangle on the FP64 tensor-core path (DMMA, mma.sync .f64).
// Shared by the CholeskyQR2 / EKF factor kernels (k_cholqr.cu) and the per-feature chi² gate (k_feature.cu).
//
// Layout: the lower triangle is cut into 8x8 tiles; tile (bi, bj), bj <= bi, lives at (bi(bi+1)/2 + bj)*64 doubles, row-major.
// Read at 2*lane that IS the DMMA accumulator fragment of the tile, so a trailing update is load / 2 DMMA / store with no
// index arithmetic. Right-hand-side rows ride along as rows n.. of the same layout: after the factorisation row n+q holds
// rhs_q L^-T, i.e. (L^-1 rhs_q')'.
//
// All multiply-adds on the dependent chains are spelled fma(): the header is also compiled with -fmad=false (k_feature.cu).
#pragma once
#include "chol.cuh"
#ifdef CQ_PROBE
#include <cstdio>
#endif

#define CT_XP 12 // pitch of the panel buffer (conflict-free 8x4 fragments)

// D(8x8) += A(8x4) B(4x8). a = A[lane>>2][lane&3], b = B[lane&3][lane>>2], d0/d1 = D[lane>>2][2*(lane&3)+{0,1}]
__device__ __forceinline__ void ct_dmma(double &d0, double &d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}
// Two m8n8k4 products that share B in one instruction: [D0; D1](16x8) += [A0; A1](16x4) B(4x8), m16n8k4. Same operand and
// accumulator fragments as ct_dmma (a0/d0/d1 of A0/D0, a1/e0/e1 of A1). It takes the FP64 pipe as long as one m8n8k4 does
// (twice the rate, tools/ubench/fp64_rate.cu) and gives the same bits as the two m8n8k4 it replaces.
__device__ __forceinline__ void ct_dmma2(double &d0, double &d1, double &e0, double &e1, double a0, double a1, double b) {
  asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
               : "+d"(d0), "+d"(d1), "+d"(e0), "+d"(e1)
               : "d"(a0), "d"(a1), "d"(b));
}
// Two 8x8x8 tile products that share B, m16n8k8: [D0; D1] += [A0; A1] B with k = 0..7. The operands are two ct_dmma
// k-steps each: a00/a01 = A0's fragments at k 0-3 / 4-7, likewise a10/a11 of A1 and b0/b1 of B. Same bits as the chain
// ct_dmma(k 0-3), ct_dmma(k 4-7) on each tile, in half the pipe time.
__device__ __forceinline__ void ct_dmma2k8(double &d0, double &d1, double &e0, double &e1, double a00, double a01, double a10, double a11, double b0, double b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+d"(d0), "+d"(d1), "+d"(e0), "+d"(e1)
               : "d"(a00), "d"(a10), "d"(a01), "d"(a11), "d"(b0), "d"(b1));
}
// [D0; D1] += [A0; A1] B with k = 0..15, m16n8k16: a[i] = A[g + 8(i&1)][q + 4(i>>1)] (A = [A0; A1], 16 x 16),
// b[j] = B[q + 4j][g]. Same bits as four chained ct_dmma2 over k 0-3, 4-7, 8-11, 12-15, and as the sixteen chained
// fma(a_k, b_k, d) of each output in ascending k (tools/ubench/fp64_rate.cu checks both), in less pipe time.
__device__ __forceinline__ void ct_dmma2k16(double &d0, double &d1, double &e0, double &e1, const double (&a)[8], const double (&b)[4]) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, "
               "{%0,%1,%2,%3};"
               : "+d"(d0), "+d"(d1), "+d"(e0), "+d"(e1)
               : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]), "d"(b[2]),
                 "d"(b[3]));
}
__device__ __forceinline__ int ct_tri(int b) { return (b * (b + 1)) >> 1; }
__device__ __forceinline__ void ct_bar_group(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }
// element (i, j), j <= i, of a tile-packed triangle
__device__ __forceinline__ size_t ct_idx(int i, int j) { return (size_t)(ct_tri(i >> 3) + (j >> 3)) * 64 + (i & 7) * 8 + (j & 7); }

// Shared-memory working set of one factorisation (NRB = row blocks incl. the right-hand-side rows):
//   T      ct_tri(NRB)*64      the triangle (zero past the edges)
//   Xp0/1  NRB*8*CT_XP each    double-buffered panel (rows of the current block column as DMMA operands); must start zeroed
//   invd   NRB*8               reciprocal pivots
//   Linv   2*64                inverse of the current / next diagonal block (row-major 8x8, lower), for the helpers' panels
//   dummyT 64, dummyX 2*CT_XP  zero tile / zero operand rows: target of the masked-out half of a tile pair
struct CtView {
  double *T, *Xp0, *Xp1, *invd, *Linv0, *Linv1, *dummyT, *dummyX;
  int *flag;
};
__host__ __device__ inline size_t ct_view_doubles(int NRB) {
  return (size_t)((NRB * (NRB + 1)) / 2) * 64 + 2 * (size_t)NRB * 8 * CT_XP + (size_t)NRB * 8 + 128 + 64 + 2 * CT_XP;
}
// carve a view out of `base` (16-byte aligned); flag_word: one int of shared memory
__device__ __forceinline__ CtView ct_view_carve(double *base, int NRB, int *flag_word) {
  CtView v;
  v.T = base;
  v.Xp0 = v.T + (size_t)((NRB * (NRB + 1)) / 2) * 64;
  v.Xp1 = v.Xp0 + (size_t)NRB * 8 * CT_XP;
  v.invd = v.Xp1 + (size_t)NRB * 8 * CT_XP;
  v.Linv0 = v.invd + (size_t)NRB * 8;
  v.Linv1 = v.Linv0 + 64;
  v.dummyT = v.Linv1 + 64;
  v.dummyX = v.dummyT + 64;
  v.flag = flag_word;
  return v;
}

// Factor a diagonal tile held by one warp in the DMMA accumulator layout: lane (g, q) = (lane>>2, lane&3) carries
// d0 = A[g][2q], d1 = A[g][2q+1]. strict: a pivot <= 0 (or NaN) raises *flag; else pivots are floored at floor_d
// (semidefinite input) and a zero pivot empties its column. Rows >= nbk of the tile (right-hand-side rows sharing the last
// diagonal tile) come out solved against the nbk x nbk factor; columns >= nbk come out zero. invd[0..8) <- 1/L_jj.
//
// What the eight pivots cost is their dependent chain (tools/ubench/diag8_bench.cu times it). It is longest when every
// lane factors the whole block in registers (~450 FP64 instructions, in-order issue puts them on the chain), shorter with
// the block spread over the lanes and column j broadcast after scaling, and shortest in the form below, where
//   * the UNSCALED column j and the next diagonal entry are broadcast at the top of the step (the shuffles run under the
//     reciprocal square root), each lane scaling what it receives (same inputs, same rounding: bit-identical), and
//   * every lane carries the next pivot itself (p' = a[j+1][j+1] - (a[j+1][j] iv)^2, exactly what the owning lane computes),
// leaves rsqrt -> multiply -> FMA per pivot on the chain.
__device__ __forceinline__ void ct_diag8_frag(double &d0, double &d1, int nbk, double *invd, bool strict, double floor_d, int *flag) {
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  bool bad = false;
  double myinv = 0.0;
  const double inv_floor = (floor_d > 0.0) ? fast_rsqrt(floor_d) : 0.0; // off the chain: known before the first pivot
  double pj = __shfl_sync(full, d0, 0);
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const int jq = j >> 1;
    const double cur = (j & 1) ? d1 : d0;
    const double ag = __shfl_sync(full, cur, 4 * g + jq);      // a[g][j]
    const double ac0 = __shfl_sync(full, cur, 8 * q + jq);     // a[2q][j]
    const double ac1 = __shfl_sync(full, cur, 8 * q + 4 + jq); // a[2q+1][j]
    double an = 0.0, dn = 0.0;
    if (j < 7) {
      an = __shfl_sync(full, cur, 4 * (j + 1) + jq);                                 // a[j+1][j]
      dn = __shfl_sync(full, ((j + 1) & 1) ? d1 : d0, 4 * (j + 1) + ((j + 1) >> 1)); // a[j+1][j+1], updated through column j-1
    }
    const double y = fast_rsqrt(pj); // unconditional; the comparisons below run beside it and only select
    const bool in = j < nbk;
    double d, iv;
    if (strict) {
      const bool pos = pj > 0.0;
      bad = bad || (in && !pos);
      d = pj;
      iv = (in && pos) ? y : 0.0;
    } else {
      const bool above = pj > floor_d; // NaN falls to the floor as well; it survives elsewhere in the row
      d = above ? pj : floor_d;
      iv = in ? (above ? y : inv_floor) : 0.0; // floor 0 (all-zero system): the column empties
    }
    if (j < 7) {
      const double ln = an * iv;
      pj = fma(-ln, ln, dn);
    }
    if (lane == j)
      myinv = iv;
    if (q == jq) { // the lanes holding column j (rows above the diagonal carry scaled padding, never read)
      if (j & 1)
        d1 = (g == j) ? d * iv : d1 * iv;
      else
        d0 = (g == j) ? d * iv : d0 * iv;
    }
    const double lg = ag * iv, lc0 = ac0 * iv, lc1 = ac1 * iv;
    if (2 * q > j)
      d0 = fma(-lg, lc0, d0);
    if (2 * q + 1 > j)
      d1 = fma(-lg, lc1, d1);
  }
  if (lane < 8)
    invd[lane] = myinv;
  if (bad && lane == 0)
    *flag = 1;
}

// L^-1 of a factored diagonal tile (zero past the columns whose reciprocal pivot is zero): lane c (and its copies in the
// other quarters of the warp) carries column c through the forward substitution L m = e_c. The whole warp calls.
__device__ __forceinline__ void ct_linv8(const double *Lt, const double *invd, double *Linv) {
  const int lane = threadIdx.x & 31, cc = lane & 7;
  double mc[8];
#pragma unroll
  for (int j = 0; j < 8; j++) {
    double s0 = (j == cc) ? 1.0 : 0.0, s1 = 0.0;
#pragma unroll
    for (int t = 0; t < j; t++) {
      if (t & 1)
        s1 = fma(-Lt[j * 8 + t], mc[t], s1);
      else
        s0 = fma(-Lt[j * 8 + t], mc[t], s0);
    }
    mc[j] = (s0 + s1) * invd[j];
  }
  if (lane < 8) {
#pragma unroll
    for (int i = 0; i < 8; i++)
      Linv[i * 8 + cc] = (i >= cc) ? mc[i] : 0.0;
  }
}

// Panel tiles (i, k) and (i1, k): X = T(i,k) L_kk^-T, each one 8x8x8 product on the tensor path (both in one m16n8k8:
// they share L_kk^-T), written back over the tile and into the operand buffer (rows 8i.. of Xb). two == false: tile i1
// does not exist; its half of the product runs on zero operands and is dropped. The whole warp calls.
__device__ __forceinline__ void ct_panel_pair(const CtView &sm, int i, int i1, bool two, int k, const double *Linv, double *Xb) {
  const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  double *t = sm.T + (size_t)(ct_tri(i) + k) * 64;
  double *t1 = sm.T + (size_t)(ct_tri(i1) + k) * 64;
  const double a0 = t[g * 8 + q], a1 = t[g * 8 + q + 4];
  const double a10 = two ? t1[g * 8 + q] : 0.0, a11 = two ? t1[g * 8 + q + 4] : 0.0;
  const double b0 = Linv[g * 8 + q], b1 = Linv[g * 8 + q + 4]; // B[k][n] = Linv[n][k]
  double2 d = make_double2(0.0, 0.0), e = make_double2(0.0, 0.0);
  ct_dmma2k8(d.x, d.y, e.x, e.y, a0, a1, a10, a11, b0, b1);
  *reinterpret_cast<double2 *>(t + 2 * lane) = d;
  *reinterpret_cast<double2 *>(Xb + (size_t)(8 * i + g) * CT_XP + 2 * q) = d;
  if (two) {
    *reinterpret_cast<double2 *>(t1 + 2 * lane) = e;
    *reinterpret_cast<double2 *>(Xb + (size_t)(8 * i1 + g) * CT_XP + 2 * q) = e;
  }
}

// rows i0, i0+stride, ... of panel k: x L_kk' = S[i][kb..kb+8) by substitution, one thread per row (backward stable row by
// row); writes x in place and into the panel buffer (zero past nbk). L_kk and the reciprocal pivots go to registers first
// so that the substitution chain never waits for shared memory.
__device__ __forceinline__ void ct_panel_rows(double *T, double *Xp, const double *invd, int i0, int stride, int nrows, int k, int nbk) {
  if (i0 >= nrows)
    return;
  const double *Lk = T + (size_t)(ct_tri(k) + k) * 64;
  double L[8][8], iv[8];
#pragma unroll
  for (int c = 0; c < 8; c++) {
    iv[c] = (c < nbk) ? invd[8 * k + c] : 0.0;
#pragma unroll
    for (int t2 = 0; t2 < 4; t2++) {
      if (2 * t2 < c) {
        const double2 v = *reinterpret_cast<const double2 *>(Lk + c * 8 + 2 * t2);
        L[c][2 * t2] = v.x;
        L[c][2 * t2 + 1] = v.y;
      }
    }
  }
  for (int i = i0; i < nrows; i += stride) {
    double *src = T + (size_t)(ct_tri(i >> 3) + k) * 64 + (i & 7) * 8;
    double v[8], x[8];
    {
      const double2 v01 = *reinterpret_cast<const double2 *>(src), v23 = *reinterpret_cast<const double2 *>(src + 2);
      const double2 v45 = *reinterpret_cast<const double2 *>(src + 4), v67 = *reinterpret_cast<const double2 *>(src + 6);
      v[0] = v01.x, v[1] = v01.y, v[2] = v23.x, v[3] = v23.y, v[4] = v45.x, v[5] = v45.y, v[6] = v67.x, v[7] = v67.y;
    }
    // right-looking: as soon as x[c] is known every later column takes its term, the next column's first
#pragma unroll
    for (int c = 0; c < 8; c++) {
      x[c] = (c < nbk) ? v[c] * iv[c] : 0.0;
#pragma unroll
      for (int t = c + 1; t < 8; t++)
        v[t] = fma(-x[c], L[t][c], v[t]);
    }
    if (nbk == 8) {
      *reinterpret_cast<double2 *>(src) = make_double2(x[0], x[1]);
      *reinterpret_cast<double2 *>(src + 2) = make_double2(x[2], x[3]);
      *reinterpret_cast<double2 *>(src + 4) = make_double2(x[4], x[5]);
      *reinterpret_cast<double2 *>(src + 6) = make_double2(x[6], x[7]);
    } else {
#pragma unroll
      for (int c = 0; c < 8; c++)
        if (c < nbk)
          src[c] = x[c];
    }
    double *xp = Xp + (size_t)i * CT_XP;
    *reinterpret_cast<double2 *>(xp) = make_double2(x[0], x[1]);
    *reinterpret_cast<double2 *>(xp + 2) = make_double2(x[2], x[3]);
    *reinterpret_cast<double2 *>(xp + 4) = make_double2(x[4], x[5]);
    *reinterpret_cast<double2 *>(xp + 6) = make_double2(x[6], x[7]);
  }
}

struct CtTileOps {
  double a0, a1, b0, b1;
  double2 c;
  double2 *cp;
};
// valid == false: the pair's second slot is empty; it is pointed at the dummy tile with zero operands so that both DMMAs of
// the pair execute unconditionally (a branch around mma.sync costs convergence code on every use)
__device__ __forceinline__ void ct_tile_load(CtTileOps &o, const CtView &sm, const double *Xp, int bi, int bj, int lane, bool valid) {
  const int g = lane >> 2, q = lane & 3;
  const double *xa = valid ? Xp + (size_t)(8 * bi + g) * CT_XP + q : sm.dummyX + q;
  const double *xb = valid ? Xp + (size_t)(8 * bj + g) * CT_XP + q : sm.dummyX + q;
  o.cp = reinterpret_cast<double2 *>((valid ? sm.T + (size_t)(ct_tri(bi) + bj) * 64 : sm.dummyT) + 2 * lane);
  o.a0 = -xa[0];
  o.a1 = -xa[4];
  o.b0 = xb[0];
  o.b1 = xb[4];
  o.c = *o.cp;
}
__device__ __forceinline__ void ct_tile_mma(CtTileOps &o) {
  ct_dmma(o.c.x, o.c.y, o.a0, o.b0);
  ct_dmma(o.c.x, o.c.y, o.a1, o.b1);
}
// two tiles of one block column (same B operands) in one m16n8k8
__device__ __forceinline__ void ct_tile_pair_mma_store(CtTileOps &o0, CtTileOps &o1) {
  ct_dmma2k8(o0.c.x, o0.c.y, o1.c.x, o1.c.y, o0.a0, o0.a1, o1.a0, o1.a1, o0.b0, o0.b1);
  *o0.cp = o0.c;
  *o1.cp = o1.c;
}

#ifdef CQ_PROBE
#define CT_PROBE_T(v) v = clock64()
#else
#define CT_PROBE_T(v) do { } while (0)
#endif

// One row of the trailing update of step k: T(bi, bj) -= X(bi,k) X(bj,k)' for j0 <= bj <= jmax. The row's own operand
// fragments stay in registers; two tiles in flight. The tiles of a row share A, not B, so they stay m8n8k4: pairing the
// two rows of a warp by block column (m16n8k8) made k_cq_chol_gram slower (74.7 -> 77.1 us per two launches, config 2).
__device__ __forceinline__ void ct_trail_row(const CtView &sm, const double *Xk, int bi, int j0, int jmax, int lane) {
  const int g = lane >> 2, q = lane & 3;
  const double *xa = Xk + (size_t)(8 * bi + g) * CT_XP + q;
  const double a0 = -xa[0], a1 = -xa[4];
  double *trow = sm.T + (size_t)ct_tri(bi) * 64 + 2 * lane;
  for (int bj = j0; bj <= jmax; bj += 2) {
    const bool two = bj + 1 <= jmax;
    const double *xb0 = Xk + (size_t)(8 * bj + g) * CT_XP + q;
    const double *xb1 = two ? xb0 + 8 * CT_XP : sm.dummyX + q;
    double2 *c0p = reinterpret_cast<double2 *>(trow + (size_t)bj * 64);
    double2 *c1p = two ? c0p + 32 : reinterpret_cast<double2 *>(sm.dummyT + 2 * lane);
    const double b00 = xb0[0], b01 = xb0[4], b10 = xb1[0], b11 = xb1[4];
    double2 c0 = *c0p, c1 = *c1p;
    ct_dmma(c0.x, c0.y, a0, b00);
    ct_dmma(c1.x, c1.y, a0, b10);
    ct_dmma(c0.x, c0.y, a1, b01);
    ct_dmma(c1.x, c1.y, a1, b11);
    *c0p = c0;
    *c1p = c1;
  }
}

// The factorisation proper, on a tile-packed lower triangle already in shared memory. n columns, nrows = n + extra rows.
// THREADS = threads of the CTA (all must call). Organised around the one chain that cannot be shortened — diagonal tile,
// its eight pivots, the rows right below it, the next diagonal tile — which warp 0 runs alone:
//   step k, warp 0 :  T(k+1,k+1) -= X(k+1,k) X(k+1,k)' (stays in registers)  ->  pivots of block k+1 (ct_diag8_frag)
//                     ->  X(k+2,k+1): the eight rows of block k+2 solved against L(k+1,k+1)
//   step k, helpers:  X(i,k) for the rows of blocks i >= k+2 (one thread per row), then T(i,k+1) -= X(i,k) X(k+1,k)' (warp
//                     0's third move needs the first of these tiles), then the rest of the trailing update
//                     T(i,j) -= X(i,k) X(j,k)', k+2 <= j <= i, by rows (rows r and R-1-r go to the same warp: equal shares).
// The helpers are the warps of sub-partitions 1-3 (wid % 4 != 0): a DMMA holds its sub-partition's FP64 pipe for 16
// cycles, and with helpers next to it warp 0's pivots ran 2-2.5x slower (tools/ubench/diag8_bench.cu: 854 cycles alone,
// 1900-2400 in the first version of this kernel); the other warps of sub-partition 0 only keep the barriers company.
// One __syncthreads per step; named barrier 1 joins the helpers after their panel rows, named barrier 2 hands block
// column k+1 to warp 0 (it has never been seen to wait there: the helpers' first two moves are shorter than eight pivots),
// named barrier 3 hands each factored diagonal block to the inverting warp.
// Block column k (tiles (i, k), i >= k, and reciprocal pivots 8k..8k+7) is final at the barrier that ends step k. With
// nine warps or more, warp 8 (on warp 0's sub-partition, otherwise idle) calls pub.column(sm, k) during step k + 1, so
// that a consumer of the factor can start on it while the chain runs; the last column is the caller's to publish.
struct CtNoPublish {
  __device__ __forceinline__ void column(const CtView &, int) const {}
};
template <int THREADS, typename PUB = CtNoPublish>
__device__ __forceinline__ void ct_chol_tiles(const CtView &sm, int n, int nrows, bool strict, double floor_d, const PUB &pub = PUB()) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  constexpr int NW = THREADS / 32, NH = NW - (NW + 3) / 4;
  static_assert(NH >= 1, "need at least one helper warp");
  const bool helper = (wid & 3) != 0;
  const int hr = wid - 1 - (wid >> 2); // rank among the helpers
  // With eight warps or more, warp 4 (idle, on warp 0's sub-partition) inverts each diagonal block as soon as warp 0 has
  // stored it (named barrier 3), and the helpers' panel tiles become one 8x8x8 DMMA product each instead of a 36-step
  // substitution per row. The explicit inverse makes the panel error proportional to cond(L_kk) (<= ~3e5 in the first
  // CholeskyQR pass, whose factor only preconditions the second; O(1..1e3) elsewhere) instead of backward stable.
  constexpr bool LINV = NW >= 8;
#ifdef CQ_PROBE
  long long p0 = 0, p1 = 0, p2 = 0, p3 = 0, p4 = 0, p5 = 0, acc[6] = {0, 0, 0, 0, 0, 0};
#endif
  const int NB = (n + 7) >> 3, NRB = (nrows + 7) >> 3;
  if (wid == 0) {
    double2 c = *reinterpret_cast<const double2 *>(sm.T + 2 * lane);
    ct_diag8_frag(c.x, c.y, min(8, n), sm.invd, strict, floor_d, sm.flag);
    *reinterpret_cast<double2 *>(sm.T + 2 * lane) = c;
    __syncwarp();
    if (LINV)
      asm volatile("bar.arrive 3, 64;" ::: "memory");
    ct_panel_rows(sm.T, sm.Xp0, sm.invd, lane < 8 ? 8 + lane : nrows, 1 << 30, nrows, 0, min(8, n)); // the eight rows of block 1 only
  } else if (LINV && wid == 4) {
    asm volatile("bar.sync 3, 64;" ::: "memory");
    ct_linv8(sm.T, sm.invd, sm.Linv0);
  }
  __syncthreads();
  for (int k = 0; k < NB; k++) {
    const int par = k & 1;
    double *Xk = par ? sm.Xp1 : sm.Xp0, *Xn = par ? sm.Xp0 : sm.Xp1;
    const bool more = k + 1 < NB;
    CT_PROBE_T(p0);
#ifdef CQ_PROBE
    p1 = p2 = p3 = p4 = p0;
#endif
    if (wid == 0) {
      if (more) {
        const int k1 = k + 1, nbk1 = min(8, n - 8 * k1);
        CtTileOps o;
        ct_tile_load(o, sm, Xk, k1, k1, lane, true);
        ct_tile_mma(o);
        CT_PROBE_T(p1);
        ct_diag8_frag(o.c.x, o.c.y, nbk1, sm.invd + 8 * k1, strict, floor_d, sm.flag);
        *o.cp = o.c;
        __syncwarp();
        if (LINV)
          asm volatile("bar.arrive 3, 64;" ::: "memory");
        CT_PROBE_T(p2);
        asm volatile("bar.sync 2, %0;" ::"r"((NH + 1) * 32) : "memory");
        CT_PROBE_T(p3);
        ct_panel_rows(sm.T, Xn, sm.invd, lane < 8 ? 8 * (k + 2) + lane : nrows, 1 << 30, nrows, k1, nbk1); // block k+2 only
        CT_PROBE_T(p4);
      }
    } else if (LINV && wid == 4) {
      if (more) {
        asm volatile("bar.sync 3, 64;" ::: "memory");
        ct_linv8(sm.T + (size_t)(ct_tri(k + 1) + k + 1) * 64, sm.invd + 8 * (k + 1), par ? sm.Linv0 : sm.Linv1);
      }
    } else if (helper) {
      if (LINV) {
        const double *Lk = par ? sm.Linv1 : sm.Linv0;
        for (int i = k + 2 + hr; i < NRB; i += 2 * NH)
          ct_panel_pair(sm, i, i + NH, i + NH < NRB, k, Lk, Xk);
      } else {
        ct_panel_rows(sm.T, Xk, sm.invd, 8 * (k + 2) + hr * 32 + lane, NH * 32, nrows, k, min(8, n - 8 * k));
      }
      if (NH > 1)
        ct_bar_group(1, NH * 32);
      else
        __syncwarp();
      CT_PROBE_T(p1);
      if (more) {
        for (int i = k + 2 + hr; i < NRB; i += 2 * NH) {
          CtTileOps o0, o1;
          ct_tile_load(o0, sm, Xk, i, k + 1, lane, true);
          ct_tile_load(o1, sm, Xk, i + NH, k + 1, lane, i + NH < NRB);
          ct_tile_pair_mma_store(o0, o1);
        }
        asm volatile("bar.arrive 2, %0;" ::"r"((NH + 1) * 32) : "memory");
        CT_PROBE_T(p2);
        const int R = NRB - (k + 2), jmaxc = NB - 1;
        for (int pr = hr; 2 * pr < R; pr += NH) {
          const int rb = R - 1 - pr;
          ct_trail_row(sm, Xk, k + 2 + rb, k + 2, min(k + 2 + rb, jmaxc), lane);
          if (rb != pr)
            ct_trail_row(sm, Xk, k + 2 + pr, k + 2, min(k + 2 + pr, jmaxc), lane);
        }
      }
      CT_PROBE_T(p3);
    } else if (wid == 8 && k > 0) {
      pub.column(sm, k - 1);
    }
    __syncthreads();
    CT_PROBE_T(p5);
#ifdef CQ_PROBE
    if (wid == 0) {
      acc[0] += p1 - p0, acc[1] += p2 - p1, acc[2] += p3 - p2, acc[3] += p4 - p3, acc[4] += p5 - p4;
    } else {
      acc[0] += p1 - p0, acc[1] += p2 - p1, acc[2] += p3 - p2, acc[3] += p5 - p3;
    }
    acc[5] += p5 - p0;
#endif
  }
#ifdef CQ_PROBE // sums over the block steps, one line per role
  if (tid == 0)
    printf("chol n=%d W0 (cycles over %d steps): diag update %lld pivots %lld wait %lld rows below %lld step tail %lld | %lld\n", n, NB, acc[0], acc[1], acc[2], acc[3],
           acc[4], acc[5]);
  if (tid == 32 || tid == THREADS - 32)
    printf("chol n=%d helper warp %d: panel rows %lld column k+1 %lld trailing %lld wait %lld | %lld\n", n, wid, acc[0], acc[1], acc[2], acc[3], acc[5]);
#endif
}
