// k_tsqr.cu — measurement compression as a communication-avoiding blocked Householder QR (TSQR/CAQR), plus the
// stacked-column bookkeeping of UpdaterMSCKF::update.
// Replaces UpdaterHelper::measurement_compress_inplace (ov_msckf/src/update/UpdaterHelper.cpp:456-487: a Givens sweep
// of 3mn² flops with stride-m accesses) and the first-seen column map of UpdaterMSCKF.cpp:237-245.
//
// Layout: the stacked system [H | r] is row-major in HBM/L2 (m x (n+1), leading dimension ldA). For each column panel
// (NB = 16 wide) the active rows are cut into chunks of CR = 256 rows; a CTA owns (chunk, column tile group):
//   1. panel factorisation in registers: one row per thread, Householder by column with ONE 16-wide block reduction
//      per column (p_j = a_k·a_j gives the column norm, all v'a_j and the reflector Gram row at once),
//   2. compact-WY application to the chunk's trailing columns as two shared-memory GEMMs (Y = V'A, A -= V Z),
//   3. the chunk's 16 x 16 R goes to a small workspace; the next level repeats 1-2 on the stacked R factors
//      (rows addressed in place through an index map), until one chunk is left.
// Chunks never exchange data inside a level (no grid-wide sync, no atomics: bitwise reproducible); Q is never formed.
// Upper levels: as soon as a level has <= QR_CLUSTER chunks, those chunks are factored TOGETHER by one thread-block
// cluster (one CTA per chunk): the 17 per-step dot products and the 16 x 32 V'A block of every trailing tile are
// summed across the cluster through distributed shared memory (st.async + mbarrier complete_tx, no cluster barrier
// in the loop), so the level finishes the panel in ONE launch instead of two or three latency-bound ones.
// The reference's Givens R has diag >= 0; rows of R (and z) are sign-flipped at the end to match.
#include "ovb_internal.cuh"
#include <math.h>
#include <cstddef>
#include <cooperative_groups.h>
namespace cg = cooperative_groups;

#define QR_NB OVB_NB
#define QR_CR OVB_CR
#define QR_CT 32
#define QR_THREADS QR_CR
#define QR_WARPS (QR_THREADS / 32)
#define QR_CLUSTER 8 // portable maximum cluster size
#define QR_XW 36     // exchange record: [0..15] dots, [16] sigma, [17] alpha, [18..33] pivot-row entries
#ifdef OVB_TSQR_TIMING
#include <cstdio>
#define TPROBE(i) do { if (tid == 0 && blockIdx.x == 0 && blockIdx.y == 0) tprobe[i] = clock64(); } while (0)
#else
#define TPROBE(i) do { } while (0)
#endif

#define QR_VPITCH 20 // pitch of Vs: conflict-free 8x4 / 4x8 double fragments (2*20 mod 32 = 8)
#define QR_APITCH 36 // pitch of At / Ys / Zs (2*36 mod 32 = 8)
struct QrSmem {
  double Vs[QR_CR][QR_VPITCH];        // reflectors, unit lower trapezoid: V[r][j] at Vs[r][j ^ ((r >> 4) & 15)] (swizzled)
  double At[QR_CR][QR_APITCH];        // trailing tile, buffer 0 (also the panel staging buffer)
  double Ys[QR_NB][QR_APITCH];        // V'A of the tile
  double Zs[QR_NB][QR_APITCH];        // -(Tt Y): the update is At + V Zs
  double G[QR_NB][QR_NB];             // strict lower: v_k'v_i
  double Rb[QR_NB][QR_NB];            // finished R entries of this chunk
  double Tt[QR_NB][QR_NB];            // reflector coupling (lower triangular): z = Tt y
  double tau[QR_NB];
  double vbuf[2][16 * 18];            // pivot column broadcast, double buffered by step parity, pitch 18
  double sc[4];                       // [2 + parity]: pivot element alpha of the current step
  int rowidx[QR_CR];
  // cluster mode only (written by the peer CTAs through DSMEM)
  double xch[2][QR_CLUSTER][QR_XW];          // per-step partial sums, double buffered by step parity
  unsigned long long mbar[4];                // [0..1] per-step exchange (by step parity), [2] tile exchange
  union {
    double At1[QR_CR][QR_APITCH];            // trailing tile, buffer 1 (next tile streams in while this one is updated)
    double Yx[QR_CLUSTER][QR_NB][QR_APITCH]; // cluster mode: per-tile partial V'A of every CTA of the cluster
  };
};

__device__ __forceinline__ void cp_async16(unsigned dst, const void *src, unsigned src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async8(unsigned dst, const void *src, unsigned src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// DSMEM exchange without a cluster barrier: the sender stores straight into the peer's shared memory and the same
// instruction credits the bytes to an mbarrier there (st.async ... mbarrier::complete_tx); the receiver only polls its
// own mbarrier (one DSMEM latency instead of latency + barrier.cluster round trip).
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ unsigned mapa_u32(unsigned addr, unsigned rank) {
  unsigned r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void st_async_f64(unsigned raddr, double v, unsigned rbar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b64 [%0], %1, [%2];" ::"r"(raddr), "l"(__double_as_longlong(v)), "r"(rbar)
               : "memory");
}
__device__ __forceinline__ void st_async_f64x2(unsigned raddr, double a, double b, unsigned rbar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v2.b64 [%0], {%1, %2}, [%3];" ::"r"(raddr), "l"(__double_as_longlong(a)),
               "l"(__double_as_longlong(b)), "r"(rbar)
               : "memory");
}
__device__ __forceinline__ void mbar_init(unsigned bar, unsigned count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity) {
  asm volatile("{\n\t.reg .pred p;\n\tOVB_WAIT:\n\tmbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%0], %1;\n\t@p bra OVB_DONE;\n\tbra OVB_WAIT;\n\tOVB_DONE:\n\t}" ::"r"(bar),
               "r"(parity)
               : "memory");
}

__device__ __forceinline__ void cluster_arrive_release() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait_acquire() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }

// D(8x8) += A(8x4) B(4x8) on the FP64 tensor-core path (DMMA). Fragments: a = A[lane>>2][lane&3], b = B[lane&3][lane>>2],
// d0/d1 = D[lane>>2][2*(lane&3) + {0,1}].
__device__ __forceinline__ void dmma884(double &d0, double &d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}

// One (panel, level) step. grid = (chunks, column-tile groups). csize > 1: the grid's x extent is one cluster of csize
// CTAs (rank = chunk) that factor their chunks as ONE tall block; chunks past the data are padded with zero rows.
__global__ void __launch_bounds__(QR_THREADS)
    k_tsqr_level(double *__restrict__ A, int ldA, int nt, int c0, int nbp, int level, int len, const double *__restrict__ Win,
                 double *__restrict__ Wout, double *__restrict__ Rout, int ldR, int is_last, int csize, int cr0) {
  extern __shared__ __align__(16) unsigned char qr_smem_raw[];
  QrSmem &sm = *reinterpret_cast<QrSmem *>(qr_smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int chunk = blockIdx.x;
#ifdef OVB_TSQR_TIMING
  long long tprobe[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
#endif
  TPROBE(0);
  // rows per chunk: cr0 (<= QR_CR, multiple of 16) at level 0 so that the chunks fill the SMs, QR_CR above
  const int crl = (level == 0) ? cr0 : QR_CR;
  const int rows_i = max(0, min(crl, len - chunk * crl));
  const int rows16 = (rows_i + 15) & ~15;
  const bool clustered = csize > 1;
  const int crank = clustered ? chunk : 0; // gridDim.x == cluster size
  const bool has_pivots = (crank == 0);    // the pivot rows of a clustered block all live in its first chunk
  // Programmatic dependent launch: let the next (panel, level) kernel of the chain be scheduled right away — its CTAs
  // run their prologue on the SMs this grid leaves idle and then block in griddepcontrol.wait until this grid has
  // completed and flushed. Everything before OUR wait below touches only shared memory.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  // my exchange slot and mbarriers as seen by the peer this lane serves (lane group index pg = tid & 15 -> peer rank)
  unsigned peer_xch = 0, peer_bar = 0, peer_yx = 0;
  if (clustered) {
    const unsigned peer = (unsigned)(tid & 15) % (unsigned)csize;
    peer_xch = mapa_u32(smem_u32(&sm.xch[0][crank][0]), peer);
    peer_bar = mapa_u32(smem_u32(&sm.mbar[0]), peer);
    peer_yx = smem_u32(&sm.Yx[crank][0][0]);
    if (tid == 0) {
      mbar_init(smem_u32(&sm.mbar[0]), 1);
      mbar_init(smem_u32(&sm.mbar[1]), 1);
      mbar_init(smem_u32(&sm.mbar[2]), 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // every CTA of the cluster is running and has its mbarriers initialised before anyone writes into a peer
    cluster_arrive_release();
    cluster_wait_acquire();
  }
  // ---- row map of this level back to rows of A
  {
    int g = chunk * crl + tid;
    for (int l = level; l >= 1; l--)
      g = (g / nbp) * (l == 1 ? cr0 : QR_CR) + (g % nbp);
    sm.rowidx[tid] = c0 + g;
  }
  asm volatile("griddepcontrol.wait;" ::: "memory"); // the previous kernel's writes to A / W are visible from here on
  // ---- panel factorisation. Ownership: thread (j = tid>>4, g = tid&15) holds rows 16g..16g+15 of panel column j in
  // registers, so a half-warp owns one column and every column dot product is 16 FMAs + a 4-level half-warp butterfly.
  // The 16 rows sit in a rotating window (after k rotations slot t holds local row (k + t) mod 16): the pivot row of
  // step k is slot 0 of group 0 and every register index is static, so the loop stays rolled (one copy in the I-cache).
  double *Bp = &sm.At[0][0]; // staging [j][t][g], pitch 257: conflict-free both ways (aliases the tile buffer)
  {
    // 8-byte cp.async straight into the transposed staging layout: every load of the CTA is in flight at once
    // (zero-filled beyond the chunk's rows / the panel's columns)
    const int lj = tid & 15, rr = tid >> 4;
#pragma unroll 4
    for (int pass = 0; pass < QR_CR / 16; pass++) {
      const int r = pass * 16 + rr;
      const bool ok = (r < rows_i) && (lj < nbp);
      const double *src = A;
      if (ok)
        src = (level == 0) ? A + (size_t)(c0 + chunk * crl + r) * ldA + c0 + lj : Win + (size_t)(chunk * QR_CR + r) * QR_NB + lj;
      cp_async8(smem_u32(&Bp[lj * 257 + (r & 15) * 16 + (r >> 4)]), src, ok ? 8u : 0u);
    }
    cp_async_commit();
    cp_async_wait_all();
  }
  __syncthreads();
  TPROBE(1);
  const int pj = tid >> 4, pg = tid & 15;
  double a[QR_NB];
#pragma unroll
  for (int t = 0; t < QR_NB; t++)
    a[t] = Bp[pj * 257 + t * 16 + pg];
  __syncthreads(); // Bp (== At) is free again
  // ---- trailing tiles of this CTA stream in with cp.async: the first one during the panel factorisation, the next one
  // while the current one is updated (cluster mode: single buffer, the second buffer holds the exchange slots)
  const int tc0 = c0 + nbp;
  const int ntiles = (nt - tc0 + QR_CT - 1) / QR_CT;
  auto prefetch_tile = [&](int tile, int buf) {
    const int col0 = tc0 + tile * QR_CT;
    const int ncol = min(QR_CT, nt - col0);
    double(*At)[QR_APITCH] = buf ? sm.At1 : sm.At;
    if (((ldA | col0) & 1) == 0 && (((size_t)A) & 15) == 0) {
      const int ch = tid & 15, rr = tid >> 4; // 16-byte chunk of the 256-byte row
      const int nb = max(0, min(16, ncol * 8 - ch * 16));
      for (int r = rr; r < rows16; r += 16) {
        const bool ok = (r < rows_i) && nb > 0;
        const double *src = ok ? A + (size_t)sm.rowidx[r] * ldA + col0 + 2 * ch : A;
        cp_async16(smem_u32(&At[r][2 * ch]), src, ok ? (unsigned)nb : 0u);
      }
    } else {
      const int cc = tid & 31, rr = tid >> 5;
      for (int r = rr; r < rows16; r += 8) {
        const bool ok = (r < rows_i) && cc < ncol;
        const double *src = ok ? A + (size_t)sm.rowidx[r] * ldA + col0 + cc : A;
        cp_async8(smem_u32(&At[r][cc]), src, ok ? 8u : 0u);
      }
    }
    cp_async_commit();
  };
  bool tile_pending = false;
  if ((int)blockIdx.y < ntiles) {
    prefetch_tile(blockIdx.y, 0);
    tile_pending = true;
  }
  // Finished rows (row k of columns j >= k after step k) leave the register window: their value goes to sm.Rb and the
  // slot is zeroed, so dot products and updates run unmasked. ONE barrier per step: the pivot column and the pivot
  // element are broadcast through (double-buffered) shared memory; every thread then derives the reflector scalars
  // itself (the column norm is reduced redundantly by every half-warp in the same butterfly as its own dot product).
#pragma unroll 1
  for (int k = 0; k < nbp; k++) {
    const int par = k & 1;
    double pv = 0.0;
    if (has_pivots && pg == 0 && pj >= k) { // pivot row k lives in group 0, window slot 0
      pv = a[0];
      a[0] = 0.0;
    }
    if (pj == k) {
#pragma unroll
      for (int t = 0; t < QR_NB; t++)
        sm.vbuf[par][pg * 18 + t] = a[t];
      if (pg == 0)
        sm.sc[2 + par] = pv;
    }
    __syncthreads();
    double v[QR_NB];
#pragma unroll
    for (int t = 0; t < QR_NB; t += 2) {
      const double2 vv = *reinterpret_cast<const double2 *>(&sm.vbuf[par][pg * 18 + t]);
      v[t] = vv.x;
      v[t + 1] = vv.y;
    }
    double alpha = sm.sc[2 + par];
    double d0 = 0.0, d1 = 0.0, d2 = 0.0, d3 = 0.0, s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
#pragma unroll
    for (int t = 0; t < QR_NB; t += 4) {
      d0 += v[t] * a[t];
      d1 += v[t + 1] * a[t + 1];
      d2 += v[t + 2] * a[t + 2];
      d3 += v[t + 3] * a[t + 3];
      s0 += v[t] * v[t];
      s1 += v[t + 1] * v[t + 1];
      s2 += v[t + 2] * v[t + 2];
      s3 += v[t + 3] * v[t + 3];
    }
    double dot = (d0 + d1) + (d2 + d3), sigma = (s0 + s1) + (s2 + s3);
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) {
      dot += __shfl_xor_sync(0xffffffffu, dot, o);
      sigma += __shfl_xor_sync(0xffffffffu, sigma, o);
    }
    // pivot-row entry of this thread's column (held by the g == 0 thread of the half-warp; for j < k it is V[k][j])
    double akj = __shfl_sync(0xffffffffu, (pj >= k) ? pv : a[0], lane & 16);
    if (clustered) {
      // every CTA adds its rows' share: post (dots, sigma[, alpha, pivot row]) into slot `crank` of every peer, wait on
      // the own mbarrier, then sum the csize slots in the same order everywhere (bitwise identical scalars cluster-wide).
      // After the butterfly every lane of the half-warp holds the column's dot: lane group pg posts it to peer pg.
      const unsigned bar_l = smem_u32(&sm.mbar[par]);
      if (tid == 0) // bytes this CTA receives in this step: (16 dots + sigma) from everybody, (alpha + 16 pivot entries) from rank 0
        mbar_expect_tx(bar_l, (unsigned)(csize * 17 * 8 + 17 * 8));
      if (pg < csize) {
        const unsigned dst = peer_xch + (unsigned)(par * (QR_CLUSTER * QR_XW) * 8);
        const unsigned rb = peer_bar + (unsigned)(par * 8);
        st_async_f64(dst + pj * 8, dot, rb);
        if (has_pivots)
          st_async_f64(dst + (18 + pj) * 8, akj, rb);
        if (pj == 0) {
          st_async_f64(dst + 16 * 8, sigma, rb);
          if (has_pivots)
            st_async_f64(dst + 17 * 8, alpha, rb);
        }
      }
      mbar_wait(bar_l, (unsigned)((k >> 1) & 1));
      double ds[QR_CLUSTER], ss[QR_CLUSTER];
#pragma unroll
      for (int r = 0; r < QR_CLUSTER; r++) {
        ds[r] = (r < csize) ? sm.xch[par][r][pj] : 0.0;
        ss[r] = (r < csize) ? sm.xch[par][r][16] : 0.0;
      }
      dot = ((ds[0] + ds[1]) + (ds[2] + ds[3])) + ((ds[4] + ds[5]) + (ds[6] + ds[7]));
      sigma = ((ss[0] + ss[1]) + (ss[2] + ss[3])) + ((ss[4] + ss[5]) + (ss[6] + ss[7]));
      alpha = sm.xch[par][0][17];
      akj = sm.xch[par][0][18 + pj];
    }
    // reflector scalars: beta = -sign(alpha) |x|, tau = (beta - alpha)/beta = 1 + |alpha|/|x|, scale = 1/(alpha - beta)
    double tk = 0.0, scale = 0.0, beta = alpha;
    if (sigma != 0.0) {
      const double n2 = alpha * alpha + sigma;
      const double aa = fabs(alpha);
      double nrm, sc;
      if (n2 > 1e-30 && n2 < 1e30) {
        // No library sqrt/divide on the critical path (FP64 dependent latency is ~19 cycles per op). Float seeds
        // (22 bits), then ONE third-order step each (22 -> 66 bits): y = 1/sqrt(n2), rc = 1/(|alpha| + |x|).
        // The reciprocal's seed comes from the float estimate of |x| so that it overlaps the rsqrt refinement.
        const float n2f = (float)n2;
        const float yf = rsqrtf(n2f);
        double rc = (double)(1.0f / ((float)aa + n2f * yf));
        double y = (double)yf;
        const double e = 1.0 - n2 * (y * y);
        y = y + y * (e * (0.5 + 0.375 * e));
        nrm = n2 * y;
        const double x = aa + nrm;
        const double f = 1.0 - x * rc;
        rc = rc + rc * (f + f * f);
        sc = rc + rc * (1.0 - x * rc); // one cheap Newton touch-up: the seed of rc saw only the float |x|
        tk = 1.0 + aa * y;
      } else {
        nrm = sqrt(n2);
        sc = 1.0 / (aa + nrm);
        tk = (aa + nrm) / nrm;
      }
      beta = (alpha >= 0.0) ? -nrm : nrm;
      scale = (alpha >= 0.0) ? sc : -sc;
    }
    const double wj = akj + dot * scale; // v'a_j (for j < k: v_k'v_j)
    if (pj > k) {
      const double tw = tk * wj * scale;
#pragma unroll
      for (int t = 0; t < QR_NB; t++)
        a[t] -= tw * v[t];
      if (pg == 0)
        sm.Rb[k][pj] = akj - tk * wj; // finished entry R[k][j]
    } else if (pj == k) {
#pragma unroll
      for (int t = 0; t < QR_NB; t++)
        a[t] = v[t] * scale;
      if (pg == 0) {
        sm.tau[k] = tk;
        sm.Rb[k][k] = beta;
      }
    } else if (pg == 0) {
      sm.G[k][pj] = wj;
    }
    {
      const double t0 = a[0];
#pragma unroll
      for (int t = 0; t < QR_NB - 1; t++)
        a[t] = a[t + 1];
      a[QR_NB - 1] = t0;
    }
  }
#pragma unroll 1
  for (int s2 = nbp; s2 < QR_NB; s2++) { // complete the cycle: slot t is local row t again
    const double t0 = a[0];
#pragma unroll
    for (int t = 0; t < QR_NB - 1; t++)
      a[t] = a[t + 1];
    a[QR_NB - 1] = t0;
  }
  __syncthreads();
  TPROBE(2);
  // ---- publish V (unit lower trapezoid; column index swizzled by the row group: conflict-free) and emit this chunk's R
#pragma unroll
  for (int t = 0; t < QR_NB; t++) {
    const int r = pg * 16 + t;
    double vv = 0.0;
    if (pj < nbp && r < rows_i)
      vv = (!has_pivots || r > pj) ? a[t] : (r == pj ? 1.0 : 0.0);
    sm.Vs[r][pj ^ pg] = vv;
  }
  if (blockIdx.y == 0 && pg == 0 && has_pivots) {
    // thread (j, g=0) emits column j of the chunk's R from sm.Rb (rows t <= j; zeros below the diagonal)
    const int nr = min(nbp, rows_i);
    for (int t = 0; t < nr; t++) {
      const double val = (pj < nbp && t <= pj) ? sm.Rb[t][pj] : 0.0;
      if (is_last) {
        if (pj < nbp)
          Rout[(size_t)(c0 + t) * ldR + c0 + pj] = val;
      } else {
        Wout[(size_t)(chunk * nbp + t) * QR_NB + pj] = val;
      }
    }
  }
  // ---- reflector coupling Tt (lower triangular 16x16): z = Tt y solves z_k = tau_k (y_k - sum_{i<k} G[k][i] z_i).
  // Column c by thread c, in the same barrier interval as the publish/emit above.
  if (tid < QR_NB) {
    const int c = tid;
    double x[QR_NB];
#pragma unroll
    for (int k = 0; k < QR_NB; k++) {
      // x[i] = 0 for i < c, so the sum runs over all i < k with static bounds; four interleaved chains
      double acc[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
      for (int i = 0; i < QR_NB; i++)
        if (i < k)
          acc[i & 3] += sm.G[k][i] * x[i];
      double val = -sm.tau[k] * ((acc[0] + acc[1]) + (acc[2] + acc[3]));
      if (k == c)
        val = sm.tau[c];
      if (k < c || c >= nbp || k >= nbp)
        val = 0.0;
      x[k] = val;
    }
#pragma unroll
    for (int k = 0; k < QR_NB; k++)
      sm.Tt[k][c] = x[k];
  }
  __syncthreads();
  // ---- apply Q' to the trailing column tiles owned by this CTA: two small GEMMs on the FP64 tensor-core path
  TPROBE(3);
  const int fr = lane >> 2, fk = lane & 3; // DMMA fragment coordinates
  int tile_it = -1, buf = 0;
  for (int tile = blockIdx.y; tile < ntiles; tile += gridDim.y) {
    tile_it++;
    const int col0 = tc0 + tile * QR_CT;
    const int ncol = min(QR_CT, nt - col0);
    double(*At)[QR_APITCH] = buf ? sm.At1 : sm.At;
    if (!tile_pending)
      prefetch_tile(tile, buf);
    cp_async_wait_all();
    __syncthreads();
    tile_pending = false;
    if (!clustered && tile + (int)gridDim.y < ntiles) {
      prefetch_tile(tile + gridDim.y, buf ^ 1);
      tile_pending = true;
    }
    if (tile == (int)blockIdx.y) TPROBE(4);
    // Y = V'At (16 x 32, K = 256): warp w owns the 8x8 output tile (w>>2, w&3); 4 interleaved accumulator pairs
    {
      const int i0 = 8 * (wid >> 2), cc0 = 8 * (wid & 3);
      double y0[4] = {0.0, 0.0, 0.0, 0.0}, y1[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll 4
      for (int r0 = 0; r0 < rows16; r0 += 16) {
        const int sw = (r0 >> 4) & 15;
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const int r = r0 + 4 * q + fk;
          dmma884(y0[q], y1[q], sm.Vs[r][(i0 + fr) ^ sw], At[r][cc0 + fr]);
        }
      }
      const double ya = (y0[0] + y0[1]) + (y0[2] + y0[3]), yb = (y1[0] + y1[1]) + (y1[2] + y1[3]);
      if (!clustered) {
        sm.Ys[i0 + fr][cc0 + 2 * fk] = ya;
        sm.Ys[i0 + fr][cc0 + 2 * fk + 1] = yb;
      } else {
        const unsigned off = (unsigned)(((i0 + fr) * QR_APITCH + cc0 + 2 * fk) * 8);
        const unsigned bar2 = smem_u32(&sm.mbar[2]);
#pragma unroll
        for (int r = 0; r < QR_CLUSTER; r++)
          if (r < csize)
            st_async_f64x2(mapa_u32(peer_yx + off, r), ya, yb, mapa_u32(bar2, r));
      }
    }
    if (clustered) {
      const unsigned bar2 = smem_u32(&sm.mbar[2]);
      if (tid == 0)
        mbar_expect_tx(bar2, (unsigned)(csize * QR_NB * QR_CT * 8));
      mbar_wait(bar2, (unsigned)(tile_it & 1));
      // Ys = sum over the cluster (fixed order), two entries per thread
      const int i = tid >> 4, c2 = (tid & 15) * 2;
      double2 acc[QR_CLUSTER];
#pragma unroll
      for (int r = 0; r < QR_CLUSTER; r++)
        acc[r] = (r < csize) ? *reinterpret_cast<const double2 *>(&sm.Yx[r][i][c2]) : make_double2(0.0, 0.0);
      sm.Ys[i][c2] = ((acc[0].x + acc[1].x) + (acc[2].x + acc[3].x)) + ((acc[4].x + acc[5].x) + (acc[6].x + acc[7].x));
      sm.Ys[i][c2 + 1] = ((acc[0].y + acc[1].y) + (acc[2].y + acc[3].y)) + ((acc[4].y + acc[5].y) + (acc[6].y + acc[7].y));
    }
    __syncthreads();
    if (tile == (int)blockIdx.y) TPROBE(5);
    // Zs = -(Tt Y) (lower triangular 16x16 times 16x32): thread = (row k, 2 columns), two interleaved chains
    {
      const int k = tid >> 4, c2 = (tid & 15) * 2;
      double z0 = 0.0, z1 = 0.0, z2 = 0.0, z3 = 0.0;
#pragma unroll
      for (int i = 0; i < QR_NB; i += 2) {
        const double t0 = (i <= k) ? sm.Tt[k][i] : 0.0, t1 = (i + 1 <= k) ? sm.Tt[k][i + 1] : 0.0;
        z0 += t0 * sm.Ys[i][c2];
        z1 += t0 * sm.Ys[i][c2 + 1];
        z2 += t1 * sm.Ys[i + 1][c2];
        z3 += t1 * sm.Ys[i + 1][c2 + 1];
      }
      sm.Zs[k][c2] = -(z0 + z2);
      sm.Zs[k][c2 + 1] = -(z1 + z3);
    }
    __syncthreads();
    if (tile == (int)blockIdx.y) TPROBE(6);
    // At + V Zs (256 x 32, K = 16): warp w owns row tiles w, w+8, w+16, w+24 (8 rows each) x 4 column tiles
    {
#pragma unroll
      for (int rq = 0; rq < 4; rq++) {
        const int r0 = 8 * (wid + 8 * rq);
        if (r0 >= rows16)
          break;
        const int sw = (r0 >> 4) & 15;
        const int r = r0 + fr;
        double va[4];
#pragma unroll
        for (int kq = 0; kq < 4; kq++)
          va[kq] = sm.Vs[r][(4 * kq + fk) ^ sw];
        double c[4][2];
        // a ragged last tile (ncol < 32) only pays for the 8-column sub-tiles it has
#pragma unroll
        for (int ct = 0; ct < 4; ct++) {
          if (8 * ct < ncol) {
            const double2 cc = *reinterpret_cast<const double2 *>(&At[r][8 * ct + 2 * fk]);
            c[ct][0] = cc.x;
            c[ct][1] = cc.y;
          }
        }
#pragma unroll
        for (int kq = 0; kq < 4; kq++)
#pragma unroll
          for (int ct = 0; ct < 4; ct++)
            if (8 * ct < ncol)
              dmma884(c[ct][0], c[ct][1], va[kq], sm.Zs[4 * kq + fk][8 * ct + fr]);
        if (r < rows_i) {
          double *dst = A + (size_t)sm.rowidx[r] * ldA + col0;
#pragma unroll
          for (int ct = 0; ct < 4; ct++) {
            const int cj = 8 * ct + 2 * fk;
            if (cj < ncol)
              dst[cj] = c[ct][0];
            if (cj + 1 < ncol)
              dst[cj + 1] = c[ct][1];
          }
        }
      }
    }
    __syncthreads();
    if (!clustered)
      buf ^= 1;
    if (clustered && tile + (int)gridDim.y < ntiles) { // Yx is reused by the next tile: nobody may still be reading it
      cluster_arrive_release();
      cluster_wait_acquire();
    }
  }
  if (clustered) { // no CTA may exit while a peer can still write into its shared memory
    cluster_arrive_release();
    cluster_wait_acquire();
  }
  TPROBE(7);
#ifdef OVB_TSQR_TIMING
  if (tid == 0 && blockIdx.x == 0 && blockIdx.y == 0)
    printf("tsqr c0=%d lvl=%d grid=(%d,%d) rows=%d | load %lld qr %lld publish+Tt %lld tileload %lld Y %lld Z %lld upd+rest %lld | total %lld\n", c0,
           level, gridDim.x, gridDim.y, rows_i, tprobe[1] - tprobe[0], tprobe[2] - tprobe[1], tprobe[3] - tprobe[2], tprobe[4] - tprobe[3],
           tprobe[5] - tprobe[4], tprobe[6] - tprobe[5], tprobe[7] - tprobe[6], tprobe[7] - tprobe[0]);
#endif
}

// copy the trailing parts of the finished R rows out of A, zero the strict lower part, normalise diag >= 0
__global__ void k_tsqr_assemble(const double *__restrict__ A, int ldA, int m, int n, double *__restrict__ Rout, int ldR) {
  OVB_PDL_ENTER();
  int i = blockIdx.x; // row of R
  if (i >= n)
    return;
  int pend = min(n, (i / QR_NB + 1) * QR_NB); // first column right of this row's panel
  for (int j = threadIdx.x; j <= n; j += blockDim.x) {
    if (j < i)
      Rout[(size_t)i * ldR + j] = 0.0;
    else if (j >= pend)
      Rout[(size_t)i * ldR + j] = (i < m) ? A[(size_t)i * ldA + j] : 0.0;
    else if (i >= m)
      Rout[(size_t)i * ldR + j] = 0.0;
  }
  __syncthreads();
  double d = Rout[(size_t)i * ldR + i];
  __syncthreads(); // everyone has read the diagonal before anyone flips it
  if (d < 0.0) {
    for (int j = threadIdx.x; j <= n; j += blockDim.x)
      Rout[(size_t)i * ldR + j] = -Rout[(size_t)i * ldR + j];
  }
}

void launch_tsqr(ovb_ctx *ctx, double *A, int m, int n, int ldA, double *Rout, int ldR) {
  if (!ctx->attr_done[0]) { // function attributes are per device: one flag per context
    cudaFuncSetAttribute(k_tsqr_level, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(QrSmem));
    if (ctx->tsqr_cluster) { // can this device co-schedule one cluster of QR_CLUSTER CTAs with this much shared memory?
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3(QR_CLUSTER, 1);
      cfg.blockDim = dim3(QR_THREADS);
      cfg.dynamicSmemBytes = sizeof(QrSmem);
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeClusterDimension;
      at[0].val.clusterDim.x = QR_CLUSTER;
      at[0].val.clusterDim.y = 1;
      at[0].val.clusterDim.z = 1;
      cfg.attrs = at;
      cfg.numAttrs = 1;
      int ncl = 0;
      if (cudaOccupancyMaxActiveClusters(&ncl, k_tsqr_level, &cfg) != cudaSuccess || ncl < 1) {
        cudaGetLastError();
        ctx->tsqr_cluster = 0; // plain three-level tree instead
      }
    }
    ctx->attr_done[0] = 1;
  }
  const int nt = n + 1;
  // panel blocks of rows that never get factored (m < n) must read as zero
  cudaMemsetAsync(Rout, 0, sizeof(double) * (size_t)n * ldR, ctx->stream);
  for (int c0 = 0; c0 < n; c0 += QR_NB) {
    int nbp = n - c0 < QR_NB ? n - c0 : QR_NB;
    int len = m - c0;
    if (len <= 0)
      break;
    int level = 0;
    const int ntiles = (nt - (c0 + nbp) + QR_CT - 1) / QR_CT;
    // level-0 chunk height: enough chunks to fill the SMs, but no more than one cluster can take over at level 1
    int cr0 = QR_CR;
    {
      int want = ctx->sm_count < QR_CLUSTER * QR_CR / QR_NB ? ctx->sm_count : QR_CLUSTER * QR_CR / QR_NB;
      if (!ctx->tsqr_cluster)
        want = ctx->sm_count;
      int h = ((len + want - 1) / want + 15) & ~15;
      if (h < 64)
        h = 64;
      if (h < QR_CR && len > QR_CLUSTER * QR_CR)
        cr0 = h;
    }
    while (true) {
      const int crl = (level == 0) ? cr0 : QR_CR;
      int chunks = (len + crl - 1) / crl;
      // 2..QR_CLUSTER chunks: one thread-block cluster factors them as a single tall block and finishes the panel
      const bool clustered = ctx->tsqr_cluster && chunks > 1 && chunks <= QR_CLUSTER;
      int last = (chunks == 1) || clustered;
      // few chunks: spread the trailing tiles over more CTAs; many chunks: one CTA walks all tiles (no redundant panels)
      // one CTA per SM (~200 KB of shared memory): fill the SMs in ONE wave; every column group of a chunk repeats the
      // panel factorisation, so never use more groups than that
      int gx = clustered ? QR_CLUSTER : chunks;
      int gy = ctx->sm_count / gx;
      if (gy > ntiles)
        gy = ntiles;
      if (gy < 1)
        gy = 1;
      const double *Win = level > 0 ? ctx->d_W[(level - 1) & 1] : nullptr;
      double *Wout = ctx->d_W[level & 1];
      const int cl = clustered ? QR_CLUSTER : 1;
      ovb_launch(ctx, k_tsqr_level, ovb_grid(dim3(gx, gy), dim3(cl)), dim3(QR_THREADS), sizeof(QrSmem), A, ldA, nt, c0, nbp, level, len, Win, Wout, Rout,
                 ldR, last, cl, cr0);
      ctx->n_launch_tsqr_level++;
      if (last)
        break;
      int rows_last = len - (chunks - 1) * crl;
      len = (chunks - 1) * nbp + (rows_last < nbp ? rows_last : nbp);
      level++;
    }
  }
  ovb_launch(ctx, k_tsqr_assemble, dim3(n), dim3(128), (size_t)(0), A, ldA, m, n, Rout, ldR);
}

// =====================================================================================================================
// stacked-column bookkeeping: which variables the accepted features touch, in which order (UpdaterMSCKF.cpp:237-245)
extern unsigned char *ovb_feat_order_ptr(ovb_ctx *ctx);

__global__ void k_column_map(const DevFrame *__restrict__ fr, const DevOpts *__restrict__ dop, const DevFeat *__restrict__ feats, int n_feats,
                             const unsigned char *__restrict__ feat_order, DevUpdateInfo *__restrict__ info, int rows_drop) {
  __shared__ unsigned int key[OVB_MAX_VARS];
  __shared__ int n_used_feats, rows_stacked;
  __shared__ int order[OVB_MAX_VARS];
  __shared__ int n_order;
  OVB_PDL_ENTER();
  const int tid = threadIdx.x;
  if (tid < OVB_MAX_VARS)
    key[tid] = 0xffffffffu;
  if (tid == 0) {
    n_used_feats = 0;
    rows_stacked = 0;
    n_order = 0;
  }
  __syncthreads();
  for (int f = tid; f < n_feats; f += blockDim.x) {
    if (feats[f].status != OVB_FEAT_OK)
      continue;
    atomicAdd(&n_used_feats, 1);
    atomicAdd(&rows_stacked, 2 * (feats[f].m1 - feats[f].m0) - rows_drop); // 3 rows lost to the nullspace projection (MSCKF), 0 (SLAM)
    const unsigned char *ord = feat_order + (size_t)f * (OVB_MAX_VARS + 1);
    int no = ord[0];
    for (int q = 0; q < no; q++)
      atomicMin(&key[ord[1 + q]], ((unsigned int)f << 7) | (unsigned int)q);
  }
  __syncthreads();
  const int n_slots = fr->n_slots;
  const bool first_seen = (dop->o.col_order == OVB_COLS_REFERENCE_FIRST_SEEN);
  if (tid < n_slots) {
    // rank among used slots: first-seen order = ascending key; canonical = ascending slot id
    int rank = 0, nused = 0;
    for (int s = 0; s < n_slots; s++) {
      bool used = key[s] != 0xffffffffu;
      nused += used ? 1 : 0;
      if (!used)
        continue;
      if (first_seen ? (key[s] < key[tid]) : (s < tid))
        rank++;
    }
    if (!first_seen)
      order[tid] = tid; // canonical layout: stacked column q IS canonical column q (unused variables stay as zero columns)
    else if (key[tid] != 0xffffffffu)
      order[rank] = tid;
    else {
      // unused slots go last, in slot order (their columns are all zero)
      int r2 = 0;
      for (int s = 0; s < tid; s++)
        if (key[s] == 0xffffffffu)
          r2++;
      order[nused + r2] = tid;
    }
    if (tid == 0)
      n_order = nused;
  }
  __syncthreads();
  if (tid == 0) {
    int col = 0, used_cols = 0;
    for (int q = 0; q < n_slots; q++) {
      int s = order[q];
      info->order_slot[q] = s;
      for (int k = 0; k < fr->slot_size[s]; k++) {
        info->col_state[col] = fr->slot_off[s] + k;
        info->col_canon[col] = fr->slot_col[s] + k;
        col++;
      }
      if (key[s] != 0xffffffffu)
        used_cols += fr->slot_size[s];
    }
    info->n_order = n_order;
    info->n_used = used_cols;
    info->n_feats_used = n_used_feats;
    info->rows_stacked = rows_stacked;
    info->neg_diag_index = -1;
    info->not_spd = 0;
    info->nonfinite = 0;
  }
}

void launch_column_map(ovb_ctx *ctx, int n_feats, BlobView bv, int rows_drop) {
  ovb_launch(ctx, k_column_map, dim3(1), dim3(256), (size_t)0, ctx->d_frame, ctx->d_opts, ctx->d_feat, n_feats, ovb_feat_order_ptr(ctx), ctx->d_info,
             rows_drop);
}

// SLAM update: the variables are the frame's slots plus one landmark per feature. A feature's landmark is the last entry of
// its Hxf_order and never seen before it (UpdaterSLAM.cpp:385-387), so its first-seen key is (f, number of frame entries
// of the feature). The counts cover the whole batch; full_map (a batch of one column group) also writes the column map of
// the group's layout exactly as k_column_map does for slots (unused variables last, in canonical order).
#define CM_MAX_ENT (OVB_MAX_VARS + OVB_MAX_COLS)
// A landmark in ANCHORED_INVERSE_DEPTH_SINGLE is 1 wide and loses 2 rows to its bearing projection; the others are 3 wide
// and keep all 2M rows.
__device__ __forceinline__ int slam_lm_width(const DevFeat &d) { return d.rep == OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE ? 1 : 3; }

__global__ void k_column_map_slam(const DevFrame *__restrict__ fr, const DevOpts *__restrict__ dop, const DevFeat *__restrict__ feats, int n_feats,
                                  const unsigned char *__restrict__ feat_order, DevUpdateInfo *__restrict__ info, int full_map) {
  __shared__ unsigned int key[OVB_MAX_VARS];
  __shared__ unsigned int ekey[CM_MAX_ENT];
  __shared__ int order[CM_MAX_ENT];
  __shared__ int n_used_feats, rows_stacked, lm_cols;
  OVB_PDL_ENTER();
  const int tid = threadIdx.x;
  if (tid < OVB_MAX_VARS)
    key[tid] = 0xffffffffu;
  if (tid == 0) {
    n_used_feats = 0;
    rows_stacked = 0;
    lm_cols = 0;
  }
  __syncthreads();
  for (int f = tid; f < n_feats; f += blockDim.x) {
    if (feats[f].status != OVB_FEAT_OK)
      continue;
    const int lmw = slam_lm_width(feats[f]);
    atomicAdd(&n_used_feats, 1);
    atomicAdd(&lm_cols, lmw);
    atomicAdd(&rows_stacked, 2 * (feats[f].m1 - feats[f].m0) - (lmw == 1 ? 2 : 0));
    const unsigned char *ord = feat_order + (size_t)f * (OVB_MAX_VARS + 1);
    int no = ord[0];
    for (int q = 0; q < no; q++)
      atomicMin(&key[ord[1 + q]], ((unsigned int)f << 7) | (unsigned int)q);
  }
  __syncthreads();
  const int n_slots = fr->n_slots;
  if (!full_map) {
    if (tid == 0) {
      int used_cols = 0, n_order = 0;
      for (int s = 0; s < n_slots; s++)
        if (key[s] != 0xffffffffu) {
          used_cols += fr->slot_size[s];
          n_order++;
        }
      info->n_order = n_order + n_used_feats;
      info->n_used = used_cols + lm_cols;
      info->n_feats_used = n_used_feats;
      info->rows_stacked = rows_stacked;
      info->neg_diag_index = -1;
      info->not_spd = 0;
      info->nonfinite = 0;
    }
    return;
  }
  const DevGroup *G = fr->groups;
  const int n_ent = G->n_ent;
  for (int i = tid; i < n_ent; i += blockDim.x) {
    const int e = G->ent[i];
    if (e >= 0) {
      ekey[i] = key[e];
    } else {
      const int f = -1 - e;
      ekey[i] = feats[f].status == OVB_FEAT_OK ? (((unsigned int)f << 7) | (unsigned int)feat_order[(size_t)f * (OVB_MAX_VARS + 1)]) : 0xffffffffu;
    }
  }
  __syncthreads();
  const bool first_seen = (dop->o.col_order == OVB_COLS_REFERENCE_FIRST_SEEN);
  for (int i = tid; i < n_ent; i += blockDim.x) {
    // rank among used variables: first-seen order = ascending key; canonical = ascending entry (covariance offset)
    int rank = 0, nused = 0, r2 = 0;
    for (int t = 0; t < n_ent; t++) {
      const bool used = ekey[t] != 0xffffffffu;
      nused += used ? 1 : 0;
      r2 += (!used && t < i) ? 1 : 0;
      if (used && (first_seen ? (ekey[t] < ekey[i]) : (t < i)))
        rank++;
    }
    if (!first_seen)
      order[i] = i; // canonical layout: stacked column q IS canonical column q (unused variables stay as zero columns)
    else if (ekey[i] != 0xffffffffu)
      order[rank] = i;
    else
      order[nused + r2] = i; // unused variables go last, in canonical order (their columns are all zero)
  }
  __syncthreads();
  if (tid == 0) {
    // canonical column of every entry, then the stacked map in the chosen order
    int c = 0;
    for (int i = 0; i < n_ent; i++) {
      const int e = G->ent[i];
      ekey[i] = (unsigned int)c; // ekey is free now: canonical start column
      c += e >= 0 ? fr->slot_size[e] : slam_lm_width(feats[-1 - e]);
    }
    int col = 0, used_cols = 0, n_order = 0;
    for (int q = 0; q < n_ent; q++) {
      const int i = order[q], e = G->ent[i];
      const int off = e >= 0 ? fr->slot_off[e] : feats[-1 - e].lm_off;
      const int sz = e >= 0 ? fr->slot_size[e] : slam_lm_width(feats[-1 - e]);
      const bool used = e >= 0 ? key[e] != 0xffffffffu : feats[-1 - e].status == OVB_FEAT_OK;
      for (int k = 0; k < sz; k++) {
        info->col_state[col] = off + k;
        info->col_canon[col] = (int)ekey[i] + k;
        col++;
      }
      if (used) {
        used_cols += sz;
        n_order++;
      }
    }
    info->n_order = n_order;
    info->n_used = used_cols;
    info->n_feats_used = n_used_feats;
    info->rows_stacked = rows_stacked;
    info->neg_diag_index = -1;
    info->not_spd = 0;
    info->nonfinite = 0;
  }
}

void launch_column_map_slam(ovb_ctx *ctx, int n_feats, bool full_map) {
  ovb_launch(ctx, k_column_map_slam, dim3(1), dim3(256), (size_t)0, ctx->d_frame, ctx->d_opts, ctx->d_feat, n_feats, ovb_feat_order_ptr(ctx),
             ctx->d_info, full_map ? 1 : 0);
}

// B[i][q] = Rin[i][col_canon[q]] for q < n_all, B[i][n_all] = Rin[i][n_all] (residual)
__global__ void k_gather_cols(const double *__restrict__ Rin, int ldRin, int n_all, const DevUpdateInfo *__restrict__ info, double *__restrict__ B,
                              int ldB) {
  OVB_PDL_ENTER();
  int i = blockIdx.x;
  for (int q = threadIdx.x; q <= n_all; q += blockDim.x) {
    int src = (q < n_all) ? info->col_canon[q] : n_all;
    B[(size_t)i * ldB + q] = Rin[(size_t)i * ldRin + src];
  }
}

void launch_reorder_R(ovb_ctx *ctx, const double *Rin, int n_all, int ldRin, double *Rout, int ldRout) {
  // permuted copy into the (now free) staging matrix, then the same TSQR re-triangularises it
  int ldB = ldRin;
  ovb_launch(ctx, k_gather_cols, dim3(n_all), dim3(128), (size_t)(0), Rin, ldRin, n_all, ctx->d_info, ctx->d_Hs, ldB);
  launch_tsqr(ctx, ctx->d_Hs, n_all, n_all, ldB, Rout, ldRout);
}
