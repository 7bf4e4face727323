// k_feature.cu — one CTA per feature: measurement Jacobians, left-nullspace projection, chi² gate, stacked write-out.
// Replaces UpdaterHelper::get_feature_jacobian_representation / get_feature_jacobian_full / nullspace_project_inplace
// (ov_msckf/src/update/UpdaterHelper.cpp:32-454), StateHelper::get_marginal_covariance for the gate
// (ov_msckf/src/state/StateHelper.cpp:226-254) and the chi² test + stacking of UpdaterMSCKF::update
// (ov_msckf/src/update/UpdaterMSCKF.cpp:196-256).
//
// GPU-first formulation (not the reference's dense Eigen path):
//  * the per-measurement Jacobian is kept block-sparse in shared memory (clone 2x6 | extrinsics 2x6 | intrinsics 2x8
//    [| anchor clone 2x6 | anchor extrinsics 2x6]) — 600 B per measurement instead of 2 x w_f doubles;
//  * the left nullspace of H_f is applied as a rank-3 compact-WY reflector (three Householder vectors) instead of
//    3(2M-1) sequential Givens rotations: Q2'[H_x r] = rows 3.. of (X - V Z). It spans the same subspace; the
//    projected block differs from the reference's by an orthogonal transform of its rows, which leaves H_o'H_o,
//    H_o'r_o, chi² and everything downstream unchanged (SURVEY.md App. A.6);
//  * the gate needs chi² = r_o'(Q2' S Q2)^-1 r_o with S = H_x P H_x' + s²I. S is accumulated from the sparse blocks
//    (≈6x fewer flops than the dense (2M-3) x w_f products) straight into a tile-packed triangle and factored ONCE,
//    unprojected, by the DMMA tile Cholesky of chol_tiles.cuh; the projection is folded into four right-hand-side rows
//    (r and the columns of Q1): chi² = a'a - (C'a)'(C'C)^-1(C'a), a = L^-1 r, C = L^-1 Q1 (see "gate" in the kernel).
//    Tracks too long for a shared-memory triangle (template parameter BIG) keep the explicit two-sided projection and the
//    scalar blocked Cholesky of chol.cuh on an L2-resident scratch slice;
//  * tracks whose per-measurement blocks do not fit one CTA either (template parameter LONG, up to OVB_MAX_MEAS_PER_FEAT
//    = 384 measurements) run the BIG algorithm with those blocks in the CTA's global scratch slice as well;
//  * rows are written straight into the stacked staging matrix in canonical column order, coalesced.
// Compiled with -fmad=false (see geom.cuh).
#include <algorithm>
#include <cstdio>
#include "geom.cuh"
#include "chol.cuh"
#include "chol_tiles.cuh"

#define FT_THREADS 256
#define FT_WARPS (FT_THREADS / 32)
#define FT_TU 2
#ifdef FT_PROBE // per-phase cycle stamps of the longest track of a launch (thread 0 of CTA 0), printed at the end of the feature
#define FT_STAMP(i) do { if (tid == 0 && blockIdx.x == 0) ft_t[i] = clock64(); } while (0)
#else
#define FT_STAMP(i) do { } while (0)
#endif      // measurements whose covariance rows are in flight together in the T = H_x P pass

// Per-measurement Jacobian blocks live in shared memory as structure-of-arrays:
//   Bsh[I][b][16]  blocks [2][8] (row stride 8): 0 clone(6) 1 extrinsics(6) 2 intrinsics(8) 3 anchor clone(6) 4 anchor extrinsics(6);
//                  blocks 3/4 exist only for the anchored representations (nblk = 5, else 3); SLAM updates add block 5 =
//                  the landmark's own 2x3 Jacobian H_f (nblk = 6)
//   Hfs[I][6], ress[I][2], mslot[I][8] (slot id per block or -1; blocks 3/4 only when their slot differs from blocks 0/1)
//   lut[I][lutw]   slot -> block index (255 = the measurement does not touch the slot)
struct MeasView {
  double *B;
  double *Hf;
  double *res;
  signed char *slot;
  unsigned char *lut;
  int nblk, lutw, bstride; // bstride = 16*nblk + 1 doubles per measurement: lanes walking measurements hit distinct banks
  __device__ __forceinline__ double *blk(int I, int b) const { return B + (size_t)I * bstride + b * 16; }
  // value of Jacobian row (I, r) in column k of slot s (0 when the measurement does not touch the slot)
  __device__ __forceinline__ double x_at(int I, int r, int s, int k) const {
    const int b = lut[(size_t)I * lutw + s];
    return (b == 255) ? 0.0 : B[(size_t)I * bstride + b * 16 + 8 * r + k];
  }
};

__device__ __forceinline__ int blk_w(int b) { return b == 2 ? 8 : (b == 5 ? 3 : 6); }

// block-wide sum of three values; every thread gets the result. red: FT_WARPS*3 doubles of shared memory.
__device__ __forceinline__ void block_sum3(double &a, double &b, double &c, double *red) {
  a = warp_sum(a);
  b = warp_sum(b);
  c = warp_sum(c);
  int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads(); // protect red from the previous use
  if (l == 0) {
    red[w * 3 + 0] = a;
    red[w * 3 + 1] = b;
    red[w * 3 + 2] = c;
  }
  __syncthreads();
  a = b = c = 0.0;
#pragma unroll
  for (int i = 0; i < FT_WARPS; i++) {
    a += red[i * 3 + 0];
    b += red[i * 3 + 1];
    c += red[i * 3 + 2];
  }
}

// block-wide sums of NV values; every thread gets the results. red: FT_WARPS*NV doubles of shared memory.
template <int NV> __device__ __forceinline__ void block_sum_n(double (&v)[NV], double *red) {
#pragma unroll
  for (int e = 0; e < NV; e++)
    v[e] = warp_sum(v[e]);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads(); // protect red from the previous use
  if (l == 0) {
#pragma unroll
    for (int e = 0; e < NV; e++)
      red[w * NV + e] = v[e];
  }
  __syncthreads();
#pragma unroll
  for (int e = 0; e < NV; e++) {
    double a = 0.0;
#pragma unroll
    for (int i = 0; i < FT_WARPS; i++)
      a += red[i * NV + e];
    v[e] = a;
  }
}

// The gate's factorisation as a real call: its register allocation (the 8x8 pivot block and the panel rows live in
// registers) is then independent of what the feature kernel keeps live around it.
__device__ __noinline__ void ft_gate_chol(double *ctbase, int NRB, int *flag, int n, int nrows) {
  const CtView cv = ct_view_carve(ctbase, NRB, flag);
  ct_chol_tiles<FT_THREADS>(cv, n, nrows, true, 0.0);
}

// ---- d p_FinG / d lambda and the anchor terms: UpdaterHelper.cpp:32-190. Returns L (3x3 row-major),
// Hanc (3x6), Hcal (3x6); has_anchor tells whether the anchored terms exist.
__device__ inline void jacobian_representation(const DevFrame *fr, const ovb_opts &op, int rep, dv3 p_FinG, dv3 p_FinG_fej, dv3 p_FinA_in,
                                               int acam, int aclone, double L[9], double Hanc[18], double Hcal[18]) {
#pragma unroll
  for (int i = 0; i < 9; i++)
    L[i] = 0.0;
  if (rep == OVB_REP_GLOBAL_3D) {
    L[0] = L[4] = L[8] = 1.0;
    return;
  }
  if (rep == OVB_REP_GLOBAL_FULL_INVERSE_DEPTH || rep == OVB_REP_ANCHORED_FULL_INVERSE_DEPTH) {
    // handled below once the linearisation point is known
  }
  dm3 Rcg;
  dv3 pA = p_FinA_in, p_IinC = mk3(0, 0, 0);
  bool anchored = (rep != OVB_REP_GLOBAL_FULL_INVERSE_DEPTH);
  if (anchored) {
    dm3 R_ItoC = ld_m3(fr->cam_R[acam]);
    p_IinC = ld_v3(fr->cam_p[acam]);
    dm3 R_GtoI = ld_m3(fr->clone_R[aclone]);
    dv3 p_IinG = ld_v3(fr->clone_p[aclone]);
    if (op.do_fej) {
      // p_FinG_best = R_GtoI' R_ItoC' (p_FinA - p_IinC) + p_IinG, then re-expressed with the FEJ anchor (:89-96)
      dm3 RtRt;
#pragma unroll
      for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++)
          RtRt.m[3 * i + j] = (R_GtoI.m[i] * R_ItoC.m[3 * j] + R_GtoI.m[3 + i] * R_ItoC.m[3 * j + 1]) + R_GtoI.m[6 + i] * R_ItoC.m[3 * j + 2];
      dv3 best = add3(mv3(RtRt, sub3(p_FinA_in, p_IinC)), p_IinG);
      R_GtoI = ld_m3(fr->clone_R_fej[aclone]);
      p_IinG = ld_v3(fr->clone_p_fej[aclone]);
      dm3 RR; // (R_GtoI' R_ItoC')' = R_ItoC R_GtoI evaluated as the transpose of the product
#pragma unroll
      for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++)
          RR.m[3 * j + i] = (R_GtoI.m[i] * R_ItoC.m[3 * j] + R_GtoI.m[3 + i] * R_ItoC.m[3 * j + 1]) + R_GtoI.m[6 + i] * R_ItoC.m[3 * j + 2];
      pA = add3(mv3(RR, sub3(best, p_IinG)), p_IinC);
    }
    // R_CtoG = R_GtoI' * R_ItoC'
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
      for (int j = 0; j < 3; j++)
        Rcg.m[3 * i + j] = (R_GtoI.m[i] * R_ItoC.m[3 * j] + R_GtoI.m[3 + i] * R_ItoC.m[3 * j + 1]) + R_GtoI.m[6 + i] * R_ItoC.m[3 * j + 2];
    // H_anc = [ -R_GtoI' * skew(R_ItoC' (p_FinA - p_IinC)) , I ]
    dm3 sk = skew3(mTv3(R_ItoC, sub3(pA, p_IinC)));
    dm3 nRt;
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
      for (int j = 0; j < 3; j++)
        nRt.m[3 * i + j] = -R_GtoI.m[3 * j + i];
    dm3 blk = mul33(nRt, sk);
#pragma unroll
    for (int r = 0; r < 3; r++)
#pragma unroll
      for (int c = 0; c < 3; c++) {
        Hanc[6 * r + c] = blk.m[3 * r + c];
        Hanc[6 * r + 3 + c] = (r == c) ? 1.0 : 0.0;
      }
    // H_calib = [ -R_CtoG * skew(p_FinA - p_IinC) , -R_CtoG ]
    dm3 nRcg;
#pragma unroll
    for (int i = 0; i < 9; i++)
      nRcg.m[i] = -Rcg.m[i];
    dm3 blk2 = mul33(nRcg, skew3(sub3(pA, p_IinC)));
#pragma unroll
    for (int r = 0; r < 3; r++)
#pragma unroll
      for (int c = 0; c < 3; c++) {
        Hcal[6 * r + c] = blk2.m[3 * r + c];
        Hcal[6 * r + 3 + c] = -Rcg.m[3 * r + c];
      }
  }
  if (rep == OVB_REP_ANCHORED_3D) {
#pragma unroll
    for (int i = 0; i < 9; i++)
      L[i] = Rcg.m[i];
    return;
  }
  dm3 d;
#pragma unroll
  for (int i = 0; i < 9; i++)
    d.m[i] = 0.0;
  if (rep == OVB_REP_GLOBAL_FULL_INVERSE_DEPTH || rep == OVB_REP_ANCHORED_FULL_INVERSE_DEPTH) {
    dv3 p = anchored ? pA : (op.do_fej ? p_FinG_fej : p_FinG);
    double rho = 1 / norm3(p);
    double phi = acos(rho * p.z);
    double theta = atan2(p.y, p.x);
    double sin_th = sin(theta), cos_th = cos(theta), sin_phi = sin(phi), cos_phi = cos(phi);
    d.m[0] = -(1.0 / rho) * sin_th * sin_phi;
    d.m[1] = (1.0 / rho) * cos_th * cos_phi;
    d.m[2] = -(1.0 / (rho * rho)) * cos_th * sin_phi;
    d.m[3] = (1.0 / rho) * cos_th * sin_phi;
    d.m[4] = (1.0 / rho) * sin_th * cos_phi;
    d.m[5] = -(1.0 / (rho * rho)) * sin_th * sin_phi;
    d.m[6] = 0.0;
    d.m[7] = -(1.0 / rho) * sin_phi;
    d.m[8] = -(1.0 / (rho * rho)) * cos_phi;
    if (!anchored) {
#pragma unroll
      for (int i = 0; i < 9; i++)
        L[i] = d.m[i];
      return;
    }
  } else { // ANCHORED_MSCKF_INVERSE_DEPTH (SINGLE is remapped to it for MSCKF features)
    double alpha = pA.x / pA.z;
    double beta = pA.y / pA.z;
    double rho = 1 / pA.z;
    d.m[0] = (1.0 / rho);
    d.m[2] = -(1.0 / (rho * rho)) * alpha;
    d.m[4] = (1.0 / rho);
    d.m[5] = -(1.0 / (rho * rho)) * beta;
    d.m[8] = -(1.0 / (rho * rho));
  }
  dm3 Lm = mul33(Rcg, d);
#pragma unroll
  for (int i = 0; i < 9; i++)
    L[i] = Lm.m[i];
}

__device__ __forceinline__ bool rep_is_relative(int rep) {
  return rep == OVB_REP_ANCHORED_3D || rep == OVB_REP_ANCHORED_FULL_INVERSE_DEPTH || rep == OVB_REP_ANCHORED_MSCKF_INVERSE_DEPTH ||
         rep == OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE;
}

// =====================================================================================================================
// mode 0: full (gate + write projected rows to Hs)   mode 1: dump pre-nullspace dense rows to `dump`
// mode 2: SLAM update (update/UpdaterSLAM.cpp:310-447): the landmark is a state variable (block 5 = H_f, slot lm_slot),
//         no nullspace projection (all 2M rows are kept), per-feature noise / gate multiplier, rows whitened by 1/sigma
// The SLAM variant is a separate instantiation so that the MSCKF hot path carries none of its code or registers.
// BIG: tracks whose gate matrix does not fit shared memory (the launcher decides): S lives in a per-CTA slice of an
// L2-resident scratch buffer and is factored by the scalar blocked Cholesky of chol.cuh after a two-sided projection.
// Otherwise the gate runs on the tile-packed triangle of chol_tiles.cuh (DMMA) with the projection folded into the
// right-hand sides (see "gate" below).
// LONG (implies BIG): the per-measurement arrays (Jacobian blocks, H_f, residuals, reflectors, slot tables) also live in
// the CTA's scratch slice, ahead of S, so shared memory no longer grows with the track; every one-thread-per-row step
// strides over the rows (up to 2 * OVB_MAX_MEAS_PER_FEAT = 3 * FT_THREADS).
// LONG runs one CTA per SM (its grid is at most the SM count), so it may use up to 255 registers per thread; ptxas still
// reports about 300 bytes of spill stores for it (against 1-1.5 KB for the 128-register variants).
// INIT (not SLAM): one new landmark of ovb_slam_delayed_init (StateHelper::initialize, UpdaterSLAM.cpp:197-233). The gate is
// the MSCKF one (the rows orthogonal to all three columns of H_f) with the feature's own representation, sigma and
// multiplier and the threshold of the initialize system's row count (2M, or 2M-2 for ANCHORED_INVERSE_DEPTH_SINGLE, whose
// bearing columns the reference projects out before the split). The projected rows go out in the feature's compact
// columns whatever the gate says, and the top rows Q1'[H_x | H_f | r] of the Householder split (the init system) go to
// `dump`, a DevInitSys. A Householder split differs from the reference's Givens split by a k x k orthogonal transform of
// the init rows, which leaves H_L^-1 H_R, H_L^-1 r and the posterior unchanged (tests/test_slam_init_cpu.py).
template <bool SLAM, bool BIG, bool LONG = false, bool INIT = false>
__global__ void __launch_bounds__(FT_THREADS, LONG ? 1 : 2)
    k_feature_system(const DevFrame *__restrict__ fr, const DevOpts *__restrict__ dop, DevFeat *__restrict__ feats, int sched_lo, int n_feats,
                     BlobView bv,
                     const double *__restrict__ P, int ldP, const double *__restrict__ chi2_table, double *__restrict__ Hs, int ldH,
                     unsigned char *__restrict__ feat_order, int mode, int maxM, int nblk, double *__restrict__ scratch,
                     size_t scratch_per_cta, double *__restrict__ dump, int ld_dump, int dump_rows) {
  static_assert(BIG || !LONG, "the long-track layout keeps S in scratch");
  static_assert(!(SLAM && INIT), "a delayed initialisation is not a SLAM update");
  static_assert(2 * OVB_MAX_MEAS_PER_FEAT <= 3 * FT_THREADS, "Householder rows per thread");
  constexpr int RPT = LONG ? 3 : 1; // rows of H_f per thread in the Householder QR
  OVB_PDL_ENTER();
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const ovb_opts &op = dop->o;
  constexpr bool slam = SLAM;
  // SLAM: the feature's own landmark is one more variable of the per-CTA tables, slot id n_slots (the frame's slots are
  // clones and calibration only), and its columns follow the frame's canonical columns: j = fr->n_all + k. Every landmark
  // has its own representation (DevFeat::rep, so its own width); the tables below are sized for the batch's widest.
  const int n_all_c = fr->n_all + (SLAM ? fr->lm_w : 0);
  const int n_slots = fr->n_slots;
  constexpr int NSV = SLAM ? OVB_MAX_VARS + 4 : OVB_MAX_VARS; // entries of the per-CTA slot tables
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int n_all8 = (n_all_c + 7) & ~7;
  // ---- shared memory carve-up (mirrors feature_smem_bytes). LONG: the per-measurement arrays go to the scratch slice
  // instead (same order, mirrored by feature_long_slice_doubles), followed by S.
  size_t o = 0, og = 0;
  unsigned char *gslice = LONG ? (unsigned char *)(scratch + (size_t)blockIdx.x * scratch_per_cta) : nullptr;
  auto carve_m = [&](size_t bytes) -> unsigned char * {
    unsigned char *p;
    if constexpr (LONG) {
      p = gslice + og;
      og += bytes;
    } else {
      p = smem_raw + o;
      o += bytes;
    }
    return p;
  };
  MeasView mv;
  mv.nblk = nblk;
  mv.bstride = 16 * nblk + 1;
  mv.lutw = (n_slots + (SLAM ? 1 : 0) + 3) & ~3;
  mv.B = (double *)carve_m(sizeof(double) * (size_t)mv.bstride * maxM);
  mv.Hf = (double *)carve_m(sizeof(double) * 6 * (size_t)maxM);
  mv.res = (double *)carve_m(sizeof(double) * 2 * (size_t)maxM);
  double *V = (double *)carve_m(sizeof(double) * 3 * 2 * (size_t)maxM); // [2M][3]
  double *Z = (double *)(smem_raw + o); // [3][n_all+1]
  o += sizeof(double) * 3 * (size_t)(n_all_c + 1);
  double *red = (double *)(smem_raw + o);
  o += sizeof(double) * (FT_WARPS * 12 + 24);
  int *slot2l = (int *)(smem_raw + o); // [NSV] compact column start of a slot or -1
  o += sizeof(int) * NSV;
  int *fslot_off = (int *)(smem_raw + o); // frame tables, staged once per CTA (SLAM: entry n_slots = the feature's landmark)
  o += sizeof(int) * NSV;
  int *ishare = (int *)(smem_raw + o); // misc ints: [0]=wf [1]=flag [2]=gated
  o += sizeof(int) * 8;
  short *lcol_slot = (short *)(smem_raw + o); // [n_all] slot of compact column c
  o += sizeof(short) * (size_t)n_all8;
  short *lcol_k = (short *)(smem_raw + o);
  o += sizeof(short) * (size_t)n_all8;
  unsigned char *ccol_slot = smem_raw + o; // [n_all] slot / offset-in-slot of canonical column j
  o += (size_t)n_all8;
  unsigned char *ccol_k = smem_raw + o;
  o += (size_t)n_all8;
  unsigned char *fslot_size = smem_raw + o;
  o += NSV;
  mv.slot = (signed char *)carve_m((size_t)maxM * 8); // [maxM][8]
  unsigned char *mcam = carve_m((size_t)((maxM + 7) & ~7)); // [maxM] camera id / clone slot of each measurement
  unsigned char *mcs = carve_m((size_t)((maxM + 7) & ~7));
  mv.lut = carve_m((size_t)maxM * mv.lutw);
  o = (o + 15) & ~(size_t)15;
  og = (og + 15) & ~(size_t)15;
  // Tw [FT_WARPS][2][n_all]: one measurement's two rows of T = H_x P per warp; then (not BIG) the gate's Cholesky working set
  double *Tw = (double *)(smem_raw + o);
  double *ctbase = Tw + (size_t)FT_WARPS * 2 * n_all_c; // 16-byte aligned: an even number of doubles after a 16-byte boundary

  // ---- frame tables -> shared memory (the bookkeeping below would otherwise chase them through L2 serially)
  for (int s = tid; s < n_slots; s += FT_THREADS) {
    fslot_off[s] = fr->slot_off[s];
    fslot_size[s] = (unsigned char)fr->slot_size[s];
    const int c0 = fr->slot_col[s], w = fr->slot_size[s];
    for (int k = 0; k < w; k++) {
      ccol_slot[c0 + k] = (unsigned char)s;
      ccol_k[c0 + k] = (unsigned char)k;
    }
  }
  if constexpr (SLAM) { // a landmark of width w reads the first w of these columns
    if (tid < fr->lm_w) {
      ccol_slot[fr->n_all + tid] = (unsigned char)n_slots;
      ccol_k[fr->n_all + tid] = (unsigned char)tid;
    }
  }

  // this launch works on entries [sched_lo, n_feats) of the longest-first schedule (one size class, see the launcher)
  for (int fi = sched_lo + blockIdx.x; fi < n_feats; fi += gridDim.x) {
    const int f = feats[fi].sched; // longest tracks first: the short ones fill the tail of the last wave
#ifdef FT_PROBE
    long long ft_t[12] = {0};
#endif
    FT_STAMP(0);
    DevFeat *F = &feats[f];
    // SLAM landmarks kept as a single inverse depth (ANCHORED_INVERSE_DEPTH_SINGLE, UpdaterSLAM.cpp:344-353): the landmark
    // variable is 1 wide (the depth column of H_f) and the two bearing columns are projected out like an MSCKF feature's three
    const bool single = (SLAM || INIT) && (F->rep == OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE);
    const int nproj = slam ? (single ? 2 : 0) : 3; // columns of H_f that are projected out = rows removed
    const int r0 = nproj;
    const int lmw = single ? 1 : 3;                // width of the landmark block (block 5)
    const int n_all = SLAM ? fr->n_all + lmw : n_all_c;
    const int m0 = F->m0, M = F->m1 - F->m0;
    const int rows = 2 * M;
    const int status_in = F->status;
    __syncthreads();
    if (mode == 1) {
      // ------------------------------------------------------------------ debug: dense pre-nullspace rows
      if (status_in != OVB_FEAT_OK || M < 2 || M > maxM)
        continue;
    } else {
      if (M < ((slam && !single) ? 1 : 2))
        continue; // no rows reserved
      if (status_in != OVB_FEAT_OK || M > maxM) {
        // rows reserved for this feature are zero (they are harmless in the QR); SLAM: the width of its group's layout
        int nr = rows - r0;
        const int n_out = SLAM ? fr->groups[F->grp].n_cols : n_all;
        for (int e = tid; e < nr * (n_out + 1); e += FT_THREADS) {
          int i = e / (n_out + 1), j = e % (n_out + 1);
          Hs[(size_t)(F->row0 + i) * ldH + j] = 0.0;
        }
        if (tid == 0 && feat_order)
          feat_order[(size_t)f * (OVB_MAX_VARS + 1)] = 0;
        continue;
      }
    }
    // SINGLE's Jacobians are those of ANCHORED_MSCKF_INVERSE_DEPTH (UpdaterSLAM.cpp:327-329), as DevOpts::rep remaps MSCKF features
    const int rep = (SLAM || INIT) ? (single ? OVB_REP_ANCHORED_MSCKF_INVERSE_DEPTH : F->rep) : dop->rep;
    const bool relative = rep_is_relative(rep);
    const int acam = F->anchor_cam, aclone = F->anchor_clone;
    const dv3 p_FinA = ld_v3(F->p_FinA);
    dv3 p_FinG = ld_v3(F->p_FinG);
    int s_anchor = -1, s_anchor_ext = -1;
    if (relative) {
      s_anchor = fr->clone_slot[aclone];
      s_anchor_ext = op.do_calib_camera_pose ? fr->cam_ext_slot[acam] : -1;
      // p_FinG = R_GtoI' R_ItoC' (p_FinA - p_IinC) + p_IinG (UpdaterHelper.cpp:269-280)
      dm3 R_ItoC = ld_m3(fr->cam_R[acam]);
      dv3 p_IinC = ld_v3(fr->cam_p[acam]);
      dm3 R_GtoI = ld_m3(fr->clone_R[aclone]);
      dv3 p_IinG = ld_v3(fr->clone_p[aclone]);
      dm3 RtRt;
#pragma unroll
      for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++)
          RtRt.m[3 * i + j] = (R_GtoI.m[i] * R_ItoC.m[3 * j] + R_GtoI.m[3 + i] * R_ItoC.m[3 * j + 1]) + R_GtoI.m[6 + i] * R_ItoC.m[3 * j + 2];
      p_FinG = add3(mv3(RtRt, sub3(p_FinA, p_IinC)), p_IinG);
    }
    // MSCKF features: p_FinG_fej = p_FinG (UpdaterMSCKF.cpp:190-193); anchored: always the "best" p_FinG
    // (UpdaterHelper.cpp:284-287); SLAM landmarks in a global representation bring their own FEJ value (UpdaterSLAM.cpp:339-340)
    const dv3 p_FinG_fej = (slam && !relative) ? ld_v3(F->p_FinG_fej) : p_FinG;
    const double sig2 = F->sigma_sq;

    for (int e = tid; e < M * mv.lutw; e += FT_THREADS)
      mv.lut[e] = 255;
    if constexpr (!BIG) { // the gate's working set starts zeroed (panel buffers, the padding of the edge tiles, the dummy tile)
      if (mode != 1) {
        const int nd = (int)ct_view_doubles((rows + 1 + nproj + 7) >> 3);
        for (int e = tid; e < nd; e += FT_THREADS)
          ctbase[e] = 0.0;
      }
    }
    // measurement metadata -> shared memory, one coalesced pass
    for (int i = tid; i < M; i += FT_THREADS) {
      mcam[i] = bv.cam[m0 + i];
      mcs[i] = (unsigned char)fr->clone_slot[bv.clone[m0 + i]];
    }
    __syncthreads();
    // ---- one thread of the last warp (it computes no Jacobian unless M is huge): slot bookkeeping
    //      (Hx_order in the reference's first-seen order + compact column map)
    const int bk_tid = (M <= FT_THREADS - 32) ? FT_THREADS - 32 : 0;
    if (tid == bk_tid) {
      unsigned long long seen = 0ull;
      unsigned char *ord = feat_order ? feat_order + (size_t)f * (OVB_MAX_VARS + 1) : nullptr;
      int no = 0;
      for (int k = F->key0; k < F->key1; k++) {
        int key = bv.keys[k];
        if (op.do_calib_camera_pose) {
          int s = fr->cam_ext_slot[key];
          if (s >= 0 && !((seen >> s) & 1ull)) {
            seen |= 1ull << s;
            if (ord)
              ord[1 + no] = (unsigned char)s;
            no++;
          }
        }
        if (op.do_calib_camera_intrinsics) {
          int s = fr->cam_intr_slot[key];
          if (s >= 0 && !((seen >> s) & 1ull)) {
            seen |= 1ull << s;
            if (ord)
              ord[1 + no] = (unsigned char)s;
            no++;
          }
        }
        for (int i = 0; i < M; i++) {
          if (mcam[i] != key)
            continue;
          int s = mcs[i];
          if (!((seen >> s) & 1ull)) {
            seen |= 1ull << s;
            if (ord)
              ord[1 + no] = (unsigned char)s;
            no++;
          }
        }
      }
      if (relative) {
        if (!((seen >> s_anchor) & 1ull)) {
          seen |= 1ull << s_anchor;
          if (ord)
            ord[1 + no] = (unsigned char)s_anchor;
          no++;
        }
        if (s_anchor_ext >= 0 && !((seen >> s_anchor_ext) & 1ull)) {
          seen |= 1ull << s_anchor_ext;
          if (ord)
            ord[1 + no] = (unsigned char)s_anchor_ext;
          no++;
        }
      }
      // SLAM: Hxf_order.push_back(landmark) is always last and never seen before (UpdaterSLAM.cpp:385-387), so the order
      // lists the frame variables only and the column map appends the landmark after them
      if (ord)
        ord[0] = (unsigned char)no;
      // compact columns in canonical slot order: the slot starts here, the per-column tables by all threads below.
      // SLAM: the landmark block goes where its covariance offset puts it among the frame's slots
      int wf = 0;
      int lm_at = 0;
      if constexpr (SLAM) {
        lm_at = F->lm_off;
        fslot_off[n_slots] = lm_at;
        fslot_size[n_slots] = (unsigned char)lmw;
      }
      for (int s = 0; s < n_slots; s++) {
        if constexpr (SLAM) {
          if (lm_at >= 0 && fslot_off[s] > lm_at) {
            slot2l[n_slots] = wf;
            wf += lmw;
            lm_at = -1;
          }
        }
        if ((seen >> s) & 1ull) {
          slot2l[s] = wf;
          wf += fslot_size[s];
        } else
          slot2l[s] = -1;
      }
      if constexpr (SLAM) {
        if (lm_at >= 0) {
          slot2l[n_slots] = wf;
          wf += lmw;
        }
      }
      ishare[0] = wf;
      ishare[1] = 0;
      ishare[2] = 0;
    }

    // ---- per-measurement Jacobian (UpdaterHelper.cpp:313-423), one thread per measurement (strided: LONG tracks exceed the block)
    for (int t = tid; t < M; t += FT_THREADS) {
      const int i = m0 + t;
      const int cam = mcam[t], cl = bv.clone[i];
      double *B0 = mv.blk(t, 0), *B1 = mv.blk(t, 1), *B2 = mv.blk(t, 2);
      double *mHf = mv.Hf + 6 * t;
      signed char *msl = mv.slot + 8 * t;
      dm3 R_ItoC = ld_m3(fr->cam_R[cam]);
      dv3 p_IinC = ld_v3(fr->cam_p[cam]);
      dm3 R_GtoIi = ld_m3(fr->clone_R[cl]);
      dv3 p_IiinG = ld_v3(fr->clone_p[cl]);
      dv3 p_FinIi = mv3(R_GtoIi, sub3(p_FinG, p_IiinG));
      dv3 p_FinCi = add3(mv3(R_ItoC, p_FinIi), p_IinC);
      double un = p_FinCi.x / p_FinCi.z, vn = p_FinCi.y / p_FinCi.z;
      double ud, vd;
      cam_distort_d(fr->cam_model[cam], fr->cam_intr[cam], un, vn, ud, vd);
      mv.res[2 * t] = (double)bv.uv[2 * i] - ud;
      mv.res[2 * t + 1] = (double)bv.uv[2 * i + 1] - vd;
      if (op.do_fej) {
        R_GtoIi = ld_m3(fr->clone_R_fej[cl]);
        p_IiinG = ld_v3(fr->clone_p_fej[cl]);
        p_FinIi = mv3(R_GtoIi, sub3(p_FinG_fej, p_IiinG));
        p_FinCi = add3(mv3(R_ItoC, p_FinIi), p_IinC);
      }
      double dz_dzn[4], dz_dzeta[16];
      cam_distort_jacobian(fr->cam_model[cam], fr->cam_intr[cam], un, vn, dz_dzn, dz_dzeta);
      double zz = p_FinCi.z * p_FinCi.z;
      double dzn_dpfc[2][3] = {{1 / p_FinCi.z, 0, -p_FinCi.x / zz}, {0, 1 / p_FinCi.z, -p_FinCi.y / zz}};
      dm3 dpfc_dpfg = mul33(R_ItoC, R_GtoIi);
      dm3 dpfc_dth = mul33(R_ItoC, skew3(p_FinIi));
      double dz_dpfc[2][3], dz_dpfg[2][3];
#pragma unroll
      for (int r = 0; r < 2; r++)
#pragma unroll
        for (int k = 0; k < 3; k++)
          dz_dpfc[r][k] = dz_dzn[2 * r + 0] * dzn_dpfc[0][k] + dz_dzn[2 * r + 1] * dzn_dpfc[1][k];
#pragma unroll
      for (int r = 0; r < 2; r++)
#pragma unroll
        for (int k = 0; k < 3; k++)
          dz_dpfg[r][k] = (dz_dpfc[r][0] * dpfc_dpfg.m[k] + dz_dpfc[r][1] * dpfc_dpfg.m[3 + k]) + dz_dpfc[r][2] * dpfc_dpfg.m[6 + k];
      double L[9], Hanc[18], Hcal[18];
      jacobian_representation(fr, op, rep, p_FinG, p_FinG_fej, p_FinA, acam, aclone, L, Hanc, Hcal);
#pragma unroll
      for (int r = 0; r < 2; r++)
#pragma unroll
        for (int k = 0; k < 3; k++)
          mHf[3 * r + k] = (dz_dpfg[r][0] * L[k] + dz_dpfg[r][1] * L[3 + k]) + dz_dpfg[r][2] * L[6 + k];
      // clone block: dz_dpfc * [R_ItoC skew(p_FinIi), -R_ItoC R_GtoIi]
#pragma unroll
      for (int r = 0; r < 2; r++)
#pragma unroll
        for (int k = 0; k < 3; k++) {
          B0[8 * r + k] = (dz_dpfc[r][0] * dpfc_dth.m[k] + dz_dpfc[r][1] * dpfc_dth.m[3 + k]) + dz_dpfc[r][2] * dpfc_dth.m[6 + k];
          B0[8 * r + 3 + k] =
              (dz_dpfc[r][0] * (-dpfc_dpfg.m[k]) + dz_dpfc[r][1] * (-dpfc_dpfg.m[3 + k])) + dz_dpfc[r][2] * (-dpfc_dpfg.m[6 + k]);
        }
      int sl[6];
      sl[5] = -1;
      if (slam) { // H_xf = [H_x, H_f]: the landmark's own columns (UpdaterSLAM.cpp:365-383)
        double *B5 = mv.blk(t, 5);
#pragma unroll
        for (int r = 0; r < 2; r++)
#pragma unroll
          for (int k = 0; k < 3; k++)
            B5[8 * r + k] = single ? mHf[3 * r + 2] : mHf[3 * r + k]; // single: only entry 0 (the depth column) is read
        sl[5] = n_slots;
      }
      sl[0] = mcs[t];
      sl[1] = op.do_calib_camera_pose ? fr->cam_ext_slot[cam] : -1;
      sl[2] = op.do_calib_camera_intrinsics ? fr->cam_intr_slot[cam] : -1;
      sl[3] = -1;
      sl[4] = -1;
#pragma unroll
      for (int k = 0; k < 16; k++)
        B1[k] = 0.0;
      // anchored extras: H(anchor clone) += dz_dpfg*H_anc ; H(anchor ext) += dz_dpfg*H_calib (:396-398)
      if (relative) {
        double *B3 = mv.blk(t, 3), *B4 = mv.blk(t, 4);
        double Ea[12], Ec[12];
#pragma unroll
        for (int r = 0; r < 2; r++)
#pragma unroll
          for (int k = 0; k < 6; k++) {
            Ea[6 * r + k] = (dz_dpfg[r][0] * Hanc[k] + dz_dpfg[r][1] * Hanc[6 + k]) + dz_dpfg[r][2] * Hanc[12 + k];
            Ec[6 * r + k] = (dz_dpfg[r][0] * Hcal[k] + dz_dpfg[r][1] * Hcal[6 + k]) + dz_dpfg[r][2] * Hcal[12 + k];
          }
        if (s_anchor == sl[0]) {
#pragma unroll
          for (int r = 0; r < 2; r++)
#pragma unroll
            for (int k = 0; k < 6; k++)
              B0[8 * r + k] += Ea[6 * r + k];
        } else {
          sl[3] = s_anchor;
#pragma unroll
          for (int r = 0; r < 2; r++)
#pragma unroll
            for (int k = 0; k < 6; k++)
              B3[8 * r + k] = Ea[6 * r + k];
        }
        if (s_anchor_ext >= 0) {
          if (s_anchor_ext == sl[1]) {
#pragma unroll
            for (int r = 0; r < 2; r++)
#pragma unroll
              for (int k = 0; k < 6; k++)
                B1[8 * r + k] += Ec[6 * r + k];
          } else {
            sl[4] = s_anchor_ext;
#pragma unroll
            for (int r = 0; r < 2; r++)
#pragma unroll
              for (int k = 0; k < 6; k++)
                B4[8 * r + k] = Ec[6 * r + k];
          }
        }
      }
      if (op.do_calib_camera_pose) {
        // dz_dpfc * [skew(p_FinCi - p_IinC), I] added onto the block (:404-413)
        dm3 sk = skew3(sub3(p_FinCi, p_IinC));
#pragma unroll
        for (int r = 0; r < 2; r++)
#pragma unroll
          for (int k = 0; k < 3; k++) {
            B1[8 * r + k] += (dz_dpfc[r][0] * sk.m[k] + dz_dpfc[r][1] * sk.m[3 + k]) + dz_dpfc[r][2] * sk.m[6 + k];
            B1[8 * r + 3 + k] += (dz_dpfc[r][0] * (k == 0 ? 1.0 : 0.0) + dz_dpfc[r][1] * (k == 1 ? 1.0 : 0.0)) + dz_dpfc[r][2] * (k == 2 ? 1.0 : 0.0);
          }
      }
      if (op.do_calib_camera_intrinsics) {
#pragma unroll
        for (int k = 0; k < 16; k++)
          B2[k] = dz_dzeta[k];
      }
#pragma unroll
      for (int b = 0; b < 6; b++) {
        msl[b] = (signed char)sl[b];
        if (sl[b] >= 0)
          mv.lut[(size_t)t * mv.lutw + sl[b]] = (unsigned char)b;
      }
    }
    __syncthreads();

    const int wf = ishare[0];
    for (int j = tid; j < n_all; j += FT_THREADS) { // compact column -> (slot, offset in slot)
      const int sj = ccol_slot[j], l0 = slot2l[sj];
      if (l0 >= 0) {
        lcol_slot[l0 + ccol_k[j]] = (short)sj;
        lcol_k[l0 + ccol_k[j]] = (short)ccol_k[j];
      }
    }
    __syncthreads();
    if (mode == 1) {
      // dense dump: [Hf rows x 3][res rows][Hx rows x ld_dump], rows indexed 2*m0 + local
      double *dHf = dump, *dres = dump + (size_t)dump_rows * 3, *dHx = dump + (size_t)dump_rows * 4;
      for (int e = tid; e < rows * (n_all + 4); e += FT_THREADS) {
        int i = e / (n_all + 4), j = e % (n_all + 4);
        size_t grow = (size_t)(2 * m0 + i);
        int r = i & 1;
        if (j < n_all)
          dHx[grow * ld_dump + j] = mv.x_at(i >> 1, r, ccol_slot[j], ccol_k[j]);
        else if (j < n_all + 3)
          dHf[grow * 3 + (j - n_all)] = mv.Hf[6 * (i >> 1) + 3 * r + (j - n_all)];
        else
          dres[grow] = mv.res[i];
      }
      continue;
    }

    FT_STAMP(1);
    // ---- Householder QR of H_f (rows x 3): V (unit lower trapezoid) and tau; one thread per row (RPT rows per thread
    // for LONG: row tid + q * FT_THREADS)
    double a[RPT][3];
#pragma unroll
    for (int q = 0; q < RPT; q++) {
      const int row = tid + q * FT_THREADS;
      a[q][0] = a[q][1] = a[q][2] = 0.0;
      if (row < rows) {
        a[q][0] = mv.Hf[3 * row];
        a[q][1] = mv.Hf[3 * row + 1];
        a[q][2] = mv.Hf[3 * row + 2];
      }
    }
    double tau[3] = {0.0, 0.0, 0.0};
    double *rowk = red + FT_WARPS * 3; // 3 doubles: the pivot row's values
    if (nproj < 3) { // fewer (or no) reflectors: the unused ones are tau = 0, V = 0, which makes their sweeps no-ops
      for (int row = tid; row < rows; row += FT_THREADS)
        V[3 * row] = V[3 * row + 1] = V[3 * row + 2] = 0.0;
      __syncthreads();
    }
#pragma unroll
    for (int k = 0; k < 3; k++) {
      if (k >= nproj)
        break;
      // g[j] = sum over rows below the pivot of a_k a_j  (g[k] = squared norm of the sub-column)
      double g[3];
#pragma unroll
      for (int q = 0; q < RPT; q++) {
        const int row = tid + q * FT_THREADS;
        const bool below = (row > k && row < rows);
#pragma unroll
        for (int j = 0; j < 3; j++) {
          const double gq = below ? a[q][k] * a[q][j] : 0.0;
          g[j] = (q == 0) ? gq : g[j] + gq;
        }
      }
      block_sum3(g[0], g[1], g[2], red);
      if (tid == k) {
        rowk[0] = a[0][0];
        rowk[1] = a[0][1];
        rowk[2] = a[0][2];
      }
      __syncthreads();
      const double alpha = rowk[k];
      const double sigma = g[k];
      double beta, scale, tk;
      if (sigma == 0.0) { // nothing below the pivot: H = I
        tk = 0.0;
        beta = alpha;
        scale = 0.0;
      } else {
        beta = sqrt(alpha * alpha + sigma);
        if (alpha >= 0.0)
          beta = -beta;
        tk = (beta - alpha) / beta;
        scale = 1.0 / (alpha - beta);
      }
      tau[k] = tk;
#pragma unroll
      for (int q = 0; q < RPT; q++) {
        const int row = tid + q * FT_THREADS;
        const bool below = (row > k && row < rows);
        const double vr = below ? a[q][k] * scale : (row == k ? 1.0 : 0.0);
        // v'a_j = a_kj + (sum_below a_k a_j)/(alpha-beta), then a_j -= tau (v'a_j) v for the remaining columns
#pragma unroll
        for (int j = 0; j < 3; j++) {
          if (j > k) {
            double wj = rowk[j] + g[j] * scale;
            if (row >= k && row < rows)
              a[q][j] -= tk * wj * vr;
          }
        }
        if (row < rows)
          V[3 * row + k] = vr;
      }
      __syncthreads();
    }
    // Gram of the reflectors: G10 = v1'v0, G20 = v2'v0, G21 = v2'v1
    double G10 = 0, G20 = 0, G21 = 0;
#pragma unroll
    for (int q = 0; q < RPT; q++) {
      const int row = tid + q * FT_THREADS;
      if (row < rows && nproj > 0) {
        double v0 = V[3 * row], v1 = V[3 * row + 1], v2 = V[3 * row + 2];
        G10 = (q == 0) ? v1 * v0 : G10 + v1 * v0;
        G20 = (q == 0) ? v2 * v0 : G20 + v2 * v0;
        G21 = (q == 0) ? v2 * v1 : G21 + v2 * v1;
      }
    }
    block_sum3(G10, G20, G21, red);

    FT_STAMP(2);
    // ---- Z[k][j]: coefficients of Q'x = x - V z for every canonical column j and the residual (j = n_all)
    for (int j = tid; j <= n_all; j += FT_THREADS) {
      double w0 = 0, w1 = 0, w2 = 0;
      if (j < n_all) {
        const int s = ccol_slot[j], kk = ccol_k[j];
        if (slot2l[s] >= 0) {
          // branch-free (a measurement that does not touch the slot adds zeros) so that the loads of several
          // measurements are in flight together
#pragma unroll 4
          for (int I = 0; I < M; I++) {
            const int b = mv.lut[(size_t)I * mv.lutw + s];
            const bool hit = (b != 255);
            const double *Bb = mv.blk(I, hit ? b : 0);
            const double x0 = hit ? Bb[kk] : 0.0, x1 = hit ? Bb[8 + kk] : 0.0;
            const double *v = V + 6 * I;
            w0 += v[0] * x0 + v[3] * x1;
            w1 += v[1] * x0 + v[4] * x1;
            w2 += v[2] * x0 + v[5] * x1;
          }
        }
      } else {
        for (int I = 0; I < M; I++) {
          const double r0 = mv.res[2 * I], r1 = mv.res[2 * I + 1];
          const double *v = V + 6 * I;
          w0 += v[0] * r0 + v[3] * r1;
          w1 += v[1] * r0 + v[4] * r1;
          w2 += v[2] * r0 + v[5] * r1;
        }
      }
      double z0 = tau[0] * w0;
      double z1 = tau[1] * (w1 - G10 * z0);
      double z2 = tau[2] * (w2 - G20 * z0 - G21 * z1);
      Z[j] = z0;
      Z[(n_all + 1) + j] = z1;
      Z[2 * (n_all + 1) + j] = z2;
    }
    __syncthreads();
    if constexpr (INIT) { // H_L = Q1' H_f: the same reflector sweep on the three columns of H_f, rows 0..2
      double wf9[9];
#pragma unroll
      for (int e = 0; e < 9; e++)
        wf9[e] = 0.0;
      for (int i = tid; i < rows; i += FT_THREADS) {
#pragma unroll
        for (int kq = 0; kq < 3; kq++)
#pragma unroll
          for (int c = 0; c < 3; c++)
            wf9[3 * kq + c] += V[3 * i + kq] * mv.Hf[3 * i + c];
      }
      block_sum_n<9>(wf9, red);
      if (tid < 9) {
        const int i = tid / 3, c = tid % 3;
        const double z0 = tau[0] * wf9[c];
        const double z1 = tau[1] * (wf9[3 + c] - G10 * z0);
        const double z2 = tau[2] * (wf9[6 + c] - G20 * z0 - G21 * z1);
        ((DevInitSys *)dump)->HL[3 * i + c] = mv.Hf[3 * i + c] - ((V[3 * i] * z0 + V[3 * i + 1] * z1) + V[3 * i + 2] * z2);
      }
    }

    const int nr = rows - r0;
    bool spd = true;
    double c2 = 0.0;
    FT_STAMP(3);
    // ---- S = H_x P_marg H_x' + s² I from the sparse blocks (rows x rows), warp per measurement row pair
    // BIG: full symmetric S in a per-CTA slice of an L2-resident scratch buffer (odd leading dimension: conflict-free row and
    // column sweeps); else the lower triangle goes straight into the tile-packed layout of the gate's Cholesky
    const int ldS = rows | 1;
    double *S = LONG ? (double *)(gslice + og) : (BIG ? scratch + (size_t)blockIdx.x * scratch_per_cta : nullptr);
    const int NRB = (rows + 1 + nproj + 7) >> 3;
    const CtView cv = ct_view_carve(ctbase, NRB, &ishare[1]);
    double *Tmy = Tw + (size_t)wid * 2 * n_all;
    // row pairs are dealt out so that every warp gets a similar share of the triangular J >= I sweep
    for (int it = 0; it * FT_WARPS < M; it++) {
      const int I = (it & 1) ? (it * FT_WARPS + (FT_WARPS - 1 - wid)) : (it * FT_WARPS + wid);
      if (I >= M)
        continue;
      const signed char *slI = mv.slot + 8 * I;
      const int s0 = slI[0], s1 = slI[1], s2 = slI[2];
      const double *B0 = mv.blk(I, 0), *B1 = mv.blk(I, 1), *B2 = mv.blk(I, 2);
      // T_I[r][c] = sum_b sum_k B_b[r][k] * P[off_b + k][state(c)]; all loads of a column are issued before their use
      // (P is L2-resident: ~20 dependent-latency round trips per column otherwise)
      for (int c = lane; c < wf; c += 32) {
        const int pc = fslot_off[lcol_slot[c]] + lcol_k[c];
        double pv[20];
        const double *P0 = P + (size_t)fslot_off[s0] * ldP + pc;
        const double *P1 = P + (size_t)fslot_off[s1 >= 0 ? s1 : s0] * ldP + pc;
        const double *P2 = P + (size_t)fslot_off[s2 >= 0 ? s2 : s0] * ldP + pc;
#pragma unroll
        for (int k = 0; k < 6; k++)
          pv[k] = __ldg(P0 + (size_t)k * ldP);
        if (s1 >= 0) {
#pragma unroll
          for (int k = 0; k < 6; k++)
            pv[6 + k] = __ldg(P1 + (size_t)k * ldP);
        }
        if (s2 >= 0) {
#pragma unroll
          for (int k = 0; k < 8; k++)
            pv[12 + k] = __ldg(P2 + (size_t)k * ldP);
        }
        double t0 = 0.0, t1 = 0.0;
#pragma unroll
        for (int k = 0; k < 6; k++) {
          t0 = fma(B0[k], pv[k], t0);
          t1 = fma(B0[8 + k], pv[k], t1);
        }
        // one accumulator pair per block: three 6..8-deep chains side by side instead of one 20-deep chain
        double u0 = 0.0, u1 = 0.0, v0 = 0.0, v1 = 0.0;
        if (s1 >= 0) {
#pragma unroll
          for (int k = 0; k < 6; k++) {
            u0 = fma(B1[k], pv[6 + k], u0);
            u1 = fma(B1[8 + k], pv[6 + k], u1);
          }
        }
        if (s2 >= 0) {
#pragma unroll
          for (int k = 0; k < 8; k++) {
            v0 = fma(B2[k], pv[12 + k], v0);
            v1 = fma(B2[8 + k], pv[12 + k], v1);
          }
        }
        t0 += u0 + v0;
        t1 += u1 + v1;
        if (nblk > 3) {
#pragma unroll
          for (int b = 3; b < 6; b++) {
            if (b >= nblk)
              break;
            const int sb = slI[b];
            if (sb < 0)
              continue;
            const double *B = mv.blk(I, b);
            const double *Pb = P + (size_t)fslot_off[sb] * ldP + pc;
            const int wb = (b == 5) ? lmw : blk_w(b);
            double pw[6];
#pragma unroll
            for (int k = 0; k < 6; k++)
              pw[k] = (k < wb) ? __ldg(Pb + (size_t)k * ldP) : 0.0;
#pragma unroll
            for (int k = 0; k < 6; k++) {
              if (k < wb) {
                t0 = fma(B[k], pw[k], t0);
                t1 = fma(B[8 + k], pw[k], t1);
              }
            }
          }
        }
        Tmy[c] = t0;
        Tmy[n_all + c] = t1;
      }
      __syncwarp();
      for (int J = I + lane; J < M; J += 32) {
        const signed char *slJ = mv.slot + 8 * J;
        double s00 = 0, s01 = 0, s10 = 0, s11 = 0;
        // block widths are compile-time (6 6 8 6 6, landmark 1 or 3): the loads of a block are issued together
#define FT_S_BLOCK(BI, W)                                                                       \
  if ((BI) < nblk) {                                                                            \
    const int sb = slJ[BI];                                                                     \
    if (sb >= 0) {                                                                              \
      const double *B = mv.blk(J, BI);                                                          \
      const double *ta_ = Tmy + slot2l[sb], *tb_ = ta_ + n_all;                                 \
      _Pragma("unroll") for (int k = 0; k < (W); k++) {                                         \
        const double ta = ta_[k], tb = tb_[k];                                                  \
        s00 = fma(ta, B[k], s00);                                                               \
        s01 = fma(ta, B[8 + k], s01);                                                           \
        s10 = fma(tb, B[k], s10);                                                               \
        s11 = fma(tb, B[8 + k], s11);                                                           \
      }                                                                                         \
    }                                                                                           \
  }
        FT_S_BLOCK(0, 6)
        FT_S_BLOCK(1, 6)
        FT_S_BLOCK(2, 8)
        FT_S_BLOCK(3, 6)
        FT_S_BLOCK(4, 6)
#undef FT_S_BLOCK
        if (nblk > 5 && slJ[5] >= 0) {
          const double *B = mv.blk(J, 5);
          const double *ta_ = Tmy + slot2l[slJ[5]], *tb_ = ta_ + n_all;
          for (int k = 0; k < lmw; k++) {
            const double ta = ta_[k], tb = tb_[k];
            s00 = fma(ta, B[k], s00);
            s01 = fma(ta, B[8 + k], s01);
            s10 = fma(tb, B[k], s10);
            s11 = fma(tb, B[8 + k], s11);
          }
        }
        if (J == I) {
          s00 += sig2;
          s11 += sig2;
          s10 = s01; // exact symmetry of the diagonal 2x2 block
        }
        if constexpr (BIG) {
          S[(2 * I) * ldS + 2 * J] = s00;
          S[(2 * I) * ldS + 2 * J + 1] = s01;
          S[(2 * I + 1) * ldS + 2 * J] = s10;
          S[(2 * I + 1) * ldS + 2 * J + 1] = s11;
          S[(2 * J) * ldS + 2 * I] = s00;
          S[(2 * J + 1) * ldS + 2 * I] = s01;
          S[(2 * J) * ldS + 2 * I + 1] = s10;
          S[(2 * J + 1) * ldS + 2 * I + 1] = s11;
        } else { // s_ab = S[2I+a][2J+b] = S[2J+b][2I+a], J >= I: the lower triangle
          cv.T[ct_idx(2 * J, 2 * I)] = s00;
          cv.T[ct_idx(2 * J + 1, 2 * I)] = s01;
          if (J != I)
            cv.T[ct_idx(2 * J, 2 * I + 1)] = s10;
          cv.T[ct_idx(2 * J + 1, 2 * I + 1)] = s11;
        }
      }
      __syncwarp();
    }
    __syncthreads();

    FT_STAMP(4);
    if constexpr (BIG) {
      // ---- S <- Q' S Q (both sides), only rows/cols 3.. are used afterwards
      for (int pass = 0; pass < 2 && nproj > 0; pass++) {
        for (int j = tid; j < rows; j += FT_THREADS) {
          // pass 0: vector = column j (stride ldS); pass 1: vector = row j (stride 1)
          const int st = (pass == 0) ? ldS : 1;
          double *x = (pass == 0) ? (S + j) : (S + (size_t)j * ldS);
          double w0 = 0, w1 = 0, w2 = 0;
          for (int i = 0; i < rows; i++) {
            double xv = x[(size_t)i * st];
            w0 += V[3 * i] * xv;
            w1 += V[3 * i + 1] * xv;
            w2 += V[3 * i + 2] * xv;
          }
          double z0 = tau[0] * w0;
          double z1 = tau[1] * (w1 - G10 * z0);
          double z2 = tau[2] * (w2 - G20 * z0 - G21 * z1);
          for (int i = 0; i < rows; i++)
            x[(size_t)i * st] -= (V[3 * i] * z0 + V[3 * i + 1] * z1) + V[3 * i + 2] * z2;
        }
        __syncthreads();
      }
      // projected residual as the extra row `rows` of S: r_o[i] = res[i] - V[i,:] z(res)
      {
        double z0 = Z[n_all], z1 = Z[(n_all + 1) + n_all], z2 = Z[2 * (n_all + 1) + n_all];
        for (int i = tid; i < rows; i += FT_THREADS) {
          double rv = mv.res[i] - ((V[3 * i] * z0 + V[3 * i + 1] * z1) + V[3 * i + 2] * z2);
          S[(size_t)rows * ldS + i] = rv;
        }
      }
      __syncthreads();
      // ---- chi² = |L^-1 r_o|² on the trailing (rows-3) block
      spd = chol_lower_block<FT_THREADS, 2>(S + r0 * ldS + r0, ldS, nr, 1, &ishare[1], red + FT_WARPS * 3 + 4);
      c2 = 0.0;
      for (int i = tid; i < nr; i += FT_THREADS) {
        double y = S[(size_t)rows * ldS + r0 + i];
        c2 += y * y;
      }
      double dummy1 = 0, dummy2 = 0;
      block_sum3(c2, dummy1, dummy2, red);
    } else {
      // ---- gate on the tile-packed triangle. chi² = r_o' (Q2' S Q2)^-1 r_o with S = H_x P_marg H_x' + s² I is evaluated
      // without projecting S: for Q = [Q1 Q2] orthogonal,
      //   (Q2' S Q2)^-1 = Q2' S^-1 Q2 - Q2' S^-1 Q1 (Q1' S^-1 Q1)^-1 Q1' S^-1 Q2,  so with S = L L', a = L^-1 r, C = L^-1 Q1:
      //   chi² = a'a - (C'a)' (C'C)^-1 (C'a)       (the generalised-least-squares residual of r against range(H_f))
      // r and the nproj columns of Q1 ride through the factorisation as right-hand-side rows. Q1 = Q E comes straight from
      // the reflectors (Q x = x - V z with the reverse recurrence), so a rank-deficient H_f behaves as in the projected form.
      const int nrows_t = rows + 1 + nproj;
      {
        double zq[3][3]; // zq[j][k]: coefficient k of Q e_j
#pragma unroll
        for (int j = 0; j < 3; j++) {
          const double w0 = V[3 * j], w1 = V[3 * j + 1], w2 = V[3 * j + 2];
          const double z2 = tau[2] * w2;
          const double z1 = tau[1] * (w1 - G21 * z2);
          const double z0 = tau[0] * (w0 - G10 * z1 - G20 * z2);
          zq[j][0] = z0, zq[j][1] = z1, zq[j][2] = z2;
        }
        for (int i = tid; i < rows; i += FT_THREADS) {
          cv.T[ct_idx(rows, i)] = mv.res[i];
          const double v0 = V[3 * i], v1 = V[3 * i + 1], v2 = V[3 * i + 2];
#pragma unroll
          for (int j = 0; j < 3; j++)
            if (j < nproj)
              cv.T[ct_idx(rows + 1 + j, i)] = ((i == j) ? 1.0 : 0.0) - ((v0 * zq[j][0] + v1 * zq[j][1]) + v2 * zq[j][2]);
        }
      }
      FT_STAMP(6);
      ft_gate_chol(ctbase, NRB, &ishare[1], rows, nrows_t);
      FT_STAMP(7);
      // a'a, C'a, C'C over the solved right-hand-side rows
      double q[10];
#pragma unroll
      for (int e = 0; e < 10; e++)
        q[e] = 0.0;
      for (int i = tid; i < rows; i += FT_THREADS) {
        const double a = cv.T[ct_idx(rows, i)];
        double cq[3] = {0.0, 0.0, 0.0};
#pragma unroll
        for (int j = 0; j < 3; j++)
          if (j < nproj)
            cq[j] = cv.T[ct_idx(rows + 1 + j, i)];
        q[0] = fma(a, a, q[0]);
        q[1] = fma(cq[0], a, q[1]);
        q[2] = fma(cq[1], a, q[2]);
        q[3] = fma(cq[2], a, q[3]);
        q[4] = fma(cq[0], cq[0], q[4]);
        q[5] = fma(cq[1], cq[0], q[5]);
        q[6] = fma(cq[1], cq[1], q[6]);
        q[7] = fma(cq[2], cq[0], q[7]);
        q[8] = fma(cq[2], cq[1], q[8]);
        q[9] = fma(cq[2], cq[2], q[9]);
      }
      block_sum_n<10>(q, red);
      {
        // (C'C) y = C'a by a 3x3 Cholesky; unused columns are the identity
        const double W00 = nproj > 0 ? q[4] : 1.0, W11 = nproj > 1 ? q[6] : 1.0, W22 = nproj > 2 ? q[9] : 1.0;
        const double l00 = sqrt(W00), l10 = q[5] / l00, l20 = q[7] / l00;
        const double l11 = sqrt(W11 - l10 * l10), l21 = (q[8] - l20 * l10) / l11;
        const double l22 = sqrt(W22 - l20 * l20 - l21 * l21);
        const double y0 = q[1] / l00, y1 = (q[2] - l10 * y0) / l11, y2 = (q[3] - l20 * y0 - l21 * y1) / l22;
        c2 = q[0] - ((y0 * y0 + y1 * y1) + y2 * y2);
      }
      spd = (ishare[1] == 0);
    }
    const double qnan = __longlong_as_double(0x7ff8000000000000LL);
    double chi2 = spd ? c2 : qnan;
    double chi2_check = chi2_table[min(INIT ? (single ? rows - 2 : rows) : nr, OVB_CHI2_TABLE_LEN - 1)];
    bool gated = !(chi2 <= F->chi2_mult * chi2_check); // UpdaterMSCKF.cpp:225, UpdaterSLAM.cpp:409 (NaN rejects)
    if (tid == 0) {
      F->chi2 = chi2;
      if (gated)
        F->status = OVB_FEAT_CHI2;
    }
    FT_STAMP(8);
    // ---- write the projected rows into the stacked matrix, canonical columns, coalesced
    if constexpr (SLAM) {
      // the group's layout: frame columns (group column -> frame canonical column), the landmark columns of the group's
      // features (this feature's own at lm_col, zero for the others), the residual last; rows whitened by 1/sigma of the
      // feature's class, the EKF update then runs with R = I (R_big of UpdaterSLAM.cpp:444 is sigma^2 I per feature)
      const DevGroup *G = fr->groups + F->grp;
      const int n_out = G->n_cols, lm_col = F->lm_col;
      const double wgt = 1.0 / sqrt(sig2);
      for (int jb = 0; jb <= n_out; jb += FT_THREADS) {
        const int jg = jb + tid;
        if (jg > n_out)
          break;
        int j = n_all; // kernel column: frame canonical column, fr->n_all + k for the landmark, n_all for the residual
        bool present = true;
        if (jg < n_out) {
          const int c = G->col_frame[jg];
          if (c >= 0)
            j = c;
          else if (jg >= lm_col && jg < lm_col + lmw)
            j = fr->n_all + (jg - lm_col);
          else
            present = false; // another feature's landmark
        }
        int s = 0, kk = 0;
        if (present && j < n_all) {
          s = ccol_slot[j];
          kk = ccol_k[j];
          present = slot2l[s] >= 0;
        }
        double *out = Hs + (size_t)F->row0 * ldH + jg;
        if (gated || !present) {
          for (int i = r0; i < rows; i++)
            out[(size_t)(i - r0) * ldH] = 0.0;
        } else {
          const double z0 = Z[j], z1 = Z[(n_all + 1) + j], z2 = Z[2 * (n_all + 1) + j];
#pragma unroll 4
          for (int i = r0; i < rows; i++) {
            const int I = i >> 1, r = i & 1;
            const int b = (j == n_all) ? 255 : mv.lut[(size_t)I * mv.lutw + s];
            const double *src = (j == n_all) ? (mv.res + i) : (mv.blk(I, b == 255 ? 0 : b) + 8 * r + kk);
            const double xl = *src;
            const double xv = (j < n_all && b == 255) ? 0.0 : xl;
            out[(size_t)(i - r0) * ldH] = (xv - ((V[3 * i] * z0 + V[3 * i + 1] * z1) + V[3 * i + 2] * z2)) * wgt;
          }
        }
      }
    } else if constexpr (INIT) {
      // compact columns c < wf (canonical order of the touched slots), the residual at c = wf. Rows 3.. are the projected
      // system at row0; rows 3-k..2 the init system (SINGLE drops the two bearing rows 0-1).
      DevInitSys *sys = (DevInitSys *)dump;
      const int i0 = single ? 2 : 0;
      for (int c = tid; c <= wf; c += FT_THREADS) {
        int s = 0, kk = 0, j = n_all;
        if (c < wf) {
          s = lcol_slot[c];
          kk = lcol_k[c];
          j = fr->slot_col[s] + kk;
          sys->col_state[c] = fslot_off[s] + kk;
        }
        const double z0 = Z[j], z1 = Z[(n_all + 1) + j], z2 = Z[2 * (n_all + 1) + j];
        double *out = Hs + (size_t)F->row0 * ldH + c;
        for (int i = i0; i < rows; i++) {
          const int I = i >> 1, r = i & 1;
          const int b = (j == n_all) ? 255 : mv.lut[(size_t)I * mv.lutw + s];
          const double xv = (j == n_all) ? mv.res[i] : (b == 255 ? 0.0 : mv.blk(I, b)[8 * r + kk]);
          const double v = xv - ((V[3 * i] * z0 + V[3 * i + 1] * z1) + V[3 * i + 2] * z2);
          if (i >= 3)
            out[(size_t)(i - 3) * ldH] = v;
          else if (c < wf)
            sys->HR[(size_t)(i - i0) * wf + c] = v;
          else
            sys->res[i] = v;
        }
      }
      if (tid == 0)
        sys->n = wf;
    } else {
      for (int jb = 0; jb <= n_all; jb += FT_THREADS) {
        int j = jb + tid;
        if (j > n_all)
          break;
        int s = 0, kk = 0;
        bool present = false;
        if (j < n_all) {
          s = ccol_slot[j];
          kk = ccol_k[j];
          present = slot2l[s] >= 0;
        }
        double z0 = Z[j], z1 = Z[(n_all + 1) + j], z2 = Z[2 * (n_all + 1) + j];
        double *out = Hs + (size_t)F->row0 * ldH + j;
        if (gated || (j < n_all && !present)) {
          for (int i = r0; i < rows; i++)
            out[(size_t)(i - r0) * ldH] = 0.0;
        } else {
#pragma unroll 4
          for (int i = r0; i < rows; i++) {
            const int I = i >> 1, r = i & 1;
            const int b = (j == n_all) ? 255 : mv.lut[(size_t)I * mv.lutw + s];
            const double *src = (j == n_all) ? (mv.res + i) : (mv.blk(I, b == 255 ? 0 : b) + 8 * r + kk);
            const double xl = *src;
            const double xv = (j < n_all && b == 255) ? 0.0 : xl;
            out[(size_t)(i - r0) * ldH] = xv - ((V[3 * i] * z0 + V[3 * i + 1] * z1) + V[3 * i + 2] * z2);
          }
        }
      }
    }
#ifdef FT_PROBE
    if (tid == 0 && blockIdx.x == 0 && fi == sched_lo && mode == 0)
      printf("feat M=%d wf=%d: jac %lld hh %lld Z %lld | S sweep %lld | rhs rows %lld chol %lld chi2 %lld write %lld | total %lld\n", M, ishare[0],
             ft_t[1] - ft_t[0], ft_t[2] - ft_t[1], ft_t[3] - ft_t[2], ft_t[4] - ft_t[3], ft_t[6] - ft_t[4], ft_t[7] - ft_t[6], ft_t[8] - ft_t[7],
             clock64() - ft_t[8], clock64() - ft_t[0]);
#endif
  }
}

// Paths of the per-feature kernel, chosen per track by its length (feature_path):
//   FT_TILE  everything in shared memory, gate on the tile-packed triangle (DMMA Cholesky)
//   FT_BIG   per-measurement blocks in shared memory, S in a per-CTA slice of ctx->d_scratch (sized at ovb_create for
//            OVB_BIG_MAX_MEAS measurements)
//   FT_LONG  per-measurement blocks and S in a per-CTA slice of ctx->d_long (grown on demand, feature_scratch_reserve)
enum { FT_TILE = 0, FT_BIG = 1, FT_LONG = 2 };
static const size_t FT_SMEM_LIMIT = 227 * 1024; // dynamic shared memory of one H100 CTA

// Column and slot counts of the per-feature kernel's tables: the frame's, plus (SLAM) the feature's own landmark as one
// more slot whose columns follow the frame's, as wide as the batch's widest landmark
struct FeatDims {
  int n_all, n_slots, nsv;
};
static FeatDims feature_dims(const ovb_ctx *ctx, bool slam) {
  if (slam)
    return {ctx->h_frame->n_all + ctx->h_frame->lm_w, ctx->h_frame->n_slots + 1, OVB_MAX_VARS + 4};
  return {ctx->h_frame->n_all, ctx->h_frame->n_slots, OVB_MAX_VARS};
}

// dynamic shared memory of one launch whose longest track has maxM measurements (mirrors the kernel's carve-up)
static size_t feature_smem_bytes(int maxM, const FeatDims &dm, int nblk, int path) {
  size_t o = 0;
  const int n_all = dm.n_all, n_slots = dm.n_slots;
  const size_t n_all8 = (size_t)((n_all + 7) & ~7);
  if (path != FT_LONG) {
    o += sizeof(double) * (size_t)(16 * nblk + 1) * maxM;
    o += sizeof(double) * 6 * (size_t)maxM;
    o += sizeof(double) * 2 * (size_t)maxM;
    o += sizeof(double) * 3 * 2 * (size_t)maxM;
  }
  o += sizeof(double) * 3 * (size_t)(n_all + 1);
  o += sizeof(double) * (FT_WARPS * 12 + 24);
  o += sizeof(int) * (size_t)dm.nsv * 2;
  o += sizeof(int) * 8;
  o += sizeof(short) * n_all8 * 2;
  o += n_all8 * 2;
  o += (size_t)dm.nsv;
  if (path != FT_LONG) {
    o += (size_t)maxM * 8;
    o += (size_t)((maxM + 7) & ~7) * 2;
    o += (size_t)maxM * (size_t)((n_slots + 3) & ~3);
  }
  o = (o + 15) & ~(size_t)15;
  o += sizeof(double) * FT_WARPS * 2 * (size_t)n_all;
  if (path == FT_TILE)
    o += sizeof(double) * ct_view_doubles((2 * maxM + 4 + 7) >> 3);
  return o;
}

// FT_LONG: doubles of one CTA's scratch slice: the per-measurement arrays (same order as the kernel's carve_m), then S
// with its extra residual row, (2 maxM + 1) x (2 maxM | 1)
static size_t feature_long_slice_doubles(int maxM, int n_slots, int nblk) {
  size_t g = sizeof(double) * (size_t)(16 * nblk + 1) * maxM;
  g += sizeof(double) * (6 + 2 + 6) * (size_t)maxM;
  g += (size_t)maxM * 8;
  g += (size_t)((maxM + 7) & ~7) * 2;
  g += (size_t)maxM * (size_t)((n_slots + 3) & ~3);
  g = (g + 15) & ~(size_t)15;
  const size_t rows = 2 * (size_t)maxM;
  return g / sizeof(double) + (rows + 1) * (rows | 1);
}

static int feature_nblk(const ovb_ctx *ctx, bool slam) {
  // anchor blocks exist only for the anchored representations (same remap as DevOpts::rep)
  const int rep = ctx->h_opts->rep;
  return slam ? 6 : ((rep == OVB_REP_GLOBAL_3D || rep == OVB_REP_GLOBAL_FULL_INVERSE_DEPTH) ? 3 : 5);
}

// the path a track of M measurements runs on; monotone in M (tile, then BIG, then LONG)
static int feature_path(int M, const FeatDims &dm, int nblk) {
  const int m = M < 2 ? 2 : M;
  if (feature_smem_bytes(m, dm, nblk, FT_TILE) <= FT_SMEM_LIMIT)
    return FT_TILE;
  if (m <= OVB_BIG_MAX_MEAS && feature_smem_bytes(m, dm, nblk, FT_BIG) <= FT_SMEM_LIMIT)
    return FT_BIG;
  return FT_LONG;
}

// the delayed initialisation's tracks carry the anchor blocks whatever the call's representation (each feature has its own)
#define FT_INIT_NBLK 5

ovb_status feature_scratch_reserve(ovb_ctx *ctx, int n_feats, bool slam, bool init) {
  const FeatDims dm = feature_dims(ctx, slam);
  const int nblk = init ? FT_INIT_NBLK : feature_nblk(ctx, slam);
  int n_long = 0, maxM = 0;
  for (int f = 0; f < n_feats; f++) {
    const int M = ctx->h_feat[f].m1 - ctx->h_feat[f].m0;
    if (feature_path(M, dm, nblk) == FT_LONG) {
      n_long++;
      maxM = M > maxM ? M : maxM;
    }
  }
  if (n_long == 0)
    return OVB_OK;
  const size_t need = feature_long_slice_doubles(maxM, dm.n_slots, nblk) * (size_t)(n_long < ctx->sm_count ? n_long : ctx->sm_count);
  if (need <= ctx->long_cap)
    return OVB_OK;
  if (ctx->d_long)
    cudaFree(ctx->d_long); // waits for the work that may still read it
  ctx->d_long = nullptr;
  ctx->long_cap = 0;
  cudaError_t e = cudaMalloc(&ctx->d_long, sizeof(double) * need);
  if (e != cudaSuccess) {
    cudaGetLastError(); // clear the (non-sticky) allocation error so that a later call does not report it
    ctx->d_long = nullptr;
    snprintf(ctx->err, sizeof(ctx->err), "long-track scratch of %zu MB: %s", sizeof(double) * need >> 20, cudaGetErrorString(e));
    return OVB_ERR_CUDA;
  }
  ctx->long_cap = need;
  return OVB_OK;
}

// feat_order buffer lives right after the DevFeat array in ctx->d_feat's allocation (see ovb_api.cu)
extern unsigned char *ovb_feat_order_ptr(ovb_ctx *ctx);

void launch_feature_system(ovb_ctx *ctx, int n_feats, BlobView bv, int ldH, int mode) {
  if (n_feats <= 0)
    return;
  const bool slam = (mode == 2);
  const FeatDims dm = feature_dims(ctx, slam);
  const int nblk = feature_nblk(ctx, slam);
  if (!ctx->attr_done[1]) { // function attributes are per device: one flag per context
    cudaFuncSetAttribute(k_feature_system<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FT_SMEM_LIMIT);
    cudaFuncSetAttribute(k_feature_system<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FT_SMEM_LIMIT);
    cudaFuncSetAttribute(k_feature_system<false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FT_SMEM_LIMIT);
    cudaFuncSetAttribute(k_feature_system<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FT_SMEM_LIMIT);
    cudaFuncSetAttribute(k_feature_system<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FT_SMEM_LIMIT);
    cudaFuncSetAttribute(k_feature_system<true, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FT_SMEM_LIMIT);
    ctx->attr_done[1] = 1;
  }
  const int dump_rows = ctx->dump_rows; // rows of the current dump (set by ovb_feature_jacobians)
  auto len = [&](int i) {
    const DevFeat &d = ctx->h_feat[ctx->h_feat[i].sched];
    return d.m1 - d.m0;
  };
  // ---- per-track routing. The schedule is sorted longest-first and the path is monotone in the track length, so every
  // path works on a contiguous range of it: [0, b_big) LONG, [b_big, b_tile) BIG, [b_tile, n_feats) tile.
  int b_big = 0, b_tile;
  while (b_big < n_feats && feature_path(len(b_big), dm, nblk) == FT_LONG)
    b_big++;
  for (b_tile = b_big; b_tile < n_feats && feature_path(len(b_tile), dm, nblk) == FT_BIG;)
    b_tile++;
  struct Launch {
    int path, lo, hi, stream;
  } list[5];
  int nl = 0;
  auto add = [&](int path, int lo, int hi, int stream) {
    if (hi > lo)
      list[nl++] = {path, lo, hi, stream};
  };
  const bool has_long = b_tile > 0;
  add(FT_LONG, 0, b_big, 0);
  add(FT_BIG, b_big, b_tile, 0);
  // ---- size classes of the tile path. Shared memory per CTA grows with the square of the track length, and one launch
  // must size it for its longest track: a single launch runs 1-2 CTAs/SM for everybody and the short tracks wait for a
  // second wave. Three launches (tracks > 32, 17..32, <= 16 measurements; contiguous ranges of the schedule) on three
  // streams let several short-track CTAs share an SM next to the long ones. When BIG / LONG tracks are present they hold
  // the main stream and the tile classes run beside them on the two side streams.
  if (mode == 0 && ctx->feat_classes && n_feats - b_tile > ctx->sm_count) {
    const int thr[2] = {32, 16};
    int bound[4] = {b_tile, n_feats, n_feats, n_feats};
    for (int i = b_tile, c = 0; i < n_feats && c < 2; i++) {
      while (c < 2 && len(i) <= thr[c])
        bound[++c] = i;
    }
    add(FT_TILE, bound[0], bound[1], has_long ? 1 : 0);
    add(FT_TILE, bound[1], bound[2], has_long ? 2 : 1);
    add(FT_TILE, bound[2], bound[3], 2);
  } else {
    add(FT_TILE, b_tile, n_feats, 0);
  }
  cudaStream_t main_stream = ctx->stream;
  cudaStream_t streams[3] = {main_stream, ctx->side_stream, ctx->side_stream2};
  cudaEvent_t joined[3] = {nullptr, ctx->ev_join, ctx->ev_join2};
  bool used[3] = {false, false, false};
  for (int l = 0; l < nl; l++)
    used[list[l].stream] = true;
  if (used[1] || used[2]) // the side streams start from the main stream's state before any of these launches
    cudaEventRecord(ctx->ev_fork, main_stream);
  for (int s = 1; s < 3; s++)
    if (used[s])
      cudaStreamWaitEvent(streams[s], ctx->ev_fork, 0);
  for (int l = 0; l < nl; l++) {
    const Launch &L = list[l];
    const int s = L.stream;
    int cM = len(L.lo);
    cM = cM < 2 ? 2 : (cM > OVB_MAX_MEAS_PER_FEAT ? OVB_MAX_MEAS_PER_FEAT : cM);
    const size_t smem = feature_smem_bytes(cM, dm, nblk, L.path);
    int grid = L.hi - L.lo;
    double *scratch = nullptr;
    size_t per_cta = ctx->scratch_per_cta;
    if (L.path == FT_BIG) {
      grid = grid < ctx->scratch_ctas ? grid : ctx->scratch_ctas;
      scratch = ctx->d_scratch;
    } else if (L.path == FT_LONG) { // feature_scratch_reserve sized d_long for this track length (pack_inputs)
      per_cta = feature_long_slice_doubles(cM, dm.n_slots, nblk);
      const int fit = (int)(ctx->long_cap / per_cta);
      grid = grid < ctx->sm_count ? grid : ctx->sm_count;
      grid = grid < fit ? grid : fit;
      scratch = ctx->d_long;
      if (grid < 1) { // pack_inputs reserves d_long for every batch it accepts, so this is never taken
        snprintf(ctx->err, sizeof(ctx->err), "long-track scratch not reserved");
        continue;
      }
    }
    void (*kern)(const DevFrame *, const DevOpts *, DevFeat *, int, int, BlobView, const double *, int, const double *, double *, int,
                 unsigned char *, int, int, int, double *, size_t, double *, int, int);
    if (slam)
      kern = L.path == FT_TILE ? k_feature_system<true, false> : (L.path == FT_BIG ? k_feature_system<true, true> : k_feature_system<true, true, true>);
    else
      kern = L.path == FT_TILE ? k_feature_system<false, false> : (L.path == FT_BIG ? k_feature_system<false, true> : k_feature_system<false, true, true>);
    ctx->stream = streams[s];
    ovb_launch(ctx, kern, dim3(grid), dim3(FT_THREADS), smem, ctx->d_frame, ctx->d_opts, ctx->d_feat, L.lo, L.hi, bv, ctx->P[ctx->cur], ctx->ldP,
               ctx->d_chi2_table, ctx->d_Hs, ldH, ovb_feat_order_ptr(ctx), mode, cM, nblk, scratch, per_cta, ctx->d_dump, OVB_MAX_COLS, dump_rows);
    ctx->stream = main_stream;
  }
  for (int s = 1; s < 3; s++)
    if (used[s]) {
      cudaEventRecord(joined[s], streams[s]);
      cudaStreamWaitEvent(main_stream, joined[s], 0);
    }
}

void launch_feature_init(ovb_ctx *ctx, int sched, BlobView bv, int ldH) {
  const FeatDims dm = feature_dims(ctx, false);
  const int nblk = FT_INIT_NBLK;
  if (!ctx->attr_done[6]) {
    cudaFuncSetAttribute(k_feature_system<false, false, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FT_SMEM_LIMIT);
    cudaFuncSetAttribute(k_feature_system<false, true, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FT_SMEM_LIMIT);
    cudaFuncSetAttribute(k_feature_system<false, true, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FT_SMEM_LIMIT);
    ctx->attr_done[6] = 1;
  }
  const DevFeat &d = ctx->h_feat[ctx->h_feat[sched].sched];
  const int cM = std::min(std::max(d.m1 - d.m0, 2), OVB_MAX_MEAS_PER_FEAT);
  const int path = feature_path(cM, dm, nblk);
  double *scratch = nullptr;
  size_t per_cta = ctx->scratch_per_cta;
  if (path == FT_BIG) {
    scratch = ctx->d_scratch;
  } else if (path == FT_LONG) { // feature_scratch_reserve(init) sized d_long for the call's longest track
    per_cta = feature_long_slice_doubles(cM, dm.n_slots, nblk);
    scratch = ctx->d_long;
  }
  auto kern = path == FT_TILE ? k_feature_system<false, false, false, true>
                              : (path == FT_BIG ? k_feature_system<false, true, false, true> : k_feature_system<false, true, true, true>);
  ovb_launch(ctx, kern, dim3(1), dim3(FT_THREADS), feature_smem_bytes(cM, dm, nblk, path), ctx->d_frame, ctx->d_opts, ctx->d_feat, sched, sched + 1,
             bv, ctx->P[ctx->cur], ctx->ldP, ctx->d_chi2_table, ctx->d_Hs, ldH, nullptr, 0, cM, nblk, scratch, per_cta, (double *)ctx->d_init,
             0, 0);
}
