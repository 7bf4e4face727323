// k_triangulate.cu — one warp per feature: linear triangulation + Levenberg–Marquardt refinement.
// Replaces ov_core::FeatureInitializer::{single_triangulation, single_triangulation_1d, single_gaussnewton,
// compute_error} (ov_core/src/feat/FeatureInitializer.cpp:30-423) and the camera-at-clone pose build of
// UpdaterMSCKF::update (ov_msckf/src/update/UpdaterMSCKF.cpp:98-115).
// Compiled with -fmad=false (see geom.cuh). Lanes stride over the feature's measurements; sums over measurements
// run in measurement order (seq_add) and end identical in all lanes, everything else is warp-uniform.
#include "geom.cuh"

// R_GtoCi = R_ItoC * R_GtoI ; p_CiinG = p_IinG - R_GtoCi' * p_IinC   (UpdaterMSCKF.cpp:106-107)
__global__ void k_cam_poses(const DevFrame *fr, DevCamPoses *cc) {
  OVB_PDL_ENTER();
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  int total = fr->n_cams * fr->n_clones;
  if (idx >= total)
    return;
  int cam = idx / fr->n_clones, cl = idx % fr->n_clones;
  dm3 R_ItoC = ld_m3(fr->cam_R[cam]);
  dv3 p_IinC = ld_v3(fr->cam_p[cam]);
  dm3 R_GtoI = ld_m3(fr->clone_R[cl]);
  dv3 p_IinG = ld_v3(fr->clone_p[cl]);
  dm3 R = mul33(R_ItoC, R_GtoI);
  dv3 p = sub3(p_IinG, mTv3(R, p_IinC));
#pragma unroll
  for (int i = 0; i < 9; i++)
    cc->cc_R[cam][cl][i] = R.m[i];
  cc->cc_p[cam][cl][0] = p.x;
  cc->cc_p[cam][cl][1] = p.y;
  cc->cc_p[cam][cl][2] = p.z;
}

void launch_cam_poses(ovb_ctx *ctx) {
  int total = OVB_MAX_CAMS * OVB_MAX_CLONES;
  ovb_launch(ctx, k_cam_poses, dim3((total + 127) / 128), dim3(128), (size_t)0, ctx->d_frame, ctx->d_cc);
}

// Sum of one contribution per measurement IN MEASUREMENT ORDER — the order of the reference's loops over
// feat->timestamps (feat/FeatureInitializer.cpp:58-85, :238-283, :391-419) — so that every accumulated double is the
// reference's bit for bit: c[] holds this lane's contribution for measurement base + lane of the current 32-wide chunk,
// `count` (warp uniform) of them are real. A butterfly sum would differ in the last bits, and the LM loop's float32 casts
// turn such a difference into 1e-8-level jumps of p_FinG now and then (SURVEY.md App. A.1, hard part 8). seq_sums hands
// every lane the same sums.
#define TRI_MAX_WARPS 8
#define TRI_PITCH 33 // doubles per component row in the staging buffer (odd: lanes reading different rows hit distinct banks)
#define TRI_NSUM 9   // widest seq_add: A, b of the linear system, or the LM's Hessian (6) and gradient (3)
#define TRI_REL 15   // doubles of one cached relative pose (Rel)
#define TRI_LM_BATCH 3 // LM trials evaluated side by side (at most TRI_NSUM: their costs share one seq_add)
// Lane k (< NV) adds component k of lanes 0..count-1 onto its running sum `a` (0.0 before the first chunk) in that order,
// reading the terms from the warp's staging buffer — the same operation sequence as the reference's loop, ~2
// instructions per term for the warp instead of the 3 NV a shuffle-per-term version issues (864 instructions per 32
// measurements at NV = 9; the kernel is one dependent instruction chain per feature, so its duration follows its
// instruction count).
template <int NV> __device__ __forceinline__ void seq_add(double &a, const double (&c)[NV], int count, double *wbuf) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < NV; k++)
    wbuf[k * TRI_PITCH + lane] = c[k];
  __syncwarp();
  if (lane < NV) {
    const double *row = wbuf + lane * TRI_PITCH;
    for (int l = 0; l < count; l++)
      a += row[l];
  }
  __syncwarp(); // the buffer is rewritten by the next call
}
// after the last chunk: component k of the sums (lane k's `a`) in every lane
template <int NV> __device__ __forceinline__ void seq_sums(double (&s)[NV], double a) {
#pragma unroll
  for (int k = 0; k < NV; k++)
    s[k] = __shfl_sync(0xffffffffu, a, k);
}

struct Rel {
  dm3 R;  // R_AtoCi
  dv3 t;  // p_CiinA
  dv3 q;  // p_AinCi
};
// feat/FeatureInitializer.cpp:245-254
__device__ __forceinline__ Rel rel_pose(const DevCamPoses *fr, int cam, int cl, const dm3 &R_GtoA, dv3 p_AinG) {
  dm3 Rc = ld_m3(fr->cc_R[cam][cl]);
  dv3 pc = ld_v3(fr->cc_p[cam][cl]);
  Rel r;
  r.R = mul33T(Rc, R_GtoA);
  r.t = mv3(R_GtoA, sub3(pc, p_AinG));
  r.q = negmv3(r.R, r.t);
  return r;
}

// The relative poses depend on the anchor only, so each feature computes them once into its warp's cache: component k of
// measurement j (= i - m0) at rc[k * pitch + j]. Lanes walk consecutive measurements (conflict-free), and every lane
// reads back only the measurements it wrote.
__device__ __forceinline__ void st_rel(double *rc, int pitch, int j, const Rel &r) {
#pragma unroll
  for (int k = 0; k < 9; k++)
    rc[k * pitch + j] = r.R.m[k];
  rc[9 * pitch + j] = r.t.x, rc[10 * pitch + j] = r.t.y, rc[11 * pitch + j] = r.t.z;
  rc[12 * pitch + j] = r.q.x, rc[13 * pitch + j] = r.q.y, rc[14 * pitch + j] = r.q.z;
}
__device__ __forceinline__ Rel ld_rel(const double *rc, int pitch, int j) {
  Rel r;
#pragma unroll
  for (int k = 0; k < 9; k++)
    r.R.m[k] = rc[k * pitch + j];
  r.t = mk3(rc[9 * pitch + j], rc[10 * pitch + j], rc[11 * pitch + j]);
  r.q = mk3(rc[12 * pitch + j], rc[13 * pitch + j], rc[14 * pitch + j]);
  return r;
}

// feat/FeatureInitializer.cpp:377-423 at K points x[k] = (alpha, beta, rho); returns lane k's sum: the cost at x[k]
template <int K>
__device__ __forceinline__ double lm_cost(const double *rc, int pitch, const BlobView &bv, int m0, int m1, int lane, const dv3 (&x)[K], double *wbuf) {
  double acc = 0.0;
  for (int base = m0; base < m1; base += 32) {
    const int i = base + lane;
    double c[K];
#pragma unroll
    for (int k = 0; k < K; k++)
      c[k] = 0.0;
    if (i < m1) {
      Rel r = ld_rel(rc, pitch, i - m0);
      const float u0 = bv.uvn[2 * i], u1 = bv.uvn[2 * i + 1];
#pragma unroll
      for (int k = 0; k < K; k++) {
        const double alpha = x[k].x, beta = x[k].y, rho = x[k].z;
        double hi1 = r.R.m[0] * alpha + r.R.m[1] * beta + r.R.m[2] + rho * r.q.x;
        double hi2 = r.R.m[3] * alpha + r.R.m[4] * beta + r.R.m[5] + rho * r.q.y;
        double hi3 = r.R.m[6] * alpha + r.R.m[7] * beta + r.R.m[8] + rho * r.q.z;
        float z0 = (float)(hi1 / hi3), z1 = (float)(hi2 / hi3);
        float r0 = __fsub_rn(u0, z0), r1 = __fsub_rn(u1, z1);
        float nrm = __fsqrt_rn(__fadd_rn(__fmul_rn(r0, r0), __fmul_rn(r1, r1)));
        c[k] = (double)nrm * (double)nrm; // exact: product of two promoted floats
      }
    }
    seq_add<K>(acc, c, min(32, m1 - base), wbuf);
  }
  return acc;
}

// feat/FeatureInitializer.cpp:238-283 — returns lane k's sum of component k of Hess 00 01 02 11 12 22 | grad 0 1 2
__device__ __forceinline__ double lm_hess(const double *rc, int pitch, const BlobView &bv, int m0, int m1, int lane, double alpha, double beta,
                                          double rho, double *wbuf) {
  double acc = 0.0;
  for (int base = m0; base < m1; base += 32) {
    const int i = base + lane;
    double c[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (i < m1) {
      Rel r = ld_rel(rc, pitch, i - m0);
      double hi1 = r.R.m[0] * alpha + r.R.m[1] * beta + r.R.m[2] + rho * r.q.x;
      double hi2 = r.R.m[3] * alpha + r.R.m[4] * beta + r.R.m[5] + rho * r.q.y;
      double hi3 = r.R.m[6] * alpha + r.R.m[7] * beta + r.R.m[8] + rho * r.q.z;
      double h3sq = hi3 * hi3;
      double H0[3], H1[3];
      H0[0] = (r.R.m[0] * hi3 - hi1 * r.R.m[6]) / h3sq;
      H0[1] = (r.R.m[1] * hi3 - hi1 * r.R.m[7]) / h3sq;
      H0[2] = (r.q.x * hi3 - hi1 * r.q.z) / h3sq;
      H1[0] = (r.R.m[3] * hi3 - hi2 * r.R.m[6]) / h3sq;
      H1[1] = (r.R.m[4] * hi3 - hi2 * r.R.m[7]) / h3sq;
      H1[2] = (r.q.y * hi3 - hi2 * r.q.z) / h3sq;
      float z0 = (float)(hi1 / hi3), z1 = (float)(hi2 / hi3);
      double rd0 = (double)__fsub_rn(bv.uvn[2 * i], z0), rd1 = (double)__fsub_rn(bv.uvn[2 * i + 1], z1);
      c[0] = H0[0] * H0[0] + H1[0] * H1[0];
      c[1] = H0[0] * H0[1] + H1[0] * H1[1];
      c[2] = H0[0] * H0[2] + H1[0] * H1[2];
      c[3] = H0[1] * H0[1] + H1[1] * H1[1];
      c[4] = H0[1] * H0[2] + H1[1] * H1[2];
      c[5] = H0[2] * H0[2] + H1[2] * H1[2];
#pragma unroll
      for (int a = 0; a < 3; a++)
        c[6 + a] = H0[a] * rd0 + H1[a] * rd1;
    }
    seq_add<9>(acc, c, min(32, m1 - base), wbuf);
  }
  return acc;
}

// doubles of one warp's dynamic shared memory: the seq_add staging rows, then the relative-pose cache (pitch = the
// launch's longest track)
__host__ __device__ __forceinline__ int tri_warp_doubles(int pitch) { return TRI_NSUM * TRI_PITCH + TRI_REL * pitch; }

__global__ void __launch_bounds__(256) k_triangulate(const DevCamPoses *__restrict__ fr, const DevOpts *__restrict__ dop,
                                                     DevFeat *__restrict__ feats, int n_feats, BlobView bv, int pitch) {
  OVB_PDL_ENTER();
  extern __shared__ double tri_smem[];
  double *wbuf = tri_smem + (size_t)(threadIdx.x >> 5) * tri_warp_doubles(pitch);
  double *rc = wbuf + TRI_NSUM * TRI_PITCH;
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (warp >= n_feats)
    return;
  DevFeat *F = &feats[warp];
  const ovb_opts &op = dop->o;
  int m0 = F->m0, m1 = F->m1;
  const double qnan = __longlong_as_double(0x7ff8000000000000LL);
  int status = OVB_FEAT_OK;
  dv3 pA = mk3(qnan, qnan, qnan), pG = pA;
  int anchor_cam = -1, anchor_clone = -1;
  if (m1 - m0 < 2) {
    status = OVB_FEAT_FEW_MEAS; // update/UpdaterMSCKF.cpp:88
  } else {
    // ---- anchor: first visited camera with the strictly largest count, its last measurement (:35-46)
    int most = 0;
    anchor_cam = 0;
    for (int k = F->key0; k < F->key1; k++) {
      int key = bv.keys[k];
      int cnt = 0;
      for (int i = m0 + lane; i < m1; i += 32)
        cnt += (bv.cam[i] == key) ? 1 : 0;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1)
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
      if (cnt > most) {
        anchor_cam = key;
        most = cnt;
      }
    }
    int ameas = -1;
    for (int i = m0 + lane; i < m1; i += 32)
      if (bv.cam[i] == anchor_cam)
        ameas = i;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
      ameas = max(ameas, __shfl_xor_sync(0xffffffffu, ameas, o));
    anchor_clone = bv.clone[ameas];
    dm3 R_GtoA = ld_m3(fr->cc_R[anchor_cam][anchor_clone]);
    dv3 p_AinG = ld_v3(fr->cc_p[anchor_cam][anchor_clone]);
    for (int i = m0 + lane; i < m1; i += 32)
      st_rel(rc, pitch, i - m0, rel_pose(fr, bv.cam[i], bv.clone[i], R_GtoA, p_AinG));
    dv3 p_f;
    if (!op.triangulate_1d) {
      // ---- A = sum Bperp'Bperp, b = sum Ai p_CiinA (:58-85)
      double acc = 0.0;
      for (int base = m0; base < m1; base += 32) {
        const int i = base + lane;
        double c[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        if (i < m1) {
          Rel r = ld_rel(rc, pitch, i - m0);
          dv3 bi = mTv3(r.R, mk3((double)bv.uvn[2 * i], (double)bv.uvn[2 * i + 1], 1.0));
          double nb = norm3(bi);
          bi = mk3(bi.x / nb, bi.y / nb, bi.z / nb);
          dm3 Bp = skew3(bi);
          dm3 Ai = mulT33(Bp, Bp);
          dv3 Aip = mv3(Ai, r.t);
          c[0] = Ai.m[0], c[1] = Ai.m[1], c[2] = Ai.m[2], c[3] = Ai.m[4], c[4] = Ai.m[5], c[5] = Ai.m[8];
          c[6] = Aip.x, c[7] = Aip.y, c[8] = Aip.z;
        }
        seq_add<9>(acc, c, min(32, m1 - base), wbuf);
      }
      double Ab[9]; // A00 A01 A02 A11 A12 A22 | b0 b1 b2
      seq_sums(Ab, acc);
      // the mirrored entries of A follow the same operation sequence as their twins
      double A[9] = {Ab[0], Ab[1], Ab[2], Ab[1], Ab[3], Ab[4], Ab[2], Ab[4], Ab[5]};
      double b[3] = {Ab[6], Ab[7], Ab[8]};
      p_f = colpiv_solve3(A, mk3(b[0], b[1], b[2]));
      double condA = cond_sym3(A);
      if (fabs(condA) > op.max_cond_number)
        status = OVB_FEAT_TRI_COND;
      else if (p_f.z < op.min_dist || p_f.z > op.max_dist)
        status = OVB_FEAT_TRI_DEPTH;
      else if (isnan(norm3(p_f)))
        status = OVB_FEAT_TRI_NAN;
    } else {
      // ---- 1d depth along the anchor bearing (:114-195)
      dv3 ba = mk3((double)bv.uvn[2 * ameas], (double)bv.uvn[2 * ameas + 1], 1.0);
      double nba = norm3(ba);
      ba = mk3(ba.x / nba, ba.y / nba, ba.z / nba);
      double acc = 0.0;
      for (int base = m0; base < m1; base += 32) {
        const int i = base + lane;
        double c[2] = {0.0, 0.0};
        if (i < m1 && i != ameas) { // the anchor observation is skipped (:150-151): adding 0.0 leaves the sums unchanged
          Rel r = ld_rel(rc, pitch, i - m0);
          dv3 bi = mTv3(r.R, mk3((double)bv.uvn[2 * i], (double)bv.uvn[2 * i + 1], 1.0));
          double nb = norm3(bi);
          bi = mk3(bi.x / nb, bi.y / nb, bi.z / nb);
          dm3 Bp = skew3(bi);
          dv3 Bb = mv3(Bp, ba);
          c[0] = dot3(Bb, Bb);
          c[1] = dot3(Bb, mv3(Bp, r.t));
        }
        seq_add<2>(acc, c, min(32, m1 - base), wbuf);
      }
      double Ab1[2];
      seq_sums(Ab1, acc);
      const double A1 = Ab1[0], b1 = Ab1[1];
      double depth = b1 / A1;
      p_f = mk3(depth * ba.x, depth * ba.y, depth * ba.z);
      if (p_f.z < op.min_dist || p_f.z > op.max_dist)
        status = OVB_FEAT_TRI_DEPTH;
      else if (isnan(norm3(p_f)))
        status = OVB_FEAT_TRI_NAN;
    }
    if (status == OVB_FEAT_OK) {
      pA = p_f;
      pG = add3(mTv3(R_GtoA, pA), p_AinG); // :109-110
    }
    // ---- Levenberg–Marquardt on (alpha, beta, rho) (:197-335)
    if (status == OVB_FEAT_OK && op.refine_features) {
      // The loop's warp-uniform values that are read only now and then are kept one component per lane (lane k: component k)
      // and shuffled back where they are read: the anchor pose (after the loop), Hess|grad (at each solve) and the trial
      // steps. This holds the kernel at 128 registers.
      double anc = 0.0;
#pragma unroll
      for (int k = 0; k < 9; k++)
        anc = (lane == k) ? R_GtoA.m[k] : anc;
      anc = (lane == 9) ? p_AinG.x : ((lane == 10) ? p_AinG.y : ((lane == 11) ? p_AinG.z : anc));
      double rho = 1 / pA.z;
      double alpha = pA.x / pA.z;
      double beta = pA.y / pA.z;
      double lam = op.init_lamda;
      double eps = 10000;
      int runs = 0;
      bool recompute = true;
      double hg = 0.0; // Hess 00 01 02 11 12 22 | grad 0 1 2, one component per lane
      double cost_old;
      {
        const dv3 x0[1] = {mk3(alpha, beta, rho)};
        cost_old = __shfl_sync(0xffffffffu, lm_cost<1>(rc, pitch, bv, m0, m1, lane, x0, wbuf), 0);
      }
      while (runs < op.max_runs && lam < op.max_lamda && eps > op.min_dx) {
        if (recompute)
          hg = lm_hess(rc, pitch, bv, m0, m1, lane, alpha, beta, rho, wbuf);
        // Until a trial is accepted, Hess, grad, the point and cost_old stay fixed and only lam grows, by lam_mult per
        // rejection; the slowest features spend most of their time in such runs of rejected trials. So the next
        // TRI_LM_BATCH trials are solved side by side (lane k with lam multiplied k times, as k rejections would leave
        // it), their costs are taken in one measurement pass, and the loop's decisions are replayed on them in order.
        double lam_k = lam;
        for (int k = 0; k < lane && k < TRI_LM_BATCH - 1; k++)
          lam_k = lam_k * op.lam_mult;
        double Hg[9];
        seq_sums(Hg, hg);
        double Hl[9] = {Hg[0] * (1.0 + lam_k), Hg[1], Hg[2], Hg[1], Hg[3] * (1.0 + lam_k), Hg[4], Hg[2], Hg[4], Hg[5] * (1.0 + lam_k)};
        const dv3 dxl = colpiv_solve3(Hl, mk3(Hg[6], Hg[7], Hg[8]));
        dv3 xt[TRI_LM_BATCH];
#pragma unroll
        for (int k = 0; k < TRI_LM_BATCH; k++)
          xt[k] = mk3(alpha + __shfl_sync(0xffffffffu, dxl.x, k), beta + __shfl_sync(0xffffffffu, dxl.y, k), rho + __shfl_sync(0xffffffffu, dxl.z, k));
        double cost[TRI_LM_BATCH];
        seq_sums(cost, lm_cost<TRI_LM_BATCH>(rc, pitch, bv, m0, m1, lane, xt, wbuf));
        bool done = false, converged = false;
#pragma unroll
        for (int k = 0; k < TRI_LM_BATCH; k++) {
          const dv3 dxk = mk3(__shfl_sync(0xffffffffu, dxl.x, k), __shfl_sync(0xffffffffu, dxl.y, k), __shfl_sync(0xffffffffu, dxl.z, k));
          if (done)
            continue;
          if (k > 0 && !(runs < op.max_runs && lam < op.max_lamda && eps > op.min_dx)) { // the loop ends before trial k
            done = true;
            continue;
          }
          if (cost[k] <= cost_old && (cost_old - cost[k]) / cost_old < op.min_dcost) {
            alpha += dxk.x;
            beta += dxk.y;
            rho += dxk.z;
            eps = 0;
            done = converged = true;
          } else if (cost[k] <= cost_old) {
            recompute = true;
            cost_old = cost[k];
            alpha += dxk.x;
            beta += dxk.y;
            rho += dxk.z;
            runs++;
            lam = lam / op.lam_mult;
            eps = norm3(dxk);
            done = true;
          } else {
            recompute = false;
            lam = lam * op.lam_mult;
          }
        }
        if (converged)
          break;
      }
      pA = mk3(alpha / rho, beta / rho, 1 / rho);
      // ---- baseline check (:338-370)
      dv3 q1, q2;
      householder_tangent3(pA, q1, q2);
      double base_line_max = 0.0;
      for (int i = m0 + lane; i < m1; i += 32) {
        const double *t_i = rc + 9 * pitch + (i - m0);
        dv3 t = mk3(t_i[0], t_i[pitch], t_i[2 * pitch]);
        double a0 = dot3(q1, t), a1 = dot3(q2, t);
        double bl = sqrt(a0 * a0 + a1 * a1);
        if (bl > base_line_max)
          base_line_max = bl;
      }
      base_line_max = warp_max(base_line_max);
      if (pA.z < op.min_dist || pA.z > op.max_dist)
        status = OVB_FEAT_GN_DEPTH;
      else if ((norm3(pA) / base_line_max) > op.max_baseline)
        status = OVB_FEAT_GN_BASELINE;
      else if (isnan(norm3(pA)))
        status = OVB_FEAT_GN_NAN;
      else {
        dm3 Ra;
#pragma unroll
        for (int k = 0; k < 9; k++)
          Ra.m[k] = __shfl_sync(0xffffffffu, anc, k);
        const dv3 pa = mk3(__shfl_sync(0xffffffffu, anc, 9), __shfl_sync(0xffffffffu, anc, 10), __shfl_sync(0xffffffffu, anc, 11));
        pG = add3(mTv3(Ra, pA), pa); // :373
      }
    }
  }
  if (lane == 0) {
    F->status = status;
    F->anchor_cam = anchor_cam;
    F->anchor_clone = anchor_clone;
    F->p_FinA[0] = pA.x;
    F->p_FinA[1] = pA.y;
    F->p_FinA[2] = pA.z;
    F->p_FinG[0] = pG.x;
    F->p_FinG[1] = pG.y;
    F->p_FinG[2] = pG.z;
    F->chi2 = qnan;
  }
}

static const size_t TRI_SMEM_LIMIT = 227 * 1024; // dynamic shared memory of one H100 CTA

void launch_triangulate(ovb_ctx *ctx, int n_feats, BlobView bv) {
  if (n_feats <= 0)
    return;
  if (!ctx->attr_done[8]) { // function attributes are per device: one flag per context
    cudaFuncSetAttribute(k_triangulate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TRI_SMEM_LIMIT);
    ctx->attr_done[8] = 1;
  }
  // the relative-pose cache holds the launch's longest track: the first of pack_inputs' longest-first schedule
  const DevFeat &longest = ctx->h_feat[ctx->h_feat[0].sched];
  const int pitch = longest.m1 - longest.m0;
  const size_t warp_bytes = sizeof(double) * (size_t)tri_warp_doubles(pitch);
  // one warp per feature; spread the warps over all SMs (each warp is one long dependent FP64 chain), as many per CTA as
  // their caches fit (at least 4 at OVB_MAX_MEAS_PER_FEAT)
  int warps_per_cta = (n_feats + ctx->sm_count - 1) / ctx->sm_count;
  warps_per_cta = warps_per_cta < 1 ? 1 : (warps_per_cta > TRI_MAX_WARPS ? TRI_MAX_WARPS : warps_per_cta);
  const int fit = (int)(TRI_SMEM_LIMIT / warp_bytes);
  warps_per_cta = warps_per_cta < fit ? warps_per_cta : fit;
  int grid = (n_feats + warps_per_cta - 1) / warps_per_cta;
  ovb_launch(ctx, k_triangulate, dim3(grid), dim3(warps_per_cta * 32), warp_bytes * warps_per_cta, ctx->d_cc, ctx->d_opts, ctx->d_feat, n_feats,
             bv, pitch);
}
