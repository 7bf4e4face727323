// anchor_change.cu — the math of UpdaterSLAM::perform_anchor_change (ov_msckf/src/update/UpdaterSLAM.cpp:506-647), compiled
// once for the host and the device. The host entry ovb_slam_anchor_change hands Phi + the variable order to
// ovb_cov_propagate (StateHelper::EKFPropagation on the resident P); k_anchor_phi runs the same source for every landmark of
// an ovb_marginalize_window call. This unit is compiled with -fmad=false: every product and sum is rounded on its own on the
// device, as the host (x86-64 without FMA contraction) computes it, so the rational representations give the same bits on
// both sides. acos / atan2 / sin / cos (ANCHORED_FULL_INVERSE_DEPTH only) are the C library's on the host and CUDA's on the
// device, which may round differently in the last ulp: ovb_marginalize_window therefore takes that representation's Phi from
// the host function and runs the kernel for the other three.
// The representation Jacobians follow UpdaterHelper::get_feature_jacobian_representation (UpdaterHelper.cpp:32-190) for
// the anchored representations, including its FEJ rule (the anchor pose is taken at its first estimate, the landmark is
// re-expressed in that FEJ anchor frame from the best global position, :89-96).
#include "ovb_internal.cuh"
#include <cmath>

namespace {

#define OVB_HD __host__ __device__ __forceinline__

// the frame arrays the math reads; the FEJ arrays are never null (the caller substitutes the current estimates)
struct AnchorFrame {
  const double *clone_R, *clone_p, *clone_R_fej, *clone_p_fej, *cam_R, *cam_p;
  const int *clone_off, *cam_ext_off;
};

struct M3 {
  double a[9];
};
OVB_HD M3 mul(const M3 &x, const M3 &y) {
  M3 r;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++)
      r.a[3 * i + j] = x.a[3 * i] * y.a[j] + x.a[3 * i + 1] * y.a[3 + j] + x.a[3 * i + 2] * y.a[6 + j];
  return r;
}
OVB_HD M3 tr(const M3 &x) {
  M3 r;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++)
      r.a[3 * i + j] = x.a[3 * j + i];
  return r;
}
OVB_HD void mv(const M3 &x, const double v[3], double out[3]) {
  for (int i = 0; i < 3; i++)
    out[i] = x.a[3 * i] * v[0] + x.a[3 * i + 1] * v[1] + x.a[3 * i + 2] * v[2];
}
OVB_HD M3 skew(const double w[3]) {
  M3 r = {{0, -w[2], w[1], w[2], 0, -w[0], -w[1], w[0], 0}};
  return r;
}
OVB_HD M3 load(const double *p) {
  M3 r;
  for (int i = 0; i < 9; i++)
    r.a[i] = p[i];
  return r;
}

// d p_FinG / d(landmark parameters) [3 x nf], d p_FinG / d(anchor clone) [3 x 6], d p_FinG / d(anchor extrinsics) [3 x 6]
OVB_HD void rep_jacobian(const AnchorFrame &fr, bool do_fej, int rep, const double p_FinA_in[3], int acam, int aclone, double Hf[9], int *nf,
                         double Hanc[18], double Hcal[18]) {
  const M3 R_ItoC = load(fr.cam_R + 9 * acam);
  const double *p_IinC = fr.cam_p + 3 * acam;
  M3 R_GtoI = load(fr.clone_R + 9 * aclone);
  double p_IinG[3] = {fr.clone_p[3 * aclone], fr.clone_p[3 * aclone + 1], fr.clone_p[3 * aclone + 2]};
  double p_FinA[3] = {p_FinA_in[0], p_FinA_in[1], p_FinA_in[2]};
  if (do_fej) {
    // best global position with the current estimates, then back into the FEJ anchor frame (:89-96)
    const M3 RtRt = mul(tr(R_GtoI), tr(R_ItoC));
    double d[3] = {p_FinA[0] - p_IinC[0], p_FinA[1] - p_IinC[1], p_FinA[2] - p_IinC[2]}, best[3];
    mv(RtRt, d, best);
    for (int i = 0; i < 3; i++)
      best[i] += p_IinG[i];
    R_GtoI = load(fr.clone_R_fej + 9 * aclone);
    const double *pf = fr.clone_p_fej + 3 * aclone;
    for (int i = 0; i < 3; i++)
      p_IinG[i] = pf[i];
    const M3 RR = tr(mul(tr(R_GtoI), tr(R_ItoC)));
    double e[3] = {best[0] - p_IinG[0], best[1] - p_IinG[1], best[2] - p_IinG[2]};
    mv(RR, e, p_FinA);
    for (int i = 0; i < 3; i++)
      p_FinA[i] += p_IinC[i];
  }
  const M3 R_CtoG = mul(tr(R_GtoI), tr(R_ItoC));
  // H_anc = [-R_GtoI' skew(R_ItoC' (p_FinA - p_IinC)), I] (:100-102)
  {
    double d[3] = {p_FinA[0] - p_IinC[0], p_FinA[1] - p_IinC[1], p_FinA[2] - p_IinC[2]}, v[3];
    mv(tr(R_ItoC), d, v);
    M3 nR = tr(R_GtoI);
    for (double &x : nR.a)
      x = -x;
    const M3 blk = mul(nR, skew(v));
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) {
        Hanc[6 * r + c] = blk.a[3 * r + c];
        Hanc[6 * r + 3 + c] = (r == c) ? 1.0 : 0.0;
      }
  }
  // H_calib = [-R_CtoG skew(p_FinA - p_IinC), -R_CtoG] (:109-115)
  {
    double d[3] = {p_FinA[0] - p_IinC[0], p_FinA[1] - p_IinC[1], p_FinA[2] - p_IinC[2]};
    M3 nR = R_CtoG;
    for (double &x : nR.a)
      x = -x;
    const M3 blk = mul(nR, skew(d));
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) {
        Hcal[6 * r + c] = blk.a[3 * r + c];
        Hcal[6 * r + 3 + c] = -R_CtoG.a[3 * r + c];
      }
  }
  *nf = 3;
  if (rep == OVB_REP_ANCHORED_3D) { // :118-121
    for (int i = 0; i < 9; i++)
      Hf[i] = R_CtoG.a[i];
    return;
  }
  M3 d = {{0, 0, 0, 0, 0, 0, 0, 0, 0}};
  if (rep == OVB_REP_ANCHORED_FULL_INVERSE_DEPTH) { // :124-150
    const double rho = 1 / sqrt(p_FinA[0] * p_FinA[0] + p_FinA[1] * p_FinA[1] + p_FinA[2] * p_FinA[2]);
    const double phi = acos(rho * p_FinA[2]);
    const double theta = atan2(p_FinA[1], p_FinA[0]);
    const double sin_th = sin(theta), cos_th = cos(theta), sin_phi = sin(phi), cos_phi = cos(phi);
    d.a[0] = -(1.0 / rho) * sin_th * sin_phi;
    d.a[1] = (1.0 / rho) * cos_th * cos_phi;
    d.a[2] = -(1.0 / (rho * rho)) * cos_th * sin_phi;
    d.a[3] = (1.0 / rho) * cos_th * sin_phi;
    d.a[4] = (1.0 / rho) * sin_th * cos_phi;
    d.a[5] = -(1.0 / (rho * rho)) * sin_th * sin_phi;
    d.a[6] = 0.0;
    d.a[7] = -(1.0 / rho) * sin_phi;
    d.a[8] = -(1.0 / (rho * rho)) * cos_phi;
  } else if (rep == OVB_REP_ANCHORED_MSCKF_INVERSE_DEPTH) { // :153-172
    const double alpha = p_FinA[0] / p_FinA[2], beta = p_FinA[1] / p_FinA[2], rho = 1 / p_FinA[2];
    d.a[0] = (1.0 / rho);
    d.a[2] = -(1.0 / (rho * rho)) * alpha;
    d.a[4] = (1.0 / rho);
    d.a[5] = -(1.0 / (rho * rho)) * beta;
    d.a[8] = -(1.0 / (rho * rho));
  } else { // ANCHORED_INVERSE_DEPTH_SINGLE (:175-186): only the depth is a parameter
    const double rho = 1.0 / p_FinA[2];
    const double v[3] = {-(1.0 / (rho * rho)) * (rho * p_FinA[0]), -(1.0 / (rho * rho)) * (rho * p_FinA[1]), -(1.0 / (rho * rho)) * (rho * p_FinA[2])};
    double out[3];
    mv(R_CtoG, v, out);
    Hf[0] = out[0];
    Hf[1] = out[1];
    Hf[2] = out[2];
    *nf = 1;
    return;
  }
  const M3 L = mul(R_CtoG, d);
  for (int i = 0; i < 9; i++)
    Hf[i] = L.a[i];
}

// inverse of a 3x3 by Gauss-Jordan with partial pivoting (the reference solves H_f_new X = I with ColPivHouseholderQR)
OVB_HD bool inv3(const double A_in[9], double Inv[9]) {
  double A[9];
  for (int i = 0; i < 9; i++)
    A[i] = A_in[i];
  for (int i = 0; i < 9; i++)
    Inv[i] = (i % 4 == 0) ? 1.0 : 0.0;
  for (int c = 0; c < 3; c++) {
    int piv = c;
    for (int i = c + 1; i < 3; i++)
      if (fabs(A[3 * i + c]) > fabs(A[3 * piv + c]))
        piv = i;
    if (!(fabs(A[3 * piv + c]) > 0.0))
      return false;
    if (piv != c)
      for (int j = 0; j < 3; j++) {
        double t = A[3 * c + j];
        A[3 * c + j] = A[3 * piv + j];
        A[3 * piv + j] = t;
        t = Inv[3 * c + j];
        Inv[3 * c + j] = Inv[3 * piv + j];
        Inv[3 * piv + j] = t;
      }
    const double d = A[3 * c + c];
    for (int j = 0; j < 3; j++) {
      A[3 * c + j] /= d;
      Inv[3 * c + j] /= d;
    }
    for (int i = 0; i < 3; i++) {
      if (i == c)
        continue;
      const double f = A[3 * i + c];
      for (int j = 0; j < 3; j++) {
        A[3 * i + j] -= f * A[3 * c + j];
        Inv[3 * i + j] -= f * Inv[3 * c + j];
      }
    }
  }
  return true;
}

OVB_HD void camera_pose(const AnchorFrame &fr, int cam, int cl, bool fej, M3 *R_GtoC, double p_CinG[3]) {
  const M3 R_GtoI = load((fej ? fr.clone_R_fej : fr.clone_R) + 9 * cl);
  const double *p_IinG = (fej ? fr.clone_p_fej : fr.clone_p) + 3 * cl;
  *R_GtoC = mul(load(fr.cam_R + 9 * cam), R_GtoI);
  double t[3];
  mv(tr(*R_GtoC), fr.cam_p + 3 * cam, t);
  for (int i = 0; i < 3; i++)
    p_CinG[i] = p_IinG[i] - t[i];
}

OVB_HD void transfer(const AnchorFrame &fr, int old_cam, int old_clone, int new_cam, int new_clone, bool fej, const double p_old[3], double p_new[3]) {
  M3 R_GtoOLD, R_GtoNEW;
  double p_OLDinG[3], p_NEWinG[3];
  camera_pose(fr, old_cam, old_clone, fej, &R_GtoOLD, p_OLDinG);
  camera_pose(fr, new_cam, new_clone, fej, &R_GtoNEW, p_NEWinG);
  const M3 R_OLDtoNEW = mul(R_GtoNEW, tr(R_GtoOLD));
  const double d[3] = {p_OLDinG[0] - p_NEWinG[0], p_OLDinG[1] - p_NEWinG[1], p_OLDinG[2] - p_NEWinG[2]};
  double p_OLDinNEW[3], r[3];
  mv(R_GtoNEW, d, p_OLDinNEW);
  mv(R_OLDtoNEW, p_old, r);
  for (int i = 0; i < 3; i++)
    p_new[i] = r[i] + p_OLDinNEW[i];
}

// the whole re-anchoring of one landmark (arguments validated by the caller); false when H_f_new is singular
OVB_HD bool anchor_change(const AnchorFrame &fr, bool do_fej, bool ext, int rep, int lm_off, const double *value, const double *value_fej, int old_cam,
                          int old_clone, int new_cam, int new_clone, double *new_value, double *new_value_fej, double *Phi, int32_t *order_off,
                          int32_t *order_sz, int32_t *n_order, int32_t *n_cols) {
  double Hf_old[9], Hf_new[9], Hanc_old[18], Hcal_old[18], Hanc_new[18], Hcal_new[18];
  int nf_old = 3, nf_new = 3;
  rep_jacobian(fr, do_fej, rep, value, old_cam, old_clone, Hf_old, &nf_old, Hanc_old, Hcal_old);
  transfer(fr, old_cam, old_clone, new_cam, new_clone, false, value, new_value);
  transfer(fr, old_cam, old_clone, new_cam, new_clone, true, value_fej, new_value_fej);
  rep_jacobian(fr, do_fej, rep, new_value, new_cam, new_clone, Hf_new, &nf_new, Hanc_new, Hcal_new);
  // phi_order_OLD = unique(x_order_old ++ x_order_new) ++ landmark (:600-617)
  int n = 0, cur = 0;
  auto place = [&](int off) {
    int c = 0;
    for (int i = 0; i < n; i++) {
      if (order_off[i] == off)
        return c;
      c += order_sz[i];
    }
    order_off[n] = off;
    order_sz[n] = 6;
    n++;
    cur += 6;
    return cur - 6;
  };
  const int c_old_anc = place(fr.clone_off[old_clone]);
  const int c_old_cal = ext ? place(fr.cam_ext_off[old_cam]) : -1;
  const int c_new_anc = place(fr.clone_off[new_clone]);
  const int c_new_cal = ext ? place(fr.cam_ext_off[new_cam]) : -1;
  const int phisize = nf_new; // 3, or 1 for the single-depth representation
  const int c_lm = cur;
  order_off[n] = lm_off;
  order_sz[n] = phisize;
  n++;
  cur += phisize;
  *n_order = n;
  *n_cols = cur;
  // H_f_new^-1: phisize x 3 (:624-629)
  double Inv[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  if (phisize == 1) {
    const double n2 = Hf_new[0] * Hf_new[0] + Hf_new[1] * Hf_new[1] + Hf_new[2] * Hf_new[2];
    for (int i = 0; i < 3; i++)
      Inv[i] = 1.0 / n2 * Hf_new[i];
  } else if (!inv3(Hf_new, Inv)) {
    return false;
  }
  for (int i = 0; i < phisize * cur; i++)
    Phi[i] = 0.0;
  auto add6 = [&](int col, const double *B, double sign) { // Phi[:, col:col+6] += sign * Inv * B (B is 3 x 6)
    for (int i = 0; i < phisize; i++)
      for (int j = 0; j < 6; j++) {
        double acc = 0.0;
        for (int k = 0; k < 3; k++)
          acc += Inv[3 * i + k] * B[6 * k + j];
        Phi[(size_t)i * cur + col + j] += sign * acc;
      }
  };
  add6(c_old_anc, Hanc_old, 1.0);
  if (ext)
    add6(c_old_cal, Hcal_old, 1.0);
  for (int i = 0; i < phisize; i++)
    for (int j = 0; j < phisize; j++) {
      double acc = 0.0;
      for (int k = 0; k < 3; k++)
        acc += Inv[3 * i + k] * Hf_old[nf_old * k + j];
      Phi[(size_t)i * cur + c_lm + j] = acc;
    }
  add6(c_new_anc, Hanc_new, -1.0);
  if (ext)
    add6(c_new_cal, Hcal_new, -1.0);
  return true;
}

// ovb_marginalize_window: one thread per re-anchored landmark writes its new values into the result block, its Phi
// (p x q, row-major) into phi + OVB_WIN_PHI * l and the covariance index of each of Phi's q columns into idx + OVB_WIN_Q * l.
// Landmarks marked `host` (ANCHORED_FULL_INVERSE_DEPTH) arrive computed by the host. A singular H_f_new sets flags[1]; the
// kernels after this one then return without reading Phi, the indices or P.
__global__ void k_anchor_phi(const DevWinFrame *__restrict__ wf, const DevWinLM *__restrict__ lms, int n, int do_fej, int ext, int *flags,
                             double *__restrict__ new_values, double *__restrict__ phi, int *__restrict__ idx, int *__restrict__ q_out) {
  OVB_PDL_ENTER();
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= n)
    return;
  const DevWinLM &lm = lms[l];
  if (lm.host)
    return;
  const AnchorFrame fr = {&wf->clone_R[0][0], &wf->clone_p[0][0], &wf->clone_R_fej[0][0], &wf->clone_p_fej[0][0],
                          &wf->cam_R[0][0],   &wf->cam_p[0][0],   wf->clone_off,          wf->cam_ext_off};
  int32_t order_off[5], order_sz[5], n_order, n_cols;
  double *nv = new_values + 6 * l;
  if (!anchor_change(fr, do_fej != 0, ext != 0, lm.rep, lm.lm_off, lm.value, lm.value_fej, lm.old_cam, lm.old_clone, lm.new_cam, lm.new_clone, nv,
                     nv + 3, phi + (size_t)OVB_WIN_PHI * l, order_off, order_sz, &n_order, &n_cols)) {
    q_out[l] = 0; // no column of this landmark is read: the kernels after this one return on flags[1]
    atomicOr(&flags[1], 1);
    return;
  }
  int *ix = idx + OVB_WIN_Q * l;
  for (int i = 0, c = 0; i < n_order; i++)
    for (int k = 0; k < order_sz[i]; k++)
      ix[c++] = order_off[i] + k;
  q_out[l] = n_cols;
}

} // namespace

void launch_anchor_phi(ovb_ctx *ctx, const DevWinFrame *wf, const DevWinLM *lms, int n, int do_fej, int ext, int *flags, double *new_values,
                       double *phi, int *idx, int *q) {
  ovb_launch(ctx, k_anchor_phi, dim3((n + 63) / 64), dim3(64), (size_t)0, wf, lms, n, do_fej, ext, flags, new_values, phi, idx, q);
}

extern "C" ovb_status ovb_slam_anchor_change(const ovb_frame *fr, const ovb_opts *op, int lm_off, const double *value, const double *value_fej,
                                             int old_cam, int old_clone, int new_cam, int new_clone, double *new_value, double *new_value_fej,
                                             double *Phi, int32_t *order_off, int32_t *order_sz, int32_t *n_order, int32_t *n_cols) {
  if (!fr || !op || !value || !value_fej || !new_value || !new_value_fej || !Phi || !order_off || !order_sz || !n_order || !n_cols)
    return OVB_ERR_ARG;
  const int rep = op->feat_rep;
  if (rep < OVB_REP_ANCHORED_3D || rep > OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE) // global representations have no anchor (:493-496)
    return OVB_ERR_ARG;
  if (old_cam < 0 || old_cam >= fr->n_cams || new_cam < 0 || new_cam >= fr->n_cams || old_clone < 0 || old_clone >= fr->n_clones || new_clone < 0 ||
      new_clone >= fr->n_clones)
    return OVB_ERR_ARG;
  const bool ext = op->do_calib_camera_pose != 0;
  if (ext && (!fr->cam_ext_off || fr->cam_ext_off[old_cam] < 0 || fr->cam_ext_off[new_cam] < 0))
    return OVB_ERR_ARG;
  const AnchorFrame af = {fr->clone_R, fr->clone_p, fr->clone_R_fej ? fr->clone_R_fej : fr->clone_R, fr->clone_p_fej ? fr->clone_p_fej : fr->clone_p,
                          fr->cam_R,   fr->cam_p,   fr->clone_off,                                    fr->cam_ext_off};
  if (!anchor_change(af, op->do_fej != 0, ext, rep, lm_off, value, value_fej, old_cam, old_clone, new_cam, new_clone, new_value, new_value_fej, Phi,
                     order_off, order_sz, n_order, n_cols))
    return OVB_ERR_ARG;
  return OVB_OK;
}
