// tests/cpp/ovo_slam_reps.cpp — TEST INFRASTRUCTURE: the CPU oracle's SLAM pieces for per-landmark representations, built on
// the oracle's own routines (oracle/ovo_core.hpp) into a separate library by tests/oracle_reps.py, with oracle/Makefile's flags.
//  ovo_slam_update_reps          UpdaterSLAM::update steps 4-5 with one representation per landmark
//  ovo_slam_single_init_system   the ANCHORED_INVERSE_DEPTH_SINGLE branch of UpdaterSLAM::delayed_init
#include "../../oracle/ovo_core.hpp"

namespace ovo {

// oracle/ovo_core.hpp's slam_update (steps 4-5 of UpdaterSLAM::update, update/UpdaterSLAM.cpp:310-470) with every landmark in
// its own representation, as the reference reads landmark->_feat_representation per landmark (:327-329): width, remap,
// bearing projection and required measurements follow each landmark. feat_rep NULL = op.feat_rep for all.
inline int slam_update_reps(const ovb_frame &fr, const ovb_feat_batch &fb, const ovb_landmarks &lm, const ovb_opts &op, const double *chi2_table,
                            double *P, int N, ovb_feat_out *out, double *dx, ovb_stats *stats, UpdateDump *dump, const int32_t *feat_rep) {
  const int F = fb.n_feats;
  std::vector<int> status(F, OVB_FEAT_OK);
  std::vector<double> chi2s(F, std::nan(""));
  size_t max_meas_size = 0;
  for (int f = 0; f < F; f++)
    max_meas_size += 2 * (size_t)(fb.meas_off[f + 1] - fb.meas_off[f]);
  std::vector<double> res_big(max_meas_size, 0.0), R_big(max_meas_size, 1.0);
  Mat Hx_big((int)max_meas_size, N);
  std::vector<Var> Hx_order_big;
  int ct_jacob = 0, ct_meas = 0, used = 0;
  double T0 = now_s();
  for (int f = 0; f < F; f++) {
    int rep = feat_rep ? feat_rep[f] : op.feat_rep;
    const bool single = (rep == OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE);
    if (single)
      rep = OVB_REP_ANCHORED_MSCKF_INVERSE_DEPTH; // :327-329
    const int lm_size = single ? 1 : 3;
    if (fb.meas_off[f + 1] - fb.meas_off[f] < (single ? 2 : 1)) { // :278-290 (too few measurements: dropped before the update)
      status[f] = OVB_FEAT_FEW_MEAS;
      continue;
    }
    // :333-341 — the landmark's value and FEJ value in the frame its representation lives in
    V3 val = v3(lm.value[3 * f], lm.value[3 * f + 1], lm.value[3 * f + 2]);
    V3 val_fej = v3(lm.value_fej[3 * f], lm.value_fej[3 * f + 1], lm.value_fej[3 * f + 2]);
    V3 p_FinG = val, p_FinG_fej = val_fej, p_FinA = val;
    int acam = -1, aclone = -1;
    if (is_relative(rep)) {
      acam = lm.anchor_cam[f];
      aclone = lm.anchor_clone[f];
    }
    FeatJac J;
    feature_jacobian_full(fr, fb, op, f, rep, p_FinG, p_FinG_fej, p_FinA, acam, aclone, J);
    // :354-361 — H_xf = [H_x, H_f], order += landmark
    FeatJac Jxf;
    Jxf.rows = J.rows;
    Jxf.order = J.order;
    Jxf.order.push_back(Var{lm.lm_off[f], lm_size});
    Jxf.res = J.res;
    Jxf.Hx.resize_zero(J.rows, J.Hx.c + lm_size);
    for (int i = 0; i < J.rows; i++) {
      for (int k = 0; k < J.Hx.c; k++)
        Jxf.Hx(i, k) = J.Hx(i, k);
      for (int k = 0; k < lm_size; k++)
        Jxf.Hx(i, J.Hx.c + k) = J.Hf(i, single ? 2 : k);
    }
    if (single) { // :344-353 — project the bearing portion (the first two columns of H_f) out of [H_x, dz/drho] and res
      Jxf.nf = 2;
      Jxf.Hf.resize_zero(J.rows, 2);
      for (int i = 0; i < J.rows; i++)
        for (int k = 0; k < 2; k++)
          Jxf.Hf(i, k) = J.Hf(i, k);
      nullspace_project_inplace(Jxf);
    }
    // :389-420 — chi² gate with the per-class noise and multiplier
    const double sigma_pix = lm.sigma_pix ? lm.sigma_pix[f] : op.sigma_pix;
    const double sigma_pix_sq = std::pow(sigma_pix, 2);
    const double mult = lm.chi2_multipler ? lm.chi2_multipler[f] : op.chi2_multipler;
    bool spd = true;
    double chi2 = feature_chi2(P, N, Jxf, sigma_pix_sq, &spd);
    chi2s[f] = chi2;
    double chi2_check = chi2_table[std::min(Jxf.rows, OVB_CHI2_TABLE_LEN - 1)];
    if (!(chi2 <= mult * chi2_check)) {
      status[f] = OVB_FEAT_CHI2;
      continue;
    }
    // :424-447 — append with the first-seen column map
    int ct_hx = 0;
    for (const Var &var : Jxf.order) {
      int col = find_var(Hx_order_big, var.off);
      if (col < 0) {
        col = ct_jacob;
        Hx_order_big.push_back(var);
        ct_jacob += var.size;
      }
      for (int k = 0; k < var.size; k++)
        for (int i = 0; i < Jxf.rows; i++)
          Hx_big(ct_meas + i, col + k) = Jxf.Hx(i, ct_hx + k);
      ct_hx += var.size;
    }
    for (int i = 0; i < Jxf.rows; i++) {
      res_big[ct_meas + i] = Jxf.res[i];
      R_big[ct_meas + i] = sigma_pix_sq;
    }
    ct_meas += Jxf.rows;
    used++;
  }
  double T1 = now_s();
  if (out) {
    for (int f = 0; f < F; f++) {
      if (out->status)
        out->status[f] = status[f];
      if (out->chi2)
        out->chi2[f] = chi2s[f];
    }
  }
  if (stats) {
    stats->n_feats_in = F;
    stats->n_feats_used = used;
    stats->rows_stacked = ct_meas;
    stats->cols_stacked = ct_jacob;
    stats->rows_update = ct_meas;
    stats->neg_diag_index = -1;
    stats->ms_total = 0;
  }
  for (int i = 0; i < N; i++)
    dx[i] = 0.0;
  if (ct_meas < 1)
    return OVB_OK;
  Mat H(ct_meas, ct_jacob);
  for (int k = 0; k < ct_jacob; k++)
    for (int i = 0; i < ct_meas; i++)
      H(i, k) = Hx_big(i, k);
  res_big.resize(ct_meas);
  R_big.resize(ct_meas);
  if (dump) {
    dump->order_big = Hx_order_big;
    dump->H_big = H;
    dump->res_big = res_big;
    dump->H_cmp = H;
    dump->res_cmp = R_big; // the SLAM path never compresses: this slot carries diag(R_big) instead
    dump->t_sys = T1 - T0;
  }
  int neg = -1;
  int st = ekf_update(P, N, Hx_order_big, H, res_big, R_big, dx, &neg);
  if (stats) {
    stats->neg_diag_index = neg;
    stats->ms_total = (float)((now_s() - T0) * 1e3);
  }
  if (dump)
    dump->t_upd = now_s() - T1;
  return st;
}

} // namespace ovo

using namespace ovo;

extern "C" {

// ovo_slam_update of oracle/ovo_capi.cpp with feat_rep: one ovb_feat_rep per landmark, NULL = op->feat_rep for all.
int ovo_slam_update_reps(const ovb_frame *fr, const ovb_feat_batch *fb, const ovb_landmarks *lm, const ovb_opts *op, const double *chi2_table,
                    double *P, int N, ovb_feat_out *out, double *dx, ovb_stats *stats, int32_t *order_off, int32_t *order_sz, int32_t *n_order,
                    double *H_big, double *res_big, double *Rdiag_big, int cap_rows,
                         const int32_t *feat_rep) {
  UpdateDump dump;
  ovb_stats st_local;
  if (!stats)
    stats = &st_local;
  int st = slam_update_reps(*fr, *fb, *lm, *op, chi2_table, P, N, out, dx, stats, &dump, feat_rep);
  if (n_order)
    *n_order = (int)dump.order_big.size();
  for (size_t i = 0; i < dump.order_big.size() && i < OVB_MAX_VARS; i++) {
    if (order_off)
      order_off[i] = dump.order_big[i].off;
    if (order_sz)
      order_sz[i] = dump.order_big[i].size;
  }
  int cols = dump.H_big.c;
  if (H_big)
    for (int i = 0; i < dump.H_big.r && i < cap_rows; i++)
      for (int k = 0; k < cols; k++)
        H_big[(size_t)i * cols + k] = dump.H_big(i, k);
  for (int i = 0; i < (int)dump.res_big.size() && i < cap_rows; i++) {
    if (res_big)
      res_big[i] = dump.res_big[i];
    if (Rdiag_big)
      Rdiag_big[i] = dump.res_cmp[i];
  }
  return st;
}

// The ANCHORED_INVERSE_DEPTH_SINGLE branch of UpdaterSLAM::delayed_init: Hf (rows x 3, the ANCHORED_MSCKF_INVERSE_DEPTH
// Jacobian), Hx (rows x n), res (rows), row-major. H_xf = [Hx | Hf[:,2]]; the bearing columns Hf[:,0:2] are projected out of
// [H_xf | res] by the oracle's nullspace_project_inplace (Givens). Outputs (rows-2 rows): H_R (x n), h_L (x 1), res_out.
int ovo_slam_single_init_system(const double *Hf, const double *Hx, const double *res, int rows, int n, double *H_R, double *h_L, double *res_out) {
  if (rows < 3)
    return OVB_ERR_ARG;
  FeatJac J;
  J.rows = rows;
  J.nf = 2;
  J.Hf.resize_zero(rows, 2);
  J.Hx.resize_zero(rows, n + 1);
  J.res.assign(res, res + rows);
  for (int i = 0; i < rows; i++) {
    J.Hf(i, 0) = Hf[(size_t)i * 3];
    J.Hf(i, 1) = Hf[(size_t)i * 3 + 1];
    for (int j = 0; j < n; j++)
      J.Hx(i, j) = Hx[(size_t)i * n + j];
    J.Hx(i, n) = Hf[(size_t)i * 3 + 2];
  }
  nullspace_project_inplace(J);
  for (int i = 0; i < J.rows; i++) {
    for (int j = 0; j < n; j++)
      H_R[(size_t)i * n + j] = J.Hx(i, j);
    h_L[i] = J.Hx(i, n);
    res_out[i] = J.res[i];
  }
  return OVB_OK;
}

} // extern "C"
