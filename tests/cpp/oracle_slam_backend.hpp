// oracle_slam_backend.hpp — TEST INFRASTRUCTURE: the SLAM calls of ovb200::CovBackend composed from the CPU oracle
// (oracle/libovoracle.so), on top of OracleCov (oracle_backend.hpp). The oracle-backed rpng_sim runner
// (tools/run_simulation.cpp built with -DOVB_SIM_ORACLE) runs on it, so SLAM runs of the engine and of the oracle consume the
// very same inputs. Only tests/ may include this file.
#pragma once
#include "oracle_backend.hpp"

#include <cmath>

extern "C" {
int ovo_slam_update(const ovb_frame *fr, const ovb_feat_batch *fb, const ovb_landmarks *lm, const ovb_opts *op, const double *chi2_table, double *P, int N,
                    ovb_feat_out *out, double *dx, ovb_stats *stats, int32_t *order_off, int32_t *order_sz, int32_t *n_order, double *H_big, double *res_big,
                    double *Rdiag_big, int cap_rows);
int ovo_triangulate(const ovb_frame *fr, const ovb_feat_batch *fb, const ovb_opts *op, ovb_feat_out *out, int32_t *gn_runs, int32_t *gn_solves,
                    double *gn_lambda);
int ovo_feature_jacobians(const ovb_frame *fr, const ovb_feat_batch *fb, const ovb_opts *op, const double *chi2_table, const double *P, int N,
                          ovb_feat_out *out, int stage, double *Hf_out, double *Hx_out, double *res_out, int32_t *row_off_out, int ncols,
                          const int32_t *col_index, int ld_out);
int ovo_cov_initialize(const double *P, int N, const int *off, const int *sz, int nvar, const double *H_R, const double *H_L, const double *res, int r,
                       int k, double sigma2, double chi2_mult, const double *chi2_table, double *Pout, int *accepted, double *dx_new, double *dx);
int ovo_anchor_change(const ovb_frame *fr, const ovb_opts *op, int lm_off, const double *value, const double *value_fej, int old_cam, int old_clone,
                      int new_cam, int new_clone, double *new_value, double *new_value_fej, double *Phi_out, int32_t *order_off, int32_t *order_sz,
                      int32_t *n_order, int32_t *ncols);
void ovo_make_givens(double p, double q, double *cs);
}

namespace ovb200 {
class OracleSlamCov : public OracleCov {
public:
  OracleSlamCov() {
    table_.resize(OVB_CHI2_TABLE_LEN);
    for (int k = 0; k < OVB_CHI2_TABLE_LEN; k++)
      table_[(size_t)k] = ovb_chi2_quantile95(k); // the table the product embeds, as OracleCov's
  }

  // UpdaterSLAM::update steps 4-5: the oracle takes one representation per call (the runner's landmarks share feat_rep_slam)
  int slam_update(const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_landmarks *landmarks, const int32_t *reps, const ovb_opts *opts,
                  ovb_feat_out *out, double *dx, ovb_stats *stats) override {
    ovb_opts o = *opts;
    for (int f = 0; f < feats->n_feats; f++)
      if (reps[f] != reps[0])
        throw Error(OVB_ERR_ARG, "oracle slam_update: one representation per call");
    o.feat_rep = reps[0];
    const int N = dim();
    std::vector<double> P = get();
    const int st = ovo_slam_update(frame, feats, landmarks, &o, table_.data(), P.data(), N, out, dx, stats, nullptr, nullptr, nullptr, nullptr, nullptr,
                                   nullptr, 0);
    if (st != OVB_OK)
      throw Error((ovb_status)st, "oracle slam_update failed");
    set(P, N);
    return st;
  }

  // UpdaterSLAM::delayed_init composed from the oracle, as tests/test_gpu_slam_init.py composes it: triangulate every track,
  // then per triangulated feature, in order, its full Jacobians at the current frame (UpdaterHelper::get_feature_jacobian_full;
  // the single-depth representation as ANCHORED_MSCKF_INVERSE_DEPTH with the bearing columns projected out),
  // StateHelper::initialize, and the callback, which moves the mean and refreshes the frame
  void slam_delayed_init(const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_opts *opts, const int32_t *reps, const double *sigma_pix,
                         const double *chi2_multipler, ovb_init_callback on_init, void *user, ovb_feat_out *out, int32_t *lm_off) override {
    ovo_triangulate(frame, feats, opts, out, nullptr, nullptr, nullptr);
    std::vector<std::pair<int32_t, int32_t>> vars; // the frame's clone and calibration variables, ascending: the Jacobian's columns
    for (int c = 0; c < frame->n_clones; c++)
      vars.push_back({frame->clone_off[c], 6});
    for (int k = 0; k < frame->n_cams; k++) {
      if (frame->cam_ext_off[k] >= 0)
        vars.push_back({frame->cam_ext_off[k], 6});
      if (frame->cam_intr_off[k] >= 0)
        vars.push_back({frame->cam_intr_off[k], 8});
    }
    std::sort(vars.begin(), vars.end());
    std::vector<int32_t> cols;
    for (const auto &v : vars)
      for (int k = 0; k < v.second; k++)
        cols.push_back(v.first + k);
    const int ncols = (int)cols.size();
    int N = dim();
    std::vector<double> P = get();
    for (int f = 0; f < feats->n_feats; f++) {
      lm_off[f] = -1;
      if (out->status[f] != OVB_FEAT_OK)
        continue;
      const int rep = reps ? reps[f] : opts->feat_rep, k = rep == OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE ? 1 : 3;
      const int m0 = feats->meas_off[f], M = feats->meas_off[f + 1] - m0, rows = 2 * M;
      const int32_t one_meas[2] = {0, M}, one_keys[2] = {0, feats->cam_keys_off[f + 1] - feats->cam_keys_off[f]};
      const ovb_feat_batch one{1, M, one_meas, feats->cam + m0, feats->clone + m0, feats->uv + 2 * m0, feats->uvn + 2 * m0, one_keys,
                               feats->cam_keys + feats->cam_keys_off[f]};
      int32_t st = OVB_FEAT_OK, acam = out->anchor_cam[f], aclone = out->anchor_clone[f], row_off[2];
      double pA[3] = {out->p_FinA[3 * f], out->p_FinA[3 * f + 1], out->p_FinA[3 * f + 2]};
      double pG[3] = {out->p_FinG[3 * f], out->p_FinG[3 * f + 1], out->p_FinG[3 * f + 2]};
      double c2 = 0;
      ovb_feat_out o1{&st, pA, pG, &acam, &aclone, &c2};
      ovb_opts of = *opts;
      of.feat_rep = rep;
      std::vector<double> Hf((size_t)rows * 3, 0.0), Hx((size_t)rows * ncols, 0.0), res((size_t)rows, 0.0);
      ovo_feature_jacobians(frame, &one, &of, table_.data(), nullptr, N, &o1, 0, Hf.data(), Hx.data(), res.data(), row_off, ncols, cols.data(), ncols);
      // H_R over the columns the feature touches, as contiguous (offset, size) runs
      std::vector<int> used, off, sz;
      for (int j = 0; j < ncols; j++) {
        bool nz = false;
        for (int i = 0; i < rows && !nz; i++)
          nz = Hx[(size_t)i * ncols + j] != 0.0;
        if (!nz)
          continue;
        if (!used.empty() && cols[(size_t)j] == cols[(size_t)used.back()] + 1)
          sz.back()++;
        else
          off.push_back(cols[(size_t)j]), sz.push_back(1);
        used.push_back(j);
      }
      const int n = (int)used.size();
      int r = rows;
      std::vector<double> H_R((size_t)rows * n), H_L((size_t)rows * k);
      for (int i = 0; i < rows; i++)
        for (int j = 0; j < n; j++)
          H_R[(size_t)i * n + j] = Hx[(size_t)i * ncols + used[(size_t)j]];
      if (k == 3)
        H_L = Hf;
      else
        single_depth_system(Hf, H_R, res, rows, n, H_L, r);
      std::vector<double> Pn((size_t)(N + k) * (N + k)), dx_new((size_t)k), dx((size_t)(N + k));
      int accepted = 0;
      const double sp = sigma_pix ? sigma_pix[f] : opts->sigma_pix, cm = chi2_multipler ? chi2_multipler[f] : opts->chi2_multipler;
      const int s = ovo_cov_initialize(P.data(), N, off.data(), sz.data(), (int)off.size(), H_R.data(), H_L.data(), res.data(), r, k, sp * sp, cm,
                                       table_.data(), Pn.data(), &accepted, dx_new.data(), dx.data());
      if (s != OVB_OK)
        throw Error((ovb_status)s, "oracle StateHelper::initialize failed");
      if (out->chi2)
        out->chi2[f] = std::nan("");
      if (!accepted) {
        out->status[f] = OVB_FEAT_CHI2;
        continue;
      }
      P.swap(Pn);
      N += k;
      set(P, N); // the covariance the callback's caller sees is the grown one
      lm_off[f] = N - k;
      on_init(user, f, N - k, k, dx_new.data(), dx.data(), N);
    }
  }

  // the anchor changes (ovo_anchor_change, then EKFPropagation with Q = 0) in the order given, then every range
  // marginalized, highest offset first: the sequence include/ovb200.h defines ovb_marginalize_window against
  void marginalize_window(const ovb_frame *frame, const ovb_opts *opts, const int32_t *marg_off, const int32_t *marg_sz, int n_marg,
                          const ovb_anchor_changes *anchors) override {
    for (int l = 0; anchors && l < anchors->n; l++) {
      ovb_opts o = *opts;
      o.feat_rep = anchors->feat_rep[l];
      double Phi[3 * 27];
      int32_t off[8], sz[8], n_order = 0, n_cols = 0;
      ovo_anchor_change(frame, &o, anchors->lm_off[l], anchors->value + 3 * l, anchors->value_fej + 3 * l, anchors->old_cam[l], anchors->old_clone[l],
                        anchors->new_cam[l], anchors->new_clone[l], anchors->new_value + 3 * l, anchors->new_value_fej + 3 * l, Phi, off, sz, &n_order,
                        &n_cols);
      const int p = sz[n_order - 1];
      propagate(anchors->lm_off[l], p, std::vector<int>(off, off + n_order), std::vector<int>(sz, sz + n_order), std::vector<double>(Phi, Phi + p * n_cols),
                std::vector<double>((size_t)p * p, 0.0));
    }
    std::vector<std::pair<int32_t, int32_t>> ranges;
    for (int i = 0; i < n_marg; i++)
      ranges.push_back({marg_off[i], marg_sz[i]});
    std::sort(ranges.rbegin(), ranges.rend());
    for (const auto &r : ranges)
      marginalize(r.first, r.second);
  }

private:
  std::vector<double> table_;

  // the ANCHORED_INVERSE_DEPTH_SINGLE branch of UpdaterSLAM::delayed_init: [H_R | Hf[:,2] | res] with the bearing columns
  // Hf[:,0:2] Givens-projected out (UpdaterHelper::nullspace_project_inplace, the oracle's rotation and convention).
  // Returns rows - 2 rows in H_R, h_L and res.
  static void single_depth_system(std::vector<double> Hf, std::vector<double> &H_R, std::vector<double> &res, int rows, int n, std::vector<double> &h_L,
                                  int &r) {
    h_L.assign((size_t)rows, 0.0);
    for (int i = 0; i < rows; i++)
      h_L[(size_t)i] = Hf[(size_t)i * 3 + 2];
    auto rot = [](const double *cs, double &x, double &y) {
      const double xi = x, yi = y;
      x = cs[0] * xi - cs[1] * yi;
      y = cs[1] * xi + cs[0] * yi;
    };
    for (int c = 0; c < 2; c++)
      for (int m = rows - 1; m > c; m--) {
        double cs[2];
        ovo_make_givens(Hf[(size_t)(m - 1) * 3 + c], Hf[(size_t)m * 3 + c], cs);
        for (int q = c; q < 2; q++)
          rot(cs, Hf[(size_t)(m - 1) * 3 + q], Hf[(size_t)m * 3 + q]);
        for (int j = 0; j < n; j++)
          rot(cs, H_R[(size_t)(m - 1) * n + j], H_R[(size_t)m * n + j]);
        rot(cs, h_L[(size_t)m - 1], h_L[(size_t)m]);
        rot(cs, res[(size_t)m - 1], res[(size_t)m]);
      }
    r = rows - 2;
    H_R.erase(H_R.begin(), H_R.begin() + 2 * n);
    h_L.erase(h_L.begin(), h_L.begin() + 2);
    res.erase(res.begin(), res.begin() + 2);
  }
};
} // namespace ovb200
