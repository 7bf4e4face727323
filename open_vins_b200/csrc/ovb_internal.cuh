// ovb_internal.cuh — context, device-side views and launch declarations shared by the .cu files of libovb200.so.
#pragma once
#include "../../include/ovb200.h"
#include <cuda_runtime.h>
#include <stdint.h>

// OVB_MAX_MEAS_PER_FEAT (include/ovb200.h): 384 = every camera in every clone pose
#define OVB_BIG_MAX_MEAS 128      // longest track of the per-feature kernel's BIG path: d_scratch is sized for it at ovb_create
#define OVB_MAX_COLS 512          // >= 6*OVB_MAX_CLONES + 14*OVB_MAX_CAMS; also the widest H of ovb_ekf_update (config 5: n = 500)
#define OVB_NB 16                 // TSQR panel width
#define OVB_CR 256                // TSQR rows per chunk
#define OVB_PROP_MAX_N 64         // widest IMU block of ovb_cov_propagate_imu (15 + IMU intrinsics is 15, 30 or 39)
#define OVB_PROP_STEPS_RESERVE 64 // IMU steps per frame the staging of ovb_cov_propagate_imu holds from ovb_create (at n = 39)
#define OVB_NO_NEG_DIAG 0x7fffffff // negative-diagonal index (DevUpdateInfo, ovb_marginalize_window's flags) when none is negative

// ---- device-resident copy of the slice of State the path reads (uploaded once per update call)
struct DevFrame {
  int n_clones, n_cams;
  int n_slots;        // variables a feature can touch (clones + calibrated extrinsics/intrinsics)
  int n_all;          // canonical column count = sum of slot sizes
  double clone_R[OVB_MAX_CLONES][9];
  double clone_p[OVB_MAX_CLONES][3];
  double clone_R_fej[OVB_MAX_CLONES][9];
  double clone_p_fej[OVB_MAX_CLONES][3];
  double cam_R[OVB_MAX_CAMS][9];
  double cam_p[OVB_MAX_CAMS][3];
  double cam_intr[OVB_MAX_CAMS][8];
  int cam_model[OVB_MAX_CAMS];
  // slots in canonical (ascending covariance offset) order
  int slot_off[OVB_MAX_VARS];  // covariance offset
  int slot_size[OVB_MAX_VARS]; // 6 or 8
  int slot_col[OVB_MAX_VARS];  // first canonical column
  int clone_slot[OVB_MAX_CLONES];
  int cam_ext_slot[OVB_MAX_CAMS];  // -1 when not calibrated
  int cam_intr_slot[OVB_MAX_CAMS]; // -1 when not calibrated
  const struct DevGroup *groups;   // SLAM update: its column groups (ctx->d_grp), else null
  int lm_w;                        // SLAM update: width of the batch's widest landmark (sizes the per-feature kernel's tables)
};

// SLAM update: one column group = a contiguous feature range whose frame columns plus landmark columns fit OVB_MAX_COLS.
// Its rows are staged in a group-local canonical layout (the frame slots and the group's landmarks in ascending
// covariance offset), compressed on their own and applied as one step of a sequential EKF update (ovb_slam_update).
// A batch of at most OVB_MAX_COLS columns is one group whose layout is the batch's canonical layout.
struct DevGroup {
  int f0, f1;      // features [f0, f1)
  int row0, rows;  // staged rows
  int n_cols;      // group-local canonical columns
  int n_ent;       // variables of the layout: frame slots and the group's landmarks, ascending covariance offset
  int ent[OVB_MAX_VARS + OVB_MAX_COLS]; // >= 0: frame slot; < 0: the landmark of feature -1 - ent
  int col_state[OVB_MAX_COLS];          // covariance index of each group column
  short col_frame[OVB_MAX_COLS];        // frame canonical column of each group column, -1 for a landmark column
};

// camera-at-clone poses (update/UpdaterMSCKF.cpp:98-115), filled on the device by k_cam_poses
struct DevCamPoses {
  double cc_R[OVB_MAX_CAMS][OVB_MAX_CLONES][9]; // R_GtoCi
  double cc_p[OVB_MAX_CAMS][OVB_MAX_CLONES][3]; // p_CiinG
};

struct DevOpts {
  ovb_opts o;
  double sigma_pix_sq;
  int rep; // effective MSCKF representation (SINGLE remapped, UpdaterMSCKF.cpp:180-183)
};

// per-feature device record (inputs derived on the host while packing + outputs)
struct DevFeat {
  int m0, m1;        // measurement range
  int row0;          // first row in the stacked staging matrix (prefix sum of max(2M-3,0))
  int key0, key1;    // camera-key range
  int status;        // ovb_feat_status
  int anchor_cam, anchor_clone;
  int sched;         // CTA i of the per-feature kernels works on feature feats[i].sched (longest tracks first)
  int rep;           // SLAM update: the landmark's ovb_feat_rep (Landmark::_feat_representation); unused otherwise
  double p_FinA[3], p_FinG[3];
  double chi2;
  // SLAM update only (landmark already in the state, update/UpdaterSLAM.cpp:333-341, :389-408)
  double p_FinG_fej[3]; // Landmark::get_xyz(true) for the global representations
  double sigma_sq;      // per-class pixel noise variance
  double chi2_mult;     // per-class gate multiplier
  int lm_off;           // covariance offset of the landmark's own variable (3 wide, or 1 for ANCHORED_INVERSE_DEPTH_SINGLE)
                        // width and rows of a landmark: 3 and 2M, or 1 and 2M-2 for ANCHORED_INVERSE_DEPTH_SINGLE
  unsigned short lm_col, grp; // first column of the landmark in its column group's layout, and that group
};

// written by the column-map kernel; read by TSQR re-order, EKF and the host (D2H with the outputs)
struct DevUpdateInfo {
  int n_used;                   // columns of the stacked H in the requested order (ct_jacob)
  int n_feats_used;             // accepted features
  int rows_stacked;             // Σ (2M-3) over accepted features
  int n_order;                  // variables in Hx_order_big
  int order_slot[OVB_MAX_VARS]; // slot id of each variable in stacked order (MSCKF updates)
  int col_state[OVB_MAX_COLS];  // covariance index of each stacked column (order applied)
  int col_canon[OVB_MAX_COLS];  // canonical column each stacked column comes from
  int neg_diag_index;           // EKF: first negative diagonal, or OVB_NO_NEG_DIAG
  int not_spd;                  // EKF: Cholesky pivot failure flag
  int nonfinite;
};

// ovb_slam_delayed_init: one feature's StateHelper::initialize system on the device. The per-feature kernel's INIT
// instantiation writes the k init rows (k = 3, or 1 for ANCHORED_INVERSE_DEPTH_SINGLE) and the column map, k_init_prep
// finishes it; the head (status .. dx_new) is what the host reads back after the feature.
struct DevInitSys {
  int status;       // the feature's status after the gate; OVB_FEAT_OK = accepted
  int skip;         // nonzero: every kernel after the gate leaves P alone (rejected, or one of the failures below)
  int fail;         // 1: H_L is rank deficient, 2: the kernel's column count differs from the host's
  int pad;
  double chi2;
  double dx_new[3]; // H_L^-1 res_init
  // ---- written by the per-feature kernel
  int n;                        // state columns the feature touches (canonical order)
  int col_state[OVB_MAX_COLS];  // covariance index of each of them
  double HL[9];                 // Q1' H_f, 3 x 3 (rows 0..2 of the Householder split; SINGLE uses entry [2][2])
  double res[3];                // Q1' r
  double HR[3 * OVB_MAX_COLS];  // Q1' H_x, k x n with leading dimension n (the rows SINGLE keeps: row 2 only)
  double Hinv[9];               // k x k, written by k_init_prep
};
#define OVB_INIT_HEAD_BYTES (4 * sizeof(int) + 4 * sizeof(double))

// ovb_slam_delayed_init_batch: what the device needs to move the frame between the features and what it hands back.
// One allocation [DevInitBatch][DevInitRec x F][dx rows]; the head is uploaded once, everything is read back once.
struct DevInitBatch {
  int N;                                // live covariance size: advances by a landmark's width when it is initialised
  int fej_R_is_value, fej_p_is_value;   // the caller passed no FEJ array: the FEJ copy follows the moved value
  int pad;
  double clone_q[OVB_MAX_CLONES][4];    // JPL [x y z w] behind DevFrame::clone_R
  double cam_q[OVB_MAX_CAMS][4];        // behind DevFrame::cam_R
};
struct DevInitRec {
  int status;          // after the gate; OVB_FEAT_OK = initialised
  int lm_off;          // the landmark's covariance id, -1 when it was not initialised
  int fail;            // 0, or what makes the call fail at this feature: 1 H_L rank deficient, 2 column count, 3 EKF update
  int n;               // columns the per-feature kernel counted (fail 2)
  int not_spd, nonfinite, neg_diag_index, pad; // the EKF update's flags (fail 3)
  double chi2;
  double dx_new[3];
};

// ovb_marginalize_window: the frame slice the anchor changes read (FEJ arrays already substituted when the caller has
// none) and one record per re-anchored landmark; uploaded with the rest of the call's inputs in one H2D copy
struct DevWinFrame {
  double clone_R[OVB_MAX_CLONES][9];
  double clone_p[OVB_MAX_CLONES][3];
  double clone_R_fej[OVB_MAX_CLONES][9];
  double clone_p_fej[OVB_MAX_CLONES][3];
  double cam_R[OVB_MAX_CAMS][9];
  double cam_p[OVB_MAX_CAMS][3];
  int clone_off[OVB_MAX_CLONES];
  int cam_ext_off[OVB_MAX_CAMS];
};
struct DevWinLM {
  double value[3], value_fej[3];
  int lm_off, rep, p; // covariance id, ovb_feat_rep, width (3, or 1 for ANCHORED_INVERSE_DEPTH_SINGLE)
  int row0;           // first of its p rows in the moved-row scratch
  int old_cam, old_clone, new_cam, new_clone;
  int host;           // 1: Phi, its column indices, q and the new values were computed on the host and uploaded
};
#define OVB_WIN_Q 27                 // widest Phi of an anchor change: 2 clones + 2 extrinsics + the landmark
#define OVB_WIN_PHI (3 * OVB_WIN_Q)  // its doubles

// packed measurement blob layout (device): [meas_off int32 (F+1)][cam u8 (M)][pad][clone u16 (M)][pad][uv f32 2M][uvn f32 2M][keys u8]
struct BlobView {
  const uint8_t *cam;
  const uint16_t *clone;
  const float *uv;
  const float *uvn;
  const uint8_t *keys;
};

// one packed batch (pack_inputs): the arena's sizes and the device view of its measurement blob
struct Packed {
  int n_feats, n_meas, m_total, ldH, n_all;
  int n_groups; // SLAM: column groups (ctx->h_grp / d_grp); n_all is then the widest group's column count
  BlobView bv;
};

struct ovb_ctx {
  ovb_config cfg;
  int device;
  cudaStream_t stream;
  int own_stream;
  cudaStream_t side_stream;      // column bookkeeping runs here, concurrently with the compression
  cudaStream_t side_stream2;     // with side_stream: the per-feature kernel's size classes run side by side
  cudaEvent_t ev_fork, ev_join, ev_join2;
  int feat_classes;              // split the per-feature kernel into size classes (OVB_FEAT_CLASSES=0 disables: A/B timing only)
  cudaEvent_t ev[8];
  char err[256];
  // covariance (double buffered for clone/marginalize), row-major with leading dimension ldP
  int N, ldP;
  double *P[2];
  int cur;
  // per-call device inputs
  // one input arena (single H2D copy per call): [DevFrame][DevOpts][DevFeat x max_feats][blob]
  unsigned char *d_arena, *h_arena;
  size_t arena_bytes, off_opts, off_feat, off_blob;
  DevFrame *d_frame;
  DevOpts *d_opts;
  DevFeat *d_feat;
  unsigned char *d_blob; // packed SoA measurements
  DevFrame *h_frame;
  DevOpts *h_opts;
  DevFeat *h_feat;
  unsigned char *h_blob;
  size_t blob_cap;
  DevCamPoses *d_cc;
  unsigned char *d_feat_order; // [max_feats][OVB_MAX_VARS+1] per-feature Hx_order (slot ids, first-seen)
  DevUpdateInfo *d_info;
  DevUpdateInfo *h_info;
  double *h_dx;
  double *h_stage; // pinned staging for dense H / Phi uploads (grown on demand)
  size_t stage_cap;
  // device work buffers
  double *d_chi2_table;
  double *d_Hs; // stacked staging matrix [max_rows][ldH]
  size_t Hs_cap; // doubles
  double *d_W[2]; // TSQR panel ping-pong workspaces
  size_t W_cap;
  double *d_R;   // TSQR output [OVB_MAX_COLS][ldR]
  double *d_R2;  // re-ordered / re-triangularised R
  double *d_M;   // EKF: P[:,cols] H'   [max_state][ldM]
  double *d_S;   // EKF: innovation covariance / Cholesky factor
  double *d_Y;   // EKF: M L^-T
  double *d_w;   // EKF: L^-1 z
  double *d_dx;
  double *d_scratch; // per-CTA scratch for large features in the gate kernel (BIG path, up to OVB_BIG_MAX_MEAS measurements)
  size_t scratch_per_cta;
  int scratch_ctas;
  double *d_long;    // per-CTA scratch of the long-track path (feature_scratch_reserve: sized by the call's tracks, grown on demand)
  size_t long_cap;   // doubles
  double *d_dump; // debug dumps for ovb_feature_jacobians
  size_t dump_cap;
  int dump_rows;
  int max_rows;
  int sm_count;
  size_t info_bytes; // DevUpdateInfo rounded up: d_dx / h_dx start right behind d_info / h_info
  int attr_done[9]; // per-context (= per-device) one-time cudaFuncSetAttribute flags: 0 tsqr, 1 feature, 2 ekf, 3 gram, 4 cholqr, 8 triangulate
  int pdl;          // programmatic dependent launch on every ovb_launch (OVB_TSQR_PDL=0 disables: A/B timing only)
  int tsqr_cluster; // upper TSQR levels as one thread-block cluster (OVB_TSQR_CLUSTER=0 disables: A/B timing only)
  int gram_cluster;  // k_cq_gram: clusters of 4 slabs pre-reduce in distributed shared memory (OVB_GRAM_CLUSTER=0 disables: A/B timing only)
  int ekf_chol_dmma; // EKF Cholesky on the DMMA kernel of k_cholqr.cu (OVB_EKF_CHOL_DMMA=0 disables: A/B timing only)
  mutable float stage_ms[6];
  mutable int stage_pending; // stage_ms[0..4] of the last update not read back from the events yet (done on demand: each read costs ~1.5 us of host time)
  double host_us[4]; // host wall clock of the last ovb_msckf_update: marshalling + H2D enqueue, kernel enqueue, wait, result unpack
  // replay of the last update on device-resident inputs (bench: `value` leg; see ovb_msckf_replay)
  // (last_pk also carries the sharded pair's batch from ovb_msckf_shard_compress to ovb_msckf_shard_finish)
  int replay_enabled, last_pk_valid;
  Packed last_pk;
  int last_col_order;
  double *P_snap;
  void *d_flush;
  // SLAM column groups (grown on demand): the group tables, and for batches of several groups the accumulated state
  // correction [max_state doubles] followed by the failure flags [not_spd, nonfinite] of the sequential EKF update
  DevGroup *d_grp, *h_grp;
  int grp_cap;
  double *d_grp_acc;
  int slam_unbounded; // ovb_set_slam_unbounded: SLAM batches beyond OVB_MAX_VARS variables (else OVB_ERR_CAPACITY, as before)
  // bookkeeping for bench.py: kernels launched by the last call (counted by ovb_launch), bytes moved by the last ovb_msckf_update
  int n_launch, n_launch_tsqr_level;
  // normal-equations compression (k_gram.cu)
  double *d_Gpart, *d_G;
  size_t Gpart_cap, G_cap;
  double *d_cqw; // wide systems (k_cholqr.cu): [G1 | G2 | packed diagonal-block factors | scalars]
  size_t cqw_cap;
  // k_cholqr.cu's factor streaming: the publication counter (device, zero at ovb_create) and the last epoch drawn
  unsigned long long *d_pub;
  unsigned long long pub_epoch;
  size_t last_h2d_bytes, last_d2h_bytes;
  // ovb_slam_delayed_init: the device system of the current feature and its pinned read-back (allocated on first use), and
  // the counters of the last call (ovb_last_init_counters)
  DevInitSys *d_init, *h_init;
  int64_t init_counters[4];
  // ovb_slam_delayed_init_batch: [DevInitBatch][DevInitRec x F][dx rows] on the device and its pinned mirror (grown on demand)
  unsigned char *d_ib, *h_ib;
  size_t ib_cap; // bytes
  // ovb_cov_propagate_imu: the per-step operands [F | G | qc | dnc_dt | old indices], one H2D copy per call; the pinned
  // side also receives Phi and Q. Reserved at ovb_create for ordinary frames, grown with headroom beyond.
  double *d_imu, *h_imu;
  size_t imu_cap; // doubles
  // per-kernel profile (ovb_set_profile): CUDA events around every ovb_launch of the last call; PDL is off while it is on.
  // The pool of prof_cap event pairs grows on demand (ovb_prof_slot).
  int prof_on, prof_n, prof_cap;
  cudaEvent_t *prof_ev; // [2 * prof_cap]
  const void **prof_fn; // [prof_cap]
};

#define OVB_CUDA_CHECK(ctx, call)                                                                                     \
  do {                                                                                                                \
    cudaError_t e_ = (call);                                                                                          \
    if (e_ != cudaSuccess) {                                                                                          \
      snprintf((ctx)->err, sizeof((ctx)->err), "%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_));    \
      return OVB_ERR_CUDA;                                                                                            \
    }                                                                                                                 \
  } while (0)

// ---- launchers (each enqueues on ctx->stream; no host sync)
void launch_cam_poses(ovb_ctx *ctx);
void launch_triangulate(ovb_ctx *ctx, int n_feats, BlobView bv);
// mode 0: normal (write post-nullspace rows to Hs, gate on chi²); mode 1: dump pre-nullspace dense rows to d_dump
// mode 2: like 0 but features keep the status/p_FinG given (no triangulation ran) — used by ovb_feature_jacobians
// Every track runs on the path it fits (shared-memory tile, BIG, or long-track; see k_feature.cu).
void launch_feature_system(ovb_ctx *ctx, int n_feats, BlobView bv, int ldH, int mode);
// grow the long-track scratch for the tracks of the packed batch (h_feat); slam: the batch is a SLAM update, init: the
// tracks run through launch_feature_init
ovb_status feature_scratch_reserve(ovb_ctx *ctx, int n_feats, bool slam, bool init = false);
// ovb_slam_delayed_init: the per-feature kernel's INIT instantiation for the one feature feats[sched].sched: the gate of
// StateHelper::initialize with the feature's own sigma / multiplier, its 2M-3 projected rows (compact columns, residual
// last) at its row0 of d_Hs, and its init system in ctx->d_init
void launch_feature_init(ovb_ctx *ctx, int sched, BlobView bv, int ldH);
// finish the init system: H_L^-1, dx_new, the column map into d_info, the skip flag; n = the host's column count
void launch_init_prep(ovb_ctx *ctx, int feat, int k, int n);
void launch_column_map(ovb_ctx *ctx, int n_feats, BlobView bv, int rows_drop = 3);
// SLAM update: counts of the whole batch; full_map: also the column map of the single group's layout (ctx->d_grp[0]).
// Each feature's landmark width and dropped rows follow its DevFeat::rep.
void launch_column_map_slam(ovb_ctx *ctx, int n_feats, bool full_map);
// TSQR of A [m x (n+1)] (last column = residual) in place; R (n x (n+1), diag>=0) to Rout with leading dimension ldR
void launch_tsqr(ovb_ctx *ctx, double *A, int m, int n, int ldA, double *Rout, int ldR);
// gather columns of Rin in the order info->col_canon (n_used of them) into Hs scratch and re-triangularise into Rout
// [R | z] <- chol([H r]'[H r]) (k_gram.cu); false when its buffers could not be allocated
bool launch_compress_gram(ovb_ctx *ctx, const double *A, int m, int n, int ldA, double *Rout, int ldR);
// [R | z] <- shifted CholeskyQR2 of A (k_cholqr.cu; A is kept up to CQ_MAXN columns, overwritten by the wider blocked
// path); false when the system is too wide for it (callers then use launch_tsqr)
bool launch_compress_cholqr2(ovb_ctx *ctx, double *A, int m, int n, int ldA, double *Rout, int ldR);
// EKF Cholesky on the DMMA kernel of k_cholqr.cu; false when r does not fit (caller uses k_ekf_chol)
// epoch_out != nullptr: the factor streams to the launch_trsm_rows that follows (epoch 0: it does not)
bool launch_chol_ekf_dmma(ovb_ctx *ctx, double *S, int ldS, int r, const double *res, double *w, double *invdiag, double **Lpk_out,
                          unsigned long long *epoch_out);
// A <- A (L')^-1 for the rows of A [m x nt] with the packed factor of the DMMA Cholesky; false when it does not fit.
// epoch != 0: the factor streams in from the launch_chol_ekf_dmma just before, which returned that epoch
bool launch_trsm_rows(ovb_ctx *ctx, double *A, int ldA, int m, int nt, const double *Lpk, unsigned long long epoch);
// wide EKF (r > 160): blocked DMMA Cholesky of S (r x r lower, residual staged in w) and Y = M L^-T in place; false when r
// exceeds OVB_MAX_COLS or the leading dimensions are odd
bool launch_chol_solve_wide(ovb_ctx *ctx, double *S, int ldS, int r, double *w, double *invdiag, double *M, int ldM, int N, bool gate_only);
void launch_reorder_R(ovb_ctx *ctx, const double *Rin, int n_all, int ldRin, double *Rout, int ldRout);
// EKF update from an upper-trapezoidal / dense H [r x (n+1)] (r <= n) whose column n holds the residual, with the
// column->state map in d_info. gate_only: stop after the Cholesky factor (d_w then holds w = L^-1 res, P is untouched).
// skip_dev (optional): a device flag read after the previous kernels; nonzero marks the update failed before it starts
// (info->not_spd), so P is left untouched and dx = 0
void launch_ekf_update(ovb_ctx *ctx, const double *H, int ldHm, int r, int n, bool gate_only, double sigma2, const double *Rdiag_dev,
                       const int *skip_dev = nullptr);
// false: the launch was refused (shared-memory footprint) or failed; the caller must not grow N.
// skip_dev (optional): the kernel returns without writing when *skip_dev is nonzero
// N_dev (optional): the covariance size is read on the device (ctx->N is then its upper bound and sizes the launch)
bool launch_cov_init_augment(ovb_ctx *ctx, int k, int n, const double *Hx_dev, const double *Hinv_dev, double sigma2,
                             const int *skip_dev = nullptr, const int *N_dev = nullptr);
// ovb_slam_delayed_init_batch, after feature `feat`'s EKF update: its record (the dx row, N0 + k doubles, at dx_row), and
// unless the feature was skipped or failed, the StateHelper::EKFUpdate mean update (⊞) of the device frame with d_dx and
// the advance of the live covariance size by k. Compiled without FMA contraction: the frame gets the host's bits.
void launch_init_commit(ovb_ctx *ctx, DevInitBatch *ib, DevInitRec *rec, double *dx_row, int k, int calib_pose, int calib_intr);
// neg_diag_dev (optional): d_info's negative-diagonal flag of a propagation enqueued before; when it is set the clone
// leaves P alone (ovb_cov_propagate_imu then does not grow N)
void launch_cov_clone(ovb_ctx *ctx, int old_off, int size, const double *dnc_dt_dev, int dt_off, const int *neg_diag_dev = nullptr);
void launch_cov_marginalize(ovb_ctx *ctx, int off, int size);
void launch_cov_propagate(ovb_ctx *ctx, int new_off, int p, int q, const int *old_idx_dev, const double *Phi_dev, const double *Q_dev);
// ovb_marginalize_window (anchor_change.cu): Phi, column indices and new values of each re-anchored landmark
void launch_anchor_phi(ovb_ctx *ctx, const DevWinFrame *wf, const DevWinLM *lms, int n, int do_fej, int ext, int *flags, double *new_values,
                       double *phi, int *idx, int *q);
// ovb_marginalize_window (k_ekf.cu): the K moved landmark rows into R [K x N] (ld ldR), their K x K blocks into B, then
// P[cur] compacted through src / mv into P[cur ^ 1]; flags = {negative diagonal index, singular}: set, P stays untouched
void launch_window_shift(ovb_ctx *ctx, int n, int K, int N2, const DevWinLM *lms, const int *row_lm, const double *phi, const int *idx,
                         const int *q, const int *src, const int *mv, int *flags, double *R, int ldR, double *B);
// Phi, Q (n x n, n <= OVB_PROP_MAX_N) accumulated over `steps` IMU steps, F [steps][n][n], G [steps][n][12], qc [steps][4];
// false when the launch failed
bool launch_prop_accumulate(ovb_ctx *ctx, int n, int steps, const double *F_dev, const double *G_dev, const double *qc_dev, double *Phi_dev,
                            double *Q_dev);

// ---- programmatic dependent launch (PDL) ----------------------------------------------------------------------------
// Every kernel starts with OVB_PDL_ENTER() (or places the two instructions itself): it lets the NEXT kernel of the
// stream be scheduled while this one runs (its CTAs become resident on idle SMs and block), then waits until the
// PREVIOUS kernel has completed and flushed. Semantics are those of ordinary stream order as long as nothing before the
// wait touches memory another kernel writes; what is saved is the launch latency between the dependent, latency-bound
// kernels of one call. Both instructions are no-ops in a kernel launched without the attribute.
#define OVB_PDL_ENTER()                                                     \
  do {                                                                      \
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");         \
    asm volatile("griddepcontrol.wait;" ::: "memory");                      \
  } while (0)

// the profile slot of the next launch of kern (the pool grows as needed), or -1 when no event could be created
int ovb_prof_slot(ovb_ctx *ctx, const void *kern);

// launch geometry: the grid, optionally as thread-block clusters of `cluster` CTAs
struct ovb_grid {
  dim3 blocks, cluster;
  ovb_grid(dim3 b, dim3 c = dim3(1, 1, 1)) : blocks(b), cluster(c) {}
};

#ifdef __CUDACC__
// The one launch site of the library: enqueues kern on ctx->stream with the PDL attribute when ctx->pdl is set and
// profiling is off, counts the launch in ctx->n_launch and, while profiling, brackets it with a pair of CUDA events.
template <typename... KArgs, typename... Args>
static inline cudaError_t ovb_launch(ovb_ctx *ctx, void (*kern)(KArgs...), ovb_grid grid, dim3 block, size_t smem, Args &&...args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid.blocks;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = ctx->stream;
  cudaLaunchAttribute at[2];
  int na = 0;
  if (ctx->pdl && !ctx->prof_on) {
    at[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[na].val.programmaticStreamSerializationAllowed = 1;
    na++;
  }
  if (grid.cluster.x * grid.cluster.y * grid.cluster.z > 1) {
    at[na].id = cudaLaunchAttributeClusterDimension;
    at[na].val.clusterDim.x = grid.cluster.x;
    at[na].val.clusterDim.y = grid.cluster.y;
    at[na].val.clusterDim.z = grid.cluster.z;
    na++;
  }
  cfg.attrs = at;
  cfg.numAttrs = na;
  const int slot = ctx->prof_on ? ovb_prof_slot(ctx, (const void *)kern) : -1;
  if (slot >= 0)
    cudaEventRecord(ctx->prof_ev[2 * slot], ctx->stream);
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
  if (slot >= 0)
    cudaEventRecord(ctx->prof_ev[2 * slot + 1], ctx->stream);
  ctx->n_launch++;
  return e;
}
#endif
