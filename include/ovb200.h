/*
 * ovb200.h — C ABI of the H100-native MSCKF update engine (libovb200.so).
 *
 * This is the drop-in boundary for the ONE hot path of rpng/open_vins that this
 * repo re-implements for sm_90a:    UpdaterMSCKF::update  →  triangulate →
 * Jacobian → nullspace → chi² gate → stack → compress → EKFUpdate,  plus the
 * covariance side of Propagator::propagate_and_clone (EKFPropagation, clone,
 * marginalize).  The reference has no FFI layer; the seam is its C++ class
 * surface (SURVEY.md §8b).  Every entry point below names the reference
 * function whose arithmetic it replaces (paths relative to the reference root).
 *
 * Conventions
 *   - plain C: pointers, ints, doubles.  No C++/Eigen/torch types.
 *   - every function returns an ovb_status; nothing calls exit() or throws.
 *   - all HOST pointers unless the name ends in _dev; the context owns all
 *     device memory; the covariance P lives on the device between calls.
 *   - matrices crossing the ABI are dense row-major doubles unless stated
 *     (P is symmetric, so row/column-major coincide for it).
 *   - rotations are 3x3 row-major; R_GtoI rotates global→IMU (JPL convention of
 *     ov_core/src/utils/quat_ops.h).
 *   - single caller per context (the reference estimator is single-threaded,
 *     ov_msckf/src/core/VioManager.cpp:323); one CUDA stream per context.
 */
#ifndef OVB200_H
#define OVB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OVB_ABI_VERSION 1
#define OVB_MAX_CAMS 8    /* cameras per rig (reference: StateOptions::num_cameras) */
#define OVB_MAX_CLONES 48 /* clone poses in the sliding window incl. the newest */
#define OVB_MAX_VARS (OVB_MAX_CLONES + 2 * OVB_MAX_CAMS) /* 6/6/8-wide state variables a feature can touch */
#define OVB_MAX_MEAS_PER_FEAT (OVB_MAX_CAMS * OVB_MAX_CLONES) /* measurements of one feature track: every camera in every clone */
#define OVB_CHI2_TABLE_LEN 2048

/* ---- status codes (replace the reference's std::exit paths, state/StateHelper.cpp:103-113,172-182) ---- */
typedef enum {
  OVB_OK = 0,
  OVB_ERR_NEG_DIAG = 1,  /* covariance diagonal went negative (reference prints and exits) */
  OVB_ERR_NONFINITE = 2, /* NaN/Inf in dx or P */
  OVB_ERR_CAPACITY = 3,  /* a size exceeds what ovb_create reserved */
  OVB_ERR_CUDA = 4,      /* CUDA runtime error; see ovb_last_error */
  OVB_ERR_ARG = 5,       /* malformed argument */
  OVB_ERR_NOT_SPD = 6    /* innovation covariance S not positive definite */
} ovb_status;

/* ---- per-feature outcome; mirrors the reject sites of the reference ---- */
typedef enum {
  OVB_FEAT_OK = 0,          /* used in the update */
  OVB_FEAT_FEW_MEAS = 1,    /* <2 measurements           update/UpdaterMSCKF.cpp:88 */
  OVB_FEAT_TRI_COND = 2,    /* cond(A) > max_cond_number feat/FeatureInitializer.cpp:103 */
  OVB_FEAT_TRI_DEPTH = 3,   /* z outside [min,max]_dist  feat/FeatureInitializer.cpp:103,187 */
  OVB_FEAT_TRI_NAN = 4,     /* NaN                       feat/FeatureInitializer.cpp:104 */
  OVB_FEAT_GN_DEPTH = 5,    /* refined z outside range   feat/FeatureInitializer.cpp:367 */
  OVB_FEAT_GN_BASELINE = 6, /* |p|/baseline > max        feat/FeatureInitializer.cpp:368 */
  OVB_FEAT_GN_NAN = 7,      /*                           feat/FeatureInitializer.cpp:368 */
  OVB_FEAT_CHI2 = 8         /* chi² gate                 update/UpdaterMSCKF.cpp:225 */
} ovb_feat_status;

/* ov_core/src/types/LandmarkRepresentation.h:38-46 (same numeric values) */
typedef enum {
  OVB_REP_GLOBAL_3D = 0,
  OVB_REP_GLOBAL_FULL_INVERSE_DEPTH = 1,
  OVB_REP_ANCHORED_3D = 2,
  OVB_REP_ANCHORED_FULL_INVERSE_DEPTH = 3,
  OVB_REP_ANCHORED_MSCKF_INVERSE_DEPTH = 4,
  OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE = 5
} ovb_feat_rep;

typedef enum { OVB_CAM_RADTAN = 0, OVB_CAM_EQUI = 1 } ovb_cam_model; /* cam/CamRadtan.h, cam/CamEqui.h */

/* Column order of the stacked/compressed Jacobian (SURVEY.md App. A.5). */
typedef enum {
  OVB_COLS_REFERENCE_FIRST_SEEN = 0, /* update/UpdaterMSCKF.cpp:237-245: first appearance over accepted features */
  OVB_COLS_CANONICAL = 1             /* ascending covariance offset; post-update state/P agree to rounding */
} ovb_col_order;

/* How UpdaterHelper::measurement_compress_inplace (update/UpdaterHelper.cpp:456-487) is carried out. All give
 * R'R = H'H and R'z = H'r (DESIGN.md §4); ovb_opts_default selects OVB_COMPRESS_CHOLQR2. */
typedef enum {
  OVB_COMPRESS_HOUSEHOLDER_TSQR = 0, /* blocked Householder TSQR; R equals the reference's Givens R row for row (diag >= 0);
                                        post-update P/x within 1e-9 of the reference in every tested setup */
  OVB_COMPRESS_NORMAL_EQUATIONS = 1, /* opt-in: [R z] = chol([H r]'[H r]), one streaming pass. Squares the condition number:
                                        with weakly observable calibration states in the update (online intrinsics /
                                        extrinsics) the posterior of those states is only good to ~1e-6 relative, so it
                                        misses the 1e-9 parity bar there (tests/test_gpu_gram.py) */
  OVB_COMPRESS_CHOLQR2 = 2           /* default. Shifted CholeskyQR2 on the FP64 tensor-core path (csrc/k_cholqr.cu): two Gram +
                                        Cholesky passes with a row-wise triangular solve in between. No condition-number
                                        loss in R'R / R'z (DESIGN.md §4), same 1e-9 bar as the Householder path, ~3x
                                        faster at the BASELINE sizes; systems wider than 159 columns use the blocked
                                        variant (up to 512 columns), beyond that the Householder TSQR */
} ovb_compress_mode;

/* ---- context ---- */
typedef struct ovb_ctx ovb_ctx;

typedef struct {
  int device;    /* CUDA device ordinal */
  int max_state; /* capacity of the covariance dimension N (State::max_covariance_size) */
  int max_feats; /* features per update call */
  int max_meas;  /* total measurements (uv pairs) per update call */
  int max_rows;  /* rows of a raw H handed to ovb_compress / ovb_ekf_update (0 = derive from max_meas) */
} ovb_config;

/* ---- options: the three option structs the path reads ---- */
typedef struct {
  /* ov_core/src/feat/FeatureInitializerOptions.h:33-69 (defaults in comments) */
  int triangulate_1d;     /* false */
  int refine_features;    /* true  */
  int max_runs;           /* 5     */
  double init_lamda;      /* 1e-3  */
  double max_lamda;       /* 1e10  */
  double min_dx;          /* 1e-6  */
  double min_dcost;       /* 1e-6  */
  double lam_mult;        /* 10    */
  double min_dist;        /* 0.10  */
  double max_dist;        /* 60    */
  double max_baseline;    /* 40    */
  double max_cond_number; /* 10000 */
  /* ov_msckf/src/update/UpdaterOptions.h:32-48 */
  double sigma_pix;      /* 1 */
  double chi2_multipler; /* 5 (rpng_sim yaml: 1) */
  /* ov_msckf/src/state/StateOptions.h:35-176 (only what the path reads) */
  int do_fej;                     /* use_fej */
  int feat_rep;                   /* ovb_feat_rep for MSCKF features (feat_rep_msckf) */
  int do_calib_camera_pose;       /* calib_cam_extrinsics */
  int do_calib_camera_intrinsics; /* calib_cam_intrinsics */
  int col_order;                  /* ovb_col_order */
  int compress;                   /* ovb_compress_mode */
} ovb_opts;

/* Fill with the reference defaults quoted above (rpng_sim: do_fej=1, GLOBAL_3D, chi2_multipler=1). */
void ovb_opts_default(ovb_opts *o);

/* ---- frame: the slice of ov_msckf::State the path reads (state/State.h:49-193) ----
 * Clones are ordered oldest→newest; index c is what ovb_feat_batch.clone refers to.
 * *_off are the variables' first row/col in the covariance (ov_type::Type::id(), types/Type.h:57);
 * -1 = "not in the state" (calibration disabled). Clone poses are 6 wide (θ, p), extrinsics 6, intrinsics 8. */
typedef struct {
  int n_clones;
  int n_cams;
  const double *clone_R;     /* [n_clones][9]  R_GtoI        PoseJPL::Rot()     */
  const double *clone_p;     /* [n_clones][3]  p_IinG        PoseJPL::pos()     */
  const double *clone_R_fej; /* [n_clones][9]                PoseJPL::Rot_fej() */
  const double *clone_p_fej; /* [n_clones][3]                PoseJPL::pos_fej() */
  const int *clone_off;      /* [n_clones] */
  const double *cam_R;       /* [n_cams][9]    R_ItoC        state->_calib_IMUtoCAM */
  const double *cam_p;       /* [n_cams][3]    p_IinC */
  const double *cam_intr;    /* [n_cams][8]    fx fy cx cy d0 d1 d2 d3 (state->_cam_intrinsics) */
  const int *cam_model;      /* [n_cams]       ovb_cam_model */
  const int *cam_ext_off;    /* [n_cams]       or -1 */
  const int *cam_intr_off;   /* [n_cams]       or -1 */
} ovb_frame;

/* ---- feature batch: SoA replacement for std::vector<std::shared_ptr<ov_core::Feature>> (feat/Feature.h:39-83) ----
 * Measurements of feature f are meas_off[f] .. meas_off[f+1]-1, grouped by camera in the order the reference's
 * `for (auto const &pair : feat->timestamps)` visits cameras (SURVEY.md App. A.4), time-ascending within a camera.
 * Measurements at non-clone times must already be removed (Feature::clean_old_measurements, UpdaterMSCKF.cpp:79).
 * cam_keys lists, per feature, the camera keys of feat->timestamps in visit order INCLUDING cameras whose list is
 * empty after cleaning (they still contribute calibration columns, update/UpdaterHelper.cpp:204-222); pass NULL to
 * derive the list from the measurements themselves.
 * A feature has at most OVB_MAX_MEAS_PER_FEAT (= OVB_MAX_CAMS * OVB_MAX_CLONES = 384) measurements: one per camera and
 * clone pose. A longer track makes the whole call return OVB_ERR_CAPACITY. Tracks of any length up to the limit may be
 * mixed in one batch; each runs on the per-feature kernel layout it fits. */
typedef struct {
  int n_feats;
  int n_meas;
  const int32_t *meas_off;     /* [n_feats+1] */
  const uint8_t *cam;          /* [n_meas] camera id */
  const uint16_t *clone;       /* [n_meas] clone index into ovb_frame */
  const float *uv;             /* [n_meas][2] raw pixel       Feature::uvs      (f32 in the reference) */
  const float *uvn;            /* [n_meas][2] normalized      Feature::uvs_norm (f32 in the reference) */
  const int32_t *cam_keys_off; /* [n_feats+1] or NULL */
  const uint8_t *cam_keys;     /* or NULL */
} ovb_feat_batch;

/* ---- per-feature results written back to ov_core::Feature by the host shim (core/VioManager.cpp:567-570) ---- */
typedef struct {
  int32_t *status;       /* [n_feats] ovb_feat_status */
  double *p_FinA;        /* [n_feats][3] */
  double *p_FinG;        /* [n_feats][3] */
  int32_t *anchor_cam;   /* [n_feats] Feature::anchor_cam_id */
  int32_t *anchor_clone; /* [n_feats] clone index of Feature::anchor_clone_timestamp */
  double *chi2;          /* [n_feats] (NaN when the feature never reached the gate) */
} ovb_feat_out;

typedef struct {
  int n_feats_in;
  int n_feats_used;   /* accepted by every gate */
  int rows_stacked;   /* ct_meas:  Σ (2M_f-3) over accepted features (UpdaterMSCKF.cpp:254) */
  int cols_stacked;   /* ct_jacob: width of the stacked H (UpdaterMSCKF.cpp:244) */
  int rows_update;    /* rows handed to EKFUpdate after compression */
  int neg_diag_index; /* -1 or first negative diagonal of P */
  float ms_total;     /* device time of the call, CUDA events */
} ovb_stats;

/* ---- lifecycle ---- */
ovb_status ovb_create(const ovb_config *cfg, ovb_ctx **out);
void ovb_destroy(ovb_ctx *ctx);
const char *ovb_last_error(const ovb_ctx *ctx);
int ovb_abi_version(void);

/* ---- covariance residency (replaces direct access to State::_Cov, state/State.h:186) ---- */
/* StateHelper::set_initial_covariance / resync: upload a full N×N P.            state/StateHelper.cpp:199-224 */
ovb_status ovb_cov_set(ovb_ctx *ctx, const double *P, int N);
/* StateHelper::get_full_covariance.                                              state/StateHelper.cpp:256-269 */
ovb_status ovb_cov_get(ovb_ctx *ctx, double *P, int N);
int ovb_cov_dim(const ovb_ctx *ctx);
/* StateHelper::get_marginal_covariance: gather the blocks (off[i],sz[i]).        state/StateHelper.cpp:226-254 */
ovb_status ovb_cov_get_marginal(ovb_ctx *ctx, const int *off, const int *sz, int nvar, double *out);
/* StateHelper::clone (+ the time-offset term of augment_clone when dnc_dt != NULL): append a copy of the
 * `size`-wide variable at old_off to the end of P.                               state/StateHelper.cpp:341-391,604-615 */
ovb_status ovb_cov_clone(ovb_ctx *ctx, int old_off, int size, const double *dnc_dt, int dt_off);
/* StateHelper::marginalize: delete rows/cols [off, off+size).                     state/StateHelper.cpp:271-339 */
ovb_status ovb_cov_marginalize(ovb_ctx *ctx, int off, int size);
/* StateHelper::EKFPropagation: P[new,:] = Phi P[old,:], P[new,new] = Phi P[old,old] Phi' + Q (Q symmetrised from its
 * upper triangle). new block = [new_off, new_off+p); old variables (old_off[i], old_sz[i]) index Phi's columns in order.
 * Phi is p×q row-major, Q is p×p row-major.                                       state/StateHelper.cpp:36-114 */
ovb_status ovb_cov_propagate(ovb_ctx *ctx, int new_off, int p, const int *old_off, const int *old_sz, int nold,
                             const double *Phi, const double *Q);
/* Propagator::propagate_and_clone, covariance side (state/Propagator.cpp:83-137), in one call. For s = 0..steps-1, in this
 * order and with the reference's arithmetic:
 *   Qd_s = sym(G_s diag(qc_s[k/3]) G_s')           (Propagator.cpp:453-464; sym(X) = 0.5 (X + X'))
 *   Phi  = F_s Phi,   Q = sym(F_s Q F_s' + Qd_s)    (Phi = I, Q = 0 before step 0; :83-99)
 * then StateHelper::EKFPropagation of [new_off, new_off+n) from the variables (old_off[i], old_sz[i]) (:130; their sizes
 * add up to n), then StateHelper::augment_clone: clone clone_size rows/cols at clone_off, with the time-offset term when
 * dnc_dt != NULL (:137).
 * F: [steps][n][n], G: [steps][n][12], qc: [steps][4] (sigma^2/dt of n_w, n_a, n_wb, n_ab), row-major. steps = 0 is legal
 * (F, G, qc may then be NULL). Phi_out / Q_out (n*n each) may be NULL.
 * Phi, Q and P are bit-identical to the host loop followed by ovb_cov_propagate and ovb_cov_clone. OVB_ERR_ARG for
 * malformed arguments and OVB_ERR_CAPACITY for n > 64 or a clone beyond max_state, with P and N untouched;
 * OVB_ERR_NEG_DIAG when the propagated diagonal goes negative: P then holds the propagated values and nothing is cloned. */
ovb_status ovb_cov_propagate_imu(ovb_ctx *ctx, int n, int steps, const double *F, const double *G, const double *qc,
                                 int new_off, const int *old_off, const int *old_sz, int nold,
                                 int clone_off, int clone_size, const double *dnc_dt, int dt_off,
                                 double *Phi_out, double *Q_out);

/* StateHelper::initialize + initialize_invertible (state/StateHelper.cpp:393-577): add a NEW `new_size`-wide variable (a SLAM
 * landmark in UpdaterSLAM::delayed_init, update/UpdaterSLAM.cpp:233) at the END of the covariance from the linear system
 *     res = H_R * dx(state variables off/sz) + H_L * dx(new) + n,   n ~ N(0, sigma2 I)      (H_R r x n, H_L r x new_size, row-major)
 * Givens split on H_L, Mahalanobis gate of the nullspace-projected part (threshold chi2_mult * quantile95(r)), covariance
 * augmentation from the invertible part, EKF update with the projected part. *accepted = 0: gate rejected, P unchanged.
 * dx_new[new_size] = H_Linit^-1 res_init (the new variable's own correction); dx[ovb_cov_dim() AFTER the call] is the EKF
 * correction of the projected part (it also moves the new variable through its cross-covariance). */
ovb_status ovb_cov_initialize(ovb_ctx *ctx, const int *off, const int *sz, int nvar, const double *H_R, const double *H_L, const double *res,
                              int r, int new_size, double sigma2, double chi2_mult, int *accepted, double *dx_new, double *dx);

/* ---- the hot path ---- */
/* UpdaterMSCKF::update steps 2-6 in one call (update/UpdaterMSCKF.cpp:98-285). P is updated in place on the device;
 * dx (length N = ovb_cov_dim) is the correction K·res that the host applies with Type::update
 * (state/StateHelper.cpp:185-188).  stats may be NULL. */
ovb_status ovb_msckf_update(ovb_ctx *ctx, const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_opts *opts,
                            ovb_feat_out *out, double *dx, ovb_stats *stats);

/* ---- SLAM landmarks: features that already live in the state (ov_type::Landmark, types/Landmark.h; State::_features_SLAM) ----
 * One entry per feature of the batch handed to ovb_slam_update. Every landmark has its own representation
 * (Landmark::_feat_representation): the feat_rep array of ovb_slam_update_reps, or ovb_opts.feat_rep for all of them. A landmark
 * in ANCHORED_INVERSE_DEPTH_SINGLE is 1 wide (the inverse depth): its column is dz/drho and the two bearing columns of its H_f
 * are nullspace-projected out (update/UpdaterSLAM.cpp:344-353), and it needs at least two measurements (:278-281); the others
 * are 3 wide and keep all their rows. */
typedef struct {
  const int32_t *lm_off;         /* [n_feats] covariance id of the landmark variable (Type::id(); 3 wide, 1 for the SINGLE rep) */
  const double *value;           /* [n_feats][3] Landmark::get_xyz(false): p_FinG (global reps) / p_FinA (anchored reps) */
  const double *value_fej;       /* [n_feats][3] Landmark::get_xyz(true) */
  const int32_t *anchor_cam;     /* [n_feats] Landmark::_anchor_cam_id            (anchored reps; else ignored) */
  const int32_t *anchor_clone;   /* [n_feats] clone index of _anchor_clone_timestamp (anchored reps; else ignored) */
  const double *sigma_pix;       /* [n_feats] or NULL: per-class pixel noise (aruco vs slam options, UpdaterSLAM.cpp:391-393) */
  const double *chi2_multipler;  /* [n_feats] or NULL: per-class gate multiplier (UpdaterSLAM.cpp:407-408) */
} ovb_landmarks;

/* UpdaterSLAM::update steps 4-5 (update/UpdaterSLAM.cpp:310-470): per-feature Jacobians with the landmark's own 3
 * columns appended (H_xf = [H_x, H_f], no nullspace projection), chi² gate on the marginal of (H_x variables + landmark),
 * stacking and ONE EKF update of the whole batch. The reference does not compress this system; the engine whitens the
 * rows by 1/sigma and compresses when rows > columns, which leaves the posterior unchanged.
 * Batch size: a new context takes at most OVB_MAX_VARS state variables (clones + calibration blocks + landmarks) per call
 * and returns OVB_ERR_CAPACITY beyond. After ovb_set_slam_unbounded(ctx, 1) any batch that fits the context's max_feats,
 * max_meas and max_state is one call, whatever its number of landmarks (max_slam_in_update as in the reference, e.g. 100
 * for SURVEY.md config 4). Every gate sees the prior P.
 * A batch wider than 512 columns (frame columns + landmark columns) is cut into column groups, contiguous feature ranges
 * whose frame plus landmark columns fit 512; the groups are applied as sequential EKF updates at the same linearization
 * point, each group's compressed residual corrected by the state change of the groups before it, which equals the single
 * update to rounding. Such a batch is updated in its groups' canonical column order whatever opts->col_order says (the
 * order only changes rounding), and on any EKF failure (not SPD, negative diagonal, non-finite) P keeps its prior and dx
 * is zero.
 * out->status: OVB_FEAT_OK, OVB_FEAT_FEW_MEAS or OVB_FEAT_CHI2; out->chi2 filled; p_FinA/p_FinG/anchor_* are not written.
 * Every landmark of the call is in ovb_opts.feat_rep; ovb_slam_update_reps below takes one representation per landmark. */
ovb_status ovb_slam_update(ovb_ctx *ctx, const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_landmarks *landmarks,
                           const ovb_opts *opts, ovb_feat_out *out, double *dx, ovb_stats *stats);
/* ovb_slam_update with feat_rep[f] (an ovb_feat_rep) the representation of landmark f, as UpdaterSLAM::update reads
 * landmark->_feat_representation per landmark; NULL = ovb_opts.feat_rep for all. Widths, row counts, anchors and the bearing
 * projection follow each landmark. OVB_ERR_ARG with P untouched (message in ovb_last_error) for an entry outside 0..5, an
 * anchored landmark without a valid anchor, or landmark blocks that overlap with their own widths. ovb_opts.feat_rep stays
 * the representation of MSCKF features. */
ovb_status ovb_slam_update_reps(ovb_ctx *ctx, const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_landmarks *landmarks,
                                const int32_t *feat_rep /* [n_feats] ovb_feat_rep or NULL */, const ovb_opts *opts, ovb_feat_out *out,
                                double *dx, ovb_stats *stats);
/* enabled = 1: ovb_slam_update accepts batches of more than OVB_MAX_VARS state variables (see above); 0: the default. */
ovb_status ovb_set_slam_unbounded(ovb_ctx *ctx, int enabled);

/* UpdaterSLAM::delayed_init (update/UpdaterSLAM.cpp:61-251) in ONE call: triangulate + Gauss-Newton every new track (:118-142),
 * then, one feature after the other like the reference (each StateHelper::initialize mutates the covariance AND the state
 * mean that the next feature's Jacobians are evaluated at): full Jacobians (:197-219) -> StateHelper::initialize (Givens
 * split, Mahalanobis gate, covariance augmentation, EKF update; state/StateHelper.cpp:393-577). After every accepted
 * feature `on_init` is called: the host applies Type::update(dx) to its State (dx has the NEW covariance size, the landmark's
 * block at lm_off included), sets the new Landmark to its triangulated value (+) dx_new, and REFRESHES the arrays `frame`
 * points to (clone poses, calibration) — the engine re-reads them for the next feature. Landmark representation: ovb_opts.feat_rep,
 * any of the six. A landmark in ANCHORED_INVERSE_DEPTH_SINGLE is initialised 1 wide: the depth column of its H_f joins the state
 * columns and the two bearing columns are nullspace-projected out of the system first; the callback's lm_size (dx_new's length)
 * is then 1 and dx has N0 + 1 entries (N0 = ovb_cov_dim() before the landmark), else 3 and N0 + 3.
 * sigma_pix / chi2_multipler: per-feature class values (aruco vs slam options, :225-228) or NULL for ovb_opts'.
 * out->status: OVB_FEAT_OK = initialised, a triangulation status, or OVB_FEAT_CHI2 (gate); out->chi2 (when non-NULL): the
 * gate's chi2 of every feature that reached it, accepted or rejected, NaN for the others; lm_off_out[f] = the new landmark's
 * covariance id or -1. */
typedef void (*ovb_init_callback)(void *user, int feat_index, int lm_off, int lm_size, const double *dx_new, const double *dx, int n_dx);
ovb_status ovb_slam_delayed_init(ovb_ctx *ctx, const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_opts *opts, const double *sigma_pix,
                                 const double *chi2_multipler, ovb_init_callback on_init, void *user, ovb_feat_out *out, int32_t *lm_off_out);
/* ovb_slam_delayed_init with feat_rep[f] (an ovb_feat_rep) the representation of feature f, the class representation
 * (feat_rep_aruco or feat_rep_slam) the reference picks by featid; NULL = ovb_opts.feat_rep for all. Each feature's Jacobians,
 * landmark width and SINGLE projection follow its own entry. OVB_ERR_ARG with P untouched for an entry outside 0..5, and for a
 * call that mixes ANCHORED_INVERSE_DEPTH_SINGLE with a 3-wide representation: whether the reference sizes such a landmark by its
 * own class or by feat_rep_slam is not pinned down, so that mix is refused rather than guessed. Mixes among the 3-wide
 * representations are accepted. */
ovb_status ovb_slam_delayed_init_reps(ovb_ctx *ctx, const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_opts *opts,
                                      const int32_t *feat_rep, const double *sigma_pix, const double *chi2_multipler,
                                      ovb_init_callback on_init, void *user, ovb_feat_out *out, int32_t *lm_off_out);

/* The quaternions behind ovb_frame's rotations (JPL, [x y z w], ov_core/src/types/JPLQuat.h). */
typedef struct {
  const double *clone_q; /* [n_clones][4]  PoseJPL::quat() of each clone; clone_R = quat_2_Rot(clone_q) */
  const double *cam_q;   /* [n_cams][4]    q_ItoC; cam_R = quat_2_Rot(cam_q) */
} ovb_frame_quat;

/* ovb_slam_delayed_init_reps without the callback: the engine moves its copy of the frame itself between the features,
 * with the reference's mean update (VioManager::apply_dx): clone and, with do_calib_camera_pose, extrinsic quaternions take
 * q <- quatnorm([dtheta/2; 1]) (x) q (JPLQuat::update) and R = quat_2_Rot(q); positions and, with
 * do_calib_camera_intrinsics, intrinsics add their entries of dx. FEJ arrays are never moved (a NULL one follows the value,
 * as ovb_frame reads it). The arithmetic is include/ovb200_math.hpp's, rounded as the host rounds it, so the features see
 * the bits a host that applies dx and marshals its frame again would pass.
 * The caller replays the records in feature order: for every f with lm_off_out[f] >= 0, the new landmark at its triangulated
 * point (out) moved by dx_new[f] (lm_size entries: 3, or 1 for ANCHORED_INVERSE_DEPTH_SINGLE), then Type::update of every
 * variable, the new landmark included, with row f of dx (lm_off_out[f] + lm_size entries). P, N, every status and chi2,
 * lm_off_out, dx_new and dx are bit-identical to ovb_slam_delayed_init_reps with a callback that does that and marshals the
 * frame again. Rows of features that are not initialised are not written.
 * Refusals (OVB_ERR_ARG or OVB_ERR_CAPACITY) are those of ovb_slam_delayed_init_reps, plus a NULL quat, dx_new or dx and
 * an ld_dx below N + the summed landmark widths of the triangulated features. The call can only launch every feature's
 * work up front when the covariance has room for every triangulated feature: N + that sum above max_state is
 * OVB_ERR_CAPACITY. On every error P and N are left as they were.
 * At most two stream synchronisations whatever the number of features: the triangulation's read-back (which feature is initialised
 * where decides the launches) and the final one of every record. */
ovb_status ovb_slam_delayed_init_batch(ovb_ctx *ctx, const ovb_frame *frame, const ovb_frame_quat *quat, const ovb_feat_batch *feats,
                                       const ovb_opts *opts, const int32_t *feat_rep, const double *sigma_pix, const double *chi2_multipler,
                                       ovb_feat_out *out, int32_t *lm_off_out, double *dx_new /* [n_feats][3] */,
                                       double *dx /* [n_feats][ld_dx] */, int ld_dx);

/* UpdaterSLAM::perform_anchor_change (update/UpdaterSLAM.cpp:506-647), host math only (no context, no GPU work): re-express an
 * anchored landmark (ovb_opts.feat_rep = one of the ANCHORED_* representations) in a new anchor camera/clone and return
 *   new_value / new_value_fej [3]  the landmark's xyz in the new anchor frame (Landmark::set_from_xyz),
 *   order_off/order_sz[*n_order]   phi_order_OLD: old anchor clone [, its extrinsics], new anchor clone [, its extrinsics], landmark
 *   Phi [phisize x *n_cols]        row-major, phisize = 3 (1 for ANCHORED_INVERSE_DEPTH_SINGLE); capacity 3 x 27 doubles.
 * The covariance step is then  ovb_cov_propagate(ctx, lm_off, phisize, order_off, order_sz, *n_order, Phi, Q = 0). */
ovb_status ovb_slam_anchor_change(const ovb_frame *frame, const ovb_opts *opts, int lm_off, const double *value, const double *value_fej,
                                  int old_cam, int old_clone, int new_cam, int new_clone, double *new_value, double *new_value_fej,
                                  double *Phi, int32_t *order_off, int32_t *order_sz, int32_t *n_order, int32_t *n_cols);

/* The landmarks ovb_marginalize_window re-anchors (UpdaterSLAM::change_anchors), one entry per landmark, in the order the
 * anchor changes are applied. */
typedef struct {
  int n;                             /* landmarks to re-anchor */
  const int32_t *lm_off;             /* [n] covariance id (3 wide; 1 for ANCHORED_INVERSE_DEPTH_SINGLE) */
  const int32_t *feat_rep;           /* [n] an anchored ovb_feat_rep */
  const double *value, *value_fej;   /* [n][3] Landmark::get_xyz(false / true) */
  const int32_t *old_cam, *old_clone, *new_cam, *new_clone; /* [n] camera ids and clone indices into the frame */
  double *new_value, *new_value_fej; /* [n][3] out: Landmark::set_from_xyz in the new anchor */
} ovb_anchor_changes;

/* The covariance side of the end of VioManager::do_feature_propagate_update in one call: StateHelper::marginalize_slam,
 * UpdaterSLAM::change_anchors and StateHelper::marginalize_old_clone (VioManager::do_feature_propagate_update). The n_marg ranges
 * (marg_off[i], marg_sz[i]) are the lost landmarks and the oldest clone; anchors (or NULL) the landmarks to re-anchor, with
 * ovb_opts' do_fej and do_calib_camera_pose. All offsets refer to the covariance before the call; afterwards N shrinks by
 * the ranges' total and the host shifts its Type::id()s exactly as it does after each ovb_cov_marginalize.
 * Result: P and N are those of this sequence of existing calls: every anchor change in the order given
 * (ovb_slam_anchor_change, then ovb_cov_propagate with Q = 0), then ovb_cov_marginalize of every range, highest offset first.
 * P, new_value and new_value_fej are bit-identical to that sequence for every anchored representation. The anchor-change
 * math of ANCHORED_3D, ANCHORED_MSCKF_INVERSE_DEPTH and ANCHORED_INVERSE_DEPTH_SINGLE runs on the device from the same source
 * as ovb_slam_anchor_change, built without FMA contraction for both sides. An ANCHORED_FULL_INVERSE_DEPTH landmark's Phi
 * goes through acos, atan2, sin and cos, whose CUDA and C-library results may differ in the last ulp, so the call computes
 * that Phi with ovb_slam_anchor_change on the host and uploads it with the other inputs.
 * Whether the lost landmarks are marginalized before or after the anchor changes (the reference calls marginalize_slam
 * and change_anchors in either order, both before marginalize_old_clone) does not change a bit when P is symmetric, as the
 * filter's covariance is: marginalization only copies entries (some read from the mirrored position, which holds the same
 * value), an anchor change writes only the rows and columns of its own landmark and reads only those and the ones of its
 * anchor clones and extrinsics, none of which a marginalization removes (a landmark may not be both re-anchored and
 * marginalized; the old anchor clone is read before marginalize_old_clone drops it, in both orders).
 * Everything is checked before any work is enqueued; on every error P, N and the outputs are left untouched:
 *   OVB_ERR_ARG       ranges that overlap or fall outside N (landmarks and marginalized ranges alike), a landmark both
 *                     re-anchored and marginalized, a global representation, an anchor camera or clone outside the frame,
 *                     a new anchor clone or an anchor's extrinsics that is being marginalized, an anchor variable that
 *                     overlaps a re-anchored landmark; and a singular H_f in the new anchor (ovb_slam_anchor_change
 *                     reports the same; for the device-computed representations it is found on the device, after the
 *                     upload, and the kernels that would read the landmark's Phi do nothing);
 *   OVB_ERR_NEG_DIAG  a propagated landmark diagonal is negative. ovb_cov_propagate writes P before it reports this; this call
 *                     does not;
 *   OVB_ERR_CAPACITY  the call's inputs (frame, landmark records, index maps, Phi slots) exceed the staging the context
 *                     reserved at ovb_create (max_rows / max_meas and max_state size it);
 *   OVB_ERR_CUDA      a CUDA runtime error (ovb_last_error).
 * One H2D copy (frame and anchor list), one D2H copy (new values and status) and one stream synchronisation. */
ovb_status ovb_marginalize_window(ovb_ctx *ctx, const ovb_frame *frame, const ovb_opts *opts, const int32_t *marg_off, const int32_t *marg_sz,
                                  int n_marg, const ovb_anchor_changes *anchors);

/* StateHelper::EKFUpdate with R = sigma2·I (UpdaterMSCKF.cpp:282) or R = diag(Rdiag) (UpdaterSLAM.cpp:444).
 * H is r×n row-major, n = Σ sz.                                                   state/StateHelper.cpp:116-197 */
ovb_status ovb_ekf_update(ovb_ctx *ctx, const int *off, const int *sz, int nvar, const double *H, int r, const double *res,
                          double sigma2, const double *Rdiag, double *dx);

/* ---- staged entry points (parity tests, configs 3 and 5) ---- */
/* FeatureInitializer::single_triangulation(_1d) + single_gaussnewton only.        feat/FeatureInitializer.cpp:30-375 */
ovb_status ovb_triangulate(ovb_ctx *ctx, const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_opts *opts,
                           ovb_feat_out *out);

/* UpdaterHelper::get_feature_jacobian_full + nullspace_project_inplace + the chi² gate for features whose
 * p_FinG (and anchor) are GIVEN in `out` (status must be OVB_FEAT_OK on entry for features to process).
 * Dense dump in the canonical column layout: column j of the dump is covariance column col_index[j].
 *   stage 0: pre-nullspace.  rows 2M_f per feature; Hf_out [rows][3], Hx_out [rows][ncols], res_out [rows]
 *   stage 1: post-nullspace. rows 2M_f-3 per feature (gated features are zero rows); Hf_out unused.
 * row_off_out[F+1] gives each feature's first row. ncols_out/col_index_out describe the layout.
 *                                                                                update/UpdaterHelper.cpp:192-454 */
ovb_status ovb_feature_jacobians(ovb_ctx *ctx, const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_opts *opts,
                                 ovb_feat_out *out, int stage, double *Hf_out, double *Hx_out, double *res_out,
                                 int32_t *row_off_out, int32_t *ncols_out, int32_t *col_index_out, int ld_out);

/* UpdaterHelper::measurement_compress_inplace as a blocked Householder TSQR: H is m×n row-major (m>n),
 * R_out n×n row-major upper triangular with diag ≥ 0 (the Givens convention of the reference), z_out = Q1' res.
 *                                                                                update/UpdaterHelper.cpp:456-487 */
ovb_status ovb_compress(ovb_ctx *ctx, const double *H, int m, int n, const double *res, double *R_out, double *z_out);

/* Same contract through the normal equations (OVB_COMPRESS_NORMAL_EQUATIONS): R upper triangular with diag >= 0,
 * rows whose pivot is at round-off level are zero. */
ovb_status ovb_compress_gram(ovb_ctx *ctx, const double *H, int m, int n, const double *res, double *R_out, double *z_out);

/* Same contract through the shifted CholeskyQR2 (OVB_COMPRESS_CHOLQR2); n <= 512, else OVB_ERR_CAPACITY. */
ovb_status ovb_compress_cholqr2(ovb_ctx *ctx, const double *H, int m, int n, const double *res, double *R_out, double *z_out);

/* chi² 0.95 quantile table used by the gate (boost::math::quantile in the reference, UpdaterMSCKF.cpp:52-55). */
double ovb_chi2_quantile95(int dof);

/* Device time (ms) of the stages of the last ovb_msckf_update:
 * [0] triangulate+GN  [1] jacobian+nullspace+gate  [2] column map  [3] TSQR  [4] EKF update  [5] total */
ovb_status ovb_last_stage_ms(const ovb_ctx *ctx, float ms[6]);

/* ---- multi-GPU: features sharded across ranks, one all-gather of the compressed [R | z] blocks (SURVEY.md §8e) ----
 * The reference is single-process; these replace nothing in it. One context per rank/GPU, each holding a replica of P.
 *  ovb_set_stream           adopt an external CUDA stream (e.g. the stream NCCL collectives are issued on).
 *  ovb_msckf_shard_compress steps 2-5 of UpdaterMSCKF::update on THIS rank's feature shard; the shard's compressed system
 *                           [R_g | z_g] (n_cols x (n_cols+1), row-major, leading dimension *ld) is written to the DEVICE
 *                           buffer R_dev. Asynchronous on the context stream. Column order is canonical.
 *  ovb_msckf_shard_finish   stacked_dev = the n_blocks all-gathered blocks, stacked by rank (DEVICE pointer, overwritten):
 *                           compress the stack, EKFUpdate on this rank's P, return dx and the shard's per-feature results. */
ovb_status ovb_set_stream(ovb_ctx *ctx, void *cuda_stream); /* cuda_stream must be an explicit stream (not the default stream 0) */
/* Contiguous feature ranges with (nearly) equal stacked-row counts: rank r works on features [bounds[r], bounds[r+1]). */
ovb_status ovb_shard_partition(const int32_t *meas_off, int n_feats, int world, int32_t *bounds /* [world+1] */);
/* ovb_msckf_shard_compress on features [f0, f1) of a full batch (no host-side copy of the subset by the caller). */
ovb_status ovb_msckf_shard_compress_range(ovb_ctx *ctx, const ovb_frame *frame, const ovb_feat_batch *feats, int f0, int f1,
                                          const ovb_opts *opts, double *R_dev, int R_cap_doubles, int *n_cols, int *ld);
ovb_status ovb_msckf_shard_compress(ovb_ctx *ctx, const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_opts *opts, double *R_dev,
                                    int R_cap_doubles, int *n_cols, int *ld);
ovb_status ovb_msckf_shard_finish(ovb_ctx *ctx, double *stacked_dev, int n_blocks, ovb_feat_out *out, double *dx, ovb_stats *stats);

/* ---- measurement support: re-run the LAST ovb_msckf_update on its device-resident inputs ----
 * ovb_set_replay(ctx,1) makes ovb_msckf_update keep a copy of the prior P; ovb_msckf_replay then restores that prior and
 * re-enqueues the identical device pipeline `steps` times (optionally flushing L2 with a 256 MiB memset between steps),
 * timing each step with CUDA events on the context stream. ms_per_step[steps]; stage_ms_sum[5] = summed stage times
 * {triangulate, feature systems, column map, compression, EKF update}. This is bench.py's kernel-only `value` leg. */
/* out[0] kernels launched by the last call that launches any (ovb_msckf_shard_finish adds to its
 * ovb_msckf_shard_compress), counted at the launch, out[1] of which TSQR level kernels,
 * out[2]/out[3] bytes copied host->device / device->host by the last ovb_msckf_update. */
ovb_status ovb_last_counters(const ovb_ctx *ctx, int64_t out[4]);
/* The last ovb_slam_delayed_init[_reps|_batch] call: out[0] features that reached StateHelper::initialize (triangulated), out[1]
 * stream synchronisations (one for the triangulation, then one per such feature, or one in all for _batch), out[2]/out[3]
 * bytes copied host->device / device->host. */
ovb_status ovb_last_init_counters(const ovb_ctx *ctx, int64_t out[4]);
/* Host wall clock (microseconds) of the last ovb_msckf_update: [0] marshalling into the pinned arena + H2D enqueue,
 * [1] kernel and D2H enqueue, [2] wait for the stream, [3] unpacking the results. */
ovb_status ovb_last_host_us(const ovb_ctx *ctx, double out[4]);
/* Per-kernel timing (measurement support): ovb_set_profile(ctx,1) brackets every kernel launch with CUDA events
 * (programmatic dependent launch is off meanwhile); ovb_profile_read returns the kernels of the last call (as counted by
 * ovb_last_counters) in launch order: NUL-separated mangled names and durations in microseconds, the first cap of them;
 * *n = the number of kernels of that call, which may exceed cap. */
ovb_status ovb_set_profile(ovb_ctx *ctx, int enabled);
ovb_status ovb_profile_read(ovb_ctx *ctx, char *names, int name_cap, float *us, int cap, int *n);
ovb_status ovb_set_replay(ovb_ctx *ctx, int enabled);
ovb_status ovb_msckf_replay(ovb_ctx *ctx, int steps, int flush_l2, float *ms_per_step, float stage_ms_sum[5]);

#ifdef __cplusplus
}
#endif
#endif /* OVB200_H */
