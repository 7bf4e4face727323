// ovb_api.cu — the C ABI of include/ovb200.h: context, host-side marshalling into one pinned arena, stream orchestration.
// No arithmetic of the path happens on the host: it packs the inputs, launches the kernels of k_*.cu and copies results back.
#include "ovb_internal.cuh"
#include <chrono>
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

static const double g_chi2_table[OVB_CHI2_TABLE_LEN] = {
#include "chi2_table.inc"
};

unsigned char *ovb_feat_order_ptr(ovb_ctx *ctx) { return ctx->d_feat_order; }

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

int ovb_prof_slot(ovb_ctx *ctx, const void *kern) {
  if (ctx->prof_n == ctx->prof_cap) { // grow the pool: twice the pairs, created one pair at a time
    const int cap = ctx->prof_cap ? 2 * ctx->prof_cap : 128;
    cudaEvent_t *ev = (cudaEvent_t *)realloc(ctx->prof_ev, sizeof(cudaEvent_t) * 2 * cap);
    if (ev)
      ctx->prof_ev = ev;
    const void **fn = (const void **)realloc(ctx->prof_fn, sizeof(const void *) * cap);
    if (fn)
      ctx->prof_fn = fn;
    for (; ev && fn && ctx->prof_cap < cap; ctx->prof_cap++) {
      cudaEvent_t *pair = ctx->prof_ev + 2 * ctx->prof_cap;
      pair[0] = pair[1] = nullptr;
      if (cudaEventCreate(&pair[0]) != cudaSuccess || cudaEventCreate(&pair[1]) != cudaSuccess) {
        cudaGetLastError();
        if (pair[0]) // the first of the pair was created
          cudaEventDestroy(pair[0]);
        break;
      }
    }
    if (ctx->prof_n == ctx->prof_cap)
      return -1; // out of memory: this launch is not profiled
  }
  ctx->prof_fn[ctx->prof_n] = kern;
  return ctx->prof_n++;
}

extern "C" {

static ovb_status ensure_stage(ovb_ctx *ctx, size_t doubles);

// Every entry point that launches kernels starts here, so that ovb_last_counters and ovb_profile_read describe its
// launches alone (ovb_msckf_shard_finish continues the count of its ovb_msckf_shard_compress).
static void begin_launches(ovb_ctx *ctx) {
  ctx->n_launch = 0;
  ctx->n_launch_tsqr_level = 0;
  ctx->prof_n = 0;
}

int ovb_abi_version(void) { return OVB_ABI_VERSION; }

double ovb_chi2_quantile95(int dof) {
  if (dof < 1)
    return 0.0;
  if (dof >= OVB_CHI2_TABLE_LEN)
    dof = OVB_CHI2_TABLE_LEN - 1;
  return g_chi2_table[dof];
}

void ovb_opts_default(ovb_opts *o) {
  memset(o, 0, sizeof(*o));
  o->triangulate_1d = 0;
  o->refine_features = 1;
  o->max_runs = 5;
  o->init_lamda = 1e-3;
  o->max_lamda = 1e10;
  o->min_dx = 1e-6;
  o->min_dcost = 1e-6;
  o->lam_mult = 10;
  o->min_dist = 0.10;
  o->max_dist = 60;
  o->max_baseline = 40;
  o->max_cond_number = 10000;
  o->sigma_pix = 1;
  o->chi2_multipler = 5;
  o->do_fej = 1;
  o->feat_rep = OVB_REP_GLOBAL_3D;
  o->do_calib_camera_pose = 0;
  o->do_calib_camera_intrinsics = 0;
  o->col_order = OVB_COLS_CANONICAL;
  o->compress = OVB_COMPRESS_CHOLQR2;
}

const char *ovb_last_error(const ovb_ctx *ctx) { return ctx ? ctx->err : "null context"; }

ovb_status ovb_create(const ovb_config *cfg, ovb_ctx **out) {
  if (!cfg || !out)
    return OVB_ERR_ARG;
  *out = nullptr;
  ovb_ctx *ctx = new (std::nothrow) ovb_ctx();
  if (!ctx)
    return OVB_ERR_CAPACITY;
  memset(ctx, 0, sizeof(*ctx));
  ctx->cfg = *cfg;
  if (ctx->cfg.max_state < 32)
    ctx->cfg.max_state = 32;
  if (ctx->cfg.max_feats < 1)
    ctx->cfg.max_feats = 1;
  if (ctx->cfg.max_meas < 2)
    ctx->cfg.max_meas = 2;
  ctx->device = cfg->device;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || cfg->device >= ndev) {
    delete ctx;
    return OVB_ERR_CUDA; // no CUDA device: there is no CPU fallback
  }
#define CK(call)                                                                                                      \
  do {                                                                                                                \
    cudaError_t e_ = (call);                                                                                          \
    if (e_ != cudaSuccess) {                                                                                          \
      fprintf(stderr, "ovb_create: %s failed: %s\n", #call, cudaGetErrorString(e_));                                  \
      ovb_destroy(ctx);                                                                                               \
      return OVB_ERR_CUDA;                                                                                            \
    }                                                                                                                 \
  } while (0)
  CK(cudaSetDevice(ctx->device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, ctx->device));
  ctx->sm_count = prop.multiProcessorCount;
  {
    const char *e = getenv("OVB_TSQR_CLUSTER");
    ctx->tsqr_cluster = e ? atoi(e) : 1;
    const char *e2 = getenv("OVB_TSQR_PDL");
    ctx->pdl = e2 ? atoi(e2) : 1;
    const char *e3 = getenv("OVB_FEAT_CLASSES");
    ctx->feat_classes = e3 ? atoi(e3) : 1;
    const char *e4 = getenv("OVB_EKF_CHOL_DMMA");
    ctx->ekf_chol_dmma = e4 ? atoi(e4) : 1;
    const char *e5 = getenv("OVB_GRAM_CLUSTER");
    ctx->gram_cluster = e5 ? atoi(e5) : 0; // measured slower on H100 (config 2: compress 238 vs 190 us), profiles/README.md
  }
  CK(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
  ctx->own_stream = 1;
  CK(cudaStreamCreateWithFlags(&ctx->side_stream, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&ctx->side_stream2, cudaStreamNonBlocking));
  CK(cudaEventCreateWithFlags(&ctx->ev_join2, cudaEventDisableTiming));
  CK(cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
  CK(cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming));
  for (int i = 0; i < 8; i++)
    CK(cudaEventCreate(&ctx->ev[i]));
  const int ms = ctx->cfg.max_state;
  ctx->ldP = ms;
  ctx->N = 0;
  ctx->cur = 0;
  CK(cudaMalloc(&ctx->P[0], sizeof(double) * (size_t)ms * ms));
  CK(cudaMalloc(&ctx->P[1], sizeof(double) * (size_t)ms * ms));
  CK(cudaMemset(ctx->P[0], 0, sizeof(double) * (size_t)ms * ms));
  CK(cudaMemset(ctx->P[1], 0, sizeof(double) * (size_t)ms * ms));
  // input arena
  ctx->off_opts = align_up(sizeof(DevFrame), 256);
  ctx->off_feat = ctx->off_opts + align_up(sizeof(DevOpts), 256);
  ctx->off_blob = ctx->off_feat + align_up(sizeof(DevFeat) * (size_t)ctx->cfg.max_feats, 256);
  ctx->blob_cap = align_up((size_t)ctx->cfg.max_meas * (1 + 2 + 8 + 8) + (size_t)ctx->cfg.max_feats * OVB_MAX_CAMS + 64, 256);
  ctx->arena_bytes = ctx->off_blob + ctx->blob_cap;
  CK(cudaMalloc(&ctx->d_arena, ctx->arena_bytes));
  CK(cudaMallocHost(&ctx->h_arena, ctx->arena_bytes));
  ctx->d_frame = (DevFrame *)ctx->d_arena;
  ctx->d_opts = (DevOpts *)(ctx->d_arena + ctx->off_opts);
  ctx->d_feat = (DevFeat *)(ctx->d_arena + ctx->off_feat);
  ctx->d_blob = ctx->d_arena + ctx->off_blob;
  ctx->h_frame = (DevFrame *)ctx->h_arena;
  ctx->h_opts = (DevOpts *)(ctx->h_arena + ctx->off_opts);
  ctx->h_feat = (DevFeat *)(ctx->h_arena + ctx->off_feat);
  ctx->h_blob = ctx->h_arena + ctx->off_blob;
  CK(cudaMalloc(&ctx->d_cc, sizeof(DevCamPoses)));
  CK(cudaMalloc(&ctx->d_feat_order, (size_t)ctx->cfg.max_feats * (OVB_MAX_VARS + 1)));
  // update info + dx live in ONE device block and ONE pinned host block: a single D2H copy returns both
  ctx->info_bytes = align_up(sizeof(DevUpdateInfo), 256);
  CK(cudaMalloc(&ctx->d_info, ctx->info_bytes + sizeof(double) * (size_t)ms));
  ctx->d_dx = (double *)((char *)ctx->d_info + ctx->info_bytes);
  CK(cudaMallocHost(&ctx->h_info, ctx->info_bytes + sizeof(double) * (size_t)ms));
  ctx->h_dx = (double *)((char *)ctx->h_info + ctx->info_bytes);
  CK(cudaMalloc(&ctx->d_chi2_table, sizeof(g_chi2_table)));
  CK(cudaMemcpy(ctx->d_chi2_table, g_chi2_table, sizeof(g_chi2_table), cudaMemcpyHostToDevice));
  // stacked staging matrix
  ctx->max_rows = ctx->cfg.max_rows > 0 ? ctx->cfg.max_rows : 2 * ctx->cfg.max_meas;
  if (ctx->max_rows < 2 * ctx->cfg.max_meas)
    ctx->max_rows = 2 * ctx->cfg.max_meas;
  int ldcap = std::min(OVB_MAX_COLS, ms) + 8;
  ctx->Hs_cap = (size_t)ctx->max_rows * ldcap;
  CK(cudaMalloc(&ctx->d_Hs, sizeof(double) * ctx->Hs_cap));
  ctx->h_stage = nullptr; // pinned dense staging is grown on demand (ensure_stage)
  ctx->stage_cap = 0;
  ctx->W_cap = ((size_t)ctx->max_rows / OVB_CR + 2 + (size_t)ctx->sm_count) * OVB_NB * OVB_NB + 4096; // level-0 chunks can be as short as max_rows / sm_count
  CK(cudaMalloc(&ctx->d_W[0], sizeof(double) * ctx->W_cap));
  CK(cudaMalloc(&ctx->d_W[1], sizeof(double) * ctx->W_cap));
  size_t rsz = (size_t)(ms + 8) * (ms + 8);
  CK(cudaMalloc(&ctx->d_R, sizeof(double) * rsz));
  CK(cudaMalloc(&ctx->d_R2, sizeof(double) * rsz));
  CK(cudaMalloc(&ctx->d_M, sizeof(double) * (size_t)ms * ms));
  CK(cudaMalloc(&ctx->d_S, sizeof(double) * (size_t)(ms + 1) * ms));
  CK(cudaMalloc(&ctx->d_Y, sizeof(double) * (size_t)ms * ms));
  CK(cudaMalloc(&ctx->d_w, sizeof(double) * (size_t)ms * 4));
  CK(cudaMalloc(&ctx->d_pub, sizeof(unsigned long long)));
  CK(cudaMemset(ctx->d_pub, 0, sizeof(unsigned long long)));
  ctx->scratch_per_cta = (size_t)(2 * OVB_BIG_MAX_MEAS + 1) * (2 * OVB_BIG_MAX_MEAS + 1);
  ctx->scratch_ctas = 2 * ctx->sm_count;
  CK(cudaMalloc(&ctx->d_scratch, sizeof(double) * ctx->scratch_per_cta * ctx->scratch_ctas));
  ctx->dump_cap = 0;
  ctx->d_dump = nullptr; // allocated on first use by ovb_feature_jacobians(stage 0)
  // ovb_cov_propagate_imu staging: OVB_PROP_STEPS_RESERVE IMU steps of the 39-wide IMU block (400 Hz IMU, 10 Hz camera: ~41)
  ctx->imu_cap = (size_t)OVB_PROP_STEPS_RESERVE * (39 * 39 + 12 * 39 + 4) + 64 + 39;
  CK(cudaMalloc(&ctx->d_imu, sizeof(double) * ctx->imu_cap));
  CK(cudaMallocHost(&ctx->h_imu, sizeof(double) * ctx->imu_cap));
#undef CK
  *out = ctx;
  return OVB_OK;
}

void ovb_destroy(ovb_ctx *ctx) {
  if (!ctx)
    return;
  cudaSetDevice(ctx->device);
  if (ctx->stream)
    cudaStreamSynchronize(ctx->stream);
  for (int i = 0; i < 2 * ctx->prof_cap; i++)
    cudaEventDestroy(ctx->prof_ev[i]);
  free(ctx->prof_ev);
  free(ctx->prof_fn);
  void *dev[] = {ctx->P[0],   ctx->P[1], ctx->d_arena, ctx->d_cc, ctx->d_feat_order, ctx->d_info, ctx->d_chi2_table, ctx->d_Hs, ctx->d_W[0],
                 ctx->d_W[1], ctx->d_R,  ctx->d_R2,    ctx->d_M,  ctx->d_S,          ctx->d_Y,    ctx->d_w,          ctx->d_scratch,
                 ctx->d_long, ctx->d_dump, ctx->P_snap, ctx->d_flush, ctx->d_Gpart, ctx->d_G, ctx->d_cqw, ctx->d_grp, ctx->d_grp_acc, ctx->d_init, ctx->d_imu, ctx->d_pub, ctx->d_ib};
  for (void *p : dev)
    if (p)
      cudaFree(p);
  void *host[] = {ctx->h_arena, ctx->h_info, ctx->h_stage, ctx->h_grp, ctx->h_init, ctx->h_imu, ctx->h_ib};
  for (void *p : host)
    if (p)
      cudaFreeHost(p);
  for (int i = 0; i < 8; i++)
    if (ctx->ev[i])
      cudaEventDestroy(ctx->ev[i]);
  if (ctx->ev_fork)
    cudaEventDestroy(ctx->ev_fork);
  if (ctx->ev_join)
    cudaEventDestroy(ctx->ev_join);
  if (ctx->ev_join2)
    cudaEventDestroy(ctx->ev_join2);
  if (ctx->side_stream2)
    cudaStreamDestroy(ctx->side_stream2);
  if (ctx->side_stream)
    cudaStreamDestroy(ctx->side_stream);
  if (ctx->stream && ctx->own_stream)
    cudaStreamDestroy(ctx->stream);
  delete ctx;
}

// ------------------------------------------------------------------------------------------------ covariance residency
int ovb_cov_dim(const ovb_ctx *ctx) { return ctx ? ctx->N : 0; }

ovb_status ovb_cov_set(ovb_ctx *ctx, const double *P, int N) {
  if (!ctx || !P || N < 1)
    return OVB_ERR_ARG;
  if (N > ctx->cfg.max_state) {
    snprintf(ctx->err, sizeof(ctx->err), "ovb_cov_set: N=%d exceeds max_state=%d", N, ctx->cfg.max_state);
    return OVB_ERR_CAPACITY;
  }
  OVB_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
  OVB_CUDA_CHECK(ctx, cudaMemcpy2DAsync(ctx->P[ctx->cur], sizeof(double) * ctx->ldP, P, sizeof(double) * N, sizeof(double) * N, N,
                                        cudaMemcpyHostToDevice, ctx->stream));
  OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  ctx->N = N;
  return OVB_OK;
}

ovb_status ovb_cov_get(ovb_ctx *ctx, double *P, int N) {
  if (!ctx || !P || N != ctx->N)
    return OVB_ERR_ARG;
  OVB_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
  OVB_CUDA_CHECK(ctx, cudaMemcpy2DAsync(P, sizeof(double) * N, ctx->P[ctx->cur], sizeof(double) * ctx->ldP, sizeof(double) * N, N,
                                        cudaMemcpyDeviceToHost, ctx->stream));
  OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  return OVB_OK;
}

ovb_status ovb_cov_get_marginal(ovb_ctx *ctx, const int *off, const int *sz, int nvar, double *out) {
  if (!ctx || !off || !sz || !out || nvar < 1)
    return OVB_ERR_ARG;
  int n = 0;
  for (int i = 0; i < nvar; i++) {
    if (off[i] < 0 || sz[i] < 1 || off[i] + sz[i] > ctx->N)
      return OVB_ERR_ARG;
    n += sz[i];
  }
  OVB_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
  // block copies (small): one strided copy per (i,k) block
  int ii = 0;
  for (int i = 0; i < nvar; i++) {
    int kk = 0;
    for (int k = 0; k < nvar; k++) {
      OVB_CUDA_CHECK(ctx, cudaMemcpy2DAsync(out + (size_t)ii * n + kk, sizeof(double) * n,
                                            ctx->P[ctx->cur] + (size_t)off[i] * ctx->ldP + off[k], sizeof(double) * ctx->ldP,
                                            sizeof(double) * sz[k], sz[i], cudaMemcpyDeviceToHost, ctx->stream));
      kk += sz[k];
    }
    ii += sz[i];
  }
  OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  return OVB_OK;
}

ovb_status ovb_cov_clone(ovb_ctx *ctx, int old_off, int size, const double *dnc_dt, int dt_off) {
  if (!ctx || size < 1 || old_off < 0 || old_off + size > ctx->N)
    return OVB_ERR_ARG;
  if (ctx->N + size > ctx->cfg.max_state) {
    snprintf(ctx->err, sizeof(ctx->err), "ovb_cov_clone: N+size=%d exceeds max_state=%d", ctx->N + size, ctx->cfg.max_state);
    return OVB_ERR_CAPACITY;
  }
  if (dnc_dt && (dt_off < 0 || dt_off >= ctx->N || size > 64))
    return OVB_ERR_ARG;
  OVB_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
  begin_launches(ctx);
  const double *dnc_dev = nullptr;
  if (dnc_dt) {
    memcpy(ctx->h_dx, dnc_dt, sizeof(double) * size);
    OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->d_w, ctx->h_dx, sizeof(double) * size, cudaMemcpyHostToDevice, ctx->stream));
    dnc_dev = ctx->d_w;
  }
  launch_cov_clone(ctx, old_off, size, dnc_dev, dt_off);
  OVB_CUDA_CHECK(ctx, cudaGetLastError());
  OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  ctx->N += size;
  return OVB_OK;
}

ovb_status ovb_cov_marginalize(ovb_ctx *ctx, int off, int size) {
  if (!ctx || size < 1 || off < 0 || off + size > ctx->N)
    return OVB_ERR_ARG;
  OVB_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
  begin_launches(ctx);
  launch_cov_marginalize(ctx, off, size);
  OVB_CUDA_CHECK(ctx, cudaGetLastError());
  OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  ctx->cur ^= 1;
  ctx->N -= size;
  return OVB_OK;
}

ovb_status ovb_marginalize_window(ovb_ctx *ctx, const ovb_frame *fr, const ovb_opts *op, const int32_t *marg_off, const int32_t *marg_sz, int n_marg,
                                  const ovb_anchor_changes *an) {
  if (!ctx || n_marg < 0 || (n_marg > 0 && (!marg_off || !marg_sz)) || (an && an->n < 0))
    return OVB_ERR_ARG;
  const int n = an ? an->n : 0, N = ctx->N;
  auto fail = [&](const char *msg, int i) {
    snprintf(ctx->err, sizeof(ctx->err), "ovb_marginalize_window: %s (entry %d)", msg, i);
    return OVB_ERR_ARG;
  };
  if (n > 0 && (!fr || !op || !an->lm_off || !an->feat_rep || !an->value || !an->value_fej || !an->old_cam || !an->old_clone || !an->new_cam ||
                !an->new_clone || !an->new_value || !an->new_value_fej))
    return OVB_ERR_ARG;
  // every range the call touches: the marginalized ones (kind 0) and the re-anchored landmarks (kind 1, entry l)
  struct Range {
    int off, sz, kind, entry;
  };
  std::vector<Range> rng;
  int removed = 0;
  for (int i = 0; i < n_marg; i++) {
    if (marg_off[i] < 0 || marg_sz[i] < 1 || marg_off[i] + marg_sz[i] > N)
      return fail("marginalized range outside the covariance", i);
    rng.push_back({marg_off[i], marg_sz[i], 0, i});
    removed += marg_sz[i];
  }
  const bool ext = n > 0 && op->do_calib_camera_pose != 0;
  if (n > 0 && (fr->n_clones < 1 || fr->n_clones > OVB_MAX_CLONES || fr->n_cams < 1 || fr->n_cams > OVB_MAX_CAMS || !fr->clone_R || !fr->clone_p ||
                !fr->clone_off || !fr->cam_R || !fr->cam_p || (ext && !fr->cam_ext_off)))
    return fail("frame without the arrays the anchor changes read", 0);
  int K = 0;
  for (int l = 0; l < n; l++) {
    const int rep = an->feat_rep[l];
    if (rep < OVB_REP_ANCHORED_3D || rep > OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE) // global representations have no anchor
      return fail("representation is not an anchored one", l);
    const int oc = an->old_cam[l], ocl = an->old_clone[l], nc = an->new_cam[l], ncl = an->new_clone[l];
    if (oc < 0 || oc >= fr->n_cams || nc < 0 || nc >= fr->n_cams || ocl < 0 || ocl >= fr->n_clones || ncl < 0 || ncl >= fr->n_clones)
      return fail("anchor camera or clone outside the frame", l);
    if (ext && (fr->cam_ext_off[oc] < 0 || fr->cam_ext_off[nc] < 0))
      return fail("do_calib_camera_pose set but the anchor camera has no extrinsics", l);
    const int p = rep == OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE ? 1 : 3;
    if (an->lm_off[l] < 0 || an->lm_off[l] + p > N)
      return fail("landmark outside the covariance", l);
    rng.push_back({an->lm_off[l], p, 1, l});
    K += p;
  }
  std::sort(rng.begin(), rng.end(), [](const Range &a, const Range &b) { return a.off < b.off; });
  for (size_t s = 1; s < rng.size(); s++)
    if (rng[s].off < rng[s - 1].off + rng[s - 1].sz)
      return fail("overlapping ranges (a landmark re-anchored and marginalized, or listed twice)", rng[s].entry);
  // the anchor variables Phi reads are none of the moved landmarks, and all but the old anchor clone stay in the state (the
  // old one is read before the marginalization drops it: re-anchoring the landmarks of the oldest clone is what the call is for)
  for (int l = 0; l < n; l++) {
    const int var[4] = {fr->clone_off[an->old_clone[l]], fr->clone_off[an->new_clone[l]], ext ? fr->cam_ext_off[an->old_cam[l]] : -1,
                        ext ? fr->cam_ext_off[an->new_cam[l]] : -1};
    for (int v = 0; v < (ext ? 4 : 2); v++) {
      if (var[v] < 0 || var[v] + 6 > N)
        return fail("anchor variable outside the covariance", l);
      for (const Range &r : rng)
        if (var[v] < r.off + r.sz && r.off < var[v] + 6 && (r.kind == 1 || v > 0))
          return fail(r.kind == 0 ? "the new anchor clone or an anchor's extrinsics is marginalized" : "a landmark overlaps an anchor variable", l);
    }
  }
  const int N2 = N - removed;
  if (N2 < 1)
    return fail("the ranges cover the whole covariance", 0);
  // one H2D block: [DevWinFrame][DevWinLM n][flags 2 int | new values 6n][src N2 | mv N | row_lm K][q n | column indices n]
  // [Phi n]. The result block goes back in the one D2H copy. k_anchor_phi fills q, the column indices, Phi and the new
  // values of a landmark on the device, except for ANCHORED_FULL_INVERSE_DEPTH: its Phi goes through acos / atan2 / sin /
  // cos, whose last bits differ between CUDA and the C library, so ovb_slam_anchor_change computes it here and it is
  // uploaded (the upload then runs to the end of the Phi slots; without such a landmark it stops before q).
  const size_t o_lm = align_up(sizeof(DevWinFrame), 256), o_res = o_lm + align_up(sizeof(DevWinLM) * n, 256);
  const size_t res_bytes = 4 * sizeof(int) + sizeof(double) * 6 * n, o_map = align_up(o_res + res_bytes, 256);
  const size_t o_q = align_up(o_map + sizeof(int) * ((size_t)N2 + N + K), 256), o_idx = o_q + sizeof(int) * n;
  const size_t o_phi = align_up(o_idx + sizeof(int) * OVB_WIN_Q * n, 256), total = o_phi + sizeof(double) * OVB_WIN_PHI * n;
  if (total > sizeof(double) * ctx->Hs_cap) {
    snprintf(ctx->err, sizeof(ctx->err), "ovb_marginalize_window: %zu bytes of inputs exceed the reserved staging matrix", total);
    return OVB_ERR_CAPACITY;
  }
  OVB_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
  begin_launches(ctx);
  {
    ovb_status es = ensure_stage(ctx, total / sizeof(double) + 1);
    if (es != OVB_OK)
      return es;
  }
  unsigned char *h = (unsigned char *)ctx->h_stage, *d = (unsigned char *)ctx->d_Hs;
  if (n > 0) {
    DevWinFrame *wf = (DevWinFrame *)h;
    const int nc = fr->n_clones;
    memcpy(wf->clone_R, fr->clone_R, sizeof(double) * 9 * nc);
    memcpy(wf->clone_p, fr->clone_p, sizeof(double) * 3 * nc);
    memcpy(wf->clone_R_fej, fr->clone_R_fej ? fr->clone_R_fej : fr->clone_R, sizeof(double) * 9 * nc);
    memcpy(wf->clone_p_fej, fr->clone_p_fej ? fr->clone_p_fej : fr->clone_p, sizeof(double) * 3 * nc);
    memcpy(wf->cam_R, fr->cam_R, sizeof(double) * 9 * fr->n_cams);
    memcpy(wf->cam_p, fr->cam_p, sizeof(double) * 3 * fr->n_cams);
    memcpy(wf->clone_off, fr->clone_off, sizeof(int) * nc);
    for (int k = 0; k < fr->n_cams; k++)
      wf->cam_ext_off[k] = fr->cam_ext_off ? fr->cam_ext_off[k] : -1;
  }
  DevWinLM *lms = (DevWinLM *)(h + o_lm);
  int *flags = (int *)(h + o_res), *src = (int *)(h + o_map), *mv = src + N2, *row_lm = mv + N;
  int *hq = (int *)(h + o_q), *hidx = (int *)(h + o_idx);
  double *hnewv = (double *)(h + o_res + 4 * sizeof(int)), *hphi = (double *)(h + o_phi);
  flags[0] = OVB_NO_NEG_DIAG; // negative diagonal index
  flags[1] = 0;               // singular H_f
  for (int x = 0; x < N; x++)
    mv[x] = -1;
  bool host_phi = false;
  for (int l = 0, row0 = 0; l < n; l++) {
    DevWinLM &w = lms[l];
    memcpy(w.value, an->value + 3 * l, sizeof(w.value));
    memcpy(w.value_fej, an->value_fej + 3 * l, sizeof(w.value_fej));
    w.lm_off = an->lm_off[l];
    w.rep = an->feat_rep[l];
    w.p = w.rep == OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE ? 1 : 3;
    w.row0 = row0;
    w.old_cam = an->old_cam[l], w.old_clone = an->old_clone[l], w.new_cam = an->new_cam[l], w.new_clone = an->new_clone[l];
    w.host = w.rep == OVB_REP_ANCHORED_FULL_INVERSE_DEPTH;
    if (w.host) {
      ovb_opts ol = *op;
      ol.feat_rep = w.rep;
      int32_t order_off[8], order_sz[8], n_order = 0, n_cols = 0;
      if (ovb_slam_anchor_change(fr, &ol, w.lm_off, w.value, w.value_fej, w.old_cam, w.old_clone, w.new_cam, w.new_clone, hnewv + 6 * l,
                                 hnewv + 6 * l + 3, hphi + (size_t)OVB_WIN_PHI * l, order_off, order_sz, &n_order, &n_cols) != OVB_OK)
        return fail("H_f in the new anchor is singular", l);
      int *ix = hidx + OVB_WIN_Q * l;
      for (int i = 0, c = 0; i < n_order; i++)
        for (int k = 0; k < order_sz[i]; k++)
          ix[c++] = order_off[i] + k;
      hq[l] = n_cols;
      host_phi = true;
    }
    for (int j = 0; j < w.p; j++) {
      mv[w.lm_off + j] = row0 + j;
      row_lm[row0 + j] = l;
    }
    row0 += w.p;
  }
  for (int x = 0, c = 0, r = 0; x < N; x++) { // rng is sorted: skip the marginalized ranges
    while (r < (int)rng.size() && (rng[r].kind != 0 || rng[r].off + rng[r].sz <= x))
      r++;
    if (r < (int)rng.size() && x >= rng[r].off)
      continue;
    src[c++] = x;
  }
  const size_t up0 = n > 0 ? 0 : o_res; // without anchors the frame and landmark records are not read
  const size_t up1 = host_phi ? total : o_q;
  OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(d + up0, h + up0, up1 - up0, cudaMemcpyHostToDevice, ctx->stream));
  int *flags_d = (int *)(d + o_res), *q_d = (int *)(d + o_q), *idx_d = (int *)(d + o_idx);
  double *newv_d = (double *)(d + o_res + 4 * sizeof(int)), *phi_d = (double *)(d + o_phi);
  const DevWinLM *lms_d = (const DevWinLM *)(d + o_lm);
  if (n > 0)
    launch_anchor_phi(ctx, (const DevWinFrame *)d, lms_d, n, op->do_fej, ext ? 1 : 0, flags_d, newv_d, phi_d, idx_d, q_d);
  const int *src_d = (const int *)(d + o_map), *mv_d = src_d + N2, *row_lm_d = mv_d + N;
  launch_window_shift(ctx, n, K, N2, lms_d, row_lm_d, phi_d, idx_d, q_d, src_d, mv_d, flags_d, ctx->d_M, ctx->ldP, ctx->d_S);
  OVB_CUDA_CHECK(ctx, cudaGetLastError());
  OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(h + o_res, d + o_res, res_bytes, cudaMemcpyDeviceToHost, ctx->stream));
  OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  if (flags[1] != 0)
    return fail("H_f in the new anchor is singular", 0);
  if (flags[0] != OVB_NO_NEG_DIAG) {
    snprintf(ctx->err, sizeof(ctx->err), "ovb_marginalize_window: propagated diagonal at %d is negative; P is unchanged", flags[0]);
    return OVB_ERR_NEG_DIAG;
  }
  const double *newv = (const double *)(h + o_res + 4 * sizeof(int));
  for (int l = 0; l < n; l++) {
    memcpy(an->new_value + 3 * l, newv + 6 * l, sizeof(double) * 3);
    memcpy(an->new_value_fej + 3 * l, newv + 6 * l + 3, sizeof(double) * 3);
  }
  ctx->cur ^= 1;
  ctx->N = N2;
  return OVB_OK;
}

ovb_status ovb_cov_propagate(ovb_ctx *ctx, int new_off, int p, const int *old_off, const int *old_sz, int nold, const double *Phi,
                             const double *Q) {
  if (!ctx || !old_off || !old_sz || !Phi || !Q || p < 1 || nold < 1 || new_off < 0 || new_off + p > ctx->N)
    return OVB_ERR_ARG; // the reference exits on empty variable lists (StateHelper.cpp:41-44)
  int q = 0;
  for (int i = 0; i < nold; i++) {
    if (old_off[i] < 0 || old_sz[i] < 1 || old_off[i] + old_sz[i] > ctx->N)
      return OVB_ERR_ARG;
    q += old_sz[i];
  }
  // d_Hs holds [Phi p*q][Q p*p] doubles, then the q int32 old indices (ceil(q/2) doubles)
  if (q > ctx->cfg.max_state || p > ctx->cfg.max_state || (size_t)p * q + (size_t)p * p + ((size_t)q + 1) / 2 > ctx->Hs_cap) {
    snprintf(ctx->err, sizeof(ctx->err), "ovb_cov_propagate: p=%d, q=%d exceed the staging matrix (max_state=%d, %zu doubles)", p, q,
             ctx->cfg.max_state, ctx->Hs_cap);
    return OVB_ERR_CAPACITY;
  }
  OVB_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
  begin_launches(ctx);
  // stage: [Phi p*q][Q p*p] doubles, then q ints
  {
    ovb_status es = ensure_stage(ctx, (size_t)p * q + (size_t)p * p + (size_t)q + 16);
    if (es != OVB_OK)
      return es;
  }
  double *hs = ctx->h_stage;
  memcpy(hs, Phi, sizeof(double) * (size_t)p * q);
  memcpy(hs + (size_t)p * q, Q, sizeof(double) * (size_t)p * p);
  int *hidx = (int *)(hs + (size_t)p * q + (size_t)p * p);
  int c = 0;
  for (int i = 0; i < nold; i++)
    for (int k = 0; k < old_sz[i]; k++)
      hidx[c++] = old_off[i] + k;
  size_t bytes = sizeof(double) * ((size_t)p * q + (size_t)p * p) + sizeof(int) * q;
  OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->d_Hs, hs, bytes, cudaMemcpyHostToDevice, ctx->stream));
  const double *Phi_dev = ctx->d_Hs;
  const double *Q_dev = ctx->d_Hs + (size_t)p * q;
  const int *idx_dev = (const int *)(ctx->d_Hs + (size_t)p * q + (size_t)p * p);
  launch_cov_propagate(ctx, new_off, p, q, idx_dev, Phi_dev, Q_dev);
  OVB_CUDA_CHECK(ctx, cudaGetLastError());
  OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->h_info, ctx->d_info, sizeof(DevUpdateInfo), cudaMemcpyDeviceToHost, ctx->stream));
  OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  if (ctx->h_info->neg_diag_index != OVB_NO_NEG_DIAG) {
    snprintf(ctx->err, sizeof(ctx->err), "EKFPropagation: diagonal at %d is negative", ctx->h_info->neg_diag_index);
    return OVB_ERR_NEG_DIAG;
  }
  return OVB_OK;
}

ovb_status ovb_cov_propagate_imu(ovb_ctx *ctx, int n, int steps, const double *F, const double *G, const double *qc, int new_off, const int *old_off,
                                 const int *old_sz, int nold, int clone_off, int clone_size, const double *dnc_dt, int dt_off, double *Phi_out,
                                 double *Q_out) {
  if (!ctx)
    return OVB_ERR_ARG;
  if (n > OVB_PROP_MAX_N) {
    snprintf(ctx->err, sizeof(ctx->err), "ovb_cov_propagate_imu: n=%d exceeds %d", n, OVB_PROP_MAX_N);
    return OVB_ERR_CAPACITY;
  }
  if (n < 1 || steps < 0 || (steps > 0 && (!F || !G || !qc)) || !old_off || !old_sz || nold < 1 || new_off < 0 || new_off + n > ctx->N)
    return OVB_ERR_ARG;
  int q = 0;
  for (int i = 0; i < nold; i++) {
    if (old_off[i] < 0 || old_sz[i] < 1 || old_off[i] + old_sz[i] > ctx->N)
      return OVB_ERR_ARG;
    q += old_sz[i];
  }
  if (q != n) // Phi is n x n: its columns are the old variables
    return OVB_ERR_ARG;
  if (clone_size < 1 || clone_off < 0 || clone_off + clone_size > ctx->N || (dnc_dt && (dt_off < 0 || dt_off >= ctx->N || clone_size > 64)))
    return OVB_ERR_ARG;
  if (ctx->N + clone_size > ctx->cfg.max_state) {
    snprintf(ctx->err, sizeof(ctx->err), "ovb_cov_propagate_imu: N+clone_size=%d exceeds max_state=%d", ctx->N + clone_size, ctx->cfg.max_state);
    return OVB_ERR_CAPACITY;
  }
  const size_t nn = (size_t)n * n;
  if (2 * nn > ctx->Hs_cap)
    return OVB_ERR_CAPACITY;
  OVB_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
  begin_launches(ctx);
  // staging (doubles): [F steps*nn][G steps*12n][qc steps*4][dnc_dt clone_size][old indices n ints]; Phi, Q come back in front
  const size_t oF = 0, oG = oF + (size_t)steps * nn, oq = oG + (size_t)steps * 12 * n, od = oq + (size_t)steps * 4,
               oi = od + (dnc_dt ? (size_t)clone_size : 0), in_doubles = oi + ((size_t)n + 1) / 2;
  const size_t need = std::max(in_doubles, 2 * nn);
  if (need > ctx->imu_cap) {
    // half as much again: a run's longer gaps between frames do not regrow it each time (cudaFree waits for the whole
    // device, other contexts' work included)
    const size_t cap = need + need / 2;
    cudaFree(ctx->d_imu);
    cudaFreeHost(ctx->h_imu);
    ctx->d_imu = nullptr, ctx->h_imu = nullptr, ctx->imu_cap = 0;
    OVB_CUDA_CHECK(ctx, cudaMalloc(&ctx->d_imu, sizeof(double) * cap));
    OVB_CUDA_CHECK(ctx, cudaMallocHost(&ctx->h_imu, sizeof(double) * cap));
    ctx->imu_cap = cap;
  }
  double *hs = ctx->h_imu;
  if (steps > 0) {
    memcpy(hs + oF, F, sizeof(double) * (size_t)steps * nn);
    memcpy(hs + oG, G, sizeof(double) * (size_t)steps * 12 * n);
    memcpy(hs + oq, qc, sizeof(double) * (size_t)steps * 4);
  }
  if (dnc_dt)
    memcpy(hs + od, dnc_dt, sizeof(double) * clone_size);
  int *hidx = (int *)(hs + oi);
  for (int i = 0, c = 0; i < nold; i++)
    for (int k = 0; k < old_sz[i]; k++)
      hidx[c++] = old_off[i] + k;
  OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->d_imu, hs, sizeof(double) * in_doubles, cudaMemcpyHostToDevice, ctx->stream));
  // Phi and Q where ovb_cov_propagate stages them, then EKFPropagation and the clone on the same stream
  double *Phi_dev = ctx->d_Hs, *Q_dev = ctx->d_Hs + nn;
  if (!launch_prop_accumulate(ctx, n, steps, ctx->d_imu + oF, ctx->d_imu + oG, ctx->d_imu + oq, Phi_dev, Q_dev)) {
    snprintf(ctx->err, sizeof(ctx->err), "ovb_cov_propagate_imu: k_prop_accumulate launch failed: %s", cudaGetErrorString(cudaGetLastError()));
    OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream)); // the staged inputs are in flight
    return OVB_ERR_CUDA;
  }
  launch_cov_propagate(ctx, new_off, n, n, (const int *)(ctx->d_imu + oi), Phi_dev, Q_dev);
  launch_cov_clone(ctx, clone_off, clone_size, dnc_dt ? ctx->d_imu + od : nullptr, dt_off, &ctx->d_info->neg_diag_index);
  OVB_CUDA_CHECK(ctx, cudaGetLastError());
  OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(&ctx->h_info->neg_diag_index, &ctx->d_info->neg_diag_index, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  if (Phi_out || Q_out)
    OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(hs, Phi_dev, sizeof(double) * 2 * nn, cudaMemcpyDeviceToHost, ctx->stream));
  OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  if (Phi_out)
    memcpy(Phi_out, hs, sizeof(double) * nn);
  if (Q_out)
    memcpy(Q_out, hs + nn, sizeof(double) * nn);
  if (ctx->h_info->neg_diag_index != OVB_NO_NEG_DIAG) {
    snprintf(ctx->err, sizeof(ctx->err), "EKFPropagation: diagonal at %d is negative", ctx->h_info->neg_diag_index);
    return OVB_ERR_NEG_DIAG;
  }
  ctx->N += clone_size;
  return OVB_OK;
}

// ------------------------------------------------------------------------------------------------ marshalling
// group tables for n groups; several groups also need the prior's snapshot and the correction accumulator
static ovb_status ensure_groups(ovb_ctx *ctx, int n) {
  if (n > 1) {
    if (!ctx->P_snap)
      OVB_CUDA_CHECK(ctx, cudaMalloc(&ctx->P_snap, sizeof(double) * (size_t)ctx->ldP * ctx->ldP));
    if (!ctx->d_grp_acc)
      OVB_CUDA_CHECK(ctx, cudaMalloc(&ctx->d_grp_acc, sizeof(double) * ((size_t)ctx->cfg.max_state + 4)));
  }
  if (n <= ctx->grp_cap)
    return OVB_OK;
  if (ctx->d_grp)
    cudaFree(ctx->d_grp);
  if (ctx->h_grp)
    cudaFreeHost(ctx->h_grp);
  ctx->d_grp = nullptr;
  ctx->h_grp = nullptr;
  ctx->grp_cap = 0;
  const int cap = std::max(n, 4);
  OVB_CUDA_CHECK(ctx, cudaMalloc(&ctx->d_grp, sizeof(DevGroup) * (size_t)cap));
  OVB_CUDA_CHECK(ctx, cudaMallocHost(&ctx->h_grp, sizeof(DevGroup) * (size_t)cap));
  ctx->grp_cap = cap;
  return OVB_OK;
}

// Column groups of a SLAM batch (h_feat / h_frame packed): features in input order, as many landmarks per group as fit
// next to the frame's columns in OVB_MAX_COLS. A group's layout is its canonical layout, the frame slots and its landmarks
// in ascending covariance offset (a batch of one group: the batch's canonical layout). Rows are stacked in input order, so
// a group's rows are contiguous.
static int slam_lm_width(int rep) { return rep == OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE ? 1 : 3; }

static ovb_status build_groups(ovb_ctx *ctx, int F, int rows_total, Packed *pk) {
  const DevFrame *hf = ctx->h_frame;
  const int room = OVB_MAX_COLS - hf->n_all; // hf->n_all <= 6 OVB_MAX_CLONES + 14 OVB_MAX_CAMS < OVB_MAX_COLS
  // group g = features [f0[g], f0[g+1]): as many landmarks as their widths fit into room
  std::vector<int> f0;
  for (int f = 0, acc = 0; f < F; f++) {
    const int w = slam_lm_width(ctx->h_feat[f].rep);
    if (f == 0 || acc + w > room) {
      f0.push_back(f);
      acc = 0;
    }
    acc += w;
  }
  const int G = (int)f0.size();
  f0.push_back(F);
  if (room < 3 || G > 0xffff) {
    snprintf(ctx->err, sizeof(ctx->err), "SLAM batch of %d landmarks: %d column groups", F, G);
    return OVB_ERR_CAPACITY;
  }
  ovb_status st = ensure_groups(ctx, G);
  if (st != OVB_OK)
    return st;
  int widest = 0;
  std::vector<std::pair<int, int>> lms; // (offset, feature)
  for (int g = 0; g < G; g++) {
    DevGroup &gr = ctx->h_grp[g];
    gr.f0 = f0[g];
    gr.f1 = f0[g + 1];
    gr.row0 = ctx->h_feat[gr.f0].row0;
    gr.rows = (gr.f1 < F ? ctx->h_feat[gr.f1].row0 : rows_total) - gr.row0;
    lms.clear();
    for (int f = gr.f0; f < gr.f1; f++)
      lms.push_back({ctx->h_feat[f].lm_off, f});
    std::sort(lms.begin(), lms.end());
    int col = 0, n_ent = 0;
    size_t l = 0;
    for (int s = 0; s < hf->n_slots || l < lms.size();) {
      if (l < lms.size() && (s == hf->n_slots || lms[l].first < hf->slot_off[s])) {
        const int f = lms[l++].second;
        gr.ent[n_ent++] = -1 - f;
        ctx->h_feat[f].lm_col = (unsigned short)col;
        ctx->h_feat[f].grp = (unsigned short)g;
        for (int k = 0; k < slam_lm_width(ctx->h_feat[f].rep); k++, col++) {
          gr.col_frame[col] = -1;
          gr.col_state[col] = ctx->h_feat[f].lm_off + k;
        }
      } else {
        gr.ent[n_ent++] = s;
        for (int k = 0; k < hf->slot_size[s]; k++, col++) {
          gr.col_frame[col] = (short)(hf->slot_col[s] + k);
          gr.col_state[col] = hf->slot_off[s] + k;
        }
        s++;
      }
    }
    gr.n_cols = col;
    gr.n_ent = n_ent;
    widest = std::max(widest, col);
  }
  if (widest + 1 > std::min(OVB_MAX_COLS, ctx->cfg.max_state) + 8)
    return OVB_ERR_CAPACITY;
  pk->n_groups = G;
  pk->n_all = widest;
  return OVB_OK;
}

// the values of the frame (poses, calibration) into the DevFrame; the variable layout is pack_inputs' work
static void copy_frame_values(DevFrame *hf, const ovb_frame *fr) {
  memcpy(hf->clone_R, fr->clone_R, sizeof(double) * 9 * fr->n_clones);
  memcpy(hf->clone_p, fr->clone_p, sizeof(double) * 3 * fr->n_clones);
  memcpy(hf->clone_R_fej, fr->clone_R_fej ? fr->clone_R_fej : fr->clone_R, sizeof(double) * 9 * fr->n_clones);
  memcpy(hf->clone_p_fej, fr->clone_p_fej ? fr->clone_p_fej : fr->clone_p, sizeof(double) * 3 * fr->n_clones);
  memcpy(hf->cam_R, fr->cam_R, sizeof(double) * 9 * fr->n_cams);
  memcpy(hf->cam_p, fr->cam_p, sizeof(double) * 3 * fr->n_cams);
  memcpy(hf->cam_intr, fr->cam_intr, sizeof(double) * 8 * fr->n_cams);
  for (int k = 0; k < fr->n_cams; k++)
    hf->cam_model[k] = fr->cam_model ? fr->cam_model[k] : OVB_CAM_RADTAN;
}

// lm != nullptr: SLAM batch — every feature brings its landmark (a 3-wide state variable, or 1-wide for
// ANCHORED_INVERSE_DEPTH_SINGLE), rows are NOT nullspace-projected (2M per feature instead of 2M-3), values/anchors come
// from the landmark. The landmarks are not frame slots: the batch is cut into column groups (DevGroup), contiguous feature
// ranges whose frame columns plus landmark columns fit OVB_MAX_COLS. lm_rep: each landmark's representation (NULL: all
// op->feat_rep).
// per_feature: the call will launch the per-feature kernel (everything but ovb_triangulate), so its scratch is reserved.
// feat_sigma / feat_chi2_mult: per-feature pixel noise and gate multiplier (NULL: op's, or the landmarks').
static ovb_status pack_inputs(ovb_ctx *ctx, const ovb_frame *fr, const ovb_feat_batch *fb, const ovb_opts *op, const ovb_feat_out *given,
                              Packed *pk, const ovb_landmarks *lm = nullptr, bool per_feature = true, const int32_t *lm_rep = nullptr,
                              const double *feat_sigma = nullptr, const double *feat_chi2_mult = nullptr) {
  if (!fr || !fb || !op)
    return OVB_ERR_ARG;
  auto rep_of = [&](int f) { return lm_rep ? lm_rep[f] : op->feat_rep; };
  if (lm && (!lm->lm_off || !lm->value || !lm->value_fej))
    return OVB_ERR_ARG;
  if (fr->n_clones < 1 || fr->n_clones > OVB_MAX_CLONES || fr->n_cams < 1 || fr->n_cams > OVB_MAX_CAMS) {
    snprintf(ctx->err, sizeof(ctx->err), "frame: n_clones=%d (max %d) n_cams=%d (max %d)", fr->n_clones, OVB_MAX_CLONES, fr->n_cams, OVB_MAX_CAMS);
    return OVB_ERR_CAPACITY;
  }
  if (fb->n_feats < 0 || fb->n_feats > ctx->cfg.max_feats || fb->n_meas < 0 || fb->n_meas > ctx->cfg.max_meas) {
    snprintf(ctx->err, sizeof(ctx->err), "batch: n_feats=%d (max %d) n_meas=%d (max %d)", fb->n_feats, ctx->cfg.max_feats, fb->n_meas,
             ctx->cfg.max_meas);
    return OVB_ERR_CAPACITY;
  }
  DevFrame *hf = ctx->h_frame;
  memset(hf, 0, sizeof(*hf));
  hf->n_clones = fr->n_clones;
  hf->n_cams = fr->n_cams;
  copy_frame_values(hf, fr);
  // ---- slots in ascending covariance offset
  struct SlotRec {
    int off, size, kind, idx;
  }; // kind 0 clone, 1 ext, 2 intr, 3 landmark
  std::vector<SlotRec> slots;
  for (int k = 0; k < fr->n_cams; k++) {
    hf->cam_ext_slot[k] = hf->cam_intr_slot[k] = -1;
    if (op->do_calib_camera_pose) {
      if (!fr->cam_ext_off || fr->cam_ext_off[k] < 0) {
        snprintf(ctx->err, sizeof(ctx->err), "do_calib_camera_pose set but cam_ext_off[%d] < 0", k);
        return OVB_ERR_ARG;
      }
      slots.push_back({fr->cam_ext_off[k], 6, 1, k});
    }
    if (op->do_calib_camera_intrinsics) {
      if (!fr->cam_intr_off || fr->cam_intr_off[k] < 0) {
        snprintf(ctx->err, sizeof(ctx->err), "do_calib_camera_intrinsics set but cam_intr_off[%d] < 0", k);
        return OVB_ERR_ARG;
      }
      slots.push_back({fr->cam_intr_off[k], 8, 2, k});
    }
  }
  for (int c = 0; c < fr->n_clones; c++)
    slots.push_back({fr->clone_off[c], 6, 0, c});
  std::sort(slots.begin(), slots.end(), [](const SlotRec &a, const SlotRec &b) { return a.off < b.off; });
  if ((int)slots.size() > OVB_MAX_VARS) { // clones + calibration: OVB_MAX_CLONES + 2 OVB_MAX_CAMS at most
    snprintf(ctx->err, sizeof(ctx->err), "%d frame variables (clones + calibration), max %d", (int)slots.size(), OVB_MAX_VARS);
    return OVB_ERR_CAPACITY;
  }
  if (lm && !ctx->slam_unbounded && (int)slots.size() + fb->n_feats > OVB_MAX_VARS) {
    snprintf(ctx->err, sizeof(ctx->err),
             "%d state variables in one update (clones + calibration + landmarks), max %d: split the batch or ovb_set_slam_unbounded",
             (int)slots.size() + fb->n_feats, OVB_MAX_VARS);
    return OVB_ERR_CAPACITY;
  }
  int col = 0;
  for (size_t s = 0; s < slots.size(); s++) {
    if (slots[s].off < 0 || slots[s].off + slots[s].size > ctx->N) {
      snprintf(ctx->err, sizeof(ctx->err), "variable offset %d(+%d) outside the covariance (N=%d)", slots[s].off, slots[s].size, ctx->N);
      return OVB_ERR_ARG;
    }
    if (s > 0 && slots[s].off < slots[s - 1].off + slots[s - 1].size) {
      snprintf(ctx->err, sizeof(ctx->err), "overlapping state variables at offset %d", slots[s].off);
      return OVB_ERR_ARG;
    }
    hf->slot_off[s] = slots[s].off;
    hf->slot_size[s] = slots[s].size;
    hf->slot_col[s] = col;
    col += slots[s].size;
    if (slots[s].kind == 0)
      hf->clone_slot[slots[s].idx] = (int)s;
    else if (slots[s].kind == 1)
      hf->cam_ext_slot[slots[s].idx] = (int)s;
    else
      hf->cam_intr_slot[slots[s].idx] = (int)s;
  }
  hf->n_slots = (int)slots.size();
  hf->n_all = col;
  hf->groups = nullptr;
  if (col > OVB_MAX_COLS || col + 1 > std::min(OVB_MAX_COLS, ctx->cfg.max_state) + 8)
    return OVB_ERR_CAPACITY;
  if (lm) { // landmarks: a known representation, inside the covariance, overlapping neither a frame variable nor each other
    for (int f = 0; f < fb->n_feats; f++) {
      hf->lm_w = std::max(hf->lm_w, slam_lm_width(rep_of(f)));
      if (rep_of(f) < OVB_REP_GLOBAL_3D || rep_of(f) > OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE) {
        snprintf(ctx->err, sizeof(ctx->err), "landmark %d: representation %d is not an ovb_feat_rep", f, rep_of(f));
        return OVB_ERR_ARG;
      }
    }
    std::vector<std::pair<int, int>> all; // (offset, size)
    for (const SlotRec &r : slots)
      all.push_back({r.off, r.size});
    for (int f = 0; f < fb->n_feats; f++)
      all.push_back({lm->lm_off[f], slam_lm_width(rep_of(f))});
    std::sort(all.begin(), all.end());
    for (size_t s = 0; s < all.size(); s++) {
      if (all[s].first < 0 || all[s].first + all[s].second > ctx->N) {
        snprintf(ctx->err, sizeof(ctx->err), "variable offset %d(+%d) outside the covariance (N=%d)", all[s].first, all[s].second, ctx->N);
        return OVB_ERR_ARG;
      }
      if (s > 0 && all[s].first < all[s - 1].first + all[s - 1].second) {
        snprintf(ctx->err, sizeof(ctx->err), "overlapping state variables at offset %d", all[s].first);
        return OVB_ERR_ARG;
      }
    }
  }
  // ---- options
  DevOpts *ho = ctx->h_opts;
  ho->o = *op;
  ho->sigma_pix_sq = std::pow(op->sigma_pix, 2);
  ho->rep = op->feat_rep == OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE ? OVB_REP_ANCHORED_MSCKF_INVERSE_DEPTH : op->feat_rep;
  if (ho->rep < 0 || ho->rep > OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE)
    return OVB_ERR_ARG;
  // ---- blob: [cam u8 M][pad2][clone u16 M][pad4][uv f32 2M][uvn f32 2M][keys u8]
  const int F = fb->n_feats, M = fb->n_meas;
  size_t o_cam = 0;
  size_t o_clone = align_up(o_cam + (size_t)M, 16);
  size_t o_uv = align_up(o_clone + 2 * (size_t)M, 16);
  size_t o_uvn = align_up(o_uv + 8 * (size_t)M, 16);
  size_t o_keys = align_up(o_uvn + 8 * (size_t)M, 16);
  unsigned char *hb = ctx->h_blob;
  if (M > 0) {
    memcpy(hb + o_cam, fb->cam, (size_t)M);
    memcpy(hb + o_clone, fb->clone, 2 * (size_t)M);
    memcpy(hb + o_uv, fb->uv, 8 * (size_t)M);
    memcpy(hb + o_uvn, fb->uvn, 8 * (size_t)M);
  }
  unsigned char *hkeys = hb + o_keys;
  size_t nkeys = 0;
  int row = 0;
  for (int f = 0; f < F; f++) {
    DevFeat &d = ctx->h_feat[f];
    d.m0 = fb->meas_off[f];
    d.m1 = fb->meas_off[f + 1];
    if (d.m0 < 0 || d.m1 < d.m0 || d.m1 > M)
      return OVB_ERR_ARG;
    int Mf = d.m1 - d.m0;
    if (Mf > OVB_MAX_MEAS_PER_FEAT) {
      snprintf(ctx->err, sizeof(ctx->err), "feature %d has %d measurements (max %d)", f, Mf, OVB_MAX_MEAS_PER_FEAT);
      return OVB_ERR_CAPACITY;
    }
    d.row0 = row;
    d.rep = rep_of(f);
    const bool lm_single = lm && d.rep == OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE; // 1-wide landmark (inverse depth only)
    if (lm)
      row += lm_single ? (Mf >= 2 ? 2 * Mf - 2 : 0) : 2 * Mf; // UpdaterSLAM.cpp:344-387: all 2M rows kept (SINGLE: 2 projected out)
    else
      row += Mf >= 2 ? 2 * Mf - 3 : 0;
    d.key0 = (int)nkeys;
    // validate BEFORE anything is stored in the pinned blob: camera ids in range, at most one key per camera (the
    // reference's feat->timestamps is a map keyed by camera id), room for the keys
    for (int i = d.m0; i < d.m1; i++)
      if (fb->cam[i] >= fr->n_cams || fb->clone[i] >= fr->n_clones) {
        snprintf(ctx->err, sizeof(ctx->err), "feature %d: measurement %d refers to camera %d / clone %d outside the frame", f, i, (int)fb->cam[i],
                 (int)fb->clone[i]);
        return OVB_ERR_ARG;
      }
    if (o_keys + nkeys + (size_t)OVB_MAX_CAMS > ctx->blob_cap)
      return OVB_ERR_CAPACITY;
    {
      unsigned seen = 0;
      if (fb->cam_keys_off && fb->cam_keys) {
        const int k0 = fb->cam_keys_off[f], k1 = fb->cam_keys_off[f + 1];
        if (k0 < 0 || k1 < k0 || k1 - k0 > fr->n_cams) {
          snprintf(ctx->err, sizeof(ctx->err), "feature %d: %d camera keys for %d cameras", f, k1 - k0, fr->n_cams);
          return OVB_ERR_ARG;
        }
        for (int k = k0; k < k1; k++) {
          const unsigned c = fb->cam_keys[k];
          if ((int)c >= fr->n_cams || (seen >> c) & 1u) {
            snprintf(ctx->err, sizeof(ctx->err), "feature %d: camera key %u out of range or repeated", f, c);
            return OVB_ERR_ARG;
          }
          seen |= 1u << c;
          hkeys[nkeys++] = (unsigned char)c;
        }
      } else {
        int last = -1;
        for (int i = d.m0; i < d.m1; i++)
          if ((int)fb->cam[i] != last) {
            last = fb->cam[i];
            if ((seen >> last) & 1u) { // measurements must be grouped by camera (include/ovb200.h, ovb_feat_batch)
              snprintf(ctx->err, sizeof(ctx->err), "feature %d: measurements are not grouped by camera", f);
              return OVB_ERR_ARG;
            }
            seen |= 1u << last;
            hkeys[nkeys++] = (unsigned char)last;
          }
      }
    }
    d.key1 = (int)nkeys;
    d.status = OVB_FEAT_OK;
    d.anchor_cam = d.anchor_clone = -1;
    d.chi2 = NAN;
    for (int k = 0; k < 3; k++)
      d.p_FinA[k] = d.p_FinG[k] = NAN;
    d.sigma_sq = std::pow(op->sigma_pix, 2);
    d.chi2_mult = op->chi2_multipler;
    if (feat_sigma)
      d.sigma_sq = std::pow(feat_sigma[f], 2);
    if (feat_chi2_mult)
      d.chi2_mult = feat_chi2_mult[f];
    d.lm_off = -1;
    d.lm_col = d.grp = 0;
    for (int k = 0; k < 3; k++)
      d.p_FinG_fej[k] = NAN;
    if (lm) {
      d.lm_off = lm->lm_off[f];
      d.status = Mf >= (lm_single ? 2 : 1) ? OVB_FEAT_OK : OVB_FEAT_FEW_MEAS; // UpdaterSLAM.cpp:278-290
      const bool rel = d.rep >= OVB_REP_ANCHORED_3D;
      d.anchor_cam = rel && lm->anchor_cam ? lm->anchor_cam[f] : -1;
      d.anchor_clone = rel && lm->anchor_clone ? lm->anchor_clone[f] : -1;
      if (rel && (d.anchor_cam < 0 || d.anchor_cam >= fr->n_cams || d.anchor_clone < 0 || d.anchor_clone >= fr->n_clones)) {
        snprintf(ctx->err, sizeof(ctx->err), "landmark %d: anchored representation without a valid anchor", f);
        return OVB_ERR_ARG;
      }
      for (int k = 0; k < 3; k++) {
        d.p_FinA[k] = lm->value[3 * f + k]; // meaning depends on the representation: the kernel reads the right one
        d.p_FinG[k] = lm->value[3 * f + k];
        d.p_FinG_fej[k] = lm->value_fej[3 * f + k];
      }
      if (lm->sigma_pix)
        d.sigma_sq = std::pow(lm->sigma_pix[f], 2);
      if (lm->chi2_multipler)
        d.chi2_mult = lm->chi2_multipler[f];
    }
    if (given) {
      d.status = given->status ? given->status[f] : OVB_FEAT_OK;
      d.anchor_cam = given->anchor_cam ? given->anchor_cam[f] : -1;
      d.anchor_clone = given->anchor_clone ? given->anchor_clone[f] : -1;
      for (int k = 0; k < 3; k++) {
        d.p_FinA[k] = given->p_FinA ? given->p_FinA[3 * f + k] : NAN;
        d.p_FinG[k] = given->p_FinG ? given->p_FinG[3 * f + k] : NAN;
      }
    }
  }
  {
    // CTA schedule of the per-feature kernels: longest tracks first (counting sort on the track length, stable)
    int cnt[OVB_MAX_MEAS_PER_FEAT + 2] = {0};
    for (int f = 0; f < F; f++)
      cnt[OVB_MAX_MEAS_PER_FEAT - (ctx->h_feat[f].m1 - ctx->h_feat[f].m0) + 1]++;
    for (int i = 1; i <= OVB_MAX_MEAS_PER_FEAT + 1; i++)
      cnt[i] += cnt[i - 1];
    for (int f = 0; f < F; f++)
      ctx->h_feat[cnt[OVB_MAX_MEAS_PER_FEAT - (ctx->h_feat[f].m1 - ctx->h_feat[f].m0)]++].sched = f;
  }
  pk->n_feats = F;
  pk->n_meas = M;
  pk->m_total = row;
  pk->n_all = col;
  pk->n_groups = 0;
  if (lm) {
    ovb_status gs = build_groups(ctx, F, row, pk);
    if (gs != OVB_OK)
      return gs;
    hf->groups = ctx->d_grp;
  }
  pk->ldH = (int)align_up((size_t)pk->n_all + 1, 4);
  if ((size_t)std::max(row, pk->n_all) * pk->ldH > ctx->Hs_cap || row > ctx->max_rows) {
    snprintf(ctx->err, sizeof(ctx->err), "stacked system %d x %d exceeds the reserved staging matrix", row, pk->ldH);
    return OVB_ERR_CAPACITY;
  }
  if (per_feature) { // long tracks: scratch of the per-feature kernel's long-track path
    ovb_status rs = feature_scratch_reserve(ctx, F, lm != nullptr);
    if (rs != OVB_OK)
      return rs;
  }
  pk->bv.cam = ctx->d_blob + o_cam;
  pk->bv.clone = (const uint16_t *)(ctx->d_blob + o_clone);
  pk->bv.uv = (const float *)(ctx->d_blob + o_uv);
  pk->bv.uvn = (const float *)(ctx->d_blob + o_uvn);
  pk->bv.keys = ctx->d_blob + o_keys;
  size_t used = ctx->off_blob + o_keys + nkeys;
  ctx->last_h2d_bytes = used;
  cudaError_t e = cudaMemcpyAsync(ctx->d_arena, ctx->h_arena, used, cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess && pk->n_groups > 0) {
    e = cudaMemcpyAsync(ctx->d_grp, ctx->h_grp, sizeof(DevGroup) * (size_t)pk->n_groups, cudaMemcpyHostToDevice, ctx->stream);
    ctx->last_h2d_bytes += sizeof(DevGroup) * (size_t)pk->n_groups;
  }
  if (e != cudaSuccess) {
    snprintf(ctx->err, sizeof(ctx->err), "H2D arena copy: %s", cudaGetErrorString(e));
    return OVB_ERR_CUDA;
  }
  return OVB_OK;
}

static void unpack_feats(ovb_ctx *ctx, int F, ovb_feat_out *out) {
  if (!out)
    return;
  for (int f = 0; f < F; f++) {
    const DevFeat &d = ctx->h_feat[f];
    if (out->status)
      out->status[f] = d.status;
    if (out->anchor_cam)
      out->anchor_cam[f] = d.anchor_cam;
    if (out->anchor_clone)
      out->anchor_clone[f] = d.anchor_clone;
    if (out->chi2)
      out->chi2[f] = d.chi2;
    for (int k = 0; k < 3; k++) {
      if (out->p_FinA)
        out->p_FinA[3 * f + k] = d.p_FinA[k];
      if (out->p_FinG)
        out->p_FinG[3 * f + k] = d.p_FinG[k];
    }
  }
}

// the status of an EKF update from its read-back failure flags, with the message in ctx->err
static ovb_status ekf_status(ovb_ctx *ctx, const DevUpdateInfo *inf) {
  if (inf->not_spd) {
    snprintf(ctx->err, sizeof(ctx->err), "EKFUpdate: innovation covariance not positive definite");
    return OVB_ERR_NOT_SPD;
  }
  if (inf->nonfinite) {
    snprintf(ctx->err, sizeof(ctx->err), "EKFUpdate: non-finite covariance entry");
    return OVB_ERR_NONFINITE;
  }
  if (inf->neg_diag_index != OVB_NO_NEG_DIAG) {
    snprintf(ctx->err, sizeof(ctx->err), "EKFUpdate: diagonal at %d is negative", inf->neg_diag_index);
    return OVB_ERR_NEG_DIAG;
  }
  return OVB_OK;
}

// the read-back of an update's F features, info and dx (the last two in one copy), enqueued behind its kernels; ev[6]
// marks its end. The caller synchronises.
static ovb_status enqueue_readback(ovb_ctx *ctx, int F) {
  const size_t info_dx = ctx->info_bytes + sizeof(double) * (size_t)ctx->N;
  OVB_CUDA_CHECK(ctx, cudaGetLastError());
  OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->h_feat, ctx->d_feat, sizeof(DevFeat) * (size_t)F, cudaMemcpyDeviceToHost, ctx->stream));
  OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->h_info, ctx->d_info, info_dx, cudaMemcpyDeviceToHost, ctx->stream));
  ctx->last_d2h_bytes = sizeof(DevFeat) * (size_t)F + info_dx;
  cudaEventRecord(ctx->ev[6], ctx->stream);
  return OVB_OK;
}

// ovb_stats of an MSCKF or SLAM update of F features that handed r rows to the EKF update, from the read-back info. The
// reference's SLAM update hands every stacked row to EKFUpdate (it never compresses there); the MSCKF update compresses.
static void fill_stats(const ovb_ctx *ctx, ovb_stats *stats, int F, int r, bool slam) {
  if (!stats)
    return;
  const DevUpdateInfo *inf = ctx->h_info;
  stats->n_feats_in = F;
  stats->n_feats_used = inf->n_feats_used;
  stats->rows_stacked = inf->rows_stacked;
  stats->cols_stacked = inf->n_used;
  stats->rows_update = slam ? inf->rows_stacked : std::min(inf->rows_stacked, inf->n_used);
  stats->neg_diag_index = (r > 0 && inf->neg_diag_index != OVB_NO_NEG_DIAG) ? inf->neg_diag_index : -1;
  stats->ms_total = ctx->stage_ms[5];
}

// ------------------------------------------------------------------------------------------------ hot path
ovb_status ovb_triangulate(ovb_ctx *ctx, const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_opts *opts, ovb_feat_out *out) {
  if (!ctx || !out)
    return OVB_ERR_ARG;
  OVB_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
  begin_launches(ctx);
  Packed pk;
  int saveN = ctx->N;
  if (ctx->N == 0)
    ctx->N = ctx->cfg.max_state; // offsets are not dereferenced by this stage
  ovb_status st = pack_inputs(ctx, frame, feats, opts, nullptr, &pk, nullptr, false);
  ctx->N = saveN;
  if (st != OVB_OK)
    return st;
  launch_cam_poses(ctx);
  launch_triangulate(ctx, pk.n_feats, pk.bv);
  OVB_CUDA_CHECK(ctx, cudaGetLastError());
  OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->h_feat, ctx->d_feat, sizeof(DevFeat) * (size_t)pk.n_feats, cudaMemcpyDeviceToHost, ctx->stream));
  OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  unpack_feats(ctx, pk.n_feats, out);
  return OVB_OK;
}

ovb_status ovb_feature_jacobians(ovb_ctx *ctx, const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_opts *opts, ovb_feat_out *out,
                                 int stage, double *Hf_out, double *Hx_out, double *res_out, int32_t *row_off_out, int32_t *ncols_out,
                                 int32_t *col_index_out, int ld_out) {
  if (!ctx || !out || !row_off_out || !ncols_out || !col_index_out)
    return OVB_ERR_ARG;
  if (ctx->N < 1) {
    snprintf(ctx->err, sizeof(ctx->err), "ovb_feature_jacobians: no covariance loaded (ovb_cov_set)");
    return OVB_ERR_ARG;
  }
  OVB_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
  begin_launches(ctx);
  Packed pk;
  ovb_status st = pack_inputs(ctx, frame, feats, opts, out, &pk);
  if (st != OVB_OK)
    return st;
  const int F = pk.n_feats, n_all = pk.n_all;
  if (ld_out < n_all)
    return OVB_ERR_ARG;
  *ncols_out = n_all;
  for (int s = 0, c = 0; s < ctx->h_frame->n_slots; s++)
    for (int k = 0; k < ctx->h_frame->slot_size[s]; k++)
      col_index_out[c++] = ctx->h_frame->slot_off[s] + k;
  launch_cam_poses(ctx);
  if (stage == 0) {
    int rows = 2 * pk.n_meas;
    size_t need = (size_t)rows * (OVB_MAX_COLS + 4);
    if (!ctx->d_dump || need > ctx->dump_cap) {
      if (ctx->d_dump)
        cudaFree(ctx->d_dump);
      ctx->dump_cap = need;
      OVB_CUDA_CHECK(ctx, cudaMalloc(&ctx->d_dump, sizeof(double) * ctx->dump_cap));
    }
    ctx->dump_rows = rows;
    OVB_CUDA_CHECK(ctx, cudaMemsetAsync(ctx->d_dump, 0, sizeof(double) * need, ctx->stream));
    launch_feature_system(ctx, F, pk.bv, pk.ldH, 1);
    OVB_CUDA_CHECK(ctx, cudaGetLastError());
    std::vector<double> host(need);
    OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(host.data(), ctx->d_dump, sizeof(double) * need, cudaMemcpyDeviceToHost, ctx->stream));
    OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    int dump_rows = rows;
    const double *dHf = host.data(), *dres = host.data() + (size_t)dump_rows * 3, *dHx = host.data() + (size_t)dump_rows * 4;
    for (int f = 0; f <= F; f++)
      row_off_out[f] = 2 * feats->meas_off[f];
    for (int i = 0; i < rows; i++) {
      if (Hf_out)
        for (int k = 0; k < 3; k++)
          Hf_out[(size_t)i * 3 + k] = dHf[(size_t)i * 3 + k];
      if (res_out)
        res_out[i] = dres[i];
      if (Hx_out)
        for (int j = 0; j < n_all; j++)
          Hx_out[(size_t)i * ld_out + j] = dHx[(size_t)i * OVB_MAX_COLS + j];
    }
    return OVB_OK;
  }
  launch_feature_system(ctx, F, pk.bv, pk.ldH, 0);
  OVB_CUDA_CHECK(ctx, cudaGetLastError());
  std::vector<double> host((size_t)pk.m_total * pk.ldH);
  if (pk.m_total > 0)
    OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(host.data(), ctx->d_Hs, sizeof(double) * host.size(), cudaMemcpyDeviceToHost, ctx->stream));
  OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->h_feat, ctx->d_feat, sizeof(DevFeat) * (size_t)F, cudaMemcpyDeviceToHost, ctx->stream));
  OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  unpack_feats(ctx, F, out);
  for (int f = 0; f < F; f++)
    row_off_out[f] = ctx->h_feat[f].row0;
  row_off_out[F] = pk.m_total;
  for (int i = 0; i < pk.m_total; i++) {
    if (res_out)
      res_out[i] = host[(size_t)i * pk.ldH + n_all];
    if (Hx_out)
      for (int j = 0; j < n_all; j++)
        Hx_out[(size_t)i * ld_out + j] = host[(size_t)i * pk.ldH + j];
  }
  return OVB_OK;
}

// JacobiRotation::makeGivens(p, q) (Eigen/src/Jacobi/Jacobi.h, real branch): G' [p; q] = [r; 0], r >= 0
static void make_givens(double p, double q, double &gc, double &gs) {
  if (q == 0.0) {
    gc = p < 0.0 ? -1.0 : 1.0;
    gs = 0.0;
  } else if (p == 0.0) {
    gc = 0.0;
    gs = q < 0.0 ? 1.0 : -1.0;
  } else if (std::fabs(p) > std::fabs(q)) {
    const double t = q / p;
    double u = std::sqrt(1.0 + t * t);
    if (p < 0.0)
      u = -u;
    gc = 1.0 / u;
    gs = -t * gc;
  } else {
    const double t = p / q;
    double u = std::sqrt(1.0 + t * t);
    if (q < 0.0)
      u = -u;
    gs = -1.0 / u;
    gc = -t * gs;
  }
}

static int compress_system(ovb_ctx *ctx, int mode, double *A, int m, int n, int ldA, double *Rout, int ldR);

// UpdaterSLAM::delayed_init in one call (see include/ovb200.h). Composition of the staged entry points with the state mean
// moved by the caller's callback between the features, exactly the reference's sequential structure.
ovb_status ovb_slam_delayed_init(ovb_ctx *ctx, const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_opts *opts, const double *sigma_pix,
                                 const double *chi2_multipler, ovb_init_callback on_init, void *user, ovb_feat_out *out, int32_t *lm_off_out) {
  return ovb_slam_delayed_init_reps(ctx, frame, feats, opts, nullptr, sigma_pix, chi2_multipler, on_init, user, out, lm_off_out);
}

// the representations of a delayed initialisation (feat_rep or opts->feat_rep): each one an ovb_feat_rep, and SINGLE not mixed
// with a 3-wide representation. Which representation sizes a SINGLE landmark when the two classes differ (the feature's own,
// or feat_rep_slam's) has not been checked against the reference source: a class mix of SINGLE with a 3-wide representation
// is refused rather than guessed. Mixes among the 3-wide representations are unaffected.
static ovb_status check_init_reps(ovb_ctx *ctx, int F, const int32_t *feat_rep, const ovb_opts *opts) {
  auto rep_of = [&](int f) { return feat_rep ? feat_rep[f] : opts->feat_rep; };
  int n_single = 0;
  for (int f = 0; f < F; f++) {
    if (rep_of(f) < OVB_REP_GLOBAL_3D || rep_of(f) > OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE) {
      snprintf(ctx->err, sizeof(ctx->err), "feature %d: representation %d is not an ovb_feat_rep", f, rep_of(f));
      return OVB_ERR_ARG;
    }
    n_single += rep_of(f) == OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE ? 1 : 0;
  }
  if (n_single > 0 && n_single < F) {
    snprintf(ctx->err, sizeof(ctx->err), "ovb_slam_delayed_init: ANCHORED_INVERSE_DEPTH_SINGLE mixed with a 3-wide representation in one call");
    return OVB_ERR_ARG;
  }
  return OVB_OK;
}

// step 1 of a delayed initialisation: pack and upload the batch once, triangulate + GN all tracks at the current state
// (UpdaterSLAM.cpp:118-142) and read the per-feature records back (one stream synchronisation). The tracks' anchors and
// positions stay on the device for the per-feature systems. sched_of: the CTA schedule entry of each feature (the launcher
// addresses a feature through it).
static ovb_status init_triangulate(ovb_ctx *ctx, const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_opts *opts, const int32_t *feat_rep,
                                   const double *sigma_pix, const double *chi2_multipler, ovb_feat_out *out, Packed *pk, std::vector<int> &sched_of) {
  const int F = feats->n_feats;
  int64_t *cnt = ctx->init_counters; // features processed, stream synchronisations, bytes H2D, bytes D2H
  cnt[0] = cnt[1] = cnt[2] = cnt[3] = 0;
  OVB_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
  begin_launches(ctx);
  const int saveN = ctx->N;
  if (ctx->N == 0)
    ctx->N = ctx->cfg.max_state; // offsets are not dereferenced before a feature is initialised (checked there)
  ovb_status st = pack_inputs(ctx, frame, feats, opts, nullptr, pk, nullptr, false, feat_rep, sigma_pix, chi2_multipler);
  ctx->N = saveN;
  if (st != OVB_OK)
    return st;
  st = feature_scratch_reserve(ctx, F, false, true);
  if (st != OVB_OK)
    return st;
  cnt[2] += (int64_t)ctx->last_h2d_bytes;
  launch_cam_poses(ctx);
  launch_triangulate(ctx, F, pk->bv);
  OVB_CUDA_CHECK(ctx, cudaGetLastError());
  OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->h_feat, ctx->d_feat, sizeof(DevFeat) * (size_t)F, cudaMemcpyDeviceToHost, ctx->stream));
  OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  cnt[1]++;
  cnt[3] += (int64_t)(sizeof(DevFeat) * (size_t)F);
  unpack_feats(ctx, F, out);
  if (!ctx->d_init) {
    OVB_CUDA_CHECK(ctx, cudaMalloc(&ctx->d_init, sizeof(DevInitSys)));
    OVB_CUDA_CHECK(ctx, cudaMallocHost(&ctx->h_init, sizeof(DevInitSys)));
  }
  sched_of.assign((size_t)F, 0);
  for (int i = 0; i < F; i++)
    sched_of[ctx->h_feat[i].sched] = i;
  return OVB_OK;
}

// the state columns a triangulated feature touches, as the per-feature kernel's bookkeeping finds them: the slots of its
// camera keys and of the clones those cameras saw it in, and the anchor's (UpdaterHelper.cpp:226-262)
static int init_columns(const ovb_ctx *ctx, const Packed &pk, const ovb_feat_batch *feats, const ovb_opts *opts, int f, int rep) {
  const DevFrame *hf = ctx->h_frame;
  const unsigned char *hkeys = ctx->h_blob + (pk.bv.keys - ctx->d_blob);
  const DevFeat &d = ctx->h_feat[f];
  unsigned long long seen = 0ull;
  for (int q = d.key0; q < d.key1; q++) {
    const int key = hkeys[q];
    if (opts->do_calib_camera_pose && hf->cam_ext_slot[key] >= 0)
      seen |= 1ull << hf->cam_ext_slot[key];
    if (opts->do_calib_camera_intrinsics && hf->cam_intr_slot[key] >= 0)
      seen |= 1ull << hf->cam_intr_slot[key];
    for (int i = d.m0; i < d.m1; i++)
      if (feats->cam[i] == key)
        seen |= 1ull << hf->clone_slot[feats->clone[i]];
  }
  if (rep >= OVB_REP_ANCHORED_3D) {
    seen |= 1ull << hf->clone_slot[d.anchor_clone];
    if (opts->do_calib_camera_pose && hf->cam_ext_slot[d.anchor_cam] >= 0)
      seen |= 1ull << hf->cam_ext_slot[d.anchor_cam];
  }
  int n = 0;
  for (int s = 0; s < hf->n_slots; s++)
    if ((seen >> s) & 1ull)
      n += hf->slot_size[s];
  return n;
}

ovb_status ovb_slam_delayed_init_reps(ovb_ctx *ctx, const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_opts *opts,
                                      const int32_t *feat_rep, const double *sigma_pix, const double *chi2_multipler, ovb_init_callback on_init,
                                      void *user, ovb_feat_out *out, int32_t *lm_off_out) {
  if (!ctx || !frame || !feats || !opts || !out || !out->status || !out->p_FinA || !out->p_FinG || !out->anchor_cam || !out->anchor_clone || !lm_off_out)
    return OVB_ERR_ARG;
  const int F = feats->n_feats;
  auto rep_of = [&](int f) { return feat_rep ? feat_rep[f] : opts->feat_rep; };
  ovb_status st = check_init_reps(ctx, F, feat_rep, opts);
  if (st != OVB_OK)
    return st;
  for (int f = 0; f < F; f++)
    lm_off_out[f] = -1;
  if (F <= 0)
    return OVB_OK;
  int64_t *cnt = ctx->init_counters;
  // 1. triangulation
  Packed pk;
  std::vector<int> sched_of;
  st = init_triangulate(ctx, frame, feats, opts, feat_rep, sigma_pix, chi2_multipler, out, &pk, sched_of);
  if (st != OVB_OK)
    return st;
  bool moved = false;
  // 2. one feature after the other: its system, gate, augmentation and EKF update on the device, one read-back of
  // {status, chi2, dx_new, dx}, then the caller's callback moves the mean that the next feature is linearised at
  for (int f = 0; f < F; f++) {
    if (out->status[f] != OVB_FEAT_OK)
      continue;
    const DevFeat &d = ctx->h_feat[f];
    const int rep = rep_of(f);
    const int k = rep == OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE ? 1 : 3;
    const int N0 = ctx->N;
    if (N0 < 1) {
      snprintf(ctx->err, sizeof(ctx->err), "ovb_slam_delayed_init: no covariance loaded (ovb_cov_set)");
      return OVB_ERR_ARG;
    }
    if (!(d.sigma_sq > 0.0))
      return OVB_ERR_ARG;
    if (N0 + k > ctx->ldP) {
      snprintf(ctx->err, sizeof(ctx->err), "initialize: covariance would grow to %d (max_state %d)", N0 + k, ctx->ldP);
      return OVB_ERR_CAPACITY;
    }
    const int n = init_columns(ctx, pk, feats, opts, f, rep);
    if (n > ctx->cfg.max_state)
      return OVB_ERR_CAPACITY;
    cnt[0]++;
    if (moved) { // the callback moved the frame: only its block is uploaded again
      copy_frame_values(ctx->h_frame, frame);
      OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->d_frame, ctx->h_frame, sizeof(DevFrame), cudaMemcpyHostToDevice, ctx->stream));
      cnt[2] += (int64_t)sizeof(DevFrame);
      launch_cam_poses(ctx);
    }
    launch_feature_init(ctx, sched_of[f], pk.bv, pk.ldH);
    launch_init_prep(ctx, f, k, n);
    const int *skip = &ctx->d_init->skip;
    if (!launch_cov_init_augment(ctx, k, n, ctx->d_init->HR, ctx->d_init->Hinv, d.sigma_sq, skip)) {
      snprintf(ctx->err, sizeof(ctx->err), "ovb_slam_delayed_init: covariance augmentation kernel could not be launched (N=%d, k=%d)", N0, k);
      return OVB_ERR_CAPACITY;
    }
    // EKFUpdate with the projected rows on the augmented covariance (StateHelper.cpp:476-479), compressed when taller than wide
    const double *Hdev = ctx->d_Hs + (size_t)d.row0 * pk.ldH;
    const int rows = 2 * (d.m1 - d.m0) - 3;
    int rr = rows;
    if (rows > n) {
      rr = compress_system(ctx, OVB_COMPRESS_CHOLQR2, ctx->d_Hs + (size_t)d.row0 * pk.ldH, rows, n, pk.ldH, ctx->d_R, pk.ldH);
      Hdev = ctx->d_R;
    }
    ctx->N = N0 + k;
    launch_ekf_update(ctx, Hdev, pk.ldH, rr, n, false, d.sigma_sq, nullptr, skip);
    ctx->N = N0;
    OVB_CUDA_CHECK(ctx, cudaGetLastError());
    const size_t flag_bytes = sizeof(DevUpdateInfo) - offsetof(DevUpdateInfo, neg_diag_index);
    OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->h_init, ctx->d_init, OVB_INIT_HEAD_BYTES, cudaMemcpyDeviceToHost, ctx->stream));
    OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(&ctx->h_info->neg_diag_index, &ctx->d_info->neg_diag_index, flag_bytes, cudaMemcpyDeviceToHost, ctx->stream));
    OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->h_dx, ctx->d_dx, sizeof(double) * (size_t)(N0 + k), cudaMemcpyDeviceToHost, ctx->stream));
    OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    cnt[1]++;
    cnt[3] += (int64_t)(OVB_INIT_HEAD_BYTES + flag_bytes + sizeof(double) * (size_t)(N0 + k));
    const DevInitSys *hs = ctx->h_init;
    if (hs->fail == 1) {
      snprintf(ctx->err, sizeof(ctx->err), "initialize: H_L is rank deficient");
      return OVB_ERR_ARG;
    }
    if (hs->fail == 2) {
      snprintf(ctx->err, sizeof(ctx->err), "ovb_slam_delayed_init: feature %d touches %d columns, the host counted %d", f, ctx->h_init->n, n);
      return OVB_ERR_CUDA;
    }
    if (out->chi2) // the gate's value, accepted or rejected (NaN: S was not positive definite)
      out->chi2[f] = hs->chi2;
    if (hs->status != OVB_FEAT_OK) {
      out->status[f] = hs->status;
      continue;
    }
    ctx->N = N0 + k;
    st = ekf_status(ctx, ctx->h_info);
    if (st != OVB_OK)
      return st;
    lm_off_out[f] = N0;
    if (on_init) {
      on_init(user, f, N0, k, hs->dx_new, ctx->h_dx, N0 + k); // the host moves its mean and refreshes the frame arrays
      moved = true;
    }
  }
  return OVB_OK;
}

// UpdaterSLAM::delayed_init without a host round trip per landmark (see include/ovb200.h). The feature after an accepted one is
// linearised at the moved mean, and whether a landmark is accepted (and so where the next one lands in P) is only known on
// the device: k_init_commit moves the device frame and advances the live size N there. Every feature's kernels are launched
// up front against the upper bound of N (N at the start plus the widths of the candidates before it): P's rows and columns
// between the live N and that bound are zero, so the EKF update over the bound gives zero rows of M and K there, zero
// entries of dx and leaves those rows zero, and every live entry gets the bits of the update over the live N.
ovb_status ovb_slam_delayed_init_batch(ovb_ctx *ctx, const ovb_frame *frame, const ovb_frame_quat *quat, const ovb_feat_batch *feats,
                                       const ovb_opts *opts, const int32_t *feat_rep, const double *sigma_pix, const double *chi2_multipler,
                                       ovb_feat_out *out, int32_t *lm_off_out, double *dx_new, double *dx, int ld_dx) {
  if (!ctx || !frame || !quat || !quat->clone_q || !quat->cam_q || !feats || !opts || !out || !out->status || !out->p_FinA || !out->p_FinG ||
      !out->anchor_cam || !out->anchor_clone || !lm_off_out || !dx_new || !dx)
    return OVB_ERR_ARG;
  const int F = feats->n_feats;
  auto rep_of = [&](int f) { return feat_rep ? feat_rep[f] : opts->feat_rep; };
  ovb_status st = check_init_reps(ctx, F, feat_rep, opts);
  if (st != OVB_OK)
    return st;
  for (int f = 0; f < F; f++)
    lm_off_out[f] = -1;
  if (F <= 0)
    return OVB_OK;
  int64_t *cnt = ctx->init_counters;
  // 1. triangulation: which features reach the initialisation decides the launches
  Packed pk;
  std::vector<int> sched_of;
  st = init_triangulate(ctx, frame, feats, opts, feat_rep, sigma_pix, chi2_multipler, out, &pk, sched_of);
  if (st != OVB_OK)
    return st;
  // 2. every candidate's width, columns, the upper bound of N in front of it and its dx row in the read-back; all refusals
  // before P is touched
  struct Cand {
    int f, k, n, bound;
    size_t row; // first double of its dx row (bound + k doubles)
  };
  std::vector<Cand> cand;
  const int N_start = ctx->N;
  int bound = N_start;
  size_t row_doubles = 0;
  for (int f = 0; f < F; f++) {
    if (out->status[f] != OVB_FEAT_OK)
      continue;
    const int k = rep_of(f) == OVB_REP_ANCHORED_INVERSE_DEPTH_SINGLE ? 1 : 3;
    if (N_start < 1) {
      snprintf(ctx->err, sizeof(ctx->err), "ovb_slam_delayed_init: no covariance loaded (ovb_cov_set)");
      return OVB_ERR_ARG;
    }
    if (!(ctx->h_feat[f].sigma_sq > 0.0))
      return OVB_ERR_ARG;
    if (bound + k > ctx->ldP) {
      snprintf(ctx->err, sizeof(ctx->err), "initialize: covariance could grow to %d (max_state %d)", bound + k, ctx->ldP);
      return OVB_ERR_CAPACITY;
    }
    if (sizeof(double) * ((size_t)bound * k + (size_t)k * k) > 200 * 1024) { // launch_cov_init_augment's one-CTA footprint
      snprintf(ctx->err, sizeof(ctx->err), "ovb_slam_delayed_init: covariance augmentation of N=%d does not fit one CTA", bound);
      return OVB_ERR_CAPACITY;
    }
    const int n = init_columns(ctx, pk, feats, opts, f, rep_of(f));
    if (n > ctx->cfg.max_state)
      return OVB_ERR_CAPACITY;
    cand.push_back({f, k, n, bound, row_doubles});
    row_doubles += (size_t)bound + k;
    bound += k;
  }
  cnt[0] = (int64_t)cand.size();
  if (cand.empty())
    return OVB_OK;
  if (ld_dx < bound) {
    snprintf(ctx->err, sizeof(ctx->err), "ovb_slam_delayed_init_batch: ld_dx = %d, the triangulated features need %d", ld_dx, bound);
    return OVB_ERR_ARG;
  }
  // 3. the batch buffer [DevInitBatch][DevInitRec x F][dx rows]: its head (live N, quaternions) up, P kept in the other
  // buffer for an error, the rows and columns P may grow into zeroed
  const size_t off_rec = sizeof(DevInitBatch), off_rows = off_rec + sizeof(DevInitRec) * (size_t)F;
  const size_t ib_bytes = off_rows + sizeof(double) * row_doubles;
  if (ib_bytes > ctx->ib_cap) {
    if (ctx->d_ib)
      cudaFree(ctx->d_ib);
    if (ctx->h_ib)
      cudaFreeHost(ctx->h_ib);
    ctx->d_ib = ctx->h_ib = nullptr;
    ctx->ib_cap = 0;
    OVB_CUDA_CHECK(ctx, cudaMalloc(&ctx->d_ib, ib_bytes));
    OVB_CUDA_CHECK(ctx, cudaMallocHost(&ctx->h_ib, ib_bytes));
    ctx->ib_cap = ib_bytes;
  }
  DevInitBatch *hb = (DevInitBatch *)ctx->h_ib, *db = (DevInitBatch *)ctx->d_ib;
  DevInitRec *drec = (DevInitRec *)(ctx->d_ib + off_rec);
  double *drows = (double *)(ctx->d_ib + off_rows);
  memset(hb, 0, sizeof(DevInitBatch));
  hb->N = N_start;
  hb->fej_R_is_value = frame->clone_R_fej == nullptr;
  hb->fej_p_is_value = frame->clone_p_fej == nullptr;
  memcpy(hb->clone_q, quat->clone_q, sizeof(double) * 4 * frame->n_clones);
  memcpy(hb->cam_q, quat->cam_q, sizeof(double) * 4 * frame->n_cams);
  OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(db, hb, sizeof(DevInitBatch), cudaMemcpyHostToDevice, ctx->stream));
  cnt[2] += (int64_t)sizeof(DevInitBatch);
  const size_t ldb = sizeof(double) * ctx->ldP;
  double *P = ctx->P[ctx->cur];
  OVB_CUDA_CHECK(ctx, cudaMemcpy2DAsync(ctx->P[ctx->cur ^ 1], ldb, P, ldb, sizeof(double) * N_start, N_start, cudaMemcpyDeviceToDevice, ctx->stream));
  OVB_CUDA_CHECK(ctx, cudaMemset2DAsync(P + (size_t)N_start * ctx->ldP, ldb, 0, sizeof(double) * bound, bound - N_start, ctx->stream));
  OVB_CUDA_CHECK(ctx, cudaMemset2DAsync(P + N_start, ldb, 0, sizeof(double) * (bound - N_start), N_start, ctx->stream));
  auto restore = [&]() { // P and N as before the call (the snapshot becomes the current buffer)
    ctx->cur ^= 1;
    ctx->N = N_start;
  };
  // 4. one feature after the other on the device: its system at the moved frame, gate, augmentation at the live N, EKF update
  // over the bound, then its record and the mean update; no host round trip in between
  const int *skip = &ctx->d_init->skip;
  for (size_t i = 0; i < cand.size(); i++) {
    const Cand &c = cand[i];
    const DevFeat &d = ctx->h_feat[c.f];
    if (i > 0)
      launch_cam_poses(ctx); // the previous feature may have moved the frame
    launch_feature_init(ctx, sched_of[c.f], pk.bv, pk.ldH);
    launch_init_prep(ctx, c.f, c.k, c.n);
    ctx->N = c.bound;
    if (!launch_cov_init_augment(ctx, c.k, c.n, ctx->d_init->HR, ctx->d_init->Hinv, d.sigma_sq, skip, &db->N)) {
      restore();
      snprintf(ctx->err, sizeof(ctx->err), "ovb_slam_delayed_init: covariance augmentation kernel could not be launched (N<=%d, k=%d)", c.bound, c.k);
      return OVB_ERR_CAPACITY;
    }
    const double *Hdev = ctx->d_Hs + (size_t)d.row0 * pk.ldH;
    const int rows = 2 * (d.m1 - d.m0) - 3;
    int rr = rows;
    if (rows > c.n) {
      rr = compress_system(ctx, OVB_COMPRESS_CHOLQR2, ctx->d_Hs + (size_t)d.row0 * pk.ldH, rows, c.n, pk.ldH, ctx->d_R, pk.ldH);
      Hdev = ctx->d_R;
    }
    ctx->N = c.bound + c.k;
    launch_ekf_update(ctx, Hdev, pk.ldH, rr, c.n, false, d.sigma_sq, nullptr, skip);
    launch_init_commit(ctx, db, drec + c.f, drows + c.row, c.k, opts->do_calib_camera_pose, opts->do_calib_camera_intrinsics);
  }
  ctx->N = N_start;
  const cudaError_t e_launch = cudaGetLastError();
  // 5. one read-back of every record
  const cudaError_t e_copy = cudaMemcpyAsync(ctx->h_ib, ctx->d_ib, ib_bytes, cudaMemcpyDeviceToHost, ctx->stream);
  const cudaError_t e_sync = cudaStreamSynchronize(ctx->stream);
  cnt[1]++;
  cnt[3] += (int64_t)ib_bytes;
  if (e_launch != cudaSuccess || e_copy != cudaSuccess || e_sync != cudaSuccess) {
    restore();
    const cudaError_t e = e_launch != cudaSuccess ? e_launch : e_copy != cudaSuccess ? e_copy : e_sync;
    snprintf(ctx->err, sizeof(ctx->err), "ovb_slam_delayed_init_batch: %s", cudaGetErrorString(e));
    return OVB_ERR_CUDA;
  }
  const DevInitRec *hrec = (const DevInitRec *)(ctx->h_ib + off_rec);
  const double *hrows = (const double *)(ctx->h_ib + off_rows);
  for (const Cand &c : cand) { // the first failure in feature order is the call's, as in ovb_slam_delayed_init_reps
    const DevInitRec &r = hrec[c.f];
    if (r.fail == 1) {
      restore();
      snprintf(ctx->err, sizeof(ctx->err), "initialize: H_L is rank deficient");
      return OVB_ERR_ARG;
    }
    if (r.fail == 2) {
      restore();
      snprintf(ctx->err, sizeof(ctx->err), "ovb_slam_delayed_init: feature %d touches %d columns, the host counted %d", c.f, r.n, c.n);
      return OVB_ERR_CUDA;
    }
    if (r.fail == 3) {
      DevUpdateInfo flags;
      flags.not_spd = r.not_spd, flags.nonfinite = r.nonfinite, flags.neg_diag_index = r.neg_diag_index;
      restore();
      return ekf_status(ctx, &flags);
    }
  }
  for (const Cand &c : cand) {
    const DevInitRec &r = hrec[c.f];
    if (out->chi2) // the gate's value, accepted or rejected (NaN: S was not positive definite)
      out->chi2[c.f] = r.chi2;
    if (r.status != OVB_FEAT_OK) {
      out->status[c.f] = r.status;
      continue;
    }
    lm_off_out[c.f] = r.lm_off;
    memcpy(dx_new + 3 * (size_t)c.f, r.dx_new, sizeof(double) * c.k);
    memcpy(dx + (size_t)c.f * ld_dx, hrows + c.row, sizeof(double) * ((size_t)r.lm_off + c.k));
  }
  ctx->N = hb->N;
  return OVB_OK;
}

ovb_status ovb_last_init_counters(const ovb_ctx *ctx, int64_t out[4]) {
  if (!ctx || !out)
    return OVB_ERR_ARG;
  for (int i = 0; i < 4; i++)
    out[i] = ctx->init_counters[i];
  return OVB_OK;
}

// dx = 0 when no row reaches the EKF update
__global__ void k_fill_zero_dx(double *dx, int N) {
  OVB_PDL_ENTER();
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N)
    dx[i] = 0.0;
}

// ---- SLAM batches of several column groups: sequential EKF updates at one linearization point. With the rows whitened
// (R = I), group g's compressed system [R_g | z_g] is applied to the mean already corrected by the groups before it,
// z_g <- z_g - R_g dx_acc[cols_g]; the result equals the joint update (tests/test_slam_batches_cpu.py).
// Copies the group's column map into info (the EKF reads it there) and writes the corrected residual over column n of R.
__global__ void k_group_take_z(double *__restrict__ R, int ldR, int rows, int n, const int *__restrict__ col_state,
                               const double *__restrict__ dx_acc, DevUpdateInfo *__restrict__ info) {
  OVB_PDL_ENTER();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n)
    info->col_state[i] = col_state[i];
  if (i < rows) {
    double *Ri = R + (size_t)i * ldR;
    double z = Ri[n];
    for (int j = 0; j < n; j++)
      z -= Ri[j] * dx_acc[col_state[j]];
    Ri[n] = z;
  }
}
// dx_acc += dx of the group; the group's failure flags are kept (the next group's EKF resets them in info)
__global__ void k_group_accumulate(const double *__restrict__ dx, double *__restrict__ dx_acc, int N, const DevUpdateInfo *__restrict__ info,
                                   int *__restrict__ flags) {
  OVB_PDL_ENTER();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N)
    dx_acc[i] += dx[i];
  if (i == 0) {
    if (info->not_spd)
      flags[0] = 1;
    if (info->nonfinite)
      flags[1] = 1;
  }
}
// after the last group: dx = dx_acc, or on any failure (not SPD, non-finite, negative diagonal) dx = 0 and P = the prior
__global__ void k_group_finish(double *__restrict__ P, int ldP, int N, const double *__restrict__ P_prior, const double *__restrict__ dx_acc,
                               double *__restrict__ dx, DevUpdateInfo *__restrict__ info, const int *__restrict__ flags) {
  OVB_PDL_ENTER();
  const bool failed = flags[0] || flags[1] || info->neg_diag_index != OVB_NO_NEG_DIAG;
  const int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y * blockDim.y + threadIdx.y;
  if (i == 0 && j < N)
    dx[j] = failed ? 0.0 : dx_acc[j];
  if (i == 0 && j == 0) {
    info->not_spd = flags[0];
    info->nonfinite = flags[1];
  }
  if (failed && i < N && j < N)
    P[(size_t)i * ldP + j] = P_prior[(size_t)i * ldP + j];
}

// measurement_compress_inplace in the requested mode; returns the number of rows of [R | z] handed to the EKF update.
// The Cholesky-based modes always produce n rows; the Householder path leaves min(m, n).
static int compress_system(ovb_ctx *ctx, int mode, double *A, int m, int n, int ldA, double *Rout, int ldR) {
  if (mode == OVB_COMPRESS_CHOLQR2 && launch_compress_cholqr2(ctx, A, m, n, ldA, Rout, ldR))
    return n;
  if (mode == OVB_COMPRESS_NORMAL_EQUATIONS && launch_compress_gram(ctx, A, m, n, ldA, Rout, ldR))
    return n;
  launch_tsqr(ctx, A, m, n, ldA, Rout, ldR);
  return std::min(m, n);
}

// The device pipeline of one update on inputs already in the arena: steps 2-6 of UpdaterMSCKF::update.
// ev (optional): ev[1] after triangulation, ev[2] after the per-feature systems, ev[3] after the column map, ev[4] after
// compression, ev[5] after the EKF update. Returns the row count handed to the EKF update.
// slam: UpdaterSLAM::update — landmarks come from the state (no triangulation), rows are kept unprojected and whitened;
// pk.n_groups column groups (ctx->h_grp). Several groups: every gate sees the prior P (the per-feature kernel runs once over
// the batch), then each group is compressed and applied in turn (ev[4] then marks the start of that loop).
static int enqueue_slam_groups(ovb_ctx *ctx, int n_groups, int ldH);
static int enqueue_update(ovb_ctx *ctx, const Packed &pk, int col_order, cudaEvent_t *ev, bool slam = false) {
  const int N = ctx->N, F = pk.n_feats, ldH = pk.ldH, m_total = pk.m_total, n_all = pk.n_all, n_groups = pk.n_groups;
  const BlobView bv = pk.bv;
  if (!slam) {
    launch_cam_poses(ctx);
    launch_triangulate(ctx, F, bv);
  }
  if (ev)
    cudaEventRecord(ev[1], ctx->stream);
  launch_feature_system(ctx, F, bv, ldH, slam ? 2 : 0);
  if (ev)
    cudaEventRecord(ev[2], ctx->stream);
  // the column bookkeeping (a single serial CTA) only feeds the re-ordering and the EKF update: it runs on the side
  // stream while the compression owns the GPU, and is joined before its first consumer
  {
    cudaEventRecord(ctx->ev_fork, ctx->stream);
    cudaStreamWaitEvent(ctx->side_stream, ctx->ev_fork, 0);
    cudaStream_t main_stream = ctx->stream;
    ctx->stream = ctx->side_stream;
    if (slam) {
      launch_column_map_slam(ctx, F, n_groups == 1);
    } else {
      launch_column_map(ctx, F, bv, 3);
    }
    ctx->stream = main_stream;
    cudaEventRecord(ctx->ev_join, ctx->side_stream);
  }
  if (ev)
    cudaEventRecord(ev[3], ctx->stream);
  if (slam && n_groups > 1) {
    cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0);
    if (ev)
      cudaEventRecord(ev[4], ctx->stream);
    const int r = enqueue_slam_groups(ctx, n_groups, ldH);
    if (ev)
      cudaEventRecord(ev[5], ctx->stream);
    return r;
  }
  const int ldR = ldH;
  const double *Rfinal = ctx->d_R;
  int r = 0;
  if (m_total > 0) {
    r = compress_system(ctx, ctx->h_opts->o.compress, ctx->d_Hs, m_total, n_all, ldH, ctx->d_R, ldR);
    cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0);
    if (col_order == OVB_COLS_REFERENCE_FIRST_SEEN) {
      launch_reorder_R(ctx, ctx->d_R, n_all, ldR, ctx->d_R2, ldR);
      Rfinal = ctx->d_R2;
    }
  }
  else
    cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0);
  if (ev)
    cudaEventRecord(ev[4], ctx->stream);
  if (r > 0)
    launch_ekf_update(ctx, Rfinal, ldR, r, n_all, false, slam ? 1.0 : ctx->h_opts->sigma_pix_sq, nullptr);
  else
    ovb_launch(ctx, k_fill_zero_dx, dim3((N + 127) / 128), dim3(128), (size_t)0, ctx->d_dx, N);
  if (ev)
    cudaEventRecord(ev[5], ctx->stream);
  return r;
}

static int enqueue_slam_groups(ovb_ctx *ctx, int n_groups, int ldH) {
  const int N = ctx->N, ld = ctx->ldP;
  double *P = ctx->P[ctx->cur];
  double *acc = ctx->d_grp_acc;
  int *flags = (int *)(acc + ctx->cfg.max_state);
  cudaMemcpyAsync(ctx->P_snap, P, sizeof(double) * (size_t)ld * N, cudaMemcpyDeviceToDevice, ctx->stream);
  cudaMemsetAsync(acc, 0, sizeof(double) * ((size_t)ctx->cfg.max_state + 4), ctx->stream);
  int r_total = 0;
  for (int g = 0; g < n_groups; g++) {
    const DevGroup &G = ctx->h_grp[g];
    if (G.rows == 0)
      continue;
    const int n = G.n_cols;
    const int r = compress_system(ctx, ctx->h_opts->o.compress, ctx->d_Hs + (size_t)G.row0 * ldH, G.rows, n, ldH, ctx->d_R, ldH);
    ovb_launch(ctx, k_group_take_z, dim3((n + 127) / 128), dim3(128), (size_t)0, ctx->d_R, ldH, r, n, (const int *)ctx->d_grp[g].col_state,
               (const double *)acc, ctx->d_info);
    launch_ekf_update(ctx, ctx->d_R, ldH, r, n, false, 1.0, nullptr);
    ovb_launch(ctx, k_group_accumulate, dim3((N + 255) / 256), dim3(256), (size_t)0, (const double *)ctx->d_dx, acc, N,
               (const DevUpdateInfo *)ctx->d_info, flags);
    r_total += r;
  }
  if (r_total > 0)
    ovb_launch(ctx, k_group_finish, dim3((N + 31) / 32, (N + 7) / 8), dim3(32, 8), (size_t)0, P, ld, N, (const double *)ctx->P_snap,
               (const double *)acc, ctx->d_dx, ctx->d_info, (const int *)flags);
  else
    ovb_launch(ctx, k_fill_zero_dx, dim3((N + 127) / 128), dim3(128), (size_t)0, ctx->d_dx, N);
  return r_total;
}

// Per-kernel timing (bench.py's roofline block): while on, every kernel launched through ovb_launch is bracketed by CUDA
// events and programmatic dependent launch is disabled, so each duration is that kernel alone, in stream order, with
// whatever the previous kernels left in L2.
ovb_status ovb_set_profile(ovb_ctx *ctx, int enabled) {
  if (!ctx)
    return OVB_ERR_ARG;
  ctx->prof_on = enabled ? 1 : 0;
  ctx->prof_n = 0;
  return OVB_OK;
}

// kernels of the last call, in launch order: names (NUL-separated, truncated to name_cap bytes in total) and their
// durations in microseconds, min(cap, *n) of them, where *n = the call's launches. Call after the call returned.
ovb_status ovb_profile_read(ovb_ctx *ctx, char *names, int name_cap, float *us, int cap, int *n) {
  if (!ctx || !names || !us || !n || name_cap < 1)
    return OVB_ERR_ARG;
  OVB_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
  int w = 0;
  for (int k = 0; k < ctx->prof_n && k < cap; k++) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, ctx->prof_ev[2 * k], ctx->prof_ev[2 * k + 1]) != cudaSuccess)
      cudaGetLastError();
    us[k] = 1e3f * ms;
    const char *nm = nullptr;
    if (cudaFuncGetName(&nm, ctx->prof_fn[k]) != cudaSuccess || !nm) {
      cudaGetLastError();
      nm = "?";
    }
    for (const char *c = nm; *c && w < name_cap - 2; c++)
      names[w++] = *c;
    names[w++] = 0;
  }
  if (w < name_cap)
    names[w] = 0;
  *n = ctx->prof_n;
  return OVB_OK;
}

ovb_status ovb_last_host_us(const ovb_ctx *ctx, double out[4]) {
  if (!ctx || !out)
    return OVB_ERR_ARG;
  for (int i = 0; i < 4; i++)
    out[i] = ctx->host_us[i];
  return OVB_OK;
}

ovb_status ovb_last_counters(const ovb_ctx *ctx, int64_t out[4]) {
  if (!ctx || !out)
    return OVB_ERR_ARG;
  out[0] = ctx->n_launch;            // kernels launched by the last call
  out[1] = ctx->n_launch_tsqr_level; // of which k_tsqr_level
  out[2] = (int64_t)ctx->last_h2d_bytes;
  out[3] = (int64_t)ctx->last_d2h_bytes;
  return OVB_OK;
}

ovb_status ovb_set_slam_unbounded(ovb_ctx *ctx, int enabled) {
  if (!ctx)
    return OVB_ERR_ARG;
  ctx->slam_unbounded = enabled ? 1 : 0;
  return OVB_OK;
}

ovb_status ovb_set_replay(ovb_ctx *ctx, int enabled) {
  if (!ctx)
    return OVB_ERR_ARG;
  OVB_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
  if (enabled && !ctx->P_snap)
    OVB_CUDA_CHECK(ctx, cudaMalloc(&ctx->P_snap, sizeof(double) * (size_t)ctx->ldP * ctx->ldP));
  ctx->replay_enabled = enabled ? 1 : 0;
  ctx->last_pk_valid = 0;
  return OVB_OK;
}

ovb_status ovb_msckf_replay(ovb_ctx *ctx, int steps, int flush_l2, float *ms_per_step, float stage_ms_sum[5]) {
  if (!ctx || steps < 1 || !ms_per_step)
    return OVB_ERR_ARG;
  if (!ctx->replay_enabled || !ctx->last_pk_valid) {
    snprintf(ctx->err, sizeof(ctx->err), "ovb_msckf_replay: call ovb_set_replay(ctx,1) and ovb_msckf_update first");
    return OVB_ERR_ARG;
  }
  OVB_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
  const size_t flush_bytes = (size_t)256 << 20; // five times the 50 MB L2 of an H100
  if (flush_l2 && !ctx->d_flush)
    OVB_CUDA_CHECK(ctx, cudaMalloc(&ctx->d_flush, flush_bytes));
  begin_launches(ctx);
  std::vector<cudaEvent_t> evs((size_t)steps * 6);
  for (auto &e : evs)
    OVB_CUDA_CHECK(ctx, cudaEventCreate(&e));
  const size_t Pbytes = sizeof(double) * (size_t)ctx->ldP * ctx->N;
  for (int s = 0; s < steps; s++) {
    if (flush_l2)
      cudaMemsetAsync(ctx->d_flush, s & 0xff, flush_bytes, ctx->stream);
    // restore the prior saved by the last ovb_msckf_update (outside the timed bracket: it is not part of an update)
    cudaMemcpyAsync(ctx->P[ctx->cur], ctx->P_snap, Pbytes, cudaMemcpyDeviceToDevice, ctx->stream);
    cudaEvent_t *ev = &evs[(size_t)s * 6];
    cudaEventRecord(ev[0], ctx->stream);
    enqueue_update(ctx, ctx->last_pk, ctx->last_col_order, ev);
  }
  OVB_CUDA_CHECK(ctx, cudaGetLastError());
  OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  if (stage_ms_sum)
    for (int k = 0; k < 5; k++)
      stage_ms_sum[k] = 0.f;
  for (int s = 0; s < steps; s++) {
    cudaEvent_t *ev = &evs[(size_t)s * 6];
    cudaEventElapsedTime(&ms_per_step[s], ev[0], ev[5]);
    if (stage_ms_sum)
      for (int k = 0; k < 5; k++) {
        float t;
        cudaEventElapsedTime(&t, ev[k], ev[k + 1]);
        stage_ms_sum[k] += t;
      }
  }
  for (auto &e : evs)
    cudaEventDestroy(e);
  return OVB_OK;
}

ovb_status ovb_msckf_update(ovb_ctx *ctx, const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_opts *opts, ovb_feat_out *out,
                            double *dx, ovb_stats *stats) {
  if (!ctx || !dx)
    return OVB_ERR_ARG;
  if (ctx->N < 1) {
    snprintf(ctx->err, sizeof(ctx->err), "ovb_msckf_update: no covariance loaded (ovb_cov_set)");
    return OVB_ERR_ARG;
  }
  OVB_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
  const int N = ctx->N;
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->neg_diag_index = -1;
  }
  for (int i = 0; i < N; i++)
    dx[i] = 0.0;
  begin_launches(ctx);
  if (!feats || feats->n_feats <= 0) // UpdaterMSCKF.cpp:61-62
    return OVB_OK;
  cudaEventRecord(ctx->ev[0], ctx->stream);
  const auto h0 = std::chrono::steady_clock::now();
  Packed pk;
  ovb_status st = pack_inputs(ctx, frame, feats, opts, nullptr, &pk);
  if (st != OVB_OK)
    return st;
  const auto h1 = std::chrono::steady_clock::now();
  const int F = pk.n_feats;
  if (ctx->replay_enabled) {
    // keep the prior so that ovb_msckf_replay can re-run this exact update on device-resident inputs
    OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->P_snap, ctx->P[ctx->cur], sizeof(double) * (size_t)ctx->ldP * N, cudaMemcpyDeviceToDevice,
                                        ctx->stream));
    ctx->last_pk_valid = 1;
    ctx->last_pk = pk;
    ctx->last_col_order = opts->col_order;
  }
  const int r = enqueue_update(ctx, pk, opts->col_order, ctx->ev);
  st = enqueue_readback(ctx, F);
  if (st != OVB_OK)
    return st;
  const auto h2 = std::chrono::steady_clock::now();
  OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  const auto h3 = std::chrono::steady_clock::now();
  unpack_feats(ctx, F, out);
  for (int i = 0; i < N; i++)
    dx[i] = ctx->h_dx[i];
  {
    const auto h4 = std::chrono::steady_clock::now();
    auto us = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
      return std::chrono::duration<double, std::micro>(b - a).count();
    };
    ctx->host_us[0] = us(h0, h1), ctx->host_us[1] = us(h1, h2), ctx->host_us[2] = us(h2, h3), ctx->host_us[3] = us(h3, h4);
  }
  ctx->stage_pending = 1; // the five stage times are read from the events when ovb_last_stage_ms asks for them
  cudaEventElapsedTime(&ctx->stage_ms[5], ctx->ev[0], ctx->ev[6]);
  fill_stats(ctx, stats, F, r, false);
  return r > 0 ? ekf_status(ctx, ctx->h_info) : OVB_OK;
}

// UpdaterSLAM::update steps 4-5 (update/UpdaterSLAM.cpp:310-470) on the device: same per-feature kernel in its SLAM mode
// (landmark block appended, no nullspace projection, per-class noise and gate), then the shared compress + EKF stages.
ovb_status ovb_slam_update(ovb_ctx *ctx, const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_landmarks *landmarks,
                           const ovb_opts *opts, ovb_feat_out *out, double *dx, ovb_stats *stats) {
  return ovb_slam_update_reps(ctx, frame, feats, landmarks, nullptr, opts, out, dx, stats);
}

ovb_status ovb_slam_update_reps(ovb_ctx *ctx, const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_landmarks *landmarks,
                                const int32_t *feat_rep, const ovb_opts *opts, ovb_feat_out *out, double *dx, ovb_stats *stats) {
  if (!ctx || !dx || !landmarks || !opts)
    return OVB_ERR_ARG;
  if (ctx->N < 1) {
    snprintf(ctx->err, sizeof(ctx->err), "ovb_slam_update: no covariance loaded (ovb_cov_set)");
    return OVB_ERR_ARG;
  }
  OVB_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
  const int N = ctx->N;
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->neg_diag_index = -1;
  }
  for (int i = 0; i < N; i++)
    dx[i] = 0.0;
  begin_launches(ctx);
  if (!feats || feats->n_feats <= 0) // UpdaterSLAM.cpp:256-257
    return OVB_OK;
  cudaEventRecord(ctx->ev[0], ctx->stream);
  Packed pk;
  ovb_status st = pack_inputs(ctx, frame, feats, opts, nullptr, &pk, landmarks, true, feat_rep);
  if (st != OVB_OK)
    return st;
  const int F = pk.n_feats;
  ctx->last_pk_valid = 0; // the replay path re-runs MSCKF updates only
  const int r = enqueue_update(ctx, pk, opts->col_order, ctx->ev, true);
  st = enqueue_readback(ctx, F);
  if (st != OVB_OK)
    return st;
  OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  if (out) {
    for (int f = 0; f < F; f++) {
      if (out->status)
        out->status[f] = ctx->h_feat[f].status;
      if (out->chi2)
        out->chi2[f] = ctx->h_feat[f].chi2;
    }
  }
  for (int i = 0; i < N; i++)
    dx[i] = ctx->h_dx[i];
  ctx->stage_pending = 1; // the five stage times are read from the events when ovb_last_stage_ms asks for them
  cudaEventElapsedTime(&ctx->stage_ms[5], ctx->ev[0], ctx->ev[6]);
  fill_stats(ctx, stats, F, r, true);
  return r > 0 ? ekf_status(ctx, ctx->h_info) : OVB_OK;
}

ovb_status ovb_last_stage_ms(const ovb_ctx *ctx, float ms[6]) {
  if (!ctx || !ms)
    return OVB_ERR_ARG;
  if (ctx->stage_pending) {
    for (int s = 0; s < 5; s++)
      cudaEventElapsedTime(&ctx->stage_ms[s], ctx->ev[s], ctx->ev[s + 1]);
    ctx->stage_pending = 0;
  }
  for (int i = 0; i < 6; i++)
    ms[i] = ctx->stage_ms[i];
  return OVB_OK;
}

// ------------------------------------------------------------------------------------------------ multi-GPU (features sharded)
// SURVEY.md §8e: stages A (triangulate, Jacobian, nullspace, gate) and the local compression run on this rank's feature
// shard; the ranks exchange their compressed [R_g | z_g] blocks with ONE all-gather (done by the caller, e.g. NCCL through
// torch.distributed on the stream adopted with ovb_set_stream); every rank then compresses the stack and performs the
// identical EKF update on its replica of P (bitwise identical kernels on identical inputs keep the replicas in sync).
ovb_status ovb_set_stream(ovb_ctx *ctx, void *cuda_stream) {
  if (!ctx)
    return OVB_ERR_ARG;
  if (!cuda_stream) {
    // the legacy default stream (handle 0) has no ordering with the engine's non-blocking streams: adopting it would
    // silently leave the engine on its own stream and race with the caller's collectives
    snprintf(ctx->err, sizeof(ctx->err), "ovb_set_stream: pass an explicit (non-default) CUDA stream handle");
    return OVB_ERR_ARG;
  }
  OVB_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
  OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  if (ctx->own_stream && ctx->stream)
    cudaStreamDestroy(ctx->stream);
  ctx->stream = (cudaStream_t)cuda_stream;
  ctx->own_stream = 0;
  return OVB_OK;
}

// contiguous feature ranges with (nearly) equal stacked-row counts sum(max(2M-3, 0)); bounds[world + 1]
ovb_status ovb_shard_partition(const int32_t *meas_off, int n_feats, int world, int32_t *bounds) {
  if (!meas_off || !bounds || n_feats < 0 || world < 1)
    return OVB_ERR_ARG;
  long long total = 0;
  for (int f = 0; f < n_feats; f++)
    total += std::max(2 * (meas_off[f + 1] - meas_off[f]) - 3, 0);
  bounds[0] = 0;
  long long cum = 0;
  int f = 0;
  for (int r = 1; r < world; r++) {
    const double target = (double)total * r / world;
    while (f < n_feats && (double)cum < target) { // first f with cum(f) >= target
      cum += std::max(2 * (meas_off[f + 1] - meas_off[f]) - 3, 0);
      f++;
    }
    bounds[r] = f;
  }
  bounds[world] = n_feats;
  return OVB_OK;
}

ovb_status ovb_msckf_shard_compress_range(ovb_ctx *ctx, const ovb_frame *frame, const ovb_feat_batch *feats, int f0, int f1, const ovb_opts *opts,
                                          double *R_dev, int R_cap_doubles, int *n_cols, int *ld) {
  if (!ctx || !feats || f0 < 0 || f1 < f0 || f1 > feats->n_feats)
    return OVB_ERR_ARG;
  // shallow view of features [f0, f1): pointers advanced, offsets rebased
  const int F = f1 - f0, m0 = feats->meas_off[f0], m1 = feats->meas_off[f1];
  std::vector<int32_t> moff((size_t)F + 1), koff;
  for (int f = 0; f <= F; f++)
    moff[(size_t)f] = feats->meas_off[f0 + f] - m0;
  ovb_feat_batch v = *feats;
  v.n_feats = F;
  v.n_meas = m1 - m0;
  v.meas_off = moff.data();
  v.cam = feats->cam + m0;
  v.clone = feats->clone + m0;
  v.uv = feats->uv + 2 * (size_t)m0;
  v.uvn = feats->uvn + 2 * (size_t)m0;
  if (feats->cam_keys_off && feats->cam_keys) {
    const int k0 = feats->cam_keys_off[f0];
    koff.resize((size_t)F + 1);
    for (int f = 0; f <= F; f++)
      koff[(size_t)f] = feats->cam_keys_off[f0 + f] - k0;
    v.cam_keys_off = koff.data();
    v.cam_keys = feats->cam_keys + k0;
  }
  return ovb_msckf_shard_compress(ctx, frame, &v, opts, R_dev, R_cap_doubles, n_cols, ld); // pack_inputs copies: the view may die here
}

ovb_status ovb_msckf_shard_compress(ovb_ctx *ctx, const ovb_frame *frame, const ovb_feat_batch *feats, const ovb_opts *opts, double *R_dev,
                                    int R_cap_doubles, int *n_cols, int *ld) {
  if (!ctx || !frame || !feats || !opts || !R_dev || !n_cols || !ld || ctx->N < 1)
    return OVB_ERR_ARG;
  OVB_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
  begin_launches(ctx);
  cudaEventRecord(ctx->ev[0], ctx->stream);
  Packed pk;
  ovb_opts o2 = *opts;
  o2.col_order = OVB_COLS_CANONICAL; // the column order must be fixed before sharding (SURVEY.md App. A.5)
  ovb_status st = pack_inputs(ctx, frame, feats, &o2, nullptr, &pk);
  if (st != OVB_OK)
    return st;
  cudaEventRecord(ctx->ev[1], ctx->stream); // inputs resident from here on
  *n_cols = pk.n_all;
  *ld = pk.ldH;
  if ((size_t)pk.n_all * pk.ldH > (size_t)R_cap_doubles)
    return OVB_ERR_CAPACITY;
  ctx->last_pk = pk;
  launch_cam_poses(ctx);
  launch_triangulate(ctx, pk.n_feats, pk.bv);
  launch_feature_system(ctx, pk.n_feats, pk.bv, pk.ldH, 0);
  launch_column_map(ctx, pk.n_feats, pk.bv);
  if (pk.m_total > 0)
    compress_system(ctx, o2.compress, ctx->d_Hs, pk.m_total, pk.n_all, pk.ldH, R_dev, pk.ldH); // unused rows of the block read as zero
  else
    OVB_CUDA_CHECK(ctx, cudaMemsetAsync(R_dev, 0, sizeof(double) * (size_t)pk.n_all * pk.ldH, ctx->stream));
  cudaEventRecord(ctx->ev[4], ctx->stream);
  OVB_CUDA_CHECK(ctx, cudaGetLastError());
  return OVB_OK;
}

ovb_status ovb_msckf_shard_finish(ovb_ctx *ctx, double *stacked_dev, int n_blocks, ovb_feat_out *out, double *dx, ovb_stats *stats) {
  if (!ctx || !stacked_dev || n_blocks < 1 || !dx || ctx->N < 1)
    return OVB_ERR_ARG;
  OVB_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
  const int N = ctx->N, n_all = ctx->last_pk.n_all, ld = ctx->last_pk.ldH, F = ctx->last_pk.n_feats;
  const double *Rfinal = stacked_dev;
  if (n_blocks > 1) {
    compress_system(ctx, ctx->h_opts->o.compress, stacked_dev, n_blocks * n_all, n_all, ld, ctx->d_R, ld);
    Rfinal = ctx->d_R;
  }
  launch_ekf_update(ctx, Rfinal, ld, n_all, n_all, false, ctx->h_opts->sigma_pix_sq, nullptr);
  cudaEventRecord(ctx->ev[5], ctx->stream);
  ovb_status st = enqueue_readback(ctx, F);
  if (st != OVB_OK)
    return st;
  OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  unpack_feats(ctx, F, out);
  for (int i = 0; i < N; i++)
    dx[i] = ctx->h_dx[i];
  ctx->stage_pending = 0;
  cudaEventElapsedTime(&ctx->stage_ms[5], ctx->ev[0], ctx->ev[6]);
  cudaEventElapsedTime(&ctx->stage_ms[3], ctx->ev[0], ctx->ev[4]);
  cudaEventElapsedTime(&ctx->stage_ms[4], ctx->ev[4], ctx->ev[5]);
  cudaEventElapsedTime(&ctx->stage_ms[0], ctx->ev[1], ctx->ev[5]); // inputs resident -> EKF update done (collective included)
  const DevUpdateInfo *inf = ctx->h_info;
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->n_feats_in = F;
    int used = 0, rows = 0;
    for (int f = 0; f < F; f++)
      if (ctx->h_feat[f].status == OVB_FEAT_OK) {
        used++;
        rows += 2 * (ctx->h_feat[f].m1 - ctx->h_feat[f].m0) - 3;
      }
    stats->n_feats_used = used; // this rank's shard
    stats->rows_stacked = rows;
    stats->cols_stacked = n_all;
    stats->rows_update = n_all;
    stats->neg_diag_index = inf->neg_diag_index != OVB_NO_NEG_DIAG ? inf->neg_diag_index : -1;
    stats->ms_total = ctx->stage_ms[5];
  }
  return ekf_status(ctx, inf);
}

// ------------------------------------------------------------------------------------------------ staged dense entry points
// rows scaled by 1/sqrt(Rdiag): whitening turns R = diag(Rdiag) into the identity so that compression applies
__global__ void k_whiten_rows(double *A, int ld, int m, int ncols) {
  OVB_PDL_ENTER();
  int i = blockIdx.x;
  double s = 1.0 / sqrt(A[(size_t)i * ld + ncols]); // the row's noise variance rides in column ncols
  __syncthreads();
  for (int j = threadIdx.x; j < ncols; j += blockDim.x)
    A[(size_t)i * ld + j] *= s;
}

// pinned staging buffer, grown on demand (dense H uploads are a test/microbench path, not the per-frame path)
static ovb_status ensure_stage(ovb_ctx *ctx, size_t doubles) {
  if (doubles <= ctx->stage_cap && ctx->h_stage)
    return OVB_OK;
  if (ctx->h_stage)
    cudaFreeHost(ctx->h_stage);
  ctx->h_stage = nullptr;
  ctx->stage_cap = 0;
  OVB_CUDA_CHECK(ctx, cudaMallocHost(&ctx->h_stage, sizeof(double) * doubles));
  ctx->stage_cap = doubles;
  return OVB_OK;
}

// [H | res | extra] rows into the device staging matrix; column n = res, column n+1 = extra (or 0)
static ovb_status stage_dense(ovb_ctx *ctx, const double *H, int m, int n, const double *res, const double *extra, int *ld_out) {
  int ld = (int)align_up((size_t)n + 2, 4);
  if ((size_t)std::max(m, n) * ld > ctx->Hs_cap) {
    snprintf(ctx->err, sizeof(ctx->err), "dense system %d x %d exceeds the reserved staging matrix (max_rows/max_state)", m, n);
    return OVB_ERR_CAPACITY;
  }
  ovb_status st = ensure_stage(ctx, (size_t)std::max(m, n) * ld);
  if (st != OVB_OK)
    return st;
  double *hs = ctx->h_stage;
  for (int i = 0; i < m; i++) {
    memcpy(hs + (size_t)i * ld, H + (size_t)i * n, sizeof(double) * n);
    hs[(size_t)i * ld + n] = res[i];
    for (int j = n + 1; j < ld; j++)
      hs[(size_t)i * ld + j] = 0.0;
    if (extra)
      hs[(size_t)i * ld + n + 1] = extra[i];
  }
  OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->d_Hs, hs, sizeof(double) * (size_t)m * ld, cudaMemcpyHostToDevice, ctx->stream));
  *ld_out = ld;
  return OVB_OK;
}

// [H | res] staged, compressed in `mode` (no fallback to another mode) and [R | z] unpacked
static ovb_status compress_dense(ovb_ctx *ctx, int mode, const double *H, int m, int n, const double *res, double *R_out, double *z_out) {
  if (!ctx || !H || !res || !R_out || !z_out || m < 1 || n < 1)
    return OVB_ERR_ARG;
  if (n > ctx->cfg.max_state)
    return OVB_ERR_CAPACITY;
  OVB_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
  begin_launches(ctx);
  int ld;
  ovb_status st = stage_dense(ctx, H, m, n, res, nullptr, &ld);
  if (st != OVB_OK)
    return st;
  if (mode == OVB_COMPRESS_HOUSEHOLDER_TSQR) {
    launch_tsqr(ctx, ctx->d_Hs, m, n, ld, ctx->d_R, ld);
  } else if (mode == OVB_COMPRESS_NORMAL_EQUATIONS) {
    if (!launch_compress_gram(ctx, ctx->d_Hs, m, n, ld, ctx->d_R, ld))
      return OVB_ERR_CUDA;
  } else if (!launch_compress_cholqr2(ctx, ctx->d_Hs, m, n, ld, ctx->d_R, ld)) {
    snprintf(ctx->err, sizeof(ctx->err), "ovb_compress_cholqr2: %d columns exceed what this path takes", n);
    return OVB_ERR_CAPACITY;
  }
  OVB_CUDA_CHECK(ctx, cudaGetLastError());
  double *hs = ctx->h_stage;
  OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(hs, ctx->d_R, sizeof(double) * (size_t)n * ld, cudaMemcpyDeviceToHost, ctx->stream));
  OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  for (int i = 0; i < n; i++) {
    for (int j = 0; j < n; j++)
      R_out[(size_t)i * n + j] = hs[(size_t)i * ld + j];
    z_out[i] = hs[(size_t)i * ld + n];
  }
  return OVB_OK;
}

ovb_status ovb_compress(ovb_ctx *ctx, const double *H, int m, int n, const double *res, double *R_out, double *z_out) {
  return compress_dense(ctx, OVB_COMPRESS_HOUSEHOLDER_TSQR, H, m, n, res, R_out, z_out);
}

ovb_status ovb_compress_gram(ovb_ctx *ctx, const double *H, int m, int n, const double *res, double *R_out, double *z_out) {
  return compress_dense(ctx, OVB_COMPRESS_NORMAL_EQUATIONS, H, m, n, res, R_out, z_out);
}

ovb_status ovb_compress_cholqr2(ovb_ctx *ctx, const double *H, int m, int n, const double *res, double *R_out, double *z_out) {
  return compress_dense(ctx, OVB_COMPRESS_CHOLQR2, H, m, n, res, R_out, z_out);
}

ovb_status ovb_ekf_update(ovb_ctx *ctx, const int *off, const int *sz, int nvar, const double *H, int r, const double *res, double sigma2,
                          const double *Rdiag, double *dx) {
  if (!ctx || !off || !sz || !H || !res || !dx || nvar < 1 || r < 1)
    return OVB_ERR_ARG;
  if (ctx->N < 1)
    return OVB_ERR_ARG;
  const int N = ctx->N;
  int n = 0;
  for (int i = 0; i < nvar; i++) {
    if (off[i] < 0 || sz[i] < 1 || off[i] + sz[i] > N)
      return OVB_ERR_ARG;
    n += sz[i];
  }
  if (n > OVB_MAX_COLS || n > ctx->cfg.max_state)
    return OVB_ERR_CAPACITY;
  OVB_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
  begin_launches(ctx);
  if (Rdiag)
    for (int i = 0; i < r; i++)
      if (!(Rdiag[i] > 0.0))
        return OVB_ERR_ARG;
  int ld;
  ovb_status st = stage_dense(ctx, H, r, n, res, Rdiag, &ld);
  if (st != OVB_OK)
    return st;
  DevUpdateInfo *hi = ctx->h_info;
  memset(hi, 0, sizeof(*hi));
  int c = 0;
  for (int i = 0; i < nvar; i++)
    for (int k = 0; k < sz[i]; k++)
      hi->col_state[c++] = off[i] + k;
  OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->d_info, hi, sizeof(DevUpdateInfo), cudaMemcpyHostToDevice, ctx->stream));
  const double *Hdev = ctx->d_Hs;
  int rr = r;
  double s2 = sigma2;
  if (Rdiag) {
    // whiten each row by 1/sqrt(R_ii) so that R = I; then compression is admissible (UpdaterSLAM.cpp:444 uses diagonal R)
    ovb_launch(ctx, k_whiten_rows, dim3(r), dim3(128), (size_t)0, ctx->d_Hs, ld, r, n + 1);
    s2 = 1.0;
  }
  if (r > n) {
    // more rows than columns: compress first (identical update, UpdaterMSCKF.cpp:275 does the same before EKFUpdate)
    rr = compress_system(ctx, OVB_COMPRESS_CHOLQR2, ctx->d_Hs, r, n, ld, ctx->d_R, ld);
    Hdev = ctx->d_R;
  }
  launch_ekf_update(ctx, Hdev, ld, rr, n, false, s2, nullptr);
  OVB_CUDA_CHECK(ctx, cudaGetLastError());
  OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->h_info, ctx->d_info, sizeof(DevUpdateInfo), cudaMemcpyDeviceToHost, ctx->stream));
  OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->h_dx, ctx->d_dx, sizeof(double) * (size_t)N, cudaMemcpyDeviceToHost, ctx->stream));
  OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
  for (int i = 0; i < N; i++)
    dx[i] = ctx->h_dx[i];
  return ekf_status(ctx, ctx->h_info);
}

// StateHelper::initialize on the device-resident covariance. The Givens split of the (tiny) system and the 3x3 inverse are
// host work in the reference's operation order; the gate, the augmentation and the update run on the GPU.
ovb_status ovb_cov_initialize(ovb_ctx *ctx, const int *off, const int *sz, int nvar, const double *H_R_in, const double *H_L_in,
                              const double *res_in, int r, int k, double sigma2, double chi2_mult, int *accepted, double *dx_new, double *dx) {
  if (!ctx || !off || !sz || !H_R_in || !H_L_in || !res_in || !accepted || !dx_new || !dx || nvar < 1 || k < 1 || k > 3 || r < k)
    return OVB_ERR_ARG;
  if (ctx->N < 1 || !(sigma2 > 0.0))
    return OVB_ERR_ARG;
  const int N = ctx->N;
  int n = 0;
  for (int i = 0; i < nvar; i++) {
    if (off[i] < 0 || sz[i] < 1 || off[i] + sz[i] > N)
      return OVB_ERR_ARG;
    n += sz[i];
  }
  if (n > OVB_MAX_COLS || n > ctx->cfg.max_state)
    return OVB_ERR_CAPACITY;
  if (N + k > ctx->ldP) {
    snprintf(ctx->err, sizeof(ctx->err), "initialize: covariance would grow to %d (max_state %d)", N + k, ctx->ldP);
    return OVB_ERR_CAPACITY;
  }
  OVB_CUDA_CHECK(ctx, cudaSetDevice(ctx->device));
  begin_launches(ctx);
  *accepted = 0;
  // ---- Givens split (StateHelper.cpp:429-440), row-major copies
  std::vector<double> HR(H_R_in, H_R_in + (size_t)r * n), HL(H_L_in, H_L_in + (size_t)r * k), res(res_in, res_in + r);
  auto rot = [](double c, double s, double &x, double &y) { // applyOnTheLeft(0, 1, G.adjoint()) on the pair (x, y)
    const double x0 = x, y0 = y;
    x = c * x0 - s * y0;
    y = s * x0 + c * y0;
  };
  for (int c0 = 0; c0 < k; ++c0) {
    for (int m = r - 1; m > c0; m--) {
      double gc, gs;
      make_givens(HL[(size_t)(m - 1) * k + c0], HL[(size_t)m * k + c0], gc, gs);
      for (int j = c0; j < k; j++)
        rot(gc, gs, HL[(size_t)(m - 1) * k + j], HL[(size_t)m * k + j]);
      rot(gc, gs, res[m - 1], res[m]);
      for (int j = 0; j < n; j++)
        rot(gc, gs, HR[(size_t)(m - 1) * n + j], HR[(size_t)m * n + j]);
    }
  }
  // ---- H_L^-1 of the invertible k x k block (Gauss-Jordan, partial pivoting)
  double A[9], Inv[9];
  for (int i = 0; i < k; i++)
    for (int j = 0; j < k; j++) {
      A[i * k + j] = HL[(size_t)i * k + j];
      Inv[i * k + j] = (i == j) ? 1.0 : 0.0;
    }
  for (int c0 = 0; c0 < k; c0++) {
    int piv = c0;
    for (int i = c0 + 1; i < k; i++)
      if (std::fabs(A[i * k + c0]) > std::fabs(A[piv * k + c0]))
        piv = i;
    if (!(std::fabs(A[piv * k + c0]) > 0.0)) {
      snprintf(ctx->err, sizeof(ctx->err), "initialize: H_L is rank deficient");
      return OVB_ERR_ARG;
    }
    if (piv != c0)
      for (int j = 0; j < k; j++) {
        std::swap(A[c0 * k + j], A[piv * k + j]);
        std::swap(Inv[c0 * k + j], Inv[piv * k + j]);
      }
    const double d = A[c0 * k + c0];
    for (int j = 0; j < k; j++) {
      A[c0 * k + j] /= d;
      Inv[c0 * k + j] /= d;
    }
    for (int i = 0; i < k; i++) {
      if (i == c0)
        continue;
      const double f = A[i * k + c0];
      for (int j = 0; j < k; j++) {
        A[i * k + j] -= f * A[c0 * k + j];
        Inv[i * k + j] -= f * Inv[c0 * k + j];
      }
    }
  }
  // ---- columns of the measuring variables
  DevUpdateInfo *hi = ctx->h_info;
  memset(hi, 0, sizeof(*hi));
  {
    int c = 0;
    for (int i = 0; i < nvar; i++)
      for (int q = 0; q < sz[i]; q++)
        hi->col_state[c++] = off[i] + q;
  }
  const int rup = r - k;
  const double *Hdev = nullptr;
  int ld = 0, rr = 0;
  if (rup > 0) {
    // ---- gate on the projected part: chi2 = resup' (Hup P Hup' + s2 I)^-1 resup (StateHelper.cpp:458-470)
    ovb_status st = stage_dense(ctx, HR.data() + (size_t)k * n, rup, n, res.data() + k, nullptr, &ld);
    if (st != OVB_OK)
      return st;
    OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->d_info, hi, sizeof(DevUpdateInfo), cudaMemcpyHostToDevice, ctx->stream));
    Hdev = ctx->d_Hs;
    rr = rup;
    double res2 = 0.0;
    for (int i = k; i < r; i++)
      res2 += res[i] * res[i];
    const bool compressed = rup > n;
    if (compressed) { // orthogonal compression keeps S's relevant block; the dropped rows add |z2|^2 / s2 to chi2
      launch_tsqr(ctx, ctx->d_Hs, rup, n, ld, ctx->d_R, ld);
      Hdev = ctx->d_R;
      rr = n;
    }
    std::vector<double> zh((size_t)rr), wh((size_t)rr);
    OVB_CUDA_CHECK(ctx, cudaMemcpy2DAsync(zh.data(), sizeof(double), Hdev + n, sizeof(double) * ld, sizeof(double), rr, cudaMemcpyDeviceToHost,
                                          ctx->stream)); // z: column n of Hdev
    launch_ekf_update(ctx, Hdev, ld, rr, n, true, sigma2, nullptr);
    OVB_CUDA_CHECK(ctx, cudaGetLastError());
    OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(wh.data(), ctx->d_w, sizeof(double) * (size_t)rr, cudaMemcpyDeviceToHost, ctx->stream));
    OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->h_info, ctx->d_info, sizeof(DevUpdateInfo), cudaMemcpyDeviceToHost, ctx->stream));
    OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    double chi2 = 0.0, z2 = 0.0;
    for (int i = 0; i < rr; i++) {
      chi2 += wh[(size_t)i] * wh[(size_t)i];
      z2 += zh[(size_t)i] * zh[(size_t)i];
    }
    if (compressed)
      chi2 += std::max(0.0, res2 - z2) / sigma2;
    if (ctx->h_info->not_spd)
      chi2 = NAN;
    const double chi2_check = g_chi2_table[std::min(r, OVB_CHI2_TABLE_LEN - 1)];
    if (!(chi2 <= chi2_mult * chi2_check))
      return OVB_OK; // rejected: nothing was modified
  } else {
    OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->d_info, hi, sizeof(DevUpdateInfo), cudaMemcpyHostToDevice, ctx->stream));
  }
  // ---- initialize_invertible: augment P (StateHelper.cpp:484-577); Hxinit | Inv staged in the free d_Y buffer
  {
    std::vector<double> stage((size_t)k * n + (size_t)k * k);
    for (int i = 0; i < k; i++)
      for (int j = 0; j < n; j++)
        stage[(size_t)i * n + j] = HR[(size_t)i * n + j];
    for (int i = 0; i < k * k; i++)
      stage[(size_t)k * n + i] = Inv[i];
    OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->d_Y, stage.data(), sizeof(double) * stage.size(), cudaMemcpyHostToDevice, ctx->stream));
    const bool launched = launch_cov_init_augment(ctx, k, n, ctx->d_Y, ctx->d_Y + (size_t)k * n, sigma2);
    OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream)); // `stage` is pageable host memory owned by this scope
    if (!launched) { // nothing was written: N and the covariance are unchanged
      snprintf(ctx->err, sizeof(ctx->err), "ovb_cov_initialize: covariance augmentation kernel could not be launched (N=%d, k=%d)", N, k);
      return OVB_ERR_CAPACITY;
    }
  }
  ctx->N = N + k;
  for (int q = 0; q < k; q++) {
    double acc = 0.0;
    for (int i = 0; i < k; i++)
      acc += Inv[q * k + i] * res[i];
    dx_new[q] = acc;
  }
  *accepted = 1;
  for (int i = 0; i < N + k; i++)
    dx[i] = 0.0;
  if (rup > 0) {
    // ---- EKFUpdate with the projected part on the augmented covariance (StateHelper.cpp:476-479)
    launch_ekf_update(ctx, Hdev, ld, rr, n, false, sigma2, nullptr);
    OVB_CUDA_CHECK(ctx, cudaGetLastError());
    OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->h_info, ctx->d_info, sizeof(DevUpdateInfo), cudaMemcpyDeviceToHost, ctx->stream));
    OVB_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->h_dx, ctx->d_dx, sizeof(double) * (size_t)(N + k), cudaMemcpyDeviceToHost, ctx->stream));
    OVB_CUDA_CHECK(ctx, cudaStreamSynchronize(ctx->stream));
    for (int i = 0; i < N + k; i++)
      dx[i] = ctx->h_dx[i];
    return ekf_status(ctx, ctx->h_info);
  }
  return OVB_OK;
}

} // extern "C"
