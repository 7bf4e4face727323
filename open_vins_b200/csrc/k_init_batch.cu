// k_init_batch.cu — the step between two landmarks of ovb_slam_delayed_init_batch: the feature's record and the mean update
// (VioManager::apply_dx, StateHelper.cpp:185-196) of the window's poses and calibration that the next feature's Jacobians
// read. JPLQuat::update, PoseJPL::update and the additive intrinsics come from include/ovb200_math.hpp, the host's source,
// and this unit is compiled with -fmad=false: every product and sum is rounded on its own, as the host (x86-64 without FMA
// contraction) rounds it, so the moved frame has the bits a host that applies dx and marshals its state again would upload.
#include "ovb_internal.cuh"
#include "../../include/ovb200_math.hpp"

namespace {

using ovb200::Mat3;
using ovb200::Vec4;

// JPLQuat::update (types/JPLQuat.h:114-126): q <- quatnorm([dθ/2; 1]) ⊗ q, then R = quat_2_Rot(q) (JPLQuat::set_value)
__device__ void jpl_update(double q[4], double R[9], const double *d) {
  const Vec4 dq = ovb200::quatnorm({.5 * d[0], .5 * d[1], .5 * d[2], 1.0});
  const Vec4 nq = ovb200::quat_multiply(dq, {q[0], q[1], q[2], q[3]});
  const Mat3 nR = ovb200::quat_2_Rot(nq);
  for (int i = 0; i < 4; i++)
    q[i] = nq[i];
  for (int i = 0; i < 9; i++)
    R[i] = nR[i];
}

#define IC_THREADS 128
#define IC_CAM0 64 // first thread of the cameras (threads 0..47 take the clones)
static_assert(OVB_MAX_CLONES <= IC_CAM0 && IC_CAM0 + OVB_MAX_CAMS <= IC_THREADS, "one thread per frame variable");

__global__ void __launch_bounds__(IC_THREADS) k_init_commit(DevFrame *__restrict__ fr, DevInitBatch *__restrict__ ib, DevInitRec *__restrict__ rec,
                                                            double *__restrict__ dx_row, const DevInitSys *__restrict__ sys,
                                                            const DevUpdateInfo *__restrict__ info, const double *__restrict__ dx, int k, int calib_pose,
                                                            int calib_intr) {
  OVB_PDL_ENTER();
  const int tid = threadIdx.x;
  const int N0 = ib->N;
  // a skipped update (gate rejection or a failure of the system) reports not_spd from k_ekf_prep: only an update that ran
  // can fail on its own
  const bool ekf_failed = !sys->skip && (info->not_spd || info->nonfinite || info->neg_diag_index != OVB_NO_NEG_DIAG);
  const bool accepted = !sys->skip && !ekf_failed;
  if (tid == 0) {
    rec->status = sys->status;
    rec->lm_off = accepted ? N0 : -1;
    rec->fail = sys->fail ? sys->fail : (ekf_failed ? 3 : 0);
    rec->n = sys->n;
    rec->not_spd = info->not_spd, rec->nonfinite = info->nonfinite, rec->neg_diag_index = info->neg_diag_index;
    rec->chi2 = sys->chi2;
    for (int q = 0; q < 3; q++)
      rec->dx_new[q] = sys->dx_new[q];
  }
  if (!accepted)
    return;
  for (int i = tid; i < N0 + k; i += IC_THREADS)
    dx_row[i] = dx[i];
  if (tid < fr->n_clones) { // PoseJPL::update (types/PoseJPL.h:74-91)
    const int c = tid, off = fr->slot_off[fr->clone_slot[c]];
    jpl_update(ib->clone_q[c], fr->clone_R[c], dx + off);
    for (int j = 0; j < 3; j++)
      fr->clone_p[c][j] += dx[off + 3 + j];
    if (ib->fej_R_is_value)
      for (int j = 0; j < 9; j++)
        fr->clone_R_fej[c][j] = fr->clone_R[c][j];
    if (ib->fej_p_is_value)
      for (int j = 0; j < 3; j++)
        fr->clone_p_fej[c][j] = fr->clone_p[c][j];
  } else if (tid >= IC_CAM0 && tid - IC_CAM0 < fr->n_cams) {
    const int c = tid - IC_CAM0;
    if (calib_pose) {
      const int off = fr->slot_off[fr->cam_ext_slot[c]];
      jpl_update(ib->cam_q[c], fr->cam_R[c], dx + off);
      for (int j = 0; j < 3; j++)
        fr->cam_p[c][j] += dx[off + 3 + j];
    }
    if (calib_intr) {
      const int off = fr->slot_off[fr->cam_intr_slot[c]];
      for (int j = 0; j < 8; j++)
        fr->cam_intr[c][j] += dx[off + j];
    }
  }
  __syncthreads(); // every thread has read N0
  if (tid == 0)
    ib->N = N0 + k;
}

} // namespace

void launch_init_commit(ovb_ctx *ctx, DevInitBatch *ib, DevInitRec *rec, double *dx_row, int k, int calib_pose, int calib_intr) {
  ovb_launch(ctx, k_init_commit, dim3(1), dim3(IC_THREADS), (size_t)0, ctx->d_frame, ib, rec, dx_row, (const DevInitSys *)ctx->d_init,
             (const DevUpdateInfo *)ctx->d_info, (const double *)ctx->d_dx, k, calib_pose, calib_intr);
}
