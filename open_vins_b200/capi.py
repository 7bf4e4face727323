"""ctypes view of include/ovb200.h and a thin handle on libovb200.so.

This module is plumbing: it mirrors the C structs field-for-field and loads the CUDA library. It never falls back
to a CPU implementation — if the library is missing, `load_library()` raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libovb200.so")

OVB_MAX_CAMS = 8
OVB_MAX_CLONES = 48
OVB_MAX_VARS = OVB_MAX_CLONES + 2 * OVB_MAX_CAMS
OVB_CHI2_TABLE_LEN = 2048

# ovb_status
OVB_OK, OVB_ERR_NEG_DIAG, OVB_ERR_NONFINITE, OVB_ERR_CAPACITY, OVB_ERR_CUDA, OVB_ERR_ARG, OVB_ERR_NOT_SPD = range(7)
# ovb_feat_status
(FEAT_OK, FEAT_FEW_MEAS, FEAT_TRI_COND, FEAT_TRI_DEPTH, FEAT_TRI_NAN, FEAT_GN_DEPTH, FEAT_GN_BASELINE, FEAT_GN_NAN,
 FEAT_CHI2) = range(9)
# ovb_feat_rep
(REP_GLOBAL_3D, REP_GLOBAL_FULL_INVERSE_DEPTH, REP_ANCHORED_3D, REP_ANCHORED_FULL_INVERSE_DEPTH,
 REP_ANCHORED_MSCKF_INVERSE_DEPTH, REP_ANCHORED_INVERSE_DEPTH_SINGLE) = range(6)
CAM_RADTAN, CAM_EQUI = 0, 1
COLS_REFERENCE_FIRST_SEEN, COLS_CANONICAL = 0, 1
COMPRESS_HOUSEHOLDER_TSQR, COMPRESS_NORMAL_EQUATIONS, COMPRESS_CHOLQR2 = 0, 1, 2

c_double_p = C.POINTER(C.c_double)
c_float_p = C.POINTER(C.c_float)
c_int_p = C.POINTER(C.c_int32)
c_u8_p = C.POINTER(C.c_uint8)
c_u16_p = C.POINTER(C.c_uint16)


class ovb_config(C.Structure):
    _fields_ = [("device", C.c_int), ("max_state", C.c_int), ("max_feats", C.c_int), ("max_meas", C.c_int),
                ("max_rows", C.c_int)]


class ovb_opts(C.Structure):
    _fields_ = [
        ("triangulate_1d", C.c_int), ("refine_features", C.c_int), ("max_runs", C.c_int),
        ("init_lamda", C.c_double), ("max_lamda", C.c_double), ("min_dx", C.c_double), ("min_dcost", C.c_double),
        ("lam_mult", C.c_double), ("min_dist", C.c_double), ("max_dist", C.c_double), ("max_baseline", C.c_double),
        ("max_cond_number", C.c_double),
        ("sigma_pix", C.c_double), ("chi2_multipler", C.c_double),
        ("do_fej", C.c_int), ("feat_rep", C.c_int), ("do_calib_camera_pose", C.c_int),
        ("do_calib_camera_intrinsics", C.c_int), ("col_order", C.c_int), ("compress", C.c_int),
    ]


def default_opts(**kw) -> ovb_opts:
    """Reference defaults (FeatureInitializerOptions.h:33-69, UpdaterOptions.h:32-48) with the rpng_sim yaml's
    use_fej=true, GLOBAL_3D, chi2_multipler=1."""
    o = ovb_opts(triangulate_1d=0, refine_features=1, max_runs=5, init_lamda=1e-3, max_lamda=1e10, min_dx=1e-6,
                 min_dcost=1e-6, lam_mult=10.0, min_dist=0.10, max_dist=60.0, max_baseline=40.0,
                 max_cond_number=10000.0, sigma_pix=1.0, chi2_multipler=1.0, do_fej=1, feat_rep=REP_GLOBAL_3D,
                 do_calib_camera_pose=0, do_calib_camera_intrinsics=0, col_order=COLS_REFERENCE_FIRST_SEEN,
                 compress=COMPRESS_CHOLQR2)
    for k, v in kw.items():
        if not hasattr(o, k):
            raise AttributeError(k)
        setattr(o, k, v)
    return o


class ovb_frame(C.Structure):
    _fields_ = [
        ("n_clones", C.c_int), ("n_cams", C.c_int),
        ("clone_R", c_double_p), ("clone_p", c_double_p), ("clone_R_fej", c_double_p), ("clone_p_fej", c_double_p),
        ("clone_off", c_int_p),
        ("cam_R", c_double_p), ("cam_p", c_double_p), ("cam_intr", c_double_p),
        ("cam_model", c_int_p), ("cam_ext_off", c_int_p), ("cam_intr_off", c_int_p),
    ]


class ovb_feat_batch(C.Structure):
    _fields_ = [
        ("n_feats", C.c_int), ("n_meas", C.c_int),
        ("meas_off", c_int_p), ("cam", c_u8_p), ("clone", c_u16_p), ("uv", c_float_p), ("uvn", c_float_p),
        ("cam_keys_off", c_int_p), ("cam_keys", c_u8_p),
    ]


class ovb_feat_out(C.Structure):
    _fields_ = [("status", c_int_p), ("p_FinA", c_double_p), ("p_FinG", c_double_p), ("anchor_cam", c_int_p),
                ("anchor_clone", c_int_p), ("chi2", c_double_p)]


class ovb_stats(C.Structure):
    _fields_ = [("n_feats_in", C.c_int), ("n_feats_used", C.c_int), ("rows_stacked", C.c_int),
                ("cols_stacked", C.c_int), ("rows_update", C.c_int), ("neg_diag_index", C.c_int),
                ("ms_total", C.c_float)]


class ovb_frame_quat(C.Structure):
    _fields_ = [("clone_q", c_double_p), ("cam_q", c_double_p)]


INIT_CALLBACK = C.CFUNCTYPE(None, C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int)


def _ptr(a: np.ndarray | None, typ):
    if a is None:
        return C.cast(None, typ)
    assert a.flags["C_CONTIGUOUS"], "array must be C-contiguous"
    return a.ctypes.data_as(typ)


class FrameArrays:
    """Owns the numpy arrays behind an ovb_frame (keeps them alive) — the slice of ov_msckf::State the path reads."""

    def __init__(self, clone_R, clone_p, clone_R_fej, clone_p_fej, clone_off, cam_R, cam_p, cam_intr, cam_model,
                 cam_ext_off, cam_intr_off):
        f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)
        i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)
        self.clone_R, self.clone_p = f64(clone_R), f64(clone_p)
        self.clone_R_fej, self.clone_p_fej = f64(clone_R_fej), f64(clone_p_fej)
        self.clone_off = i32(clone_off)
        self.cam_R, self.cam_p, self.cam_intr = f64(cam_R), f64(cam_p), f64(cam_intr)
        self.cam_model, self.cam_ext_off, self.cam_intr_off = i32(cam_model), i32(cam_ext_off), i32(cam_intr_off)
        self.n_clones = int(self.clone_off.shape[0])
        self.n_cams = int(self.cam_model.shape[0])

    def struct(self) -> ovb_frame:
        if getattr(self, "_st", None) is None:
            self._st = self._make_struct()
        return self._st

    def _make_struct(self) -> ovb_frame:
        return ovb_frame(self.n_clones, self.n_cams, _ptr(self.clone_R, c_double_p), _ptr(self.clone_p, c_double_p),
                         _ptr(self.clone_R_fej, c_double_p), _ptr(self.clone_p_fej, c_double_p),
                         _ptr(self.clone_off, c_int_p), _ptr(self.cam_R, c_double_p), _ptr(self.cam_p, c_double_p),
                         _ptr(self.cam_intr, c_double_p), _ptr(self.cam_model, c_int_p),
                         _ptr(self.cam_ext_off, c_int_p), _ptr(self.cam_intr_off, c_int_p))


class FeatArrays:
    """Owns the SoA arrays behind an ovb_feat_batch — the marshalled std::vector<std::shared_ptr<Feature>>."""

    def __init__(self, meas_off, cam, clone, uv, uvn, cam_keys_off=None, cam_keys=None):
        self.meas_off = np.ascontiguousarray(meas_off, dtype=np.int32)
        self.cam = np.ascontiguousarray(cam, dtype=np.uint8)
        self.clone = np.ascontiguousarray(clone, dtype=np.uint16)
        self.uv = np.ascontiguousarray(uv, dtype=np.float32).reshape(-1, 2)
        self.uvn = np.ascontiguousarray(uvn, dtype=np.float32).reshape(-1, 2)
        self.cam_keys_off = None if cam_keys_off is None else np.ascontiguousarray(cam_keys_off, dtype=np.int32)
        self.cam_keys = None if cam_keys is None else np.ascontiguousarray(cam_keys, dtype=np.uint8)
        self.n_feats = int(self.meas_off.shape[0] - 1)
        self.n_meas = int(self.cam.shape[0])
        assert int(self.meas_off[-1]) == self.n_meas

    def struct(self) -> ovb_feat_batch:
        if getattr(self, "_st", None) is None:
            self._st = self._make_struct()
        return self._st

    def _make_struct(self) -> ovb_feat_batch:
        return ovb_feat_batch(self.n_feats, self.n_meas, _ptr(self.meas_off, c_int_p), _ptr(self.cam, c_u8_p),
                              _ptr(self.clone, c_u16_p), _ptr(self.uv, c_float_p), _ptr(self.uvn, c_float_p),
                              _ptr(self.cam_keys_off, c_int_p), _ptr(self.cam_keys, c_u8_p))

    def subset(self, idx) -> "FeatArrays":
        """Feature subset/reorder (used for sharding across ranks)."""
        idx = np.asarray(idx, dtype=np.int64)
        lens = (self.meas_off[1:] - self.meas_off[:-1])[idx]
        off = np.zeros(len(idx) + 1, dtype=np.int32)
        np.cumsum(lens, out=off[1:])
        sel = np.concatenate([np.arange(self.meas_off[i], self.meas_off[i + 1]) for i in idx]) if len(idx) else \
            np.zeros(0, dtype=np.int64)
        ko = kk = None
        if self.cam_keys_off is not None:
            klens = (self.cam_keys_off[1:] - self.cam_keys_off[:-1])[idx]
            ko = np.zeros(len(idx) + 1, dtype=np.int32)
            np.cumsum(klens, out=ko[1:])
            kk = np.concatenate([self.cam_keys[self.cam_keys_off[i]:self.cam_keys_off[i + 1]] for i in idx]) \
                if len(idx) else np.zeros(0, dtype=np.uint8)
        return FeatArrays(off, self.cam[sel], self.clone[sel], self.uv[sel], self.uvn[sel], ko, kk)


class ovb_landmarks(C.Structure):
    _fields_ = [("lm_off", c_int_p), ("value", c_double_p), ("value_fej", c_double_p), ("anchor_cam", c_int_p),
                ("anchor_clone", c_int_p), ("sigma_pix", c_double_p), ("chi2_multipler", c_double_p)]


class LandmarkArrays:
    """Owns the arrays behind an ovb_landmarks: the SLAM landmarks (ov_type::Landmark) of the features in a batch."""

    def __init__(self, lm_off, value, value_fej, anchor_cam=None, anchor_clone=None, sigma_pix=None, chi2_multipler=None):
        n = len(lm_off)
        self.lm_off = np.ascontiguousarray(lm_off, dtype=np.int32)
        self.value = np.ascontiguousarray(value, dtype=np.float64).reshape(n, 3)
        self.value_fej = np.ascontiguousarray(value_fej, dtype=np.float64).reshape(n, 3)
        self.anchor_cam = np.full(n, -1, dtype=np.int32) if anchor_cam is None else np.ascontiguousarray(anchor_cam, dtype=np.int32)
        self.anchor_clone = np.full(n, -1, dtype=np.int32) if anchor_clone is None else np.ascontiguousarray(anchor_clone, dtype=np.int32)
        self.sigma_pix = None if sigma_pix is None else np.ascontiguousarray(sigma_pix, dtype=np.float64)
        self.chi2_multipler = None if chi2_multipler is None else np.ascontiguousarray(chi2_multipler, dtype=np.float64)

    def struct(self) -> ovb_landmarks:
        return ovb_landmarks(_ptr(self.lm_off, c_int_p), _ptr(self.value, c_double_p), _ptr(self.value_fej, c_double_p),
                             _ptr(self.anchor_cam, c_int_p), _ptr(self.anchor_clone, c_int_p), _ptr(self.sigma_pix, c_double_p),
                             _ptr(self.chi2_multipler, c_double_p))


class ovb_anchor_changes(C.Structure):
    _fields_ = [("n", C.c_int), ("lm_off", c_int_p), ("feat_rep", c_int_p), ("value", c_double_p), ("value_fej", c_double_p),
                ("old_cam", c_int_p), ("old_clone", c_int_p), ("new_cam", c_int_p), ("new_clone", c_int_p),
                ("new_value", c_double_p), ("new_value_fej", c_double_p)]


class AnchorChanges:
    """Owns the arrays behind an ovb_anchor_changes: the landmarks ovb_marginalize_window re-anchors, in order. new_value /
    new_value_fej are written by the call."""

    def __init__(self, lm_off, feat_rep, value, value_fej, old_cam, old_clone, new_cam, new_clone):
        n = len(lm_off)
        i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32).reshape(n)
        self.lm_off, self.feat_rep = i32(lm_off), i32(feat_rep)
        self.value = np.ascontiguousarray(value, dtype=np.float64).reshape(n, 3)
        self.value_fej = np.ascontiguousarray(value_fej, dtype=np.float64).reshape(n, 3)
        self.old_cam, self.old_clone, self.new_cam, self.new_clone = i32(old_cam), i32(old_clone), i32(new_cam), i32(new_clone)
        self.new_value = np.full((n, 3), np.nan)
        self.new_value_fej = np.full((n, 3), np.nan)

    def struct(self) -> ovb_anchor_changes:
        if getattr(self, "_st", None) is None:  # new_value / new_value_fej are written in place: the pointers stay valid
            self._st = ovb_anchor_changes(len(self.lm_off), _ptr(self.lm_off, c_int_p), _ptr(self.feat_rep, c_int_p), _ptr(self.value, c_double_p),
                                          _ptr(self.value_fej, c_double_p), _ptr(self.old_cam, c_int_p), _ptr(self.old_clone, c_int_p),
                                          _ptr(self.new_cam, c_int_p), _ptr(self.new_clone, c_int_p), _ptr(self.new_value, c_double_p),
                                          _ptr(self.new_value_fej, c_double_p))
        return self._st


class FeatOut:
    def __init__(self, n_feats: int):
        self.status = np.zeros(n_feats, dtype=np.int32)
        self.p_FinA = np.full((n_feats, 3), np.nan)
        self.p_FinG = np.full((n_feats, 3), np.nan)
        self.anchor_cam = np.full(n_feats, -1, dtype=np.int32)
        self.anchor_clone = np.full(n_feats, -1, dtype=np.int32)
        self.chi2 = np.full(n_feats, np.nan)

    def struct(self) -> ovb_feat_out:
        if getattr(self, "_st", None) is None:  # the arrays are written in place by the library: the pointers stay valid
            self._st = ovb_feat_out(_ptr(self.status, c_int_p), _ptr(self.p_FinA, c_double_p), _ptr(self.p_FinG, c_double_p),
                                    _ptr(self.anchor_cam, c_int_p), _ptr(self.anchor_clone, c_int_p), _ptr(self.chi2, c_double_p))
        return self._st

    def copy(self) -> "FeatOut":
        o = FeatOut(len(self.status))
        for k in ("status", "p_FinA", "p_FinG", "anchor_cam", "anchor_clone", "chi2"):
            getattr(o, k)[...] = getattr(self, k)
        return o


_LIB = None


def load_library(path: str | None = None) -> C.CDLL:
    """Load libovb200.so (built by open_vins_b200.build). Raises if it is missing: there is no CPU fallback."""
    global _LIB
    if _LIB is not None and path is None:
        return _LIB
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise RuntimeError(f"{p} not found — run `python -m open_vins_b200.build` (nvcc, sm_90a). "
                           "The engine has no CPU fallback.")
    lib = C.CDLL(p)
    vp = C.c_void_p
    lib.ovb_create.argtypes = [C.POINTER(ovb_config), C.POINTER(vp)]
    lib.ovb_destroy.argtypes = [vp]
    lib.ovb_destroy.restype = None
    lib.ovb_last_error.argtypes = [vp]
    lib.ovb_last_error.restype = C.c_char_p
    lib.ovb_abi_version.restype = C.c_int
    lib.ovb_opts_default.argtypes = [C.POINTER(ovb_opts)]
    lib.ovb_opts_default.restype = None
    lib.ovb_cov_set.argtypes = [vp, c_double_p, C.c_int]
    lib.ovb_cov_get.argtypes = [vp, c_double_p, C.c_int]
    lib.ovb_cov_dim.argtypes = [vp]
    lib.ovb_cov_get_marginal.argtypes = [vp, c_int_p, c_int_p, C.c_int, c_double_p]
    lib.ovb_cov_clone.argtypes = [vp, C.c_int, C.c_int, c_double_p, C.c_int]
    lib.ovb_cov_marginalize.argtypes = [vp, C.c_int, C.c_int]
    lib.ovb_cov_propagate.argtypes = [vp, C.c_int, C.c_int, c_int_p, c_int_p, C.c_int, c_double_p, c_double_p]
    lib.ovb_cov_propagate_imu.argtypes = [vp, C.c_int, C.c_int, c_double_p, c_double_p, c_double_p, C.c_int, c_int_p, c_int_p, C.c_int,
                                          C.c_int, C.c_int, c_double_p, C.c_int, c_double_p, c_double_p]
    lib.ovb_msckf_update.argtypes = [vp, C.POINTER(ovb_frame), C.POINTER(ovb_feat_batch), C.POINTER(ovb_opts),
                                     C.POINTER(ovb_feat_out), c_double_p, C.POINTER(ovb_stats)]
    lib.ovb_ekf_update.argtypes = [vp, c_int_p, c_int_p, C.c_int, c_double_p, C.c_int, c_double_p, C.c_double,
                                   c_double_p, c_double_p]
    lib.ovb_cov_initialize.argtypes = [vp, c_int_p, c_int_p, C.c_int, c_double_p, c_double_p, c_double_p, C.c_int, C.c_int, C.c_double,
                                       C.c_double, c_int_p, c_double_p, c_double_p]
    lib.ovb_slam_anchor_change.argtypes = [C.POINTER(ovb_frame), C.POINTER(ovb_opts), C.c_int, c_double_p, c_double_p, C.c_int, C.c_int, C.c_int,
                                           C.c_int, c_double_p, c_double_p, c_double_p, c_int_p, c_int_p, c_int_p, c_int_p]
    lib.ovb_marginalize_window.argtypes = [vp, C.POINTER(ovb_frame), C.POINTER(ovb_opts), c_int_p, c_int_p, C.c_int, C.POINTER(ovb_anchor_changes)]
    lib.ovb_slam_update.argtypes = [vp, C.POINTER(ovb_frame), C.POINTER(ovb_feat_batch), C.POINTER(ovb_landmarks), C.POINTER(ovb_opts),
                                    C.POINTER(ovb_feat_out), c_double_p, C.POINTER(ovb_stats)]
    lib.ovb_slam_delayed_init.argtypes = [vp, C.POINTER(ovb_frame), C.POINTER(ovb_feat_batch), C.POINTER(ovb_opts), c_double_p, c_double_p, INIT_CALLBACK,
                                          C.c_void_p, C.POINTER(ovb_feat_out), c_int_p]
    lib.ovb_slam_update_reps.argtypes = [vp, C.POINTER(ovb_frame), C.POINTER(ovb_feat_batch), C.POINTER(ovb_landmarks), c_int_p, C.POINTER(ovb_opts),
                                         C.POINTER(ovb_feat_out), c_double_p, C.POINTER(ovb_stats)]
    lib.ovb_slam_delayed_init_reps.argtypes = [vp, C.POINTER(ovb_frame), C.POINTER(ovb_feat_batch), C.POINTER(ovb_opts), c_int_p, c_double_p, c_double_p,
                                               INIT_CALLBACK, C.c_void_p, C.POINTER(ovb_feat_out), c_int_p]
    lib.ovb_slam_delayed_init_batch.argtypes = [vp, C.POINTER(ovb_frame), C.POINTER(ovb_frame_quat), C.POINTER(ovb_feat_batch), C.POINTER(ovb_opts),
                                                c_int_p, c_double_p, c_double_p, C.POINTER(ovb_feat_out), c_int_p, c_double_p, c_double_p, C.c_int]
    lib.ovb_triangulate.argtypes = [vp, C.POINTER(ovb_frame), C.POINTER(ovb_feat_batch), C.POINTER(ovb_opts),
                                    C.POINTER(ovb_feat_out)]
    lib.ovb_feature_jacobians.argtypes = [vp, C.POINTER(ovb_frame), C.POINTER(ovb_feat_batch), C.POINTER(ovb_opts),
                                          C.POINTER(ovb_feat_out), C.c_int, c_double_p, c_double_p, c_double_p,
                                          c_int_p, c_int_p, c_int_p, C.c_int]
    lib.ovb_compress.argtypes = [vp, c_double_p, C.c_int, C.c_int, c_double_p, c_double_p, c_double_p]
    lib.ovb_compress_gram.argtypes = [vp, c_double_p, C.c_int, C.c_int, c_double_p, c_double_p, c_double_p]
    lib.ovb_compress_cholqr2.argtypes = [vp, c_double_p, C.c_int, C.c_int, c_double_p, c_double_p, c_double_p]
    lib.ovb_chi2_quantile95.argtypes = [C.c_int]
    lib.ovb_chi2_quantile95.restype = C.c_double
    lib.ovb_last_stage_ms.argtypes = [vp, C.POINTER(C.c_float * 6)]
    lib.ovb_last_counters.argtypes = [vp, C.POINTER(C.c_int64 * 4)]
    lib.ovb_last_init_counters.argtypes = [vp, C.POINTER(C.c_int64 * 4)]
    lib.ovb_last_host_us.argtypes = [vp, C.POINTER(C.c_double * 4)]
    lib.ovb_set_stream.argtypes = [vp, C.c_void_p]
    lib.ovb_msckf_shard_compress.argtypes = [vp, C.POINTER(ovb_frame), C.POINTER(ovb_feat_batch), C.POINTER(ovb_opts), C.c_void_p,
                                             C.c_int, c_int_p, c_int_p]
    lib.ovb_msckf_shard_compress_range.argtypes = [vp, C.POINTER(ovb_frame), C.POINTER(ovb_feat_batch), C.c_int, C.c_int, C.POINTER(ovb_opts),
                                                   C.c_void_p, C.c_int, c_int_p, c_int_p]
    lib.ovb_shard_partition.argtypes = [c_int_p, C.c_int, C.c_int, c_int_p]
    lib.ovb_msckf_shard_finish.argtypes = [vp, C.c_void_p, C.c_int, C.POINTER(ovb_feat_out), c_double_p, C.POINTER(ovb_stats)]
    lib.ovb_set_profile.argtypes = [vp, C.c_int]
    lib.ovb_profile_read.argtypes = [vp, C.c_char_p, C.c_int, c_float_p, C.c_int, c_int_p]
    lib.ovb_set_replay.argtypes = [vp, C.c_int]
    lib.ovb_set_slam_unbounded.argtypes = [vp, C.c_int]
    lib.ovb_msckf_replay.argtypes = [vp, C.c_int, C.c_int, c_float_p, C.POINTER(C.c_float * 5)]
    if path is None:
        _LIB = lib
    return lib


EXPORTED_SYMBOLS = [
    "ovb_create", "ovb_destroy", "ovb_last_error", "ovb_abi_version", "ovb_opts_default", "ovb_cov_set", "ovb_cov_get",
    "ovb_cov_dim", "ovb_cov_get_marginal", "ovb_cov_clone", "ovb_cov_marginalize", "ovb_cov_propagate", "ovb_cov_propagate_imu", "ovb_cov_initialize",
    "ovb_msckf_update", "ovb_slam_update", "ovb_slam_update_reps", "ovb_set_slam_unbounded", "ovb_slam_delayed_init", "ovb_slam_delayed_init_reps",
    "ovb_slam_delayed_init_batch",
    "ovb_slam_anchor_change", "ovb_marginalize_window", "ovb_ekf_update", "ovb_triangulate", "ovb_feature_jacobians", "ovb_compress", "ovb_compress_gram", "ovb_compress_cholqr2",
    "ovb_chi2_quantile95", "ovb_last_stage_ms", "ovb_set_replay", "ovb_msckf_replay", "ovb_last_counters", "ovb_last_init_counters", "ovb_last_host_us", "ovb_set_profile", "ovb_profile_read",
    "ovb_set_stream", "ovb_msckf_shard_compress", "ovb_msckf_shard_compress_range", "ovb_shard_partition", "ovb_msckf_shard_finish",
]


def slam_anchor_change(frame: "FrameArrays", opts: ovb_opts, lm_off, value, value_fej, old_cam, old_clone, new_cam, new_clone, lib=None):
    """UpdaterSLAM::perform_anchor_change host math (no context, no GPU). Returns (new_value, new_value_fej, off, sz, Phi)."""
    lib = lib or load_library()
    value = np.ascontiguousarray(value, dtype=np.float64)
    value_fej = np.ascontiguousarray(value_fej, dtype=np.float64)
    nv, nvf = np.zeros(3), np.zeros(3)
    Phi = np.zeros(3 * 27)
    off, sz = np.zeros(8, dtype=np.int32), np.zeros(8, dtype=np.int32)
    n_order, n_cols = np.zeros(1, dtype=np.int32), np.zeros(1, dtype=np.int32)
    fs = frame.struct()
    st = lib.ovb_slam_anchor_change(C.byref(fs), C.byref(opts), int(lm_off), _ptr(value, c_double_p), _ptr(value_fej, c_double_p), int(old_cam),
                                    int(old_clone), int(new_cam), int(new_clone), _ptr(nv, c_double_p), _ptr(nvf, c_double_p), _ptr(Phi, c_double_p),
                                    _ptr(off, c_int_p), _ptr(sz, c_int_p), _ptr(n_order, c_int_p), _ptr(n_cols, c_int_p))
    if st != OVB_OK:
        raise OvbError(st, "ovb_slam_anchor_change: invalid arguments")
    no, nc = int(n_order[0]), int(n_cols[0])
    phisize = int(sz[no - 1])
    return nv, nvf, off[:no].copy(), sz[:no].copy(), Phi[:phisize * nc].reshape(phisize, nc).copy()


def shard_partition(meas_off, world: int, lib=None):
    """ovb_shard_partition: [(f0, f1)] * world, contiguous feature ranges balanced by stacked rows."""
    lib = lib or load_library()
    mo = np.ascontiguousarray(meas_off, dtype=np.int32)
    bounds = np.zeros(world + 1, dtype=np.int32)
    st = lib.ovb_shard_partition(_ptr(mo, c_int_p), len(mo) - 1, int(world), _ptr(bounds, c_int_p))
    if st != OVB_OK:
        raise OvbError(st, "ovb_shard_partition")
    return [(int(bounds[i]), int(bounds[i + 1])) for i in range(world)]


class OvbError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"ovb status {code}: {msg}")
        self.code = code


class Engine:
    """One ovb_ctx (one GPU, one stream). Methods are 1:1 with the C ABI."""

    def __init__(self, max_state=640, max_feats=1024, max_meas=1024 * 48, max_rows=0, device=0, lib=None):
        self.lib = lib or load_library()
        cfg = ovb_config(device, max_state, max_feats, max_meas, max_rows)
        h = C.c_void_p()
        st = self.lib.ovb_create(C.byref(cfg), C.byref(h))
        if st != OVB_OK:
            raise OvbError(st, "ovb_create failed (is a CUDA device visible?)")
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.lib.ovb_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, st, allow=()):
        if st != OVB_OK and st not in allow:
            raise OvbError(st, (self.lib.ovb_last_error(self.h) or b"").decode())
        return st

    # ---- covariance
    def cov_set(self, P):
        P = np.ascontiguousarray(P, dtype=np.float64)
        self._check(self.lib.ovb_cov_set(self.h, _ptr(P, c_double_p), P.shape[0]))

    def cov_dim(self) -> int:
        return int(self.lib.ovb_cov_dim(self.h))

    def cov_get(self):
        N = self.cov_dim()
        P = np.zeros((N, N))
        self._check(self.lib.ovb_cov_get(self.h, _ptr(P, c_double_p), N))
        return P

    def cov_get_marginal(self, off, sz):
        off = np.ascontiguousarray(off, dtype=np.int32)
        sz = np.ascontiguousarray(sz, dtype=np.int32)
        n = int(sz.sum())
        out = np.zeros((n, n))
        self._check(self.lib.ovb_cov_get_marginal(self.h, _ptr(off, c_int_p), _ptr(sz, c_int_p), len(off),
                                                  _ptr(out, c_double_p)))
        return out

    def cov_clone(self, old_off, size, dnc_dt=None, dt_off=-1):
        d = None if dnc_dt is None else np.ascontiguousarray(dnc_dt, dtype=np.float64)
        self._check(self.lib.ovb_cov_clone(self.h, old_off, size, _ptr(d, c_double_p), dt_off))

    def cov_marginalize(self, off, size):
        self._check(self.lib.ovb_cov_marginalize(self.h, off, size))

    def marginalize_window(self, frame, opts, marg_off, marg_sz, anchors=None):
        """ovb_marginalize_window: frame is a FrameArrays (or None without anchors), anchors an AnchorChanges (or None).
        Returns the status (OVB_OK or OVB_ERR_NEG_DIAG; other errors raise); the new values land in anchors."""
        marg_off = np.ascontiguousarray(marg_off, dtype=np.int32)
        marg_sz = np.ascontiguousarray(marg_sz, dtype=np.int32)
        fs = None if frame is None else C.byref(frame.struct())
        an = None if anchors is None else C.byref(anchors.struct())
        return self._check(self.lib.ovb_marginalize_window(self.h, fs, None if opts is None else C.byref(opts), _ptr(marg_off, c_int_p),
                                                           _ptr(marg_sz, c_int_p), len(marg_off), an), allow=(OVB_ERR_NEG_DIAG,))

    def cov_propagate(self, new_off, Phi, Q, old_off, old_sz):
        Phi = np.ascontiguousarray(Phi, dtype=np.float64)
        Q = np.ascontiguousarray(Q, dtype=np.float64)
        old_off = np.ascontiguousarray(old_off, dtype=np.int32)
        old_sz = np.ascontiguousarray(old_sz, dtype=np.int32)
        return self._check(self.lib.ovb_cov_propagate(self.h, new_off, Phi.shape[0], _ptr(old_off, c_int_p),
                                                      _ptr(old_sz, c_int_p), len(old_off), _ptr(Phi, c_double_p),
                                                      _ptr(Q, c_double_p)), allow=(OVB_ERR_NEG_DIAG,))

    def cov_propagate_imu(self, F, G, qc, new_off, old_off, old_sz, clone_off, clone_size, dnc_dt=None, dt_off=-1):
        """ovb_cov_propagate_imu: F [steps, n, n], G [steps, n, 12], qc [steps, 4]. Returns (status, Phi, Q); OVB_ERR_NEG_DIAG is
        returned, not raised (P then holds the propagated values and nothing was cloned)."""
        F = np.ascontiguousarray(F, dtype=np.float64)
        G = np.ascontiguousarray(G, dtype=np.float64)
        qc = np.ascontiguousarray(qc, dtype=np.float64)
        if F.ndim != 3 or F.shape[1] != F.shape[2] or G.shape != (F.shape[0], F.shape[1], 12) or qc.shape != (F.shape[0], 4):
            raise ValueError(f"F [steps, n, n], G [steps, n, 12], qc [steps, 4] expected, got {F.shape}, {G.shape}, {qc.shape}")
        steps, n = F.shape[0], F.shape[1]
        old_off = np.ascontiguousarray(old_off, dtype=np.int32)
        old_sz = np.ascontiguousarray(old_sz, dtype=np.int32)
        if old_off.shape != old_sz.shape or old_off.ndim != 1:
            raise ValueError("old_off and old_sz must be 1-D and of the same length")
        d = None if dnc_dt is None else np.ascontiguousarray(dnc_dt, dtype=np.float64)
        if d is not None and d.shape != (int(clone_size),):
            raise ValueError(f"dnc_dt must hold clone_size = {clone_size} values, got shape {d.shape}")
        Phi, Q = np.zeros((n, n)), np.zeros((n, n))
        st = self.lib.ovb_cov_propagate_imu(self.h, n, steps, _ptr(F, c_double_p), _ptr(G, c_double_p), _ptr(qc, c_double_p), int(new_off),
                                            _ptr(old_off, c_int_p), _ptr(old_sz, c_int_p), len(old_off), int(clone_off), int(clone_size),
                                            _ptr(d, c_double_p), int(dt_off), _ptr(Phi, c_double_p), _ptr(Q, c_double_p))
        self._check(st, allow=(OVB_ERR_NEG_DIAG,))
        return st, Phi, Q

    def cov_initialize(self, off, sz, H_R, H_L, res, sigma2=1.0, chi2_mult=1.0):
        """StateHelper::initialize: returns (status, accepted, dx_new[k], dx[N after the call])."""
        off = np.ascontiguousarray(off, dtype=np.int32)
        sz = np.ascontiguousarray(sz, dtype=np.int32)
        H_R = np.ascontiguousarray(H_R, dtype=np.float64)
        H_L = np.ascontiguousarray(H_L, dtype=np.float64)
        res = np.ascontiguousarray(res, dtype=np.float64)
        r, k = H_L.shape
        acc = np.zeros(1, dtype=np.int32)
        dx_new = np.zeros(k)
        dx = np.zeros(self.cov_dim() + k)
        st = self.lib.ovb_cov_initialize(self.h, _ptr(off, c_int_p), _ptr(sz, c_int_p), len(off), _ptr(H_R, c_double_p), _ptr(H_L, c_double_p),
                                         _ptr(res, c_double_p), r, k, float(sigma2), float(chi2_mult), _ptr(acc, c_int_p), _ptr(dx_new, c_double_p),
                                         _ptr(dx, c_double_p))
        self._check(st, allow=(OVB_ERR_NEG_DIAG,))
        return st, bool(acc[0]), dx_new, dx[:self.cov_dim()]

    # ---- hot path
    def msckf_update(self, frame: FrameArrays, feats: FeatArrays, opts: ovb_opts, out: FeatOut | None = None, dx: np.ndarray | None = None):
        """out / dx: caller-owned result buffers to reuse across calls (a host filter keeps them); allocated here when omitted."""
        out = out or FeatOut(feats.n_feats)
        if dx is None:
            dx = np.zeros(self.cov_dim())
        stats = ovb_stats()
        fs, bs, os_ = frame.struct(), feats.struct(), out.struct()
        st = self.lib.ovb_msckf_update(self.h, C.byref(fs), C.byref(bs), C.byref(opts), C.byref(os_),
                                       _ptr(dx, c_double_p), C.byref(stats))
        self._check(st, allow=(OVB_ERR_NEG_DIAG,))
        return st, out, dx, stats

    def slam_update(self, frame: FrameArrays, feats: FeatArrays, landmarks: "LandmarkArrays", opts: ovb_opts, feat_rep=None):
        """feat_rep: one ovb_feat_rep per landmark (Landmark::_feat_representation), or None for opts.feat_rep."""
        out = FeatOut(feats.n_feats)
        dx = np.zeros(self.cov_dim())
        stats = ovb_stats()
        fs, bs, ls, os_ = frame.struct(), feats.struct(), landmarks.struct(), out.struct()
        reps = None if feat_rep is None else np.ascontiguousarray(feat_rep, dtype=np.int32)
        st = self.lib.ovb_slam_update_reps(self.h, C.byref(fs), C.byref(bs), C.byref(ls), _ptr(reps, c_int_p), C.byref(opts), C.byref(os_),
                                           _ptr(dx, c_double_p), C.byref(stats))
        self._check(st, allow=(OVB_ERR_NEG_DIAG,))
        return st, out, dx, stats

    def set_slam_unbounded(self, enabled=True):
        """slam_update accepts batches of more than OVB_MAX_VARS state variables (off by default)"""
        self._check(self.lib.ovb_set_slam_unbounded(self.h, int(enabled)))

    def slam_delayed_init(self, frame: FrameArrays, feats: FeatArrays, opts: ovb_opts, on_init=None, sigma_pix=None, chi2_multipler=None,
                          feat_rep=None):
        """UpdaterSLAM::delayed_init in one call. on_init(feat_index, lm_off, dx_new, dx) must apply dx to the caller's state and
        refresh the arrays of `frame` IN PLACE. feat_rep: one ovb_feat_rep per feature (its class representation), or None for
        opts.feat_rep. Returns (FeatOut, lm_off array)."""
        out = FeatOut(feats.n_feats)
        lm_off = np.full(feats.n_feats, -1, dtype=np.int32)

        def _cb(user, f, off, size, dxn, dx, n):
            if on_init is not None:
                on_init(int(f), int(off), np.ctypeslib.as_array(dxn, shape=(size,)).copy(), np.ctypeslib.as_array(dx, shape=(n,)).copy())
        cb = INIT_CALLBACK(_cb)
        sp = None if sigma_pix is None else np.ascontiguousarray(sigma_pix, dtype=np.float64)
        cm = None if chi2_multipler is None else np.ascontiguousarray(chi2_multipler, dtype=np.float64)
        reps = None if feat_rep is None else np.ascontiguousarray(feat_rep, dtype=np.int32)
        self._check(self.lib.ovb_slam_delayed_init_reps(self.h, C.byref(frame.struct()), C.byref(feats.struct()), C.byref(opts), _ptr(reps, c_int_p),
                                                        _ptr(sp, c_double_p), _ptr(cm, c_double_p), cb, None, C.byref(out.struct()),
                                                        _ptr(lm_off, c_int_p)))
        return out, lm_off

    def slam_delayed_init_batch(self, frame: FrameArrays, clone_q, cam_q, feats: FeatArrays, opts: ovb_opts, sigma_pix=None, chi2_multipler=None,
                                feat_rep=None):
        """UpdaterSLAM::delayed_init in one call without a callback: the engine moves its copy of the frame between the
        features itself, from the JPL quaternions clone_q [n_clones][4] and cam_q [n_cams][4] behind frame.clone_R / cam_R.
        Returns (FeatOut, lm_off, dx_new [F][3], dx [F][N + 3F]); the caller replays them in feature order: for every f with
        lm_off[f] >= 0, the landmark at its triangulated point moved by dx_new[f][:lm_size], then every variable moved by
        dx[f][:lm_off[f] + lm_size]. Rows of features that were not initialised stay NaN."""
        F = feats.n_feats
        out = FeatOut(F)
        lm_off = np.full(F, -1, dtype=np.int32)
        ld = self.cov_dim() + 3 * F
        dx_new = np.full((F, 3), np.nan)
        dx = np.full((F, max(ld, 1)), np.nan)
        cq = np.ascontiguousarray(clone_q, dtype=np.float64).reshape(frame.n_clones, 4)
        kq = np.ascontiguousarray(cam_q, dtype=np.float64).reshape(frame.n_cams, 4)
        quat = ovb_frame_quat(_ptr(cq, c_double_p), _ptr(kq, c_double_p))
        sp = None if sigma_pix is None else np.ascontiguousarray(sigma_pix, dtype=np.float64)
        cm = None if chi2_multipler is None else np.ascontiguousarray(chi2_multipler, dtype=np.float64)
        reps = None if feat_rep is None else np.ascontiguousarray(feat_rep, dtype=np.int32)
        self._check(self.lib.ovb_slam_delayed_init_batch(self.h, C.byref(frame.struct()), C.byref(quat), C.byref(feats.struct()), C.byref(opts),
                                                         _ptr(reps, c_int_p), _ptr(sp, c_double_p), _ptr(cm, c_double_p), C.byref(out.struct()),
                                                         _ptr(lm_off, c_int_p), _ptr(dx_new, c_double_p), _ptr(dx, c_double_p), int(dx.shape[1])))
        return out, lm_off, dx_new, dx

    def triangulate(self, frame: FrameArrays, feats: FeatArrays, opts: ovb_opts):
        out = FeatOut(feats.n_feats)
        fs, bs, os_ = frame.struct(), feats.struct(), out.struct()
        self._check(self.lib.ovb_triangulate(self.h, C.byref(fs), C.byref(bs), C.byref(opts), C.byref(os_)))
        return out

    def feature_jacobians(self, frame: FrameArrays, feats: FeatArrays, opts: ovb_opts, out: FeatOut, stage: int):
        M = feats.meas_off[1:] - feats.meas_off[:-1]
        rows = int((2 * M).sum()) if stage == 0 else int(np.maximum(2 * M - 3, 0).sum())
        ld = OVB_MAX_VARS * 8
        Hf = np.zeros((rows, 3))
        Hx = np.zeros((rows, ld))
        res = np.zeros(rows)
        row_off = np.zeros(feats.n_feats + 1, dtype=np.int32)
        ncols = np.zeros(1, dtype=np.int32)
        col_index = np.full(ld, -1, dtype=np.int32)
        fs, bs, os_ = frame.struct(), feats.struct(), out.struct()
        self._check(self.lib.ovb_feature_jacobians(self.h, C.byref(fs), C.byref(bs), C.byref(opts), C.byref(os_),
                                                   stage, _ptr(Hf, c_double_p), _ptr(Hx, c_double_p),
                                                   _ptr(res, c_double_p), _ptr(row_off, c_int_p),
                                                   _ptr(ncols, c_int_p), _ptr(col_index, c_int_p), ld))
        n = int(ncols[0])
        return Hf, np.ascontiguousarray(Hx[:, :n]), res, row_off, col_index[:n].copy()

    def compress(self, H, res, mode=COMPRESS_HOUSEHOLDER_TSQR):
        H = np.ascontiguousarray(H, dtype=np.float64)
        res = np.ascontiguousarray(res, dtype=np.float64)
        m, n = H.shape
        R = np.zeros((n, n))
        z = np.zeros(n)
        fn = {COMPRESS_HOUSEHOLDER_TSQR: self.lib.ovb_compress, COMPRESS_NORMAL_EQUATIONS: self.lib.ovb_compress_gram,
              COMPRESS_CHOLQR2: self.lib.ovb_compress_cholqr2}[mode]
        self._check(fn(self.h, _ptr(H, c_double_p), m, n, _ptr(res, c_double_p), _ptr(R, c_double_p), _ptr(z, c_double_p)))
        return R, z

    def ekf_update(self, off, sz, H, res, sigma2=1.0, Rdiag=None, allow=()):
        off = np.ascontiguousarray(off, dtype=np.int32)
        sz = np.ascontiguousarray(sz, dtype=np.int32)
        H = np.ascontiguousarray(H, dtype=np.float64)
        res = np.ascontiguousarray(res, dtype=np.float64)
        Rd = None if Rdiag is None else np.ascontiguousarray(Rdiag, dtype=np.float64)
        dx = np.zeros(self.cov_dim())
        st = self.lib.ovb_ekf_update(self.h, _ptr(off, c_int_p), _ptr(sz, c_int_p), len(off), _ptr(H, c_double_p),
                                     H.shape[0], _ptr(res, c_double_p), float(sigma2), _ptr(Rd, c_double_p),
                                     _ptr(dx, c_double_p))
        self._check(st, allow=(OVB_ERR_NEG_DIAG,) + tuple(allow))
        return st, dx

    # ---- multi-GPU staged calls (device pointers are raw ints, e.g. torch.Tensor.data_ptr())
    def set_stream(self, cuda_stream_handle: int):
        self._check(self.lib.ovb_set_stream(self.h, C.c_void_p(cuda_stream_handle)))

    def shard_compress(self, frame: FrameArrays, feats: FeatArrays, opts: ovb_opts, R_dev_ptr: int, R_cap_doubles: int):
        n = np.zeros(1, dtype=np.int32)
        ld = np.zeros(1, dtype=np.int32)
        fs, bs = frame.struct(), feats.struct()
        self._keep = (frame, feats, fs, bs)  # the call is asynchronous: keep the host arrays alive until shard_finish
        self._check(self.lib.ovb_msckf_shard_compress(self.h, C.byref(fs), C.byref(bs), C.byref(opts), C.c_void_p(R_dev_ptr),
                                                      int(R_cap_doubles), _ptr(n, c_int_p), _ptr(ld, c_int_p)))
        return int(n[0]), int(ld[0])

    def shard_compress_range(self, frame: FrameArrays, feats: FeatArrays, f0: int, f1: int, opts: ovb_opts, R_dev_ptr: int, R_cap_doubles: int):
        n = C.c_int(0)
        ld = C.c_int(0)
        self._check(self.lib.ovb_msckf_shard_compress_range(self.h, C.byref(frame.struct()), C.byref(feats.struct()), int(f0), int(f1), C.byref(opts),
                                                            C.c_void_p(R_dev_ptr), int(R_cap_doubles), C.byref(n), C.byref(ld)))
        return n.value, ld.value

    def shard_finish(self, stacked_dev_ptr: int, n_blocks: int, n_feats: int):
        out = FeatOut(n_feats)
        dx = np.zeros(self.cov_dim())
        stats = ovb_stats()
        os_ = out.struct()
        st = self.lib.ovb_msckf_shard_finish(self.h, C.c_void_p(stacked_dev_ptr), int(n_blocks), C.byref(os_), _ptr(dx, c_double_p),
                                             C.byref(stats))
        self._check(st, allow=(OVB_ERR_NEG_DIAG,))
        return st, out, dx, stats

    def last_counters(self):
        a = (C.c_int64 * 4)()
        self._check(self.lib.ovb_last_counters(self.h, C.byref(a)))
        return dict(launches=int(a[0]), tsqr_level_launches=int(a[1]), h2d_bytes=int(a[2]), d2h_bytes=int(a[3]))

    def last_init_counters(self):
        """Counters of the last slam_delayed_init call: features that reached the initialisation, stream synchronisations,
        bytes host->device and device->host."""
        a = (C.c_int64 * 4)()
        self._check(self.lib.ovb_last_init_counters(self.h, C.byref(a)))
        return dict(features=int(a[0]), syncs=int(a[1]), h2d_bytes=int(a[2]), d2h_bytes=int(a[3]))

    def last_host_us(self):
        """Host wall clock of the last msckf_update in microseconds."""
        a = (C.c_double * 4)()
        self._check(self.lib.ovb_last_host_us(self.h, C.byref(a)))
        return dict(marshal_h2d_enqueue=float(a[0]), kernel_enqueue=float(a[1]), wait=float(a[2]), unpack=float(a[3]))

    def set_profile(self, enabled=True):
        self._check(self.lib.ovb_set_profile(self.h, int(bool(enabled))))

    def profile_read(self):
        """[(kernel name, microseconds)] of every kernel the last call launched, in launch order."""
        cap = 128
        while True:
            buf = C.create_string_buffer(512 * cap)  # mangled names of templated kernels run to a few hundred bytes
            us = np.zeros(cap, dtype=np.float32)
            n = np.zeros(1, dtype=np.int32)
            self._check(self.lib.ovb_profile_read(self.h, buf, len(buf), _ptr(us, c_float_p), cap, _ptr(n, c_int_p)))
            if int(n[0]) <= cap:
                break
            cap = int(n[0])
        names = buf.raw.split(b"\0")[: int(n[0])]
        return [(nm.decode(), float(us[i])) for i, nm in enumerate(names)]

    def set_replay(self, enabled=True):
        self._check(self.lib.ovb_set_replay(self.h, int(enabled)))

    def msckf_replay(self, steps, flush_l2=True):
        """Re-run the last msckf_update `steps` times on device-resident inputs. Returns (ms_per_step, stage_ms_sum)."""
        ms = np.zeros(steps, dtype=np.float32)
        st5 = (C.c_float * 5)()
        self._check(self.lib.ovb_msckf_replay(self.h, steps, int(flush_l2), _ptr(ms, c_float_p), C.byref(st5)))
        return ms, np.array([float(x) for x in st5])

    def last_stage_ms(self):
        a = (C.c_float * 6)()
        self.lib.ovb_last_stage_ms(self.h, C.byref(a))
        return [float(x) for x in a]
