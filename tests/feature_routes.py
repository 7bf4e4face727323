"""Pure-Python mirror of the host-side routing of the per-feature kernel k_feature_system (csrc/k_feature.cu), so that
tests can choose track lengths that reach a given layout (tile, BIG, long-track) of a given instantiation, and an
extended-precision reference of the kernel's Mahalanobis gate.

Mirrored, line for line:
  ct_view_doubles        doubles of the tile Cholesky's working set          chol_tiles.cuh:37-39
  feature_dims           column / slot counts of the per-CTA tables          k_feature.cu:1247-1254
  feature_smem_bytes     dynamic shared memory of one launch                 k_feature.cu:1256-1284
  feature_nblk           Jacobian blocks per measurement (3, 5 or 6)         k_feature.cu:1299-1303
  FT_INIT_NBLK           the delayed initialisation's blocks (5)             k_feature.cu:1316
  feature_path           tile / BIG / long-track layout of one track         k_feature.cu:1306-1313
  FT_SMEM_LIMIT          dynamic shared memory of one CTA                    k_feature.cu:1243
  launch_feature_system  the schedule split into launches, the size classes
                         of the tile layout and the BIG / long grid clamps   k_feature.cu:1372-1441
  feature_long_slice_doubles, feature_scratch_reserve (the long-track slice) k_feature.cu:1288-1297, 1318-1331
  the frame's n_all and slot count (clones + calibration blocks)             ovb_api.cu:497-551
A change to any of them has to be repeated here; tests/test_feature_routes_cpu.py checks the mirror's invariants.
"""
from __future__ import annotations

from functools import lru_cache
from typing import NamedTuple

import numpy as np

FT_THREADS = 256
FT_WARPS = FT_THREADS // 32
FT_SMEM_LIMIT = 227 * 1024
CT_XP = 12
OVB_MAX_VARS = 64
OVB_BIG_MAX_MEAS = 128
OVB_MAX_MEAS_PER_FEAT = 384
FT_INIT_NBLK = 5

TILE, BIG, LONG = 0, 1, 2
ROUTE_NAMES = {TILE: "tile", BIG: "big", LONG: "long"}

# ovb_feat_rep (include/ovb200.h)
REP_GLOBAL_3D, REP_ANCHORED_3D, REP_ANCHORED_MSCKF_INVERSE_DEPTH, REP_SINGLE = 0, 2, 4, 5


class Instance(NamedTuple):
    """One way the per-feature kernel is instantiated and fed: MSCKF (ovb_msckf_update / ovb_feature_jacobians), SLAM
    (ovb_slam_update) or INIT (ovb_slam_delayed_init), with the representation the tests give its features."""
    name: str
    kind: str  # "msckf", "slam" or "init"
    rep: int
    lm_w: int  # SLAM: the widest landmark of the batch (the frame tables grow by it)

    @property
    def slam(self) -> bool:
        return self.kind == "slam"

    @property
    def nblk(self) -> int:
        if self.kind == "init":
            return FT_INIT_NBLK
        return 6 if self.slam else (3 if self.rep in (REP_GLOBAL_3D, 1) else 5)

    @property
    def single(self) -> bool:
        return self.rep == REP_SINGLE and self.kind != "msckf"

    def dof(self, M: int) -> int:
        """Degrees of freedom of the gate's threshold, as the oracle counts them (oracle/ovo_core.hpp:1047, 1205, 1319):
        the rows of the nullspace-projected MSCKF system (2M - 3), of the SLAM system (2M; SINGLE: 2M - 2 after the bearing
        projection) and of StateHelper::initialize's input (2M; SINGLE: 2M - 2)."""
        if self.kind == "msckf":
            return 2 * M - 3
        return 2 * M - 2 if self.single else 2 * M

    @property
    def mangled(self) -> str:
        """The template arguments <SLAM, BIG, LONG, INIT> of every layout as they appear in the mangled kernel name."""
        b = lambda v: f"Lb{int(v)}E"
        return {r: "k_feature_systemI" + b(self.slam) + b(r != TILE) + b(r == LONG) + b(self.kind == "init") + "E" for r in (TILE, BIG, LONG)}


INSTANCES = (
    Instance("msckf_global", "msckf", REP_GLOBAL_3D, 0),
    Instance("msckf_anchored", "msckf", REP_ANCHORED_3D, 0),
    Instance("slam_3wide", "slam", REP_ANCHORED_MSCKF_INVERSE_DEPTH, 3),
    Instance("slam_single", "slam", REP_SINGLE, 1),
    Instance("init_3wide", "init", REP_ANCHORED_3D, 0),
    Instance("init_single", "init", REP_SINGLE, 0),
)
INSTANCE = {i.name: i for i in INSTANCES}


class FeatDims(NamedTuple):
    n_all: int
    n_slots: int
    nsv: int


def frame_dims(frame, do_calib_camera_pose: bool, do_calib_camera_intrinsics: bool) -> tuple[int, int]:
    """(n_all, n_slots) of a FrameArrays: one slot per clone (6 columns) and per calibrated camera block (6 / 8). A camera
    without a block while its calibration is on is refused, as the host refuses the frame."""
    n_slots, n_all = frame.n_clones, 6 * frame.n_clones
    for k in range(frame.n_cams):
        if do_calib_camera_pose:
            assert frame.cam_ext_off[k] >= 0, f"do_calib_camera_pose set but cam_ext_off[{k}] < 0"
            n_slots, n_all = n_slots + 1, n_all + 6
        if do_calib_camera_intrinsics:
            assert frame.cam_intr_off[k] >= 0, f"do_calib_camera_intrinsics set but cam_intr_off[{k}] < 0"
            n_slots, n_all = n_slots + 1, n_all + 8
    return n_all, n_slots


def window_dims(n_cams: int, n_clones: int, calib: bool = True) -> tuple[int, int]:
    """frame_dims of a window of n_clones clone poses and n_cams cameras, all calibrated or none"""
    return 6 * n_clones + (14 * n_cams if calib else 0), n_clones + (2 * n_cams if calib else 0)


def ct_view_doubles(NRB: int) -> int:
    return (NRB * (NRB + 1)) // 2 * 64 + 2 * NRB * 8 * CT_XP + NRB * 8 + 128 + 64 + 2 * CT_XP


def feature_dims(n_all: int, n_slots: int, inst: Instance) -> FeatDims:
    if inst.slam:
        return FeatDims(n_all + inst.lm_w, n_slots + 1, OVB_MAX_VARS + 4)
    return FeatDims(n_all, n_slots, OVB_MAX_VARS)


def feature_smem_bytes(maxM: int, dm: FeatDims, nblk: int, path: int) -> int:
    o = 0
    n_all8 = (dm.n_all + 7) & ~7
    if path != LONG:
        o += 8 * (16 * nblk + 1) * maxM
        o += 8 * 6 * maxM
        o += 8 * 2 * maxM
        o += 8 * 3 * 2 * maxM
    o += 8 * 3 * (dm.n_all + 1)
    o += 8 * (FT_WARPS * 12 + 24)
    o += 4 * dm.nsv * 2
    o += 4 * 8
    o += 2 * n_all8 * 2
    o += n_all8 * 2
    o += dm.nsv
    if path != LONG:
        o += maxM * 8
        o += ((maxM + 7) & ~7) * 2
        o += maxM * ((dm.n_slots + 3) & ~3)
    o = (o + 15) & ~15
    o += 8 * FT_WARPS * 2 * dm.n_all
    if path == TILE:
        o += 8 * ct_view_doubles((2 * maxM + 4 + 7) >> 3)
    return o


def feature_long_slice_doubles(maxM: int, n_slots: int, nblk: int) -> int:
    g = 8 * (16 * nblk + 1) * maxM
    g += 8 * (6 + 2 + 6) * maxM
    g += maxM * 8
    g += ((maxM + 7) & ~7) * 2
    g += maxM * ((n_slots + 3) & ~3)
    g = (g + 15) & ~15
    rows = 2 * maxM
    return g // 8 + (rows + 1) * (rows | 1)


def feature_path(M: int, dm: FeatDims, nblk: int, smem_limit: int = FT_SMEM_LIMIT) -> int:
    m = max(M, 2)
    if feature_smem_bytes(m, dm, nblk, TILE) <= smem_limit:
        return TILE
    if m <= OVB_BIG_MAX_MEAS and feature_smem_bytes(m, dm, nblk, BIG) <= smem_limit:
        return BIG
    return LONG


def path_of(inst: Instance, M: int, n_all: int, n_slots: int) -> int:
    return feature_path(M, feature_dims(n_all, n_slots, inst), inst.nblk)


def find_M(inst: Instance, route: int, n_all: int, n_slots: int, last: bool = False) -> int | None:
    """The shortest (last=True: longest) track, 2..OVB_MAX_MEAS_PER_FEAT measurements, that runs on `route`, or None."""
    Ms = [M for M in range(2, OVB_MAX_MEAS_PER_FEAT + 1) if path_of(inst, M, n_all, n_slots) == route]
    return (Ms[-1] if last else Ms[0]) if Ms else None


def tile_headroom(inst: Instance, n_all: int, n_slots: int) -> int:
    """Bytes of shared memory left below the limit by the last tile length"""
    MT = find_M(inst, TILE, n_all, n_slots, last=True)
    return FT_SMEM_LIMIT - feature_smem_bytes(MT, feature_dims(n_all, n_slots, inst), inst.nblk, TILE)


@lru_cache(maxsize=None)
def tight_window(inst: Instance, below: int = 1024) -> tuple[int, int]:
    """The calibrated window (cameras, clone poses) of fewest measurements per full track that holds a track one longer
    than the last tile length and whose last tile length leaves less than `below` bytes of headroom: there, a limit or a
    byte count that is off by that much moves the tile / BIG boundary."""
    best = None
    for n_cams in range(1, 9):
        for n_clones in range(2, 49):
            n_all, n_slots = window_dims(n_cams, n_clones)
            if n_cams * n_clones <= find_M(inst, TILE, n_all, n_slots, last=True) or tile_headroom(inst, n_all, n_slots) >= below:
                continue
            if best is None or n_cams * n_clones < best[0] * best[1]:
                best = (n_cams, n_clones)
    return best


class Launch(NamedTuple):
    path: int
    lo: int
    hi: int
    stream: int
    grid: int
    maxM: int


def launch_plan(lengths, inst: Instance, n_all: int, n_slots: int, sm_count: int, feat_classes: int = 1,
                long_cap: int | None = None) -> list[Launch]:
    """The launches launch_feature_system makes for a batch of tracks of `lengths` measurements (input order); the
    schedule is longest-first. long_cap: doubles of the long-track scratch (default: what feature_scratch_reserve makes
    for this batch in a fresh context)."""
    assert inst.kind != "init", "the delayed initialisation launches one CTA per feature (launch_feature_init)"
    dm = feature_dims(n_all, n_slots, inst)
    nblk = inst.nblk
    sched = sorted(lengths, reverse=True)
    n = len(sched)
    path = [feature_path(M, dm, nblk) for M in sched]
    b_big = sum(1 for p in path if p == LONG)
    b_tile = b_big + sum(1 for p in path if p == BIG)
    assert path == sorted(path, reverse=True), "the path is monotone in the track length"
    lst = []

    def add(p, lo, hi, stream):
        if hi > lo:
            lst.append((p, lo, hi, stream))
    add(LONG, 0, b_big, 0)
    add(BIG, b_big, b_tile, 0)
    has_long = b_tile > 0
    if not inst.slam and feat_classes and n - b_tile > sm_count:
        thr = (32, 16)
        bound = [b_tile, n, n, n]
        c = 0
        for i in range(b_tile, n):
            if c >= 2:
                break
            while c < 2 and sched[i] <= thr[c]:
                c += 1
                bound[c] = i
        add(TILE, bound[0], bound[1], 1 if has_long else 0)
        add(TILE, bound[1], bound[2], 2 if has_long else 1)
        add(TILE, bound[2], bound[3], 2)
    else:
        add(TILE, b_tile, n, 0)
    if long_cap is None and b_big:
        long_cap = feature_long_slice_doubles(sched[0], dm.n_slots, nblk) * min(b_big, sm_count)
    out = []
    for p, lo, hi, s in lst:
        cM = min(max(sched[lo], 2), OVB_MAX_MEAS_PER_FEAT)
        grid = hi - lo
        if p == BIG:
            grid = min(grid, 2 * sm_count)  # ctx->scratch_ctas (ovb_api.cu:170)
        elif p == LONG:
            grid = min(grid, sm_count, long_cap // feature_long_slice_doubles(cM, dm.n_slots, nblk))
        out.append(Launch(p, lo, hi, s, grid, cM))
    return out


# ------------------------------------------------------------------------------------------------------------ tracks
def cut_tracks(feats, lengths, prefix: bool = False):
    """A FeatArrays whose feature f keeps exactly lengths[f] of its measurements: evenly spread over the track (every
    camera and clone pose it has, for a wide baseline), or its first lengths[f] (prefix=True: the first camera's oldest
    clone poses, a short baseline). The kept measurements stay in their order, so every camera's measurements stay
    contiguous and the camera grouping remains valid (the index technique of test_track_over_the_limit_is_refused)."""
    from open_vins_b200 import capi
    idx, meas_off = [], [0]
    for f, M in enumerate(lengths):
        a, b = int(feats.meas_off[f]), int(feats.meas_off[f + 1])
        L = b - a
        assert 1 <= M <= L, f"feature {f}: {M} measurements wanted, the track has {L}"
        keep = np.arange(M) if prefix else np.rint(np.linspace(0, L - 1, M)).astype(np.int64)  # distinct: spacing >= 1
        idx.append(a + keep)
        meas_off.append(meas_off[-1] + M)
    idx = np.concatenate(idx)
    return capi.FeatArrays(np.array(meas_off, dtype=np.int64), feats.cam[idx], feats.clone[idx], feats.uv[idx], feats.uvn[idx])


# ------------------------------------------------------------------------------------------------------------ reference
LD = np.longdouble


def _chol_rhs(S, R):
    """Upper Cholesky factor U (U'U = S) of an SPD long-double matrix, with the right-hand sides R carried along:
    returns U^-T R. Asserts positive pivots."""
    m = S.shape[0]
    A = np.concatenate([np.array(S, dtype=LD), np.array(R, dtype=LD).reshape(m, -1)], axis=1)
    for k in range(m):
        d = A[k, k]
        assert d > 0, "reference matrix not positive definite"
        A[k, k:] /= np.sqrt(d)
        A[k + 1:, k + 1:] -= np.outer(A[k, k + 1:m], A[k, k + 1:])
    return A[:, m:]


def gate_chi2_ref(H, B, res, P, sig2):
    """chi2 = r_o' (Q2' S Q2)^-1 r_o in long double, with S = H P H' + sig2 I and Q2 an orthonormal basis of the complement
    of range(B) (B: the projected-out columns of H_f; none for a 3-wide SLAM landmark), evaluated as
    a'a - (C'a)' (C'C)^-1 (C'a) with a = L^-1 r, C = L^-1 B, S = L L'.
    Returns (chi2, kappa): kappa the 2-norm condition number of Q2' S Q2 (float64)."""
    Hl, Pl = np.array(H, dtype=LD), np.array(P, dtype=LD)
    m = Hl.shape[0]
    S = (Hl @ Pl) @ Hl.T + LD(sig2) * np.eye(m, dtype=LD)
    k = 0 if B is None else B.shape[1]
    rhs = np.array(res, dtype=LD).reshape(m, 1) if k == 0 else np.concatenate([np.array(res, dtype=LD).reshape(m, 1), np.array(B, dtype=LD)], axis=1)
    X = _chol_rhs(S, rhs)
    a = X[:, 0]
    chi2 = a @ a
    if k:
        C = X[:, 1:]
        y = _chol_rhs(C.T @ C, C.T @ a)[:, 0]
        chi2 -= y @ y
    S64 = S.astype(np.float64)
    if k:
        Q = np.linalg.qr(np.asarray(B, dtype=np.float64), mode="complete")[0][:, k:]
        S64 = Q.T @ S64 @ Q
    return float(chi2), float(np.linalg.cond(S64))


def projected_invariants_ref(Hx, Hf, res):
    """Ho'Ho, Ho'ro, ro'ro of the MSCKF nullspace projection in long double: Ho = Pi Hx, ro = Pi r with Pi the orthogonal
    projector onto the complement of range(Hf) (independent of the basis the kernel's reflectors pick)."""
    Hxl, Hfl, rl = (np.array(a, dtype=LD) for a in (Hx, Hf, res))
    X = np.concatenate([Hxl, rl.reshape(-1, 1)], axis=1)
    Y = _chol_rhs(Hfl.T @ Hfl, Hfl.T @ X)  # U^-T Hf' X: X' Hf (Hf'Hf)^-1 Hf' X = Y'Y
    G = X.T @ X - Y.T @ Y
    n = Hx.shape[1]
    return G[:n, :n], G[:n, n], G[n, n]


def gate_threshold(dof: int) -> float:
    from oracle import ovo_py
    tab = ovo_py.chi2_table()
    return float(tab[min(dof, len(tab) - 1)])
