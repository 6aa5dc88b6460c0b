"""CPU restatement of module::frame_tracker::motion_based_track (test infrastructure): loads tests/motion_track_oracle.c, compiled on first
use into a temporary directory (the tree is never written), and composes it with the oracle's stages.

  reproject(camera, pose_cw, pos_w, bounds)   camera::*::reproject_to_image for all four models
  direction(pose_cw, last_pose_cw, ...)       assume_forward / assume_backward of projection.cc:98-116
  motion_based_track(camera, kps, desc, ...)  undistort_keypoints -> query build -> match_guided mode 1 (twice when short) ->
                                              pose_optimize -> discard_outliers, stage by stage
"""
import ctypes as C

import numpy as np

from oracle import pyoracle as O

import camera_models_oracle as CMO
import cbuild

_lib = None


def lib():
    global _lib
    if _lib is None:
        L = cbuild.load("motion_track_oracle.c")
        L.mto_reproject.argtypes = [C.c_int] + [C.c_double] * 7 + [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.mto_reproject.restype = None
        _lib = L
    return _lib


def _g(camera, k):
    return float(camera.get(k, 0.0))


def default_bounds(camera):
    return tuple(float(v) for v in CMO.image_bounds(camera)) if CMO.model_of(camera) >= 2 else (0.0, _g(camera, "cols"), 0.0, _g(camera, "rows"))


def reproject(camera, pose_cw, pos_w, bounds):
    """(in_image bool (n,), reproj (n, 2) float64, x_right (n,) float32)."""
    pos = np.ascontiguousarray(pos_w, np.float64).reshape(-1, 3)
    n = len(pos)
    T = np.asarray(pose_cw, np.float64).reshape(4, 4)
    Rt = np.ascontiguousarray(np.concatenate([T[:3, :3].reshape(9), T[:3, 3]]))
    b = np.ascontiguousarray(bounds, np.float32)
    ok, rp, xr = np.zeros(max(n, 1), np.uint8), np.zeros((max(n, 1), 2)), np.zeros(max(n, 1), np.float32)
    lib().mto_reproject(CMO.model_of(camera), *[_g(camera, k) for k in ("fx", "fy", "cx", "cy", "fxb", "cols", "rows")], b.ctypes.data, Rt.ctypes.data,
                        n, pos.ctypes.data, ok.ctypes.data, rp.ctypes.data, xr.ctypes.data)
    return ok[:n].astype(bool), rp[:n], xr[:n]


def direction(pose_cw, last_pose_cw, true_baseline, monocular):
    """(assume_forward, assume_backward) of projection.cc:98-116, in the order of the reference's Eigen products (Python floats: IEEE
    double, one rounding per operation)."""
    if monocular:
        return False, False
    T, Lp = np.asarray(pose_cw, np.float64).reshape(4, 4), np.asarray(last_pose_cw, np.float64).reshape(4, 4)
    R, t = T[:3, :3].tolist(), T[:3, 3].tolist()
    tw = [(-R[0][r]) * t[0] + (-R[1][r]) * t[1] + (-R[2][r]) * t[2] for r in range(3)]
    L = Lp.tolist()
    z = L[2][0] * tw[0] + L[2][1] * tw[1] + L[2][2] * tw[2] + L[2][3]
    return z > true_baseline, -z > true_baseline


def motion_based_track(camera, kps, desc, frame, scale_factors, inv_level_sigma_sq, margin=20.0, num_matches_thr=10, true_baseline=0.0,
                       monocular=True, img_bounds=None, grid=(64, 48), thr=100, num_trials_robust=2, num_trials=2, num_each_iter=10,
                       undistort_fn=None, match_fn=None, pose_fn=None):
    """frame_tracker::motion_based_track with match::projection(0.9, true), stage by stage.  kps / desc: the current frame's (distorted)
    keypoints and descriptors; frame: the dict stella_vslam_b200.tracking.frame_tracker.pack takes.  Returns the dict of
    frame_tracker.motion_based_track.  undistort_fn / match_fn / pose_fn replace the oracle's undistort_keypoints, match_guided and
    pose_optimize (same arguments and results), e.g. by the stage-by-stage device ABI."""
    kps = np.ascontiguousarray(kps, O.KP_DTYPE)
    n_kp = len(kps)
    tb = frame["table"]
    pos = np.asarray(tb["pos_w"], np.float64).reshape(-1, 3)
    n_lm = len(pos)
    sf = np.asarray(scale_factors, np.float32)
    num_levels = len(sf)
    und, _ = (undistort_fn or CMO.undistort_keypoints)(camera, kps)
    bounds = tuple(float(v) for v in img_bounds) if img_bounds is not None else default_bounds(camera)
    pose = np.asarray(frame["pose_cw"], np.float64).reshape(4, 4)
    fwd, bwd = direction(pose, frame.get("last_pose_cw"), true_baseline, monocular)
    ok, rp, xr_q = reproject(camera, pose, pos, bounds)
    octv = np.asarray(tb["octave"], np.int64)
    lo, hi = np.maximum(0, octv - 1), np.minimum(num_levels - 1, octv + 1)
    if fwd:
        lo = octv.copy()
    elif bwd:
        hi = octv.copy()
    has_obs = np.ones(n_lm, np.uint8) if tb.get("has_observation") is None else np.asarray(tb["has_observation"], np.uint8)
    xr = frame.get("kp_x_right")

    def search(m):
        pr = dict(t_x=und["x"], t_y=und["y"], t_octave=und["octave"].astype(np.uint8), t_angle=und["angle"], t_desc=np.ascontiguousarray(desc, np.uint8),
                  t_x_right=xr, t_occupied=np.zeros(n_kp, np.uint8), bounds=bounds, grid=grid,
                  q_desc=np.ascontiguousarray(tb["desc"], np.uint8).reshape(-1, 32), q_x=rp[:, 0].astype(np.float32), q_y=rp[:, 1].astype(np.float32),
                  q_margin=np.float32(m) * sf[octv], q_min_level=lo, q_max_level=hi, q_x_right=xr_q, q_angle=np.asarray(tb["angle"], np.float32),
                  q_valid=ok.astype(np.uint8), q_has_observation=has_obs)
        out, _, n = (match_fn or O.match_guided)(pr, 1, thr=thr, lowe_ratio=0.9, check_orientation=True)
        return out, int(n)

    match_out, n_first = search(margin)
    n_matches, retried = n_first, n_first < num_matches_thr
    if retried:                                                  # frame_tracker.cc:32-36: erase_landmarks, twice the margin
        match_out, n_matches = search(np.float32(2 * np.float32(margin)))
    kp_lm = np.full(n_kp, -1, np.int32)
    for q in range(n_lm):                                        # curr_frm.add_landmark in iteration order (projection.cc:202)
        if match_out[q] >= 0:
            kp_lm[match_out[q]] = q
    out_pose = pose.copy()
    gate = n_matches >= num_matches_thr
    idx = np.nonzero(kp_lm >= 0)[0]
    if gate and len(idx) >= 5:                                   # pose_optimizer_g2o.cc:116-118 below 5 edges
        xrk = np.full(n_kp, -1.0, np.float32) if xr is None else np.asarray(xr, np.float32)
        isig = np.asarray(inv_level_sigma_sq, np.float32)
        chi = np.float32(np.sqrt(np.float32(5.99146))) if monocular else np.float32(np.sqrt(np.float32(7.81473)))
        cam = dict(model=1 if CMO.model_of(camera) == 1 else 0, fx=_g(camera, "fx"), fy=_g(camera, "fy"), cx=_g(camera, "cx"), cy=_g(camera, "cy"),
                   fxb=_g(camera, "fxb"), cols=_g(camera, "cols"), rows=_g(camera, "rows"))
        ne = len(idx)
        pp = dict(pose_cw=pose.reshape(1, 4, 4), pose_fixed=np.zeros(1, np.uint8), points=pos[kp_lm[idx]].reshape(-1, 3), point_fixed=np.ones(ne, np.uint8),
                  e_pose=np.zeros(ne, np.int32), e_point=np.arange(ne, dtype=np.int32), e_cam=np.zeros(ne, np.uint8),
                  e_obs=np.stack([und["x"][idx], und["y"][idx], xrk[idx]], 1).astype(np.float32), e_inv_sigma_sq=isig[und["octave"][idx].astype(np.int64)],
                  e_delta=np.full(ne, chi, np.float32), e_robust=None, e_can_be_outlier=None, cams=[cam])
        _, out_pose, flags = (pose_fn or O.pose_optimize)(pp, num_trials_robust, num_trials, num_each_iter)
        kp_lm[idx[flags]] = -1                                   # discard_outliers (frame_tracker.cc:133-150)
    n_valid = int((kp_lm >= 0).sum())
    return dict(kp_landmark=kp_lm, pose_cw=out_pose, n_keypoints=n_kp, n_matches_first=n_first, n_matches=n_matches, retried=bool(retried),
                n_valid=n_valid, tracked=bool(gate and n_valid >= num_matches_thr))
