"""CPU restatement of module::frame_tracker::robust_match_based_track (test infrastructure), composed from the existing oracles stage by
stage:

  undistort_keypoints + bearings           camera_models_oracle.undistort_keypoints (all four camera models)
  robust::brute_force_match(0.8, true)     pyoracle.brute_force_match
  create_random_array(5, ...) x 1000       solve.draw_min_sets on the frame's engine (b200_draw_min_sets, host code)
  essential_solver::find_via_ransac        essential_oracle.essential_ransac(recompute=True)
  pose_optimizer::optimize                 pyoracle.pose_optimize from the last pose
  discard_outliers                         frame_tracker.cc:133-150
"""
import numpy as np

from oracle import pyoracle as O

import camera_models_oracle as CMO
import essential_oracle as EO

N_ITER = 1000  # find_via_ransac(1000, true) (robust.cc:211)


def _g(camera, k):
    return float(camera.get(k, 0.0))


def _engine(frame):
    from stella_vslam_b200 import solve
    e = frame.get("engine")
    return solve.mt19937() if e is None else solve.Mt19937.from_buffer_copy(e)


def robust_match_based_track(camera, kps, desc, frame, inv_level_sigma_sq, num_matches_thr=10, monocular=True, lowe_ratio=0.8,
                             num_trials_robust=2, num_trials=2, num_each_iter=10, undistort_fn=None, match_fn=None, draw_fn=None, ransac_fn=None,
                             pose_fn=None):
    """frame_tracker::robust_match_based_track with match::robust(lowe_ratio, true).  kps / desc: the current frame's (distorted)
    keypoints and descriptors; frame: the dict stella_vslam_b200.tracking.frame_tracker.pack_robust takes (a frame without an engine
    draws from a default-constructed one).  Returns the dict of frame_tracker.robust_match_based_track plus pairs, inlier_flags and E_21.
    undistort_fn / match_fn / draw_fn / ransac_fn / pose_fn replace the stages (same arguments and results), e.g. by the stage-by-stage
    device ABI."""
    from stella_vslam_b200 import solve
    kps = np.ascontiguousarray(kps, O.KP_DTYPE)
    n_kp = len(kps)
    kf = frame["keyframe"]
    und, bear = (undistort_fn or CMO.undistort_keypoints)(camera, kps)
    bear = np.asarray(bear, np.float64).reshape(-1, 3)
    pairs = (match_fn or O.brute_force_match)(np.ascontiguousarray(desc, np.uint8).reshape(-1, 32), und["angle"], kf["desc"], kf["angle"], kf["valid"],
                                             lowe_ratio, True)
    pairs = np.asarray(pairs, np.int32).reshape(-1, 2)
    n = len(pairs)
    valid, status, flags, E = False, 0, None, None
    if n >= 5:                                                   # find_via_ransac returns before drawing below the minimal set
        ms = (draw_fn or (lambda nn, e: solve.draw_min_sets(nn, N_ITER, e, set_size=5)))(n, _engine(frame))
        kb = np.asarray(kf["bearings"], np.float64).reshape(-1, 3)
        r = (ransac_fn or EO.essential_ransac)(bear[pairs[:, 0]], kb[pairs[:, 1]], ms, True)
        valid, status, E = bool(r["valid"]), int(r["status"]), r["E_21"]
        flags = np.asarray(r["inlier_flags"], bool) if valid else None
    n_inliers = int(flags.sum()) if valid else 0
    applied = n_inliers >= num_matches_thr
    out = dict(n_keypoints=n_kp, n_matches=n, essential_valid=valid, status=0 if status == 0 else -1, n_inliers=n_inliers, applied=applied,
               n_valid=0, tracked=False, kp_landmark=None, pose_cw=None, pairs=pairs, inlier_flags=flags, E_21=E)
    if not applied:                                              # frame_tracker.cc:105-108: the frame is not touched
        return out
    kp_lm = np.full(n_kp, -1, np.int32)                          # set_landmarks (:111)
    inl = pairs[flags]
    kp_lm[inl[:, 0]] = inl[:, 1]
    pose = np.asarray(frame["last_pose_cw"], np.float64).reshape(4, 4)
    out_pose = pose.copy()
    idx = np.nonzero(kp_lm >= 0)[0]
    if len(idx) >= 5:                                            # pose_optimizer_g2o.cc:116-118 below 5 edges
        xr = frame.get("kp_x_right")
        xrk = np.full(n_kp, -1.0, np.float32) if xr is None else np.asarray(xr, np.float32)
        isig = np.asarray(inv_level_sigma_sq, np.float32)
        chi = np.float32(np.sqrt(np.float32(5.99146))) if monocular else np.float32(np.sqrt(np.float32(7.81473)))
        cam = dict(model=1 if CMO.model_of(camera) == 1 else 0, fx=_g(camera, "fx"), fy=_g(camera, "fy"), cx=_g(camera, "cx"), cy=_g(camera, "cy"),
                   fxb=_g(camera, "fxb"), cols=_g(camera, "cols"), rows=_g(camera, "rows"))
        ne = len(idx)
        pos = np.asarray(kf["pos_w"], np.float64).reshape(-1, 3)
        pp = dict(pose_cw=pose.reshape(1, 4, 4), pose_fixed=np.zeros(1, np.uint8), points=pos[kp_lm[idx]].reshape(-1, 3), point_fixed=np.ones(ne, np.uint8),
                  e_pose=np.zeros(ne, np.int32), e_point=np.arange(ne, dtype=np.int32), e_cam=np.zeros(ne, np.uint8),
                  e_obs=np.stack([und["x"][idx], und["y"][idx], xrk[idx]], 1).astype(np.float32), e_inv_sigma_sq=isig[und["octave"][idx].astype(np.int64)],
                  e_delta=np.full(ne, chi, np.float32), e_robust=None, e_can_be_outlier=None, cams=[cam])
        _, out_pose, oflags = (pose_fn or O.pose_optimize)(pp, num_trials_robust, num_trials, num_each_iter)
        kp_lm[idx[np.asarray(oflags, bool)]] = -1                # discard_outliers (frame_tracker.cc:133-150)
    n_valid = int((kp_lm >= 0).sum())
    out.update(kp_landmark=kp_lm, pose_cw=out_pose, n_valid=n_valid, tracked=n_valid >= num_matches_thr)
    return out
