"""CPU restatement of module::frame_tracker::bow_match_based_track (test infrastructure), composed from the existing oracles stage by
stage:

  undistort_keypoints                           camera_models_oracle.undistort_keypoints (all four camera models)
  bow_tree(0.7, true)::match_frame_and_keyframe pyoracle.match_pairs(variant 0): the keyframe is side 1, the frame side 2
  gate                                          num_matches >= num_matches_thr (frame_tracker.cc:69-72)
  pose_optimizer::optimize                      pyoracle.pose_optimize from the last pose
  discard_outliers                              frame_tracker.cc:133-150

A node id of -1 means that no node of the BoW vector lists the keypoint: such a keypoint takes part in no node's merge-join step.
"""
import numpy as np

from oracle import pyoracle as O

import camera_models_oracle as CMO


def _g(camera, k):
    return float(camera.get(k, 0.0))


def pairs_problem(frame, desc, angle):
    """The b200_match_pairs problem of match_frame_and_keyframe: rows are the keyframe's keypoints whose landmark is live and that a node
    lists, candidates the frame's keypoints (desc / angle: the frame's descriptors and undistorted angles)."""
    kf = frame["keyframe"]
    knode = np.asarray(kf["node"], np.int32)
    valid = (np.asarray(kf["valid"], np.uint8) != 0) & (knode >= 0)
    return dict(desc1=np.asarray(kf["desc"], np.uint8).reshape(-1, 32), angle1=np.asarray(kf["angle"], np.float32), valid1=valid.astype(np.uint8),
                node1=knode, desc2=np.ascontiguousarray(desc, np.uint8).reshape(-1, 32), angle2=np.asarray(angle, np.float32),
                node2=np.asarray(frame["kp_node"], np.int32))


def optimize_and_discard(camera, und, kp_lm, pose, pos_w, kp_x_right, inv_level_sigma_sq, monocular, num_trials_robust, num_trials, num_each_iter,
                         pose_fn=None):
    """pose_optimizer::optimize on the keypoints that carry a landmark (the < 5 observations early return included), then
    discard_outliers.  kp_lm is updated in place; returns the pose."""
    n_kp = len(kp_lm)
    idx = np.nonzero(kp_lm >= 0)[0]
    if len(idx) < 5:                                             # pose_optimizer_g2o.cc:116-118 below 5 edges
        return pose.copy()
    xrk = np.full(n_kp, -1.0, np.float32) if kp_x_right is None else np.asarray(kp_x_right, np.float32)
    isig = np.asarray(inv_level_sigma_sq, np.float32)
    chi = np.float32(np.sqrt(np.float32(5.99146))) if monocular else np.float32(np.sqrt(np.float32(7.81473)))
    cam = dict(model=1 if CMO.model_of(camera) == 1 else 0, fx=_g(camera, "fx"), fy=_g(camera, "fy"), cx=_g(camera, "cx"), cy=_g(camera, "cy"),
               fxb=_g(camera, "fxb"), cols=_g(camera, "cols"), rows=_g(camera, "rows"))
    ne = len(idx)
    pos = np.asarray(pos_w, np.float64).reshape(-1, 3)
    pp = dict(pose_cw=pose.reshape(1, 4, 4), pose_fixed=np.zeros(1, np.uint8), points=pos[kp_lm[idx]].reshape(-1, 3), point_fixed=np.ones(ne, np.uint8),
              e_pose=np.zeros(ne, np.int32), e_point=np.arange(ne, dtype=np.int32), e_cam=np.zeros(ne, np.uint8),
              e_obs=np.stack([und["x"][idx], und["y"][idx], xrk[idx]], 1).astype(np.float32), e_inv_sigma_sq=isig[und["octave"][idx].astype(np.int64)],
              e_delta=np.full(ne, chi, np.float32), e_robust=None, e_can_be_outlier=None, cams=[cam])
    _, out_pose, oflags = (pose_fn or O.pose_optimize)(pp, num_trials_robust, num_trials, num_each_iter)
    kp_lm[idx[np.asarray(oflags, bool)]] = -1                    # discard_outliers (frame_tracker.cc:133-150)
    return np.asarray(out_pose, np.float64).reshape(4, 4)


def bow_match_based_track(camera, kps, desc, frame, inv_level_sigma_sq, num_matches_thr=10, monocular=True, lowe_ratio=0.7, num_trials_robust=2,
                          num_trials=2, num_each_iter=10, undistort_fn=None, match_fn=None, pose_fn=None):
    """frame_tracker::bow_match_based_track with match::bow_tree(lowe_ratio, true).  kps / desc: the current frame's (distorted) keypoints
    and descriptors; frame: the dict stella_vslam_b200.tracking.frame_tracker.pack_bow takes.  Returns the dict of
    frame_tracker.bow_match_based_track plus match_out (keyframe keypoint -> frame keypoint).  undistort_fn / match_fn / pose_fn replace
    the stages (same arguments and results), e.g. by the stage-by-stage device ABI."""
    kps = np.ascontiguousarray(kps, O.KP_DTYPE)
    n_kp = len(kps)
    kf = frame["keyframe"]
    und, _ = (undistort_fn or CMO.undistort_keypoints)(camera, kps)
    prob = pairs_problem(frame, desc, und["angle"])
    mo, n = (match_fn or (lambda p: O.match_pairs(p, 0, lowe_ratio, True)))(prob)
    mo = np.asarray(mo, np.int32)
    applied = int(n) >= num_matches_thr
    out = dict(n_keypoints=n_kp, n_matches=int(n), applied=applied, n_valid=0, tracked=False, kp_landmark=None, pose_cw=None, match_out=mo)
    if not applied:                                              # frame_tracker.cc:69-72: the frame is not touched
        return out
    kp_lm = np.full(n_kp, -1, np.int32)                          # set_landmarks (:75)
    rows = np.nonzero(mo >= 0)[0]
    kp_lm[mo[rows]] = rows
    pose = np.asarray(frame["last_pose_cw"], np.float64).reshape(4, 4)
    out_pose = optimize_and_discard(camera, und, kp_lm, pose, kf["pos_w"], frame.get("kp_x_right"), inv_level_sigma_sq, monocular, num_trials_robust,
                                    num_trials, num_each_iter, pose_fn)
    n_valid = int((kp_lm >= 0).sum())
    out.update(kp_landmark=kp_lm, pose_cw=out_pose, n_valid=n_valid, tracked=n_valid >= num_matches_thr)
    return out
