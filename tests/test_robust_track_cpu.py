"""The CPU restatement of frame_tracker::robust_match_based_track (tests/robust_track_oracle.py) that the device chain is checked against:
pose recovery on clean scenes, inlier flags against check_inliers, the gates of the reference (fewer than 5 matches, too few inliers),
and the ctypes mirror of b200_robust_track_frame_t against the header."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import essential_oracle as EO  # noqa: E402
import robust_track_oracle as RT  # noqa: E402

CAM = dict(model="perspective", fx=718.856, fy=718.856, cx=320.0, cy=185.2157, fxb=386.1448, cols=640.0, rows=376.0)


@pytest.fixture(scope="module")
def frame():
    from oracle import pyoracle as O
    from workloads import synth
    img = synth.make_frame(640, 376, seed=11)
    r = O.orb_extract(img, min_area=800)
    _, _, _, isig = O.scale_factors()
    return r["kps"], r["desc"], isig


def _clean(frame, seed, **kw):
    from workloads import synth
    kps, desc, _ = frame
    return synth.make_robust_frame(kps, desc, CAM, seed=seed, rotated_frac=0.0, erased_frac=0.0, wrong_depth_frac=0.0, clutter_frac=0.0, **kw)


@pytest.mark.parametrize("seed", [1, 2])
def test_recovers_the_true_pose_on_clean_scenes(frame, seed):
    kps, desc, isig = frame
    fr = _clean(frame, seed)
    r = RT.robust_match_based_track(CAM, kps, desc, fr, isig)
    assert r["essential_valid"] and r["applied"] and r["tracked"]
    assert r["n_inliers"] >= 0.8 * r["n_matches"]
    assert np.abs(r["pose_cw"] - fr["gt_pose_cw"]).max() < 1e-2
    assert np.abs(r["pose_cw"] - fr["gt_pose_cw"]).max() < np.abs(fr["last_pose_cw"] - fr["gt_pose_cw"]).max()


def test_inlier_flags_are_check_inliers_of_the_returned_E(frame):
    kps, desc, isig = frame
    from workloads import synth
    import camera_models_oracle as CMO
    fr = synth.make_robust_frame(kps, desc, CAM, seed=5)
    r = RT.robust_match_based_track(CAM, kps, desc, fr, isig)
    assert r["essential_valid"]
    _, bear = CMO.undistort_keypoints(CAM, kps)
    p = r["pairs"]
    num, flags, _ = EO.check_inliers(bear[p[:, 0]], np.asarray(fr["keyframe"]["bearings"])[p[:, 1]], r["E_21"])
    assert np.array_equal(flags, r["inlier_flags"]) and num == r["n_inliers"]


def test_wrong_depth_matches_pass_the_essential_test_and_fail_the_pose(frame):
    kps, desc, isig = frame
    from workloads import synth
    fr = synth.make_robust_frame(kps, desc, CAM, seed=7, wrong_depth_frac=0.2, rotated_frac=0.0, clutter_frac=0.0, erased_frac=0.0)
    r = RT.robust_match_based_track(CAM, kps, desc, fr, isig)
    assert r["applied"] and r["tracked"]
    assert r["n_valid"] < r["n_inliers"]                         # the discard removed the landmarks at a wrong depth


def test_gates(frame):
    kps, desc, isig = frame
    fr = _clean(frame, 3)
    kf = fr["keyframe"]
    few = dict(fr, keyframe={k: v[:4] for k, v in kf.items()})
    r = RT.robust_match_based_track(CAM, kps, desc, few, isig)
    assert r["n_matches"] < 5 and not r["essential_valid"] and r["n_inliers"] == 0 and not r["applied"]
    assert r["kp_landmark"] is None and r["pose_cw"] is None
    full = RT.robust_match_based_track(CAM, kps, desc, fr, isig)
    high = RT.robust_match_based_track(CAM, kps, desc, fr, isig, num_matches_thr=full["n_inliers"] + 1)
    assert high["essential_valid"] and high["n_inliers"] == full["n_inliers"] and not high["applied"] and not high["tracked"]


def test_seeded_engine_changes_the_draws_not_the_contract(frame):
    from stella_vslam_b200 import solve
    kps, desc, isig = frame
    fr = _clean(frame, 4)
    a = RT.robust_match_based_track(CAM, kps, desc, fr, isig)
    b = RT.robust_match_based_track(CAM, kps, desc, dict(fr, engine=solve.mt19937([1, 2, 3])), isig)
    assert a["applied"] and b["applied"] and a["n_matches"] == b["n_matches"]


def test_struct_layout(tmp_path):
    import test_abi_layout as T
    from stella_vslam_b200 import tracking
    T._check(tmp_path, os.path.join(T.ROOT, "include"), "b200vslam.h", {"b200_robust_track_frame_t": tracking.RobustTrackFrame})
