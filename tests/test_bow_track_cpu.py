"""The CPU restatement of frame_tracker::bow_match_based_track (tests/bow_track_oracle.py) that the device chain is checked against: its
match against a literal walk of frame_tracker.cc:61-95 / bow_tree.cc:169-256 over the std::map merge-join (test_pairs_cpu.literal_pairs),
the gate at the threshold, the < 5 observations early return, pose recovery on clean scenes and the ctypes mirror of
b200_bow_track_frame_t against the header."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bow_track_oracle as BT  # noqa: E402
import camera_models_oracle as CMO  # noqa: E402

CAM = dict(model="perspective", fx=718.856, fy=718.856, cx=320.0, cy=185.2157, fxb=386.1448, cols=640.0, rows=376.0)


@pytest.fixture(scope="module")
def frame():
    from oracle import pyoracle as O
    from workloads import synth
    img = synth.make_frame(640, 376, seed=11)
    r = O.orb_extract(img, min_area=800)
    _, _, _, isig = O.scale_factors()
    return r["kps"], r["desc"], isig


def literal_bow_match_based_track(kps, desc, fr, num_matches_thr):
    """frame_tracker.cc:61-72 with bow_tree::match_frame_and_keyframe walked over ordered node -> indices maps.  A keypoint that no node
    lists is in neither map: it gets a key of its own side (-3 keyframe, -2 frame) that the other side never has."""
    import test_pairs_cpu as TP
    und, _ = CMO.undistort_keypoints(CAM, kps)
    kf = fr["keyframe"]
    knode = np.where(np.asarray(kf["node"]) < 0, -3, kf["node"])
    fnode = np.where(np.asarray(fr["kp_node"]) < 0, -2, fr["kp_node"])
    pr = dict(desc1=np.asarray(kf["desc"], np.uint8), angle1=np.asarray(kf["angle"], np.float32), valid1=np.asarray(kf["valid"], np.uint8),
              node1=knode, desc2=np.asarray(desc, np.uint8), angle2=np.asarray(und["angle"], np.float32), node2=fnode)
    mo = TP.literal_pairs(pr, 0, 0.7, True)
    n = int((mo >= 0).sum())
    if n < num_matches_thr:
        return mo, n, None
    kp_lm = np.full(len(kps), -1, np.int32)                      # matched_lms_in_frm, then set_landmarks
    for row, j in enumerate(mo):
        if j >= 0:
            kp_lm[j] = row
    return mo, n, kp_lm


@pytest.mark.parametrize("seed,n_nodes", [(1, 64), (2, 16), (3, 64), (4, 8)])
def test_oracle_equals_the_literal_merge_join(frame, seed, n_nodes):
    from workloads import synth
    kps, desc, isig = frame
    fr = synth.make_bow_frame(kps, desc, CAM, seed=seed, n_nodes=n_nodes, rotated_frac=0.1, erased_frac=0.1, lookalike_frac=0.2)
    r = BT.bow_match_based_track(CAM, kps, desc, fr, isig)
    mo, n, kp_lm = literal_bow_match_based_track(kps, desc, fr, 10)
    assert np.array_equal(r["match_out"], mo) and r["n_matches"] == n
    assert r["applied"] == (kp_lm is not None)
    # the scene has what the walk must get right: erased and unnoded rows never match, unnoded frame keypoints are never matched, and
    # the ratio test rejects look-alikes
    kf = fr["keyframe"]
    rows = np.nonzero(mo >= 0)[0]
    assert (np.asarray(kf["valid"])[rows] == 1).all() and (np.asarray(kf["node"])[rows] >= 0).all()
    assert (np.asarray(fr["kp_node"])[mo[rows]] >= 0).all()
    assert (np.asarray(fr["kp_node"]) < 0).any() and (np.asarray(kf["node"]) < 0).any() and (np.asarray(kf["valid"]) == 0).any()
    from oracle import pyoracle as O
    und, _ = CMO.undistort_keypoints(CAM, kps)
    _, n_no_ratio = O.match_pairs(BT.pairs_problem(fr, desc, und["angle"]), 0, 1.0, True)
    assert n_no_ratio > n
    # the discard after the optimisation works on the same landmarks
    if kp_lm is not None:
        kept = r["kp_landmark"] >= 0
        assert np.array_equal(r["kp_landmark"][kept], kp_lm[kept])


def test_gate_at_the_threshold(frame):
    from workloads import synth
    kps, desc, isig = frame
    fr = synth.make_bow_frame(kps, desc, CAM, seed=5)
    n = BT.bow_match_based_track(CAM, kps, desc, fr, isig)["n_matches"]
    assert n > 10
    at = BT.bow_match_based_track(CAM, kps, desc, fr, isig, num_matches_thr=n)
    above = BT.bow_match_based_track(CAM, kps, desc, fr, isig, num_matches_thr=n + 1)
    assert at["applied"] and at["kp_landmark"] is not None and at["pose_cw"] is not None
    assert not above["applied"] and above["n_matches"] == n and above["kp_landmark"] is None and above["pose_cw"] is None
    assert above["n_valid"] == 0 and not above["tracked"]
    # thr - 1 passes like thr
    assert BT.bow_match_based_track(CAM, kps, desc, fr, isig, num_matches_thr=n - 1)["applied"]


def test_fewer_than_five_observations_keep_the_last_pose(frame):
    from workloads import synth
    kps, desc, isig = frame
    fr = synth.make_bow_frame(kps, desc, CAM, seed=6, erased_frac=0.0, rotated_frac=0.0)
    full = BT.bow_match_based_track(CAM, kps, desc, fr, isig)
    rows = np.nonzero(full["match_out"] >= 0)[0][:3]
    few = dict(fr, keyframe={k: np.asarray(v)[rows] for k, v in fr["keyframe"].items()})
    r = BT.bow_match_based_track(CAM, kps, desc, few, isig, num_matches_thr=2)
    assert r["n_matches"] == 3 and r["applied"] and r["n_valid"] == 3 and r["tracked"]
    assert np.array_equal(r["pose_cw"], np.asarray(fr["last_pose_cw"]))


@pytest.mark.parametrize("seed", [1, 2])
def test_recovers_the_true_pose_on_clean_scenes(frame, seed):
    from workloads import synth
    kps, desc, isig = frame
    fr = synth.make_bow_frame(kps, desc, CAM, seed=seed, split_frac=0.0, lookalike_frac=0.0, unnoded_frac=0.0, kf_unnoded_frac=0.0, rotated_frac=0.0,
                              erased_frac=0.0, wrong_depth_frac=0.0, clutter_frac=0.0)
    r = BT.bow_match_based_track(CAM, kps, desc, fr, isig)
    assert r["applied"] and r["tracked"]
    assert np.abs(r["pose_cw"] - fr["gt_pose_cw"]).max() < 1e-2
    assert np.abs(r["pose_cw"] - fr["gt_pose_cw"]).max() < np.abs(fr["last_pose_cw"] - fr["gt_pose_cw"]).max()


def test_struct_layout(tmp_path):
    import test_abi_layout as T
    from stella_vslam_b200 import tracking
    T._check(tmp_path, os.path.join(T.ROOT, "include"), "b200vslam.h", {"b200_bow_track_frame_t": tracking.BowTrackFrame})
