"""The CPU restatement of frame_tracker::motion_based_track (tests/motion_track_oracle.py) that the device chain is checked against: the
retry on a short first search, the forward / backward octave windows, failed frames, discard_outliers, the reprojection of all four
camera models against numpy, and the ctypes mirror of b200_motion_track_frame_t against the header."""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import camera_models_oracle as CM  # noqa: E402
import motion_track_oracle as MT  # noqa: E402

KITTI = dict(model="perspective", fx=718.856, fy=718.856, cx=607.1928, cy=185.2157, fxb=386.1448, cols=1241.0, rows=376.0)


@pytest.fixture(scope="module")
def frame():
    from oracle import pyoracle as O
    from workloads import synth
    img = synth.make_frame(640, 376, seed=11)
    r = O.orb_extract(img, min_area=800)
    sf, _, _, isig = O.scale_factors()
    return r["kps"], r["desc"], sf, isig


def _run(frame, cam, fr, **kw):
    kps, desc, sf, isig = frame
    return MT.motion_based_track(cam, kps, desc, fr, sf, isig, **kw)


def test_short_first_search_retries_on_an_empty_frame(frame, monkeypatch):
    from oracle import pyoracle as O
    from workloads import synth
    kps, desc, sf, isig = frame
    cam = dict(KITTI, cols=640.0, cx=320.0, setup="monocular")
    fr = synth.make_motion_frame(kps, desc, cam, sf, seed=3, shift_px=25.0, landmark_frac=0.05)
    calls = []
    real = O.match_guided

    def spy(pr, mode, **kw):
        calls.append((pr["q_margin"].copy(), pr["t_occupied"].copy()))
        return real(pr, mode, **kw)

    monkeypatch.setattr(O, "match_guided", spy)
    r = _run(frame, cam, fr, margin=10.0)
    assert r["retried"] and r["n_matches_first"] < 10 <= r["n_matches"]
    assert len(calls) == 2
    assert np.array_equal(calls[1][0], np.float32(20.0) * sf[fr["table"]["octave"].astype(np.int64)])
    assert not calls[1][1].any()                                   # the second search starts from a frame without landmarks
    assert r["tracked"] and r["n_valid"] >= 10
    assert np.abs(r["pose_cw"] - fr["gt_pose_cw"]).max() < np.abs(fr["pose_cw"] - fr["gt_pose_cw"]).max()


def test_direction_windows_only_for_non_monocular(frame):
    from workloads import synth
    kps, desc, sf, _ = frame
    for motion, want in (("forward", (True, False)), ("backward", (False, True)), ("sideways", (False, False))):
        fr = synth.make_motion_frame(kps, desc, KITTI, sf, seed=4, stereo=True, motion=motion)
        assert MT.direction(fr["pose_cw"], fr["last_pose_cw"], fr["true_baseline"], monocular=False) == want, motion
        assert MT.direction(fr["pose_cw"], fr["last_pose_cw"], fr["true_baseline"], monocular=True) == (False, False)


def test_failed_frame_keeps_the_predicted_pose(frame):
    from workloads import synth
    kps, desc, sf, _ = frame
    cam = dict(KITTI, cols=640.0, cx=320.0)
    fr = synth.make_motion_frame(kps, desc, cam, sf, seed=5, shift_px=200.0, landmark_frac=0.05)
    r = _run(frame, cam, fr, margin=10.0)
    assert r["retried"] and r["n_matches"] < 10 and not r["tracked"]
    assert np.array_equal(r["pose_cw"], fr["pose_cw"])
    assert r["n_valid"] == int((r["kp_landmark"] >= 0).sum())


def test_discarded_keypoints_carry_no_landmark(frame):
    from workloads import synth
    kps, desc, sf, _ = frame
    cam = dict(KITTI, cols=640.0, cx=320.0)
    fr = synth.make_motion_frame(kps, desc, cam, sf, seed=6, pixel_sigma=3.0)
    r = _run(frame, cam, fr, margin=10.0)
    assert not r["retried"] and r["tracked"]
    assert r["n_valid"] == int((r["kp_landmark"] >= 0).sum()) < r["n_matches"]   # some matches were outliers and lost their landmark


def _numpy_reproject(cam, pose, pos, bounds):
    R, t = pose[:3, :3], pose[:3, 3]
    pc = pos @ R.T + t
    if cam["model"] == "equirectangular":
        b = pc / np.linalg.norm(pc, axis=1, keepdims=True)
        u = cam["cols"] * (0.5 + np.arctan2(b[:, 0], b[:, 2]) / (2 * math.pi))
        v = cam["rows"] * (0.5 + np.arcsin(b[:, 1]) / math.pi)
        return np.ones(len(pos), bool), np.stack([u, v], 1), np.zeros(len(pos), np.float32)
    u = cam["fx"] * pc[:, 0] / pc[:, 2] + cam["cx"]
    v = cam["fy"] * pc[:, 1] / pc[:, 2] + cam["cy"]
    xr = (u - cam.get("fxb", 0.0) / pc[:, 2]).astype(np.float32)
    b = [float(np.float32(x)) for x in bounds]
    if cam["model"] == "radial_division":
        ok = (pc[:, 2] > 0) & (u >= b[0]) & (u <= b[1]) & (v >= b[2]) & (v <= b[3])
    else:
        ok = (pc[:, 2] > 0) & (u > b[0]) & (u < b[1]) & (v > b[2]) & (v < b[3])
    return ok, np.stack([u, v], 1), xr


@pytest.mark.parametrize("model", ["perspective", "equirectangular", "fisheye", "radial_division"])
def test_reprojection_matches_numpy(model):
    cam = {"perspective": dict(KITTI), "equirectangular": dict(model="equirectangular", cols=1920.0, rows=960.0), "fisheye": dict(CM.AIST, fxb=30.0),
           "radial_division": dict(model="radial_division", fx=612.3, fy=611.7, cx=480.5, cy=270.2, distortion=-0.15, cols=960.0, rows=540.0)}[model]
    rng = np.random.default_rng(7)
    pos = np.concatenate([rng.normal(0, 3, (500, 3)) + [0, 0, 8], rng.normal(0, 3, (50, 3)) - [0, 0, 8]])
    pose = np.eye(4)
    pose[:3, :3] = np.array([[math.cos(0.1), 0, math.sin(0.1)], [0, 1, 0], [-math.sin(0.1), 0, math.cos(0.1)]])
    pose[:3, 3] = [0.1, -0.2, 0.3]
    bounds = MT.default_bounds(cam)
    ok, rp, xr = MT.reproject(cam, pose, pos, bounds)
    ok_n, rp_n, xr_n = _numpy_reproject(cam, pose, pos, bounds)
    # numpy's matrix product may round differently in the last bit: agree within 1e-9 px, and on the verdict away from the bounds
    assert np.abs(rp - rp_n).max() <= 1e-9 * max(1.0, np.abs(rp_n).max())
    assert np.abs(xr.astype(np.float64) - xr_n).max() <= 1e-3
    margin = np.minimum.reduce([np.abs(rp_n[:, 0] - bounds[0]), np.abs(rp_n[:, 0] - bounds[1]), np.abs(rp_n[:, 1] - bounds[2]),
                                np.abs(rp_n[:, 1] - bounds[3])]) > 1e-6
    assert np.array_equal(ok[margin], ok_n[margin])
    if model != "equirectangular":
        assert 0 < ok.sum() < len(pos) and not ok[500:].any()     # some inside, nothing behind the camera


def test_ctypes_mirror_matches_the_header(tmp_path):
    import test_abi_layout as T
    from stella_vslam_b200 import tracking
    T._check(tmp_path, os.path.join(T.ROOT, "include"), "b200vslam.h", {"b200_motion_track_frame_t": tracking.MotionTrackFrame})
