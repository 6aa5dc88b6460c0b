"""GPU parity of the motion-model tracking chain (b200_motion_based_track) against the CPU restatement (tests/motion_track_oracle.py) and
against the stage-by-stage device ABI: kp_landmark_out, n_matches_first, n_matches, retried, n_valid and tracked bit-exact, the pose within
1e-5 (the local-map chain's tolerance)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import camera_models_oracle as CM  # noqa: E402
import motion_track_oracle as MT  # noqa: E402

pytestmark = pytest.mark.gpu

KITTI = dict(model="perspective", fx=718.856, fy=718.856, cx=607.1928, cy=185.2157, fxb=386.1448, cols=1241.0, rows=376.0)
EUROC = dict(model="perspective", fx=458.654, fy=457.296, cx=367.215, cy=248.375, k1=-0.28340811, k2=0.07395907, p1=0.00019359, p2=1.76187114e-05,
             k3=0.0, fxb=0.0, cols=752.0, rows=480.0)
RADIAL = dict(model="radial_division", fx=612.3, fy=611.7, cx=480.5, cy=270.2, distortion=-0.15, fxb=0.0, cols=960.0, rows=540.0)
KEYS = ("n_keypoints", "n_matches_first", "n_matches", "retried", "n_valid", "tracked")


@pytest.fixture(scope="module")
def mods():
    from stella_vslam_b200 import feature, tracking
    from workloads import synth
    return feature, tracking, synth


def _extract(feature, synth, w, h, seeds, n=800):
    ex = feature.orb_extractor(feature.orb_params(), n, max_batch=len(seeds))
    kps, descs = ex.extract_batch(np.stack([synth.make_frame(w, h, seed=s) for s in seeds]))
    return ex, kps, descs


def _check(ex, tr, cam, kps, descs, frames, monocular, **kw):
    got = tr.motion_based_track(frames)
    prm = ex.orb_params_
    bounds = tuple(tr._prm.img_bounds)
    for f, (fr, g) in enumerate(zip(frames, got)):
        i = fr.get("frame", f)
        ref = MT.motion_based_track(cam, kps[i], descs[i], fr, prm.scale_factors_, prm.inv_level_sigma_sq_, margin=tr._prm.margin,
                                    num_matches_thr=tr.num_matches_thr, true_baseline=tr.true_baseline, monocular=monocular, img_bounds=bounds,
                                    grid=(tr._prm.grid_cols, tr._prm.grid_rows), **kw)
        for k in KEYS:
            assert g[k] == ref[k], (f, k, g[k], ref[k])
        assert np.array_equal(g["kp_landmark"], ref["kp_landmark"]), f
        assert np.abs(g["pose_cw"] - ref["pose_cw"]).max() <= 1e-5 * max(1.0, np.abs(ref["pose_cw"]).max()), f
    return got


@pytest.mark.parametrize("motion", ["forward", "backward"])
def test_kitti_stereo(mods, motion):
    feature, tracking, synth = mods
    ex, kps, descs = _extract(feature, synth, 1241, 376, (50, 51, 52))
    cam = dict(KITTI, setup="stereo")
    frames = [dict(synth.make_motion_frame(kps[i], descs[i], cam, ex.orb_params_.scale_factors_, seed=70 + i, stereo=True, motion=motion), frame=i)
              for i in range(3)]
    tr = tracking.frame_tracker(ex, cam, margin=10.0)
    got = _check(ex, tr, cam, kps, descs, frames, monocular=False)
    for fr, g in zip(frames, got):
        assert g["tracked"] and not g["retried"]
        assert np.abs(g["pose_cw"] - fr["gt_pose_cw"]).max() < np.abs(fr["pose_cw"] - fr["gt_pose_cw"]).max()
    assert MT.direction(frames[0]["pose_cw"], frames[0]["last_pose_cw"], tr.true_baseline, False) == (motion == "forward", motion == "backward")
    ms = tr.stage_ms()
    assert ms["chain"] > 0


def test_euroc_distortion_out_of_order_subset(mods):
    feature, tracking, synth = mods
    ex, kps, descs = _extract(feature, synth, 752, 480, (80, 81, 82, 83))
    und = [CM.undistort_keypoints(EUROC, k)[0] for k in kps]
    bounds = (-30.0, 790.0, -25.0, 510.0)
    frames = [dict(synth.make_motion_frame(und[i], descs[i], EUROC, ex.orb_params_.scale_factors_, seed=90 + i), frame=i) for i in (2, 0)]
    tr = tracking.frame_tracker(ex, EUROC, margin=20.0, img_bounds=bounds)
    got = _check(ex, tr, EUROC, kps, descs, frames, monocular=True)
    assert all(g["tracked"] for g in got)


def test_equirectangular(mods):
    feature, tracking, synth = mods
    ex, kps, descs = _extract(feature, synth, 1920, 960, (40, 41), n=2500)
    cam = dict(model="equirectangular", cols=1920.0, rows=960.0, fxb=0.0, setup="monocular")
    frames = [dict(synth.make_motion_frame(kps[i], descs[i], cam, ex.orb_params_.scale_factors_, seed=45 + i), frame=i) for i in range(2)]
    tr = tracking.frame_tracker(ex, cam)
    got = _check(ex, tr, cam, kps, descs, frames, monocular=True)
    assert all(g["tracked"] for g in got)


@pytest.mark.parametrize("model", ["fisheye", "radial_division"])
def test_fisheye_and_radial_division(mods, model):
    feature, tracking, synth = mods
    # the frames of test_camera_models_gpu: their device undistortion equals the oracle's bit for bit (checked below)
    cam, w, h, grid, seed = (dict(CM.TUM_VI, fxb=0.0), 512, 512, (16, 16), 300) if model == "fisheye" else (RADIAL, 960, 540, (64, 48), 500)
    ex, kps, descs = _extract(feature, synth, w, h, (seed, seed + 1))
    und = [CM.undistort_keypoints(cam, k)[0] for k in kps]
    for k, u in zip(kps, und):
        assert np.array_equal(ex.undistort_keypoints(cam, k)[0], u)
    frames = [dict(synth.make_motion_frame(und[i], descs[i], cam, ex.orb_params_.scale_factors_, seed=seed + 10 + i), frame=i) for i in range(2)]
    tr = tracking.frame_tracker(ex, cam, grid=grid)
    got = _check(ex, tr, cam, kps, descs, frames, monocular=True)
    assert all(g["tracked"] for g in got)


def test_rgbd_x_right(mods):
    # an RGB-D frame carries stereo_x_right_ from its depth map (b200_rgbd_depths): a non-monocular setup with kp_x_right
    feature, tracking, synth = mods
    ex, kps, descs = _extract(feature, synth, 640, 480, (60, 61))
    cam = dict(model="perspective", fx=525.0, fy=525.0, cx=319.5, cy=239.5, fxb=40.0, cols=640.0, rows=480.0, setup="rgbd")
    frames = [dict(synth.make_motion_frame(kps[i], descs[i], cam, ex.orb_params_.scale_factors_, seed=65 + i, stereo=True, motion=m), frame=i)
              for i, m in ((0, "sideways"), (1, "forward"))]
    tr = tracking.frame_tracker(ex, cam)
    got = _check(ex, tr, cam, kps, descs, frames, monocular=False)
    assert all(g["tracked"] for g in got)


def test_mixed_batch_pass_retry_fail(mods):
    feature, tracking, synth = mods
    ex, kps, descs = _extract(feature, synth, 640, 376, (11, 11, 11, 11))  # the image of test_motion_track_cpu
    cam = dict(KITTI, cols=640.0, cx=320.0, setup="monocular")
    sf = ex.orb_params_.scale_factors_
    frames = [dict(synth.make_motion_frame(kps[0], descs[0], cam, sf, seed=1), frame=0),                                    # at once
              dict(synth.make_motion_frame(kps[1], descs[1], cam, sf, seed=3, shift_px=25.0, landmark_frac=0.05), frame=1),  # retries
              dict(synth.make_motion_frame(kps[2], descs[2], cam, sf, seed=5, shift_px=200.0, landmark_frac=0.05), frame=2),  # fails
              dict(synth.make_motion_frame(kps[3], descs[3], cam, sf, seed=7, shift_px=40.0), frame=3)]                      # optimised, then short
    tr = tracking.frame_tracker(ex, cam, margin=10.0)
    got = _check(ex, tr, cam, kps, descs, frames, monocular=True)
    assert got[0]["tracked"] and not got[0]["retried"]
    assert got[1]["retried"] and got[1]["n_matches_first"] < 10 <= got[1]["n_matches"]
    assert got[2]["retried"] and not got[2]["tracked"] and np.array_equal(got[2]["pose_cw"], frames[2]["pose_cw"])
    assert [g["tracked"] for g in got] != [True] * 4


def test_degenerate_frames(mods):
    feature, tracking, synth = mods
    ex = feature.orb_extractor(feature.orb_params(), 800, max_batch=2)
    kps, descs = ex.extract_batch(np.stack([synth.make_frame(640, 480, seed=3), np.full((480, 640), 90, np.uint8)]))
    assert len(kps[1]) == 0
    cam = dict(model="perspective", fx=500.0, fy=500.0, cx=320.0, cy=240.0, fxb=0.0, cols=640.0, rows=480.0)
    f0 = synth.make_motion_frame(kps[0], descs[0], cam, ex.orb_params_.scale_factors_, seed=5)
    tb = f0["table"]
    prm = ex.orb_params_
    full = MT.motion_based_track(cam, kps[0], descs[0], f0, prm.scale_factors_, prm.inv_level_sigma_sq_)
    rows = np.sort(full["kp_landmark"][full["kp_landmark"] >= 0])
    rows = rows[tb["has_observation"][rows] == 1][:4]
    few = dict(f0, table={k: v[rows] for k, v in tb.items()})                    # matched, but fewer than 5 edges: the pose stays
    none = dict(f0, table={k: v[:0] for k, v in tb.items()})
    frames = [dict(f0, frame=0), dict(few, frame=0), dict(none, frame=0), dict(f0, frame=1)]
    tr = tracking.frame_tracker(ex, cam, num_matches_thr=3)
    got = _check(ex, tr, cam, kps, descs, frames, monocular=True)
    assert got[1]["n_matches"] >= 3 and np.array_equal(got[1]["pose_cw"], few["pose_cw"])
    assert got[2]["n_matches"] == 0 and got[2]["retried"] and not got[2]["tracked"]
    assert got[3]["n_keypoints"] == 0 and got[3]["n_matches"] == 0


def test_error_paths(mods):
    feature, tracking, synth = mods
    from stella_vslam_b200._lib import B200Error
    ex, kps, descs = _extract(feature, synth, 1241, 376, (50,))
    cam = dict(KITTI, setup="stereo")
    fr = dict(synth.make_motion_frame(kps[0], descs[0], cam, ex.orb_params_.scale_factors_, seed=70, stereo=True), frame=0)
    tr = tracking.frame_tracker(ex, cam, margin=10.0)
    for bad in (dict(fr, kp_x_right=fr["kp_x_right"][:-3]), dict(fr, last_pose_cw=None), dict(fr, frame=1),
                dict(fr, table=dict(fr["table"], octave=np.full(len(fr["table"]["octave"]), 8, np.uint8)))):
        with pytest.raises(B200Error):
            tr.motion_based_track([bad])
    with pytest.raises(B200Error):
        tr.motion_based_track([fr], kp_cap=len(kps[0]) - 1)
    with pytest.raises(B200Error):
        tracking.frame_tracker(ex, cam, margin=10.0, max_candidates=1).motion_based_track([fr])
    mono = tracking.frame_tracker(ex, dict(cam, setup="monocular"), margin=10.0)   # monocular: no last pose needed
    mono.motion_based_track([dict(fr, last_pose_cw=None, kp_x_right=None)])


def test_chain_vs_stage_by_stage_abi(mods):
    # today's path: host reprojection + b200_match_guided mode 1 (twice when short) + b200_pose_optimize, on the device undistortion
    feature, tracking, synth = mods
    from stella_vslam_b200 import match, optimize
    ex, kps, descs = _extract(feature, synth, 1241, 376, (50, 51))
    cam = dict(KITTI, setup="stereo")
    sf = ex.orb_params_.scale_factors_
    frames = [dict(synth.make_motion_frame(kps[0], descs[0], cam, sf, seed=70, stereo=True), frame=0),
              dict(synth.make_motion_frame(kps[1], descs[1], cam, sf, seed=3, stereo=True, shift_px=25.0, landmark_frac=0.05), frame=1)]
    tr = tracking.frame_tracker(ex, cam, margin=10.0)
    got = tr.motion_based_track(frames)
    po = optimize.pose_optimizer()
    for i, (fr, g) in enumerate(zip(frames, got)):
        ref = MT.motion_based_track(cam, kps[i], descs[i], fr, sf, ex.orb_params_.inv_level_sigma_sq_, margin=10.0, true_baseline=tr.true_baseline,
                                    monocular=False, img_bounds=tuple(tr._prm.img_bounds),
                                    undistort_fn=lambda c, k: ex.undistort_keypoints(c, k),
                                    match_fn=lambda pr, mode, thr, lowe_ratio, check_orientation: match.match_guided_batch([pr], mode, thr, lowe_ratio,
                                                                                                                       check_orientation)[0],
                                    pose_fn=lambda pp, a, b, c: po.optimize(pp))
        for k in KEYS:
            assert g[k] == ref[k], (i, k)
        assert np.array_equal(g["kp_landmark"], ref["kp_landmark"]), i
        assert np.abs(g["pose_cw"] - ref["pose_cw"]).max() <= 1e-5 * max(1.0, np.abs(ref["pose_cw"]).max()), i
