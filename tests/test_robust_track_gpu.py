"""GPU parity of the robust-match tracking chain (b200_robust_match_based_track) against the CPU restatement (tests/robust_track_oracle.py)
and against the stage-by-stage device ABI: kp_landmark_out, n_matches, essential_valid, n_inliers, applied, n_valid and tracked bit-exact,
the pose within 1e-5.  The device minimal-set sampler against b200_draw_min_sets, bit for bit."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import camera_models_oracle as CM  # noqa: E402
import robust_track_oracle as RT  # noqa: E402

pytestmark = pytest.mark.gpu

KITTI = dict(model="perspective", fx=718.856, fy=718.856, cx=607.1928, cy=185.2157, fxb=386.1448, cols=1241.0, rows=376.0)
EUROC = dict(model="perspective", fx=458.654, fy=457.296, cx=367.215, cy=248.375, k1=-0.28340811, k2=0.07395907, p1=0.00019359, p2=1.76187114e-05,
             k3=0.0, fxb=0.0, cols=752.0, rows=480.0)
RADIAL = dict(model="radial_division", fx=612.3, fy=611.7, cx=480.5, cy=270.2, distortion=-0.15, fxb=0.0, cols=960.0, rows=540.0)
KEYS = ("n_keypoints", "n_matches", "essential_valid", "n_inliers", "applied", "n_valid", "tracked")


@pytest.fixture(scope="module")
def mods():
    from stella_vslam_b200 import feature, tracking
    from workloads import synth
    return feature, tracking, synth


def _extract(feature, synth, w, h, seeds, n=800):
    ex = feature.orb_extractor(feature.orb_params(), n, max_batch=len(seeds))
    kps, descs = ex.extract_batch(np.stack([synth.make_frame(w, h, seed=s) for s in seeds]))
    return ex, kps, descs


def _same(g, ref, tag):
    for k in KEYS:
        assert g[k] == ref[k], (tag, k, g[k], ref[k])
    assert g["status"] == ref["status"], tag
    if ref["applied"]:
        assert np.array_equal(g["kp_landmark"], ref["kp_landmark"]), tag
        assert np.abs(g["pose_cw"] - ref["pose_cw"]).max() <= 1e-5 * max(1.0, np.abs(ref["pose_cw"]).max()), tag
    else:
        assert g["kp_landmark"] is None and g["pose_cw"] is None, tag


def _check(ex, tr, cam, kps, descs, frames, monocular, **kw):
    got = tr.robust_match_based_track(frames)
    isig = ex.orb_params_.inv_level_sigma_sq_
    for f, (fr, g) in enumerate(zip(frames, got)):
        i = fr.get("frame", f)
        ref = RT.robust_match_based_track(cam, kps[i], descs[i], fr, isig, num_matches_thr=tr.num_matches_thr, monocular=monocular, **kw)
        _same(g, ref, f)
    return got


@pytest.mark.parametrize("seeded", [False, True])
@pytest.mark.parametrize("n", [5, 6, 7, 8, 9, 50, 2000])
def test_device_sampler_matches_the_host_sampler(n, seeded):
    from stella_vslam_b200 import solve
    seeds = ([7, 11, 13], [1, 2, 3, 4, 5, 6, 7, 8, 9, 10]) if seeded else (None, None)
    engines = [solve.mt19937(s) for s in seeds]
    got = solve.draw_min_sets_batch([n, n], 1000, engines if seeded else None, set_size=5)
    for p in range(2):
        want = solve.draw_min_sets(n, 1000, solve.mt19937(seeds[p]), set_size=5)
        assert np.array_equal(got[p], want), p


def test_device_sampler_continues_an_advanced_engine():
    from stella_vslam_b200 import solve
    e = solve.mt19937([42])
    solve.draw_min_sets(9, 37, e, set_size=5)                   # index mid-block: the next twist comes during the device draws
    ref = solve.Mt19937.from_buffer_copy(e)
    got = solve.draw_min_sets_batch([9], 1000, [e], set_size=5)[0]
    assert np.array_equal(got, solve.draw_min_sets(9, 1000, ref, set_size=5))


def test_kitti_stereo(mods):
    feature, tracking, synth = mods
    ex, kps, descs = _extract(feature, synth, 1241, 376, (50, 51, 52))
    cam = dict(KITTI, setup="stereo")
    frames = [dict(synth.make_robust_frame(kps[i], descs[i], cam, seed=70 + i, stereo=True), frame=i) for i in range(3)]
    tr = tracking.frame_tracker(ex, cam, use_fixed_seed=True)
    got = _check(ex, tr, cam, kps, descs, frames, monocular=False)
    for fr, g in zip(frames, got):
        assert g["tracked"]
        assert np.abs(g["pose_cw"] - fr["gt_pose_cw"]).max() < np.abs(fr["last_pose_cw"] - fr["gt_pose_cw"]).max()
    assert tr.robust_stage_ms()["chain"] > 0


def test_euroc_distortion_out_of_order_subset_seeded(mods):
    feature, tracking, synth = mods
    from stella_vslam_b200 import solve
    ex, kps, descs = _extract(feature, synth, 752, 480, (80, 81, 82, 83))
    und = [CM.undistort_keypoints(EUROC, k)[0] for k in kps]
    frames = [dict(synth.make_robust_frame(und[i], descs[i], EUROC, seed=90 + i), frame=i, engine=solve.mt19937([i, 5])) for i in (2, 0)]
    tr = tracking.frame_tracker(ex, EUROC)
    got = _check(ex, tr, EUROC, kps, descs, frames, monocular=True)
    assert all(g["tracked"] for g in got)


def test_equirectangular(mods):
    feature, tracking, synth = mods
    ex, kps, descs = _extract(feature, synth, 1920, 960, (40, 41), n=2500)
    cam = dict(model="equirectangular", cols=1920.0, rows=960.0, fxb=0.0, setup="monocular")
    frames = [dict(synth.make_robust_frame(kps[i], descs[i], cam, seed=45 + i), frame=i) for i in range(2)]
    tr = tracking.frame_tracker(ex, cam, use_fixed_seed=True)
    got = _check(ex, tr, cam, kps, descs, frames, monocular=True)
    assert all(g["applied"] for g in got)


@pytest.mark.parametrize("model", ["fisheye", "radial_division"])
def test_fisheye_and_radial_division(mods, model):
    feature, tracking, synth = mods
    cam, w, h, seed = (dict(CM.TUM_VI, fxb=0.0), 512, 512, 300) if model == "fisheye" else (RADIAL, 960, 540, 500)
    ex, kps, descs = _extract(feature, synth, w, h, (seed, seed + 1))
    und = [CM.undistort_keypoints(cam, k)[0] for k in kps]
    frames = [dict(synth.make_robust_frame(und[i], descs[i], cam, seed=seed + 10 + i), frame=i) for i in range(2)]
    tr = tracking.frame_tracker(ex, cam, use_fixed_seed=True)
    got = _check(ex, tr, cam, kps, descs, frames, monocular=True)
    assert all(g["applied"] for g in got)


def test_rgbd_x_right(mods):
    feature, tracking, synth = mods
    ex, kps, descs = _extract(feature, synth, 640, 480, (60, 61))
    cam = dict(model="perspective", fx=525.0, fy=525.0, cx=319.5, cy=239.5, fxb=40.0, cols=640.0, rows=480.0, setup="rgbd")
    frames = [dict(synth.make_robust_frame(kps[i], descs[i], cam, seed=65 + i, stereo=True), frame=i) for i in range(2)]
    tr = tracking.frame_tracker(ex, cam, use_fixed_seed=True)
    got = _check(ex, tr, cam, kps, descs, frames, monocular=False)
    assert all(g["tracked"] for g in got)


def test_mixed_batch(mods):
    feature, tracking, synth = mods
    ex, kps, descs = _extract(feature, synth, 1241, 376, (50, 51, 52, 53))
    cam = dict(KITTI, setup="monocular")
    fr = [synth.make_robust_frame(kps[i], descs[i], cam, seed=20 + i) for i in range(4)]
    few = dict(fr[1], keyframe={k: v[:4] for k, v in fr[1]["keyframe"].items()})          # < 5 brute-force matches
    short = dict(fr[2], keyframe={k: v[:30] for k, v in fr[2]["keyframe"].items()})        # n_inliers below the threshold
    wrong = synth.make_robust_frame(kps[3], descs[3], cam, seed=23, wrong_depth_frac=0.9, rotated_frac=0.0, clutter_frac=0.0, landmark_frac=0.05)
    frames = [dict(fr[0], frame=0), dict(few, frame=1), dict(short, frame=2), dict(wrong, frame=3)]
    tr = tracking.frame_tracker(ex, cam, num_matches_thr=30, use_fixed_seed=True)
    got = _check(ex, tr, cam, kps, descs, frames, monocular=True)
    assert got[0]["tracked"]
    assert got[1]["n_matches"] < 5 and not got[1]["essential_valid"] and not got[1]["applied"]
    assert 0 < got[2]["n_inliers"] < 30 and not got[2]["applied"] and got[2]["kp_landmark"] is None
    assert got[3]["applied"] and not got[3]["tracked"] and got[3]["pose_cw"] is not None


def test_not_applied_leaves_the_callers_buffers(mods):
    feature, tracking, synth = mods
    ex, kps, descs = _extract(feature, synth, 1241, 376, (50,))
    cam = dict(KITTI, setup="monocular")
    fr = dict(synth.make_robust_frame(kps[0], descs[0], cam, seed=20), frame=0)
    tr = tracking.frame_tracker(ex, cam, num_matches_thr=100000, use_fixed_seed=True)
    packed = tr.pack_robust([fr], len(kps[0]))
    packed[2][0]["kp_landmark"][:] = 7
    T = packed[0][0]
    for k in range(16):
        T.pose_cw_out[k] = 3.0
    tr.run_robust_packed(packed)
    assert not T.applied and T.n_inliers > 0
    assert (packed[2][0]["kp_landmark"] == 7).all() and list(T.pose_cw_out) == [3.0] * 16


def test_batch_of_64(mods):
    feature, tracking, synth = mods
    seeds = tuple(range(200, 208))
    ex = feature.orb_extractor(feature.orb_params(), 2000, max_batch=64)
    imgs = [synth.make_frame(1241, 376, seed=s) for s in seeds]
    kps, descs = ex.extract_batch(np.stack([imgs[i % 8] for i in range(64)]))
    cam = dict(KITTI, setup="stereo")
    frames = [dict(synth.make_robust_frame(kps[i], descs[i], cam, seed=300 + i, stereo=True), frame=i) for i in range(64)]
    tr = tracking.frame_tracker(ex, cam, use_fixed_seed=True)
    got = tr.robust_match_based_track(frames)
    isig = ex.orb_params_.inv_level_sigma_sq_
    for i in (0, 9, 31, 63):
        _same(got[i], RT.robust_match_based_track(cam, kps[i], descs[i], frames[i], isig, monocular=False), i)
    assert sum(g["tracked"] for g in got) >= 60


def test_chain_vs_stage_by_stage_abi(mods):
    # b200_keypoints_undistort -> b200_match_bruteforce -> b200_draw_min_sets -> b200_essential_ransac -> b200_pose_optimize
    feature, tracking, synth = mods
    from stella_vslam_b200 import match, optimize, solve
    ex, kps, descs = _extract(feature, synth, 752, 480, (80, 81))
    frames = [dict(synth.make_robust_frame(CM.undistort_keypoints(EUROC, kps[i])[0], descs[i], EUROC, seed=95 + i), frame=i,
                   engine=solve.mt19937([9, i])) for i in range(2)]
    tr = tracking.frame_tracker(ex, EUROC)
    got = tr.robust_match_based_track(frames)
    rb = match.robust(0.8, True)
    po = optimize.pose_optimizer()
    for i, (fr, g) in enumerate(zip(frames, got)):
        ref = RT.robust_match_based_track(EUROC, kps[i], descs[i], fr, ex.orb_params_.inv_level_sigma_sq_,
                                          undistort_fn=lambda c, k: ex.undistort_keypoints(c, k),
                                          match_fn=lambda d1, a1, d2, a2, v2, lowe, ori: rb.brute_force_match(d1, a1, d2, a2, v2),
                                          ransac_fn=lambda b1, b2, ms, rc: solve.essential_ransac_batch([dict(bearings_1=b1, bearings_2=b2, min_sets=ms,
                                                                                                              recompute=rc)])[0],
                                          pose_fn=lambda pp, a, b, c: po.optimize(pp))
        _same(g, ref, i)
        assert g["tracked"]


def test_error_paths(mods):
    feature, tracking, synth = mods
    from stella_vslam_b200._lib import B200Error
    ex, kps, descs = _extract(feature, synth, 1241, 376, (50,))
    cam = dict(KITTI, setup="stereo")
    fr = dict(synth.make_robust_frame(kps[0], descs[0], cam, seed=70, stereo=True), frame=0)
    tr = tracking.frame_tracker(ex, cam, use_fixed_seed=True)
    for bad in (dict(fr, kp_x_right=fr["kp_x_right"][:-3]), dict(fr, frame=1)):
        with pytest.raises(B200Error):
            tr.robust_match_based_track([bad])
    with pytest.raises(B200Error):
        tr.robust_match_based_track([fr], kp_cap=len(kps[0]) - 1)
    packed = tr.pack_robust([fr], len(kps[0]))
    packed[0][0].kf_bearings = None
    with pytest.raises(B200Error):
        tr.run_robust_packed(packed)
    packed = tr.pack_robust([fr], len(kps[0]))
    packed[0][0].last_pose_cw = None
    with pytest.raises(B200Error):
        tr.run_robust_packed(packed)
    assert tr.robust_match_based_track([fr])[0]["tracked"]      # the handles still work
