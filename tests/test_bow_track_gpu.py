"""GPU parity of the BoW-match tracking chain (b200_bow_match_based_track) against the CPU restatement (tests/bow_track_oracle.py) and
against the stage-by-stage device ABI (b200_keypoints_undistort -> b200_match_pairs -> b200_pose_optimize): kp_landmark_out, n_matches,
applied, n_valid and tracked bit-exact, the pose within 1e-5."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bow_track_oracle as BT  # noqa: E402
import camera_models_oracle as CM  # noqa: E402

pytestmark = pytest.mark.gpu

KITTI = dict(model="perspective", fx=718.856, fy=718.856, cx=607.1928, cy=185.2157, fxb=386.1448, cols=1241.0, rows=376.0)
EUROC = dict(model="perspective", fx=458.654, fy=457.296, cx=367.215, cy=248.375, k1=-0.28340811, k2=0.07395907, p1=0.00019359, p2=1.76187114e-05,
             k3=0.0, fxb=0.0, cols=752.0, rows=480.0)
RADIAL = dict(model="radial_division", fx=612.3, fy=611.7, cx=480.5, cy=270.2, distortion=-0.15, fxb=0.0, cols=960.0, rows=540.0)
KEYS = ("n_keypoints", "n_matches", "applied", "n_valid", "tracked")


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
    if ref["applied"]:
        assert np.array_equal(g["kp_landmark"], ref["kp_landmark"]), tag
        assert np.abs(g["pose_cw"] - ref["pose_cw"]).max() <= 1e-5 * max(1.0, np.abs(ref["pose_cw"]).max()), tag
    else:
        assert g["kp_landmark"] is None and g["pose_cw"] is None, tag


def _check(ex, tr, cam, kps, descs, frames, monocular, **kw):
    got = tr.bow_match_based_track(frames)
    isig = ex.orb_params_.inv_level_sigma_sq_
    for f, (fr, g) in enumerate(zip(frames, got)):
        i = fr.get("frame", f)
        ref = BT.bow_match_based_track(cam, kps[i], descs[i], fr, isig, num_matches_thr=tr.num_matches_thr, monocular=monocular, **kw)
        _same(g, ref, f)
    return got


def test_kitti_stereo(mods):
    feature, tracking, synth = mods
    ex, kps, descs = _extract(feature, synth, 1241, 376, (50, 51, 52))
    cam = dict(KITTI, setup="stereo")
    frames = [dict(synth.make_bow_frame(kps[i], descs[i], cam, seed=70 + i, stereo=True), frame=i) for i in range(3)]
    tr = tracking.frame_tracker(ex, cam)
    got = _check(ex, tr, cam, kps, descs, frames, monocular=False)
    for fr, g in zip(frames, got):
        assert g["tracked"]
        assert np.abs(g["pose_cw"] - fr["gt_pose_cw"]).max() < np.abs(fr["last_pose_cw"] - fr["gt_pose_cw"]).max()
    assert tr.bow_stage_ms()["chain"] > 0


def test_euroc_distortion_out_of_order_subset(mods):
    feature, tracking, synth = mods
    ex, kps, descs = _extract(feature, synth, 752, 480, (80, 81, 82, 83))
    und = [CM.undistort_keypoints(EUROC, k)[0] for k in kps]
    frames = [dict(synth.make_bow_frame(und[i], descs[i], EUROC, seed=90 + i), frame=i) for i in (2, 0)]
    tr = tracking.frame_tracker(ex, EUROC)
    got = _check(ex, tr, EUROC, kps, descs, frames, monocular=True)
    assert all(g["tracked"] for g in got)


def test_equirectangular(mods):
    feature, tracking, synth = mods
    ex, kps, descs = _extract(feature, synth, 1920, 960, (40, 41), n=2500)
    cam = dict(model="equirectangular", cols=1920.0, rows=960.0, fxb=0.0, setup="monocular")
    frames = [dict(synth.make_bow_frame(kps[i], descs[i], cam, seed=45 + i), frame=i) for i in range(2)]
    tr = tracking.frame_tracker(ex, cam)
    got = _check(ex, tr, cam, kps, descs, frames, monocular=True)
    assert all(g["applied"] for g in got)


@pytest.mark.parametrize("model", ["fisheye", "radial_division"])
def test_fisheye_and_radial_division(mods, model):
    feature, tracking, synth = mods
    cam, w, h, seed = (dict(CM.TUM_VI, fxb=0.0), 512, 512, 300) if model == "fisheye" else (RADIAL, 960, 540, 500)
    ex, kps, descs = _extract(feature, synth, w, h, (seed, seed + 1))
    und = [CM.undistort_keypoints(cam, k)[0] for k in kps]
    frames = [dict(synth.make_bow_frame(und[i], descs[i], cam, seed=seed + 10 + i), frame=i) for i in range(2)]
    tr = tracking.frame_tracker(ex, cam)
    got = _check(ex, tr, cam, kps, descs, frames, monocular=True)
    assert all(g["applied"] for g in got)


def test_rgbd_x_right(mods):
    feature, tracking, synth = mods
    ex, kps, descs = _extract(feature, synth, 640, 480, (60, 61))
    cam = dict(model="perspective", fx=525.0, fy=525.0, cx=319.5, cy=239.5, fxb=40.0, cols=640.0, rows=480.0, setup="rgbd")
    frames = [dict(synth.make_bow_frame(kps[i], descs[i], cam, seed=65 + i, stereo=True), frame=i) for i in range(2)]
    tr = tracking.frame_tracker(ex, cam)
    got = _check(ex, tr, cam, kps, descs, frames, monocular=False)
    assert all(g["tracked"] for g in got)


def test_mixed_batch(mods):
    feature, tracking, synth = mods
    ex, kps, descs = _extract(feature, synth, 1241, 376, (50, 51, 52))
    cam = dict(KITTI, setup="monocular")
    isig = ex.orb_params_.inv_level_sigma_sq_
    fr = [synth.make_bow_frame(kps[i], descs[i], cam, seed=20 + i) for i in range(2)]
    short = dict(fr[1], keyframe={k: np.asarray(v)[:30] for k, v in fr[1]["keyframe"].items()})    # n_matches below the threshold
    wrong = synth.make_bow_frame(kps[2], descs[2], cam, seed=23, wrong_depth_frac=0.9, rotated_frac=0.0, clutter_frac=0.0, landmark_frac=0.1)
    # the threshold is the wrong-depth frame's match count: it is applied, and any landmark the discard removes leaves it untracked
    thr = BT.bow_match_based_track(cam, kps[2], descs[2], wrong, isig, num_matches_thr=0)["n_matches"]
    assert thr > 30
    frames = [dict(fr[0], frame=0), dict(short, frame=1), dict(wrong, frame=2)]
    tr = tracking.frame_tracker(ex, cam, num_matches_thr=thr)
    got = _check(ex, tr, cam, kps, descs, frames, monocular=True)
    assert got[0]["tracked"]
    assert got[1]["n_matches"] < thr and not got[1]["applied"] and got[1]["kp_landmark"] is None
    assert got[2]["applied"] and not got[2]["tracked"] and got[2]["pose_cw"] is not None and got[2]["n_valid"] < thr


def test_single_node_is_all_pairs(mods):
    feature, tracking, synth = mods
    ex, kps, descs = _extract(feature, synth, 640, 480, (61,), n=500)
    cam = dict(model="perspective", fx=525.0, fy=525.0, cx=319.5, cy=239.5, fxb=0.0, cols=640.0, rows=480.0, setup="monocular")
    frames = [dict(synth.make_bow_frame(kps[0], descs[0], cam, seed=66, n_nodes=1, unnoded_frac=0.0, kf_unnoded_frac=0.0), frame=0)]
    tr = tracking.frame_tracker(ex, cam, max_candidates=1024)
    got = _check(ex, tr, cam, kps, descs, frames, monocular=True)
    assert got[0]["applied"]


def test_not_applied_leaves_the_callers_buffers(mods):
    feature, tracking, synth = mods
    ex, kps, descs = _extract(feature, synth, 1241, 376, (50,))
    cam = dict(KITTI, setup="monocular")
    fr = dict(synth.make_bow_frame(kps[0], descs[0], cam, seed=20), frame=0)
    tr = tracking.frame_tracker(ex, cam, num_matches_thr=100000)
    packed = tr.pack_bow([fr], len(kps[0]))
    packed[2][0]["kp_landmark"][:] = 7
    T = packed[0][0]
    for k in range(16):
        T.pose_cw_out[k] = 3.0
    tr.run_bow_packed(packed)
    assert not T.applied and T.n_matches > 0 and T.n_valid == 0 and not T.tracked
    assert (packed[2][0]["kp_landmark"] == 7).all() and list(T.pose_cw_out) == [3.0] * 16


def test_batch_of_64(mods):
    feature, tracking, synth = mods
    seeds = tuple(range(200, 208))
    ex = feature.orb_extractor(feature.orb_params(), 2000, max_batch=64)
    imgs = [synth.make_frame(1241, 376, seed=s) for s in seeds]
    kps, descs = ex.extract_batch(np.stack([imgs[i % 8] for i in range(64)]))
    cam = dict(KITTI, setup="stereo")
    frames = [dict(synth.make_bow_frame(kps[i], descs[i], cam, seed=300 + i, stereo=True), frame=i) for i in range(64)]
    tr = tracking.frame_tracker(ex, cam)
    got = tr.bow_match_based_track(frames)
    isig = ex.orb_params_.inv_level_sigma_sq_
    for i in (0, 9, 31, 63):
        _same(got[i], BT.bow_match_based_track(cam, kps[i], descs[i], frames[i], isig, monocular=False), i)
    assert sum(g["tracked"] for g in got) >= 60
    one = tr.bow_match_based_track([frames[31]])[0]                  # a frame's result does not depend on its batch
    _same(one, got[31], "alone")


def test_chain_vs_stage_by_stage_abi(mods):
    feature, tracking, synth = mods
    from stella_vslam_b200 import match, optimize
    ex, kps, descs = _extract(feature, synth, 752, 480, (80, 81))
    frames = [dict(synth.make_bow_frame(CM.undistort_keypoints(EUROC, kps[i])[0], descs[i], EUROC, seed=95 + i), frame=i) for i in range(2)]
    tr = tracking.frame_tracker(ex, EUROC)
    got = tr.bow_match_based_track(frames)
    po = optimize.pose_optimizer()

    def pairs_fn(p):
        return match.match_pairs_batch([p], match.PAIRS_BOW, 0.7, True)[0]
    for i, (fr, g) in enumerate(zip(frames, got)):
        ref = BT.bow_match_based_track(EUROC, kps[i], descs[i], fr, ex.orb_params_.inv_level_sigma_sq_,
                                       undistort_fn=lambda c, k: ex.undistort_keypoints(c, k), match_fn=pairs_fn,
                                       pose_fn=lambda pp, a, b, c: po.optimize(pp))
        _same(g, ref, i)
        assert g["tracked"]


def test_error_paths(mods):
    feature, tracking, synth = mods
    from stella_vslam_b200._lib import ERR_CAPACITY, ERR_INVALID, B200Error
    ex, kps, descs = _extract(feature, synth, 1241, 376, (50,))
    cam = dict(KITTI, setup="stereo")
    fr = dict(synth.make_bow_frame(kps[0], descs[0], cam, seed=70, stereo=True), frame=0)
    tr = tracking.frame_tracker(ex, cam)
    n = len(kps[0])
    bads = (dict(fr, kp_node=fr["kp_node"][:-3], kp_x_right=fr["kp_x_right"][:-3]), dict(fr, kp_node=fr["kp_node"][:-3], kp_x_right=None),
            dict(fr, frame=1))
    for bad in bads:
        with pytest.raises(B200Error) as e:
            tr.bow_match_based_track([bad])
        assert e.value.code == ERR_INVALID
    with pytest.raises(B200Error) as e:
        tr.bow_match_based_track([fr], kp_cap=n - 1)
    assert e.value.code == ERR_INVALID
    packed = tr.pack_bow([fr], n)
    packed[0][0].kf_node = None
    with pytest.raises(B200Error) as e:
        tr.run_bow_packed(packed)
    assert e.value.code == ERR_INVALID
    # a candidate-list overflow: CAPACITY, nothing written
    one = dict(fr, kp_node=np.zeros(n, np.int32), keyframe=dict(fr["keyframe"], node=np.zeros(len(fr["keyframe"]["node"]), np.int32)))
    small = tracking.frame_tracker(ex, cam, max_candidates=1)
    packed = small.pack_bow([one], n)
    packed[2][0]["kp_landmark"][:] = 7
    T = packed[0][0]
    T.n_matches, T.applied = -5, -5
    with pytest.raises(B200Error) as e:
        small.run_bow_packed(packed)
    assert e.value.code == ERR_CAPACITY
    assert (packed[2][0]["kp_landmark"] == 7).all() and T.n_matches == -5 and T.applied == -5
    assert tr.bow_match_based_track([fr])[0]["tracked"]          # the handles still work


def test_four_chains_interleaved_on_one_matcher(mods):
    """The local-map, motion, robust and BoW chains, interleaved on one matcher handle at 1, 8 and 2 frames, forward and then in reverse,
    give bit for bit what the same call gives on a fresh handle."""
    import test_staging_gpu as SG
    feature, tracking, synth = mods
    from stella_vslam_b200 import solve
    ex, kps, descs = _extract(feature, synth, 1241, 376, tuple(range(200, 208)), n=2000)
    cam = dict(KITTI, setup="stereo")
    sf = ex.orb_params_.scale_factors_
    local = [dict(synth.make_tracking_frame(kps[i], descs[i], cam, sf, seed=70 + i, stereo=True), frame=i) for i in range(8)]
    motion = [dict(synth.make_motion_frame(kps[i], descs[i], cam, sf, seed=170 + i, stereo=True), frame=i) for i in range(8)]
    robust = [dict(synth.make_robust_frame(kps[i], descs[i], cam, seed=300 + i, stereo=True), frame=i) for i in range(8)]
    bow = [dict(synth.make_bow_frame(kps[i], descs[i], cam, seed=400 + i, stereo=True), frame=i) for i in range(8)]
    lm, ft = tracking.local_map_tracker(ex, cam), tracking.frame_tracker(ex, cam, use_fixed_seed=True)
    calls = []
    for n in (1, 8, 2):
        calls += [lambda n=n: ft.bow_match_based_track(bow[:n]), lambda n=n: lm.track(local[:n]), lambda n=n: ft.motion_based_track(motion[:n]),
                  lambda n=n: ft.robust_match_based_track([dict(fr, engine=solve.mt19937([i, 7])) for i, fr in enumerate(robust[:n])]),
                  lambda n=n: ft.bow_match_based_track(bow[8 - n:])]
    want = []
    for call in calls:
        with SG._matcher_handle():
            want.append(call())
    assert sum(r["tracked"] for r in want[5]) >= 6                  # the 8-frame BoW call tracks
    with SG._matcher_handle() as h:
        for call, w in zip(calls, want):
            with SG._matcher_handle(h):
                SG._same(call(), w)
        for call, w in zip(reversed(calls), reversed(want)):
            with SG._matcher_handle(h):
                SG._same(call(), w)
