"""GPU parity of the RGB-D frame step (b200_rgbd_depths) and the depth-seeded landmarks (b200_depth_landmarks) against the CPU
restatement (tests/rgbd_oracle.py), their agreement with b200_keypoints_undistort and b200_landmark_geometry, an RGB-D frame through
b200_track_local_map, and the rejections."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import rgbd_oracle as RO  # noqa: E402

pytestmark = pytest.mark.gpu

CAMERAS = {
    "tum_rgbd": RO.TUM_RGBD,
    "fisheye": dict(model="fisheye", fx=300.5, fy=301.2, cx=320.4, cy=240.7, k1=-3.07e-02, k2=-3.34e-03, k3=-2.88e-03, k4=-5.92e-04, cols=640.0,
                    rows=480.0),
    "radial_division": dict(model="radial_division", fx=402.3, fy=401.7, cx=321.2, cy=239.9, distortion=-0.12, cols=640.0, rows=480.0),
}
FACTOR = 5000.0


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


@pytest.fixture(scope="module")
def mods():
    from stella_vslam_b200 import _lib, feature, mapping, match, tracking
    from workloads import synth
    return _lib, feature, mapping, match, tracking, synth


@pytest.fixture(scope="module")
def batches(mods):
    """64 RGB-D frames of 640x480: gray (64, h, w), u16 depth maps at FACTOR, f32 depth maps in metres with NaN / negative / +inf."""
    synth = mods[5]
    frames = [synth.make_rgbd_frames(seed=s) for s in range(64)]
    g = np.stack([f[0] for f in frames])
    return g, np.stack([f[1] for f in frames]), np.stack([f[2] for f in frames])


def _extract(feature, gray, n):
    ex = feature.orb_extractor(feature.orb_params(), 800, max_batch=n)
    kps, descs = ex.extract_batch(gray[:n])
    return ex, kps, descs


@pytest.mark.parametrize("n", [1, 64])
@pytest.mark.parametrize("cam_name", sorted(CAMERAS))
def test_rgbd_depths_vs_oracle(mods, batches, cam_name, n):
    _, feature, _, _, _, _ = mods
    gray, d16, d32 = batches
    ex, kps, _ = _extract(feature, gray, n)
    cam = CAMERAS[cam_name]
    for maps, factor in ((d16, FACTOR), (d32, 1.0), (d32, FACTOR)):
        got = ex.rgbd_depths(cam, maps[:n], factor, RO.TUM_FXB)
        assert len(got) == n
        n_valid = 0
        for f in range(n):
            want = RO.rgbd_frame(cam, kps[f], maps[f], factor, RO.TUM_FXB)
            g = got[f]
            assert len(g["depths"]) == len(kps[f]) > 100
            for fld in ("x", "y", "size", "angle", "response", "octave"):
                assert np.array_equal(_bits(g["undist_keypts"][fld]), _bits(want["undist_keypts"][fld])), (f, fld)
            assert np.array_equal(_bits(g["bearings"]), _bits(want["bearings"])), f
            assert np.array_equal(_bits(g["depths"]), _bits(want["depths"])), f
            assert np.array_equal(_bits(g["x_right"]), _bits(want["x_right"])), f
            n_valid += int((g["depths"] > 0).sum())
        assert n_valid > 0.5 * sum(len(k) for k in kps[:n])
        if n == 1:  # the undistortion is b200_keypoints_undistort's, bit for bit
            und, b = ex.undistort_keypoints(cam, kps[0])
            assert np.array_equal(np.ascontiguousarray(und).view(np.uint8), np.ascontiguousarray(got[0]["undist_keypts"]).view(np.uint8))
            assert np.array_equal(_bits(b), _bits(got[0]["bearings"]))


def test_rgbd_depths_frame_subset_and_strided_maps(mods, batches):
    _, feature, _, _, _, _ = mods
    gray, d16, _ = batches
    ex, kps, _ = _extract(feature, gray, 4)
    cam = CAMERAS["tum_rgbd"]
    padded = np.zeros((4, 480, 700), np.uint16)  # rows 1400 bytes apart
    padded[:, :, :640] = d16[:4]
    got = ex.rgbd_depths(cam, padded[:, :, :640], FACTOR, RO.TUM_FXB, n_frames=2)
    assert len(got) == 2
    for f in range(2):
        want = RO.rgbd_frame(cam, kps[f], d16[f], FACTOR, RO.TUM_FXB)
        assert np.array_equal(_bits(got[f]["depths"]), _bits(want["depths"])) and np.array_equal(_bits(got[f]["x_right"]), _bits(want["x_right"]))


def _random_problem(mode, n, seed, n_invalid_frac=0.3, thr=3.0):
    rng = np.random.default_rng(seed)
    depth = rng.uniform(0.3, 9.0, n).astype(np.float32)
    depth[rng.random(n) < n_invalid_frac] = -1
    if n:
        depth[rng.integers(0, n, max(1, n // 20))] = depth[rng.integers(0, n)]  # ties
    a = rng.normal(0, 0.5, 3)
    th = np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]]) / th
    pose = np.eye(4)
    pose[:3, :3] = np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K
    pose[:3, 3] = rng.normal(0, 3, 3)
    sf = np.cumprod(np.concatenate([[np.float32(1.0)], np.full(7, np.float32(1.2))])).astype(np.float32)
    return dict(mode=mode, pose_wc=pose, fx_inv=1.0 / 517.306408, fy_inv=1.0 / 516.469215, cx=318.643040, cy=255.313989, depth_thr=thr,
                x=rng.uniform(0, 640, n).astype(np.float32), y=rng.uniform(0, 480, n).astype(np.float32), octave=rng.integers(0, 8, n).astype(np.int32),
                depth=depth, has_landmark=(rng.random(n) < 0.15).astype(np.uint8) if mode == 0 else None, scale_factors=sf,
                inv_scale_factor_last=np.float32(np.float32(1.0) / sf[-1]))


def _check_landmarks(got, want):
    assert np.array_equal(got["idx"], want["idx"])
    for f in ("pos_w", "mean_normal", "min_valid_dist", "max_valid_dist"):
        assert np.array_equal(_bits(got[f]), _bits(want[f])), f


def test_depth_landmarks_vs_oracle_mixed_batch(mods):
    mapping = mods[2]
    sizes = [0, 1, 50, 101, 102, 250, 2000, 2000, 4000, 9000, 17]
    probs = [_random_problem(k % 2, n, 100 + k) for k, n in enumerate(sizes)]
    probs.append(_random_problem(0, 3000, 7, thr=100.0))  # every valid depth below depth_thr: the walk covers all of them
    probs.append(_random_problem(0, 3000, 8, thr=0.0))    # none below: exactly the first 101 positions
    got = mapping.depth_landmarks(probs)
    for k, (g, pr) in enumerate(zip(got, probs)):
        assert g["status"] == 0
        _check_landmarks(g, RO.depth_landmarks(pr))
    assert len(got[-1]["idx"]) <= 101 and len(got[-2]["idx"]) > 1500
    # results do not depend on the batch
    for k in (3, 6):
        _check_landmarks(mapping.depth_landmarks([probs[k]])[0], got[k])


def test_depth_landmarks_geometry_is_landmark_geometry(mods):
    _, _, mapping, match, _, _ = mods
    pr = _random_problem(1, 1500, 21)
    g = mapping.depth_landmarks([pr])[0]
    c = pr["pose_wc"][:3, 3]
    n = len(g["idx"])
    mn, mx, mi = match.landmark_geometry(g["pos_w"], [c[None]] * n, np.tile(c, (n, 1)), pr["scale_factors"][pr["octave"][g["idx"]]],
                                         pr["inv_scale_factor_last"])
    assert np.array_equal(_bits(mn), _bits(g["mean_normal"]))
    assert np.array_equal(_bits(mx), _bits(g["max_valid_dist"])) and np.array_equal(_bits(mi), _bits(g["min_valid_dist"]))


def test_depth_landmarks_from_rgbd_frames(mods, batches):
    # the keyframe path end to end: extract, b200_rgbd_depths, then both landmark modes on the returned undistorted keypoints and depths
    _, feature, mapping, _, _, _ = mods
    gray, d16, _ = batches
    ex, kps, _ = _extract(feature, gray, 8)
    cam = CAMERAS["tum_rgbd"]
    frames = ex.rgbd_depths(cam, d16[:8], FACTOR, RO.TUM_FXB)
    prm = ex.orb_params_
    probs = []
    for f, fr in enumerate(frames):
        pose = np.eye(4)
        pose[:3, 3] = [0.1 * f, 0.0, -0.05 * f]
        probs.append(dict(mode=f % 2, pose_wc=pose, fx_inv=1.0 / cam["fx"], fy_inv=1.0 / cam["fy"], cx=cam["cx"], cy=cam["cy"], depth_thr=RO.TUM_DEPTH_THR,
                          x=fr["undist_keypts"]["x"], y=fr["undist_keypts"]["y"], octave=fr["undist_keypts"]["octave"], depth=fr["depths"],
                          has_landmark=None, scale_factors=prm.scale_factors_, inv_scale_factor_last=prm.inv_scale_factors_[-1]))
    got = mapping.depth_landmarks(probs)
    for g, pr in zip(got, probs):
        _check_landmarks(g, RO.depth_landmarks(pr))
        assert len(g["idx"]) > 100


def test_rgbd_frame_through_the_tracking_chain(mods, batches):
    _lib, feature, _, _, tracking, synth = mods
    from oracle import pyoracle as O
    gray, d16, _ = batches
    ex, kps, descs = _extract(feature, gray, 3)
    cam = dict(RO.TUM_RGBD, fxb=RO.TUM_FXB, setup="RGBD")
    rgbd = ex.rgbd_depths(cam, d16[:3], FACTOR, RO.TUM_FXB)
    bounds = (-30.0, 670.0, -25.0, 505.0)
    frames = []
    for i in range(3):
        fr = synth.make_tracking_frame(rgbd[i]["undist_keypts"], descs[i], cam, ex.orb_params_.scale_factors_, seed=300 + i)
        fr["kp_x_right"] = rgbd[i]["x_right"]
        frames.append(dict(fr, frame=i))
    tr = tracking.local_map_tracker(ex, cam, margin=10.0, img_bounds=bounds)
    got = tr.track(frames)
    prm = ex.orb_params_
    total = 0
    for i, (fr, g) in enumerate(zip(frames, got)):
        ref = O.track_local_map(cam, kps[i], descs[i], fr, prm.scale_factors_, prm.inv_level_sigma_sq_, prm.log_scale_factor_, margin=10.0,
                                monocular=False, img_bounds=bounds)
        assert np.array_equal(g["kp_landmark"], ref["kp_landmark"]), i
        assert np.array_equal(g["kp_outlier"], ref["kp_outlier"]), i
        assert g["n_matches"] == ref["n_matches"] and g["n_valid"] == ref["n_valid"], i
        assert np.abs(g["pose_cw"] - ref["pose_cw"]).max() <= 1e-5 * max(1.0, np.abs(ref["pose_cw"]).max()), i
        assert (fr["kp_x_right"] >= 0).sum() > 100
        total += g["n_matches"]
    assert total > 200


def test_rejections(mods, batches):
    _lib, feature, mapping, _, _, _ = mods
    gray, d16, d32 = batches
    ex, kps, _ = _extract(feature, gray, 2)
    cam = CAMERAS["tum_rgbd"]
    with pytest.raises(ValueError):  # neither CV_16UC1 nor CV_32FC1
        ex.rgbd_depths(cam, d16[:2].astype(np.float64), FACTOR, RO.TUM_FXB)
    with pytest.raises(_lib.B200Error) as e:  # another depth type through the ABI
        _raw_rgbd(_lib, ex, cam, d16[:2], depth_type=0)
    assert e.value.code == _lib.ERR_INVALID
    for bad in (d16[:2, :, :600], d16[:2, :400]):  # size differs from the extracted frames
        with pytest.raises(_lib.B200Error) as e:
            ex.rgbd_depths(cam, np.ascontiguousarray(bad), FACTOR, RO.TUM_FXB)
        assert e.value.code == _lib.ERR_INVALID
    with pytest.raises(_lib.B200Error) as e:  # equirectangular
        ex.rgbd_depths(dict(model="equirectangular", cols=640.0, rows=480.0), d16[:2], FACTOR, RO.TUM_FXB)
    assert e.value.code == _lib.ERR_INVALID
    with pytest.raises(_lib.B200Error) as e:  # capacity: the counts are still written
        ex.rgbd_depths(cam, d16[:2], FACTOR, RO.TUM_FXB, cap=10)
    assert e.value.code == _lib.ERR_CAPACITY
    counts = _raw_rgbd(_lib, ex, cam, d16[:2], cap=10, expect=_lib.ERR_CAPACITY)
    assert counts.tolist() == [len(k) for k in kps]
    with pytest.raises(_lib.B200Error):  # more frames than the last extract holds
        ex.rgbd_depths(cam, np.concatenate([d16[:2], d16[:1]]), FACTOR, RO.TUM_FXB)
    # depth landmarks: the bad problem is reported, the good one still runs
    good = _random_problem(0, 500, 1)
    eq = dict(_random_problem(1, 200, 2), model=1)
    oct_bad = _random_problem(0, 200, 3)
    oct_bad["octave"] = oct_bad["octave"].copy()
    oct_bad["octave"][np.nonzero(oct_bad["depth"] > 0)[0][0]] = 8
    eq_no_depth = dict(_random_problem(1, 50, 4), model=1)
    eq_no_depth["depth"] = np.full(50, -1, np.float32)  # no valid depth: nothing to unproject, nothing thrown
    big = _random_problem(0, 9000, 5, n_invalid_frac=0.0)  # more valid depths than one CTA sorts
    res = mapping.depth_landmarks([good, eq, oct_bad, eq_no_depth, big], raise_on_error=False)
    assert [r["status"] for r in res] == [0, _lib.ERR_INVALID, _lib.ERR_INVALID, 0, _lib.ERR_CAPACITY]
    _check_landmarks(res[0], RO.depth_landmarks(good))
    assert all(len(r["idx"]) == 0 for r in res[1:])
    with pytest.raises(_lib.B200Error) as e:
        mapping.depth_landmarks([good, eq])
    assert e.value.code == _lib.ERR_INVALID
    assert mapping.DEPTH_LANDMARKS_MAX_SORT == 8192
    ok = _random_problem(0, 8192, 6, n_invalid_frac=0.0)  # exactly at the limit: runs
    _check_landmarks(mapping.depth_landmarks([ok])[0], RO.depth_landmarks(ok))


def _raw_rgbd(_lib, ex, cam, maps, depth_type=2, cap=4000, expect=None):
    import ctypes as C
    n = maps.shape[0]
    und = np.zeros((n, cap), _lib.KP_DTYPE)
    b = np.zeros((n, cap, 3))
    d, xr, counts = np.zeros((n, cap), np.float32), np.zeros((n, cap), np.float32), np.zeros(n, np.int32)
    ci = _lib.camera_intrinsics(cam)
    rc = _lib.lib().b200_rgbd_depths(ex._h, n, C.byref(ci), RO.TUM_FXB, FACTOR, depth_type, _lib.ptr(maps), maps.shape[2], maps.shape[1],
                                     maps.strides[1], maps.strides[0], cap, _lib.ptr(und), _lib.ptr(b), _lib.ptr(d), _lib.ptr(xr), _lib.ptr(counts))
    if expect is None:
        _lib.check(rc)
    else:
        assert rc == expect
    return counts
