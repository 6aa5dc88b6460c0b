"""GPU parity of the fisheye and radial-division camera models against the CPU restatement (tests/camera_models_oracle.py):
b200_keypoints_undistort (keypoints and bearings), b200_frame_can_observe with landmarks on the image bounds, the keyframe blob export,
feature.camera_image_bounds, b200_track_local_map on TUM-VI-like and AIST-like fisheye frames, and the rejections."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import camera_models_oracle as CM  # noqa: E402

pytestmark = pytest.mark.gpu

TUM_VI, AIST, on_bound_landmarks = CM.TUM_VI, CM.AIST, CM.on_bound_landmarks

RADIAL = dict(model="radial_division", fx=612.3, fy=611.7, cx=641.2, cy=361.9, distortion=-0.15, cols=1280.0, rows=720.0)
STRONG = dict(TUM_VI, k1=-0.5, k2=0.1, k3=0.0, k4=0.0)  # sends many points to the (-1e6, -1e6) sentinel
EUROC = dict(model="perspective", fx=458.654, fy=457.296, cx=367.215, cy=248.375, k1=-0.28340811, k2=0.07395907, p1=0.00019359, p2=1.76187114e-05,
             k3=0.0, cols=752.0, rows=480.0)


@pytest.fixture(scope="module")
def mods():
    from stella_vslam_b200 import _lib, data, feature, tracking
    from workloads import synth
    return _lib, data, feature, tracking, synth


@pytest.fixture(scope="module")
def ex(mods):
    _, _, feature, _, _ = mods
    return feature.orb_extractor(feature.orb_params(), 800, max_batch=2)


def _keypoints(cam, n, seed):
    from oracle import pyoracle as O
    rng = np.random.default_rng(seed)
    k = np.zeros(n, O.KP_DTYPE)
    k["x"] = rng.uniform(-40, cam["cols"] + 40, n).astype(np.float32)
    k["y"] = rng.uniform(-40, cam["rows"] + 40, n).astype(np.float32)
    if n >= 3:
        k["x"][:3] = [0.0, np.float32(cam["cx"]), np.float32(cam["cols"])]
        k["y"][:3] = [0.0, np.float32(cam["cy"]), np.float32(cam["rows"])]
    k["size"] = rng.uniform(7, 40, n).astype(np.float32)
    k["angle"] = rng.uniform(0, 360, n).astype(np.float32)
    k["response"] = rng.uniform(1, 90, n).astype(np.float32)
    k["octave"] = rng.integers(0, 8, n)
    return k


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


def _check_undistorted(cam, got, want, label):
    """Radial division: bit for bit.  Fisheye: bit for bit except where CUDA's tan and glibc's differ, by at most one float ulp."""
    d = np.maximum(_ulps(got["x"], want["x"]), _ulps(got["y"], want["y"]))
    for f in ("size", "angle", "response", "octave"):
        assert np.array_equal(got[f], want[f]), (label, f)
    assert (got["response"] == 0).all()
    if cam["model"] == "radial_division":
        assert (d == 0).all(), (label, int((d != 0).sum()))
    else:
        assert d.max(initial=0) <= 1, (label, int(d.max()))
        print(f"{label}: {int((d != 0).sum())} of {len(d)} keypoints one float ulp apart (CUDA tan vs glibc tan)")
    return d == 0


@pytest.mark.parametrize("cam_name", ["tum_vi", "aist", "strong", "radial"])
@pytest.mark.parametrize("n", [0, 1, 37, 20000])
def test_undistort_and_bearings_vs_oracle(mods, ex, cam_name, n):
    cam = {"tum_vi": TUM_VI, "aist": AIST, "strong": STRONG, "radial": RADIAL}[cam_name]
    kps = _keypoints(cam, n, seed=n + 17)
    got, gb = ex.undistort_keypoints(cam, kps)
    want, wb = CM.undistort_keypoints(cam, kps)
    assert len(got) == n and gb.shape == (n, 3)
    same = _check_undistorted(cam, got, want, f"{cam_name} n={n}")
    assert np.array_equal(gb[same], wb[same])  # bearings: the perspective formula on the same float keypoint, bit for bit
    if cam_name == "strong" and n == 20000:
        assert (got["x"] == CM.SENTINEL).sum() > 100


def test_undistort_without_bearings_and_response_of_old_models(mods, ex):
    """The perspective model still zeroes the response, equirectangular still copies the keypoints."""
    from oracle import pyoracle as O
    kps = _keypoints(EUROC, 500, 3)
    got, b = ex.undistort_keypoints(EUROC, kps, want_bearings=False)
    assert b is None and (got["response"] == 0).all()
    want, _ = O.undistort_keypoints(EUROC, kps)
    assert np.array_equal(got, want)
    eq = dict(model="equirectangular", cols=EUROC["cols"], rows=EUROC["rows"])
    got, _ = ex.undistort_keypoints(eq, kps)
    assert np.array_equal(got, kps)


def test_camera_image_bounds(mods, ex):
    _, _, feature, _, _ = mods
    for cam in (TUM_VI, AIST, RADIAL, dict(RADIAL, distortion=0.0), dict(AIST, k1=0.0, k2=0.0, k3=0.0, k4=0.0)):
        got, want = feature.camera_image_bounds(cam, ex), CM.image_bounds(cam)
        assert _ulps(got, want).max() <= (0 if cam["model"] == "radial_division" else 1), (cam, got, want)
    persp = dict(model="perspective", fx=500.0, fy=500.0, cx=320.0, cy=240.0, cols=640.0, rows=480.0)
    assert feature.camera_image_bounds(persp, ex) == (0.0, 640.0, 0.0, 480.0)


def test_can_observe_on_bound_landmarks(mods, ex):
    cam, bounds, lms, on, inside = on_bound_landmarks()
    for model in ("fisheye", "radial_division"):
        c = dict(cam, model=model)
        got = ex.can_observe(c, np.eye(4), lms, img_bounds=bounds)
        want = CM.can_observe(c, np.eye(4), lms, img_bounds=bounds, num_levels=8, log_scale_factor=ex.orb_params_.log_scale_factor_)
        for k in ("observable", "reproj", "x_right", "pred_scale_level"):
            assert np.array_equal(got[k], want[k]), (model, k)
        assert np.array_equal(got["observable"], inside | on if model == "radial_division" else inside)


@pytest.mark.parametrize("cam_name", ["tum_vi", "aist", "radial"])
def test_can_observe_local_map_default_bounds(mods, ex, cam_name):
    _, _, feature, _, synth = mods
    cam = {"tum_vi": TUM_VI, "aist": AIST, "radial": RADIAL}[cam_name]
    kps = _keypoints(cam, 3000, 5)
    und, _ = CM.undistort_keypoints(cam, kps)
    desc = np.random.default_rng(5).integers(0, 256, (len(kps), 32), dtype=np.uint8)
    fr = synth.make_tracking_frame(und, desc, dict(cam, fxb=0.0), ex.orb_params_.scale_factors_, seed=9)
    bounds = feature.camera_image_bounds(cam, ex)  # the default of can_observe for these models (within an ulp of the oracle's)
    got = ex.can_observe(cam, fr["pose_cw"], fr["landmarks"])
    want = CM.can_observe(cam, fr["pose_cw"], fr["landmarks"], img_bounds=bounds, log_scale_factor=ex.orb_params_.log_scale_factor_)
    for k in ("observable", "reproj", "x_right", "pred_scale_level"):
        assert np.array_equal(got[k], want[k]), k
    assert got["observable"].sum() > 500


@pytest.mark.parametrize("cam_name", ["aist", "radial"])
def test_keyframe_blob_undistorts_the_new_models(mods, ex, cam_name):
    _, data, _, _, synth = mods
    cam = {"aist": AIST, "radial": RADIAL}[cam_name]
    img = synth.make_frame(int(cam["cols"]), int(cam["rows"]), seed=21)
    kps, _ = ex.extract(img)
    blob, _ = data.export_keyframe_blobs(ex, 0, cam)
    want, _ = CM.undistort_keypoints(cam, kps)
    assert len(blob) == len(kps) > 100
    assert (blob["class_id"] == -1).all() and (blob["response"] == 0).all()
    got = np.zeros(len(blob), want.dtype)
    for f in want.dtype.names:
        got[f] = blob[f]
    _check_undistorted(cam, got, want, f"keyframe blob {cam_name}")


def _chain(mods, cam, w, h, grid, seed):
    from oracle import pyoracle as O
    _, _, feature, tracking, synth = mods
    imgs = np.stack([synth.make_frame(w, h, seed=seed + i) for i in range(2)])
    ex = feature.orb_extractor(feature.orb_params(), 800, max_batch=2)
    kps, descs = ex.extract_batch(imgs)
    und = [CM.undistort_keypoints(cam, k)[0] for k in kps]
    for k, u in zip(kps, und):  # the chain's undistortion is the same device function as b200_keypoints_undistort
        got, _ = ex.undistort_keypoints(cam, k)
        assert np.array_equal(got, u)
    c = dict(cam, fxb=0.0, setup="monocular")
    frames = [dict(synth.make_tracking_frame(und[i], descs[i], c, ex.orb_params_.scale_factors_, seed=seed + 10 + i), frame=i) for i in range(2)]
    tr = tracking.local_map_tracker(ex, c, grid=grid)
    got = tr.track(frames)
    prm = ex.orb_params_
    total = 0
    for i, (fr, g) in enumerate(zip(frames, got)):
        ref = CM.track_local_map(c, kps[i], descs[i], fr, prm.scale_factors_, prm.inv_level_sigma_sq_, prm.log_scale_factor_, grid=grid,
                                 img_bounds=tuple(tr._prm.img_bounds))
        assert g["n_keypoints"] == ref["n_keypoints"] == len(kps[i])
        assert np.array_equal(g["observable"], ref["observable"]), i
        assert np.array_equal(g["kp_landmark"], ref["kp_landmark"]), i
        assert g["n_matches"] == ref["n_matches"] and g["n_valid"] == ref["n_valid"], i
        assert np.array_equal(g["kp_outlier"], ref["kp_outlier"]), i
        assert np.abs(g["pose_cw"] - ref["pose_cw"]).max() <= 1e-5 * max(1.0, np.abs(ref["pose_cw"]).max()), i
        assert np.abs(g["pose_cw"] - fr["gt_pose_cw"]).max() < np.abs(fr["pose_cw"] - fr["gt_pose_cw"]).max()
        total += g["n_matches"]
    return total, sum(len(k) for k in kps)


def test_chain_tum_vi_fisheye(mods):
    total, n = _chain(mods, TUM_VI, 512, 512, (16, 16), seed=300)
    assert total > 0.2 * n


def test_chain_aist_fisheye(mods):
    total, n = _chain(mods, AIST, 960, 540, (64, 48), seed=400)
    assert total > 0.2 * n


def test_chain_radial_division(mods):
    total, n = _chain(mods, dict(RADIAL, cols=960.0, rows=540.0, cx=480.5, cy=270.2), 960, 540, (64, 48), seed=500)
    assert total > 0.2 * n


def test_rejections(mods, ex):
    _lib, data, feature, tracking, synth = mods
    from stella_vslam_b200._lib import B200Error, CameraIntrinsics, check, lib, ptr
    import ctypes as C
    kps = _keypoints(AIST, 10, 1)
    out, b = np.zeros(10, kps.dtype), np.zeros((10, 3))
    bad = [_lib.camera_intrinsics(AIST), _lib.camera_intrinsics(dict(AIST, k4=float("nan"))), _lib.camera_intrinsics(dict(RADIAL, distortion=float("inf")))]
    bad[0].model = 4
    pose = np.eye(4)
    lm = np.zeros((1, 3)), np.zeros(1, np.float32)
    flags = np.zeros(1, np.uint8), np.zeros((1, 2)), np.zeros(1, np.float32), np.zeros(1, np.uint32)
    bounds = np.array([0, 960, 0, 540], np.float32)
    ex.extract(synth.make_frame(960, 540, seed=1))
    for cam in bad:
        assert lib().b200_keypoints_undistort(ex._h, C.byref(cam), ptr(kps), 10, ptr(out), ptr(b)) == _lib.ERR_INVALID
        assert lib().b200_frame_can_observe(ex._h, C.byref(cam), 0.0, ptr(bounds), ptr(pose), 1, ptr(lm[0]), ptr(lm[0]), ptr(lm[1]), ptr(lm[1]), 0.5,
                                            8, 0.18, *[ptr(f) for f in flags]) == _lib.ERR_INVALID
        L = lib()
        L.b200_orb_export_keyframe_blobs.argtypes = [C.c_void_p, C.c_int, C.POINTER(CameraIntrinsics), C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int32)]
        n = C.c_int32()
        assert L.b200_orb_export_keyframe_blobs(ex._h, 0, C.byref(cam), None, None, 0, C.byref(n)) == _lib.ERR_INVALID
    tr = tracking.local_map_tracker(ex, dict(AIST, fxb=0.0))
    kp0, d0 = ex.extract(synth.make_frame(960, 540, seed=1))
    fr = synth.make_tracking_frame(kp0, d0, dict(AIST, fxb=0.0), ex.orb_params_.scale_factors_, seed=2)
    for cam in bad:
        tr._prm.cam = cam
        with pytest.raises(B200Error):
            tr.track([fr])
    with pytest.raises(ValueError):
        ex.undistort_keypoints(dict(AIST, model="omnidirectional"), kps)
