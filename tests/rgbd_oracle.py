"""CPU restatement of the RGB-D frame step and of the depth-seeded landmarks (test infrastructure): loads tests/rgbd_oracle.c, compiled on
first use into a temporary directory (the tree is never written).

  rgbd_frame(camera, kps, depth_map, factor, fxb)   system::create_RGBD_frame after the extraction (undistortion and bearings from the
                                                     camera oracles, depth and x_right from rgbd_oracle.c)
  depth_landmarks(problem)                           keyframe_inserter (mode 0) / create_map_for_stereo (mode 1) with triangulate_stereo
"""
import ctypes as C

import numpy as np

import camera_models_oracle as CM
import cbuild

DEPTH_TYPES = {np.dtype(np.uint16): 2, np.dtype(np.float32): 5}  # cv::Mat::type() codes
# TUM RGB-D (fr1 / freiburg1 calibration of the reference's example/tum_rgbd configs), 640x480
TUM_RGBD = dict(model="perspective", fx=517.306408, fy=516.469215, cx=318.643040, cy=255.313989, k1=0.262383, k2=-0.953104, p1=-0.005358,
                p2=0.002628, k3=1.163314, cols=640.0, rows=480.0)
TUM_FXB = 40.0           # focal_x_baseline of the TUM RGB-D configs (Camera.focal_x_baseline)
TUM_DEPTH_THR = (40.0 / 517.306408) * 40.0  # camera::base::depth_thr_ = true_baseline (fxb / fx) x depth_threshold (40)
_lib = None


def lib():
    global _lib
    if _lib is None:
        L = cbuild.load("rgbd_oracle.c")
        vp, f32, f64, i32 = C.c_void_p, C.c_float, C.c_double, C.c_int
        L.rgo_depths.argtypes = [vp, vp, vp, i32, vp, i32, i32, i32, C.c_size_t, f64, f64, vp, vp]
        L.rgo_depths.restype = None
        L.rgo_depth_landmarks.argtypes = [i32, vp, f64, f64, f64, f64, f64, i32, vp, vp, vp, vp, vp, vp, f32, vp, vp, vp, vp, vp]
        L.rgo_depth_landmarks.restype = i32
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data


def depths(kps, undist_x, depth_map, factor, fxb):
    """(depths, x_right) float32 for keypoints `kps` (distorted, KP_DTYPE) whose undistorted x is `undist_x`."""
    dm = np.ascontiguousarray(depth_map)
    kx = np.ascontiguousarray(kps["x"], np.float32)
    ky = np.ascontiguousarray(kps["y"], np.float32)
    ux = np.ascontiguousarray(undist_x, np.float32)
    n = len(kx)
    d, xr = np.zeros(max(n, 1), np.float32), np.zeros(max(n, 1), np.float32)
    lib().rgo_depths(_p(kx), _p(ky), _p(ux), n, _p(dm), DEPTH_TYPES[dm.dtype], dm.shape[1], dm.shape[0], dm.strides[0], float(factor), float(fxb),
                     _p(d), _p(xr))
    return d[:n], xr[:n]


def rgbd_frame(camera, kps, depth_map, factor, fxb):
    """dict(undist_keypts, bearings, depths, x_right) as feature.orb_extractor.rgbd_depths returns it for one frame."""
    und, b = CM.undistort_keypoints(camera, kps)
    d, xr = depths(kps, und["x"], depth_map, factor, fxb)
    return dict(undist_keypts=und, bearings=b, depths=d, x_right=xr)


def depth_landmarks(pr):
    """pr: the dict mapping.depth_landmarks takes.  Returns dict(idx, pos_w, mean_normal, min_valid_dist, max_valid_dist)."""
    x = np.ascontiguousarray(pr["x"], np.float32)
    y = np.ascontiguousarray(pr["y"], np.float32)
    octv = np.ascontiguousarray(pr["octave"], np.int32)
    dep = np.ascontiguousarray(pr["depth"], np.float32)
    hl = None if pr.get("has_landmark") is None else np.ascontiguousarray(pr["has_landmark"], np.uint8)
    sf = np.ascontiguousarray(pr["scale_factors"], np.float32)
    pose = np.ascontiguousarray(pr["pose_wc"], np.float64).reshape(16)
    n = len(x)
    m = max(n, 1)
    idx, pos, mn = np.zeros(m, np.int32), np.zeros((m, 3)), np.zeros((m, 3))
    lo, hi = np.zeros(m, np.float32), np.zeros(m, np.float32)
    k = lib().rgo_depth_landmarks(int(pr["mode"]), _p(pose), float(pr["fx_inv"]), float(pr["fy_inv"]), float(pr["cx"]), float(pr["cy"]),
                                  float(pr.get("depth_thr", 0.0)), n, _p(x), _p(y), _p(octv), _p(dep), _p(hl), _p(sf),
                                  float(pr["inv_scale_factor_last"]), _p(idx), _p(pos), _p(mn), _p(lo), _p(hi))
    return dict(idx=idx[:k].copy(), pos_w=pos[:k].copy(), mean_normal=mn[:k].copy(), min_valid_dist=lo[:k].copy(), max_valid_dist=hi[:k].copy())
