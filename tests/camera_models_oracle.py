"""CPU restatement of the fisheye and radial-division camera steps (test infrastructure): loads tests/camera_models_oracle.c, compiled on
first use into a temporary directory (the tree is never written).  Perspective and equirectangular cameras go to oracle/pyoracle.py.

  undistort_keypoints(camera, kps)     camera::*::undistort_keypoints + convert_keypoints_to_bearings
  image_bounds(camera)                 camera::*::compute_image_bounds, with this module's undistortion
  can_observe(camera, pose_cw, lms)    data::frame::can_observe
  track_local_map(camera, ...)         the per-frame chain of pyoracle.track_local_map for all four models
"""
import ctypes as C
import math

import numpy as np

from oracle import pyoracle as O

import cbuild

MODELS = {"perspective": 0, "equirectangular": 1, "fisheye": 2, "radial_division": 3}
SENTINEL = np.float32(-1000000.0)
# example/tum_vi/TUM_VI_mono.yaml and example/aist/fisheye.yaml of the reference
TUM_VI = dict(model="fisheye", fx=190.97847715128717, fy=190.9733070521226, cx=254.93170605935475, cy=256.8974428996504, k1=0.0034823894022493434,
              k2=0.0007150348452162257, k3=-0.0020532361418706202, k4=0.00020293673591811182, cols=512.0, rows=512.0)
AIST = dict(model="fisheye", fx=441.730011169, fy=442.520822476, cx=480.35667528, cy=275.490228646, k1=-3.068701296607466433e-02,
            k2=-3.343454364086094217e-03, k3=-2.881735840896060968e-03, k4=-5.917420310474077278e-04, cols=960.0, rows=540.0)
_lib = None


def lib():
    global _lib
    if _lib is None:
        L = cbuild.load("camera_models_oracle.c")
        vp, f32, f64, i32 = C.c_void_p, C.c_float, C.c_double, C.c_int
        L.cmo_fisheye_undistort.argtypes = [vp, i32, f32, f32, f32, f32, vp, vp]
        L.cmo_fisheye_undistort.restype = None
        L.cmo_radial_undistort.argtypes = [vp, i32, f64, f64, f64, f64, f64, vp]
        L.cmo_radial_undistort.restype = None
        L.cmo_can_observe.argtypes = ([i32] + [f64] * 5 + [vp, vp, vp, i32, vp, vp, vp, vp, f32, C.c_uint, f32, vp, vp, vp, vp])
        L.cmo_can_observe.restype = None
        _lib = L
    return _lib


def model_of(camera):
    return MODELS[camera.get("model", "perspective")]


def _g(camera, k):
    return float(camera.get(k, 0.0))


def undistort_points(camera, xy):
    """(n, 2) float32 distorted points -> (n, 2) float32 undistorted points (fisheye / radial division)."""
    xy = np.ascontiguousarray(xy, np.float32).reshape(-1, 2)
    out = np.zeros_like(xy)
    n = len(xy)
    if n == 0:
        return out
    m = model_of(camera)
    if m == 2:
        d = np.array([_g(camera, k) for k in ("k1", "k2", "k3", "k4")], np.float32)
        lib().cmo_fisheye_undistort(xy.ctypes.data, n, *[float(np.float32(_g(camera, k))) for k in ("fx", "fy", "cx", "cy")], d.ctypes.data,
                                    out.ctypes.data)
    elif m == 3:
        lib().cmo_radial_undistort(xy.ctypes.data, n, *[_g(camera, k) for k in ("fx", "fy", "cx", "cy", "distortion")], out.ctypes.data)
    else:
        raise ValueError("undistort_points: fisheye or radial_division")
    return out


def undistort_keypoints(camera, kps):
    """(undist_kps, bearings) as feature.orb_extractor.undistort_keypoints returns them."""
    m = model_of(camera)
    if m < 2:
        return O.undistort_keypoints(camera, kps)
    kps = np.ascontiguousarray(kps, O.KP_DTYPE)
    n = len(kps)
    und = undistort_points(camera, np.stack([kps["x"], kps["y"]], 1))
    out = kps.copy()
    out["x"], out["y"] = und[:, 0], und[:, 1]
    out["response"] = 0  # undist_keypts.resize(): default cv::KeyPoint (fisheye.cc:300-306, base.cc:124-150)
    b = np.zeros((n, 3))
    if n:  # fisheye.cc:156-161, radial_division.cc:100-105: the perspective formula with the double intrinsics
        xy = np.ascontiguousarray(und, np.float32)
        O.lib().orc_points_to_bearings.argtypes = [C.c_void_p, C.c_int, C.c_int] + [C.c_double] * 6 + [C.c_void_p]
        O.lib().orc_points_to_bearings(xy.ctypes.data, n, 0, *[_g(camera, k) for k in ("fx", "fy", "cx", "cy", "cols", "rows")], b.ctypes.data)
    return out, b


def image_bounds(camera):
    """camera::*::compute_image_bounds as floats (min_x, max_x, min_y, max_y) with this oracle's undistortion (fisheye.cc:68-135,
    radial_division.cc:61-81; perspective / equirectangular without distortion: (0, cols, 0, rows))."""
    m = model_of(camera)
    f = lambda v: np.float32(v)
    cols, rows = f(int(_g(camera, "cols"))), f(int(_g(camera, "rows")))
    coeffs = {0: ("k1", "k2", "p1", "p2", "k3"), 1: (), 2: ("k1", "k2", "k3", "k4"), 3: ("distortion",)}[m]
    if all(_g(camera, k) == 0 for k in coeffs):
        return (f(0.0), cols, f(0.0), rows)
    if m < 2:
        raise ValueError("image_bounds: distorted perspective cameras are not restated here")
    fx, fy, cx, cy = (_g(camera, k) for k in ("fx", "fy", "cx", "cy"))
    if m == 2:
        px, py = (0.0 - cx) / fx, (0.0 - cy) / fy
        if math.sqrt(px * px + py * py) > math.pi / 2:
            u = undistort_points(camera, [[f(cx), 0.0], [cols, f(cy)], [0.0, f(cy)], [f(cx), rows]])
            t = math.tan(5.0 * math.pi / 180.0)  # constexpr float deg_thr = 5.0, promoted to double
            dx, dy = f(fx / t), f(fy / t)
            thr = (f(-float(dx) + cx), f(float(dx) + cx), f(-float(dy) + cy), f(float(dy) + cy))
            vals = (u[2, 0], u[1, 0], u[0, 1], u[3, 1])
            c = (cx, cx, cy, cy)
            res = []
            for k, (v, th, cc) in enumerate(zip(vals, thr, c)):
                out_of_range = (float(v) < float(th) or float(v) > cc) if k % 2 == 0 else (float(v) > float(th) or float(v) < cc)
                res.append(th if out_of_range else v)
            return tuple(res)
    u = undistort_points(camera, [[0.0, 0.0], [cols, 0.0], [0.0, rows], [cols, rows]])
    return (min(u[0, 0], u[2, 0]), max(u[1, 0], u[3, 0]), min(u[0, 1], u[1, 1]), max(u[2, 1], u[3, 1]))


def can_observe(camera, pose_cw, landmarks, ray_cos_thr=0.5, img_bounds=None, num_levels=8, log_scale_factor=None):
    """data::frame::can_observe, same arguments / result as pyoracle.can_observe.  Default bounds: image_bounds(camera)."""
    m = model_of(camera)
    if m < 2:
        return O.can_observe(camera, pose_cw, landmarks, ray_cos_thr, img_bounds, num_levels, log_scale_factor)
    pos = np.ascontiguousarray(landmarks["pos_w"], np.float64).reshape(-1, 3)
    nml = np.ascontiguousarray(landmarks["mean_normal"], np.float64).reshape(-1, 3)
    lo = np.ascontiguousarray(landmarks["min_valid_dist"], np.float32)
    hi = np.ascontiguousarray(landmarks["max_valid_dist"], np.float32)
    n = len(pos)
    bounds = np.ascontiguousarray(img_bounds if img_bounds is not None else image_bounds(camera), np.float32)
    T = np.ascontiguousarray(pose_cw, np.float64).reshape(4, 4)
    Rt = np.ascontiguousarray(np.concatenate([T[:3, :3].reshape(9), T[:3, 3]]))
    twc = np.array([-((T[0, r] * T[0, 3] + T[1, r] * T[1, 3]) + T[2, r] * T[2, 3]) for r in range(3)])
    if log_scale_factor is None:
        log_scale_factor = np.float32(np.log(np.float32(1.2)))
    ok, rp = np.zeros(max(n, 1), np.uint8), np.zeros((max(n, 1), 2))
    xr, lv = np.zeros(max(n, 1), np.float32), np.zeros(max(n, 1), np.uint32)
    p = lambda a: a.ctypes.data
    lib().cmo_can_observe(1 if m == 3 else 0, _g(camera, "fx"), _g(camera, "fy"), _g(camera, "cx"), _g(camera, "cy"), _g(camera, "fxb"), p(bounds),
                          p(Rt), p(twc), n, p(pos), p(nml), p(lo), p(hi), float(ray_cos_thr), int(num_levels), float(log_scale_factor), p(ok), p(rp),
                          p(xr), p(lv))
    return dict(observable=ok[:n].astype(bool), reproj=rp[:n], x_right=xr[:n], pred_scale_level=lv[:n])


def track_local_map(camera, kps, desc, frame, scale_factors, inv_level_sigma_sq, log_scale_factor, margin=5.0, lowe_ratio=0.8, thr=100,
                    ray_cos_thr=0.5, img_bounds=None, grid=(64, 48), monocular=True, num_trials_robust=2, num_trials=2, num_each_iter=10):
    """pyoracle.track_local_map with this module's undistortion and can_observe; the guided match and the pose optimiser are the
    oracle's (fisheye and radial division use the perspective edges).  Default bounds: image_bounds(camera) for models 2 and 3."""
    if model_of(camera) < 2:
        return O.track_local_map(camera, kps, desc, frame, scale_factors, inv_level_sigma_sq, log_scale_factor, margin, lowe_ratio, thr, ray_cos_thr,
                                 img_bounds, grid, monocular, num_trials_robust, num_trials, num_each_iter)
    kps = np.ascontiguousarray(kps, O.KP_DTYPE)
    n_kp = len(kps)
    lm = frame["landmarks"]
    n_lm = len(np.asarray(lm["pos_w"]).reshape(-1, 3))
    sf = np.asarray(scale_factors, np.float32)
    num_levels = len(sf)
    und, _ = undistort_keypoints(camera, kps)
    bounds = tuple(float(v) for v in (img_bounds if img_bounds is not None else image_bounds(camera)))
    co = can_observe(camera, frame["pose_cw"], lm, ray_cos_thr, bounds, num_levels, log_scale_factor)
    skip = np.zeros(n_lm, bool) if lm.get("skip") is None else np.asarray(lm["skip"]).astype(bool)
    has_obs = np.ones(n_lm, bool) if lm.get("has_observation") is None else np.asarray(lm["has_observation"]).astype(bool)
    observable = co["observable"] & ~skip
    kp_lm = np.full(n_kp, -1, np.int32) if frame.get("kp_landmark") is None else np.asarray(frame["kp_landmark"], np.int32).copy()
    occupied = np.array([(l >= 0 and has_obs[l]) for l in kp_lm], np.uint8)
    lvl = co["pred_scale_level"].astype(np.int64)
    pr = dict(t_x=und["x"], t_y=und["y"], t_octave=und["octave"].astype(np.uint8), t_desc=np.ascontiguousarray(desc, np.uint8),
              t_x_right=frame.get("kp_x_right"), t_occupied=occupied, bounds=bounds, grid=grid,
              q_desc=np.ascontiguousarray(lm["desc"], np.uint8), q_x=co["reproj"][:, 0].astype(np.float32), q_y=co["reproj"][:, 1].astype(np.float32),
              q_margin=np.float32(margin) * sf[lvl], q_min_level=np.maximum(0, lvl - 1), q_max_level=np.minimum(num_levels - 1, lvl + 1),
              q_x_right=co["x_right"], q_valid=observable.astype(np.uint8), q_has_observation=has_obs.astype(np.uint8))
    match_out, _, n_matches = O.match_guided(pr, 0, thr=thr, lowe_ratio=lowe_ratio, check_orientation=False)
    for q in range(n_lm):
        if match_out[q] >= 0:
            kp_lm[match_out[q]] = q
    idx = np.nonzero(kp_lm >= 0)[0]
    xr = np.full(n_kp, -1.0, np.float32) if frame.get("kp_x_right") is None else np.asarray(frame["kp_x_right"], np.float32)
    isig = np.asarray(inv_level_sigma_sq, np.float32)
    chi = np.float32(np.sqrt(np.float32(5.99146))) if monocular else np.float32(np.sqrt(np.float32(7.81473)))
    pos = np.asarray(lm["pos_w"], np.float64).reshape(-1, 3)
    cam = dict(model=0, fx=_g(camera, "fx"), fy=_g(camera, "fy"), cx=_g(camera, "cx"), cy=_g(camera, "cy"), fxb=_g(camera, "fxb"),
               cols=_g(camera, "cols"), rows=_g(camera, "rows"))
    ne = len(idx)
    pp = dict(pose_cw=np.asarray(frame["pose_cw"], np.float64).reshape(1, 4, 4), pose_fixed=np.zeros(1, np.uint8), points=pos[kp_lm[idx]].reshape(-1, 3),
              point_fixed=np.ones(ne, np.uint8), e_pose=np.zeros(ne, np.int32), e_point=np.arange(ne, dtype=np.int32), e_cam=np.zeros(ne, np.uint8),
              e_obs=np.stack([und["x"][idx], und["y"][idx], xr[idx]], 1).astype(np.float32), e_inv_sigma_sq=isig[und["octave"][idx].astype(np.int64)],
              e_delta=np.full(ne, chi, np.float32), e_robust=None, e_can_be_outlier=None, cams=[cam])
    outlier = np.zeros(n_kp, bool)
    if ne >= 5:
        n_valid, pose, flags = O.pose_optimize(pp, num_trials_robust, num_trials, num_each_iter)
        outlier[idx] = flags
    else:
        n_valid, pose = 0, np.asarray(frame["pose_cw"], np.float64).reshape(4, 4).copy()
    return dict(observable=observable, kp_landmark=kp_lm, kp_outlier=outlier, pose_cw=pose, n_matches=int(n_matches), n_valid=int(n_valid),
                n_keypoints=n_kp)


def on_bound_landmarks():
    """Landmarks in front of an identity pose (fx = fy = 256, cx = 266, cy = 276, z = 1) whose reprojection lands exactly on a bound of
    (10, 500, 20, 400), exactly inside and exactly outside.  Returns (camera fields, bounds, landmarks, on-bound mask, inside mask)."""
    cam = dict(fx=256.0, fy=256.0, cx=266.0, cy=276.0, cols=512.0, rows=420.0)
    bounds = (10.0, 500.0, 20.0, 400.0)
    uv = [(10.0, 200.0), (500.0, 200.0), (250.0, 20.0), (250.0, 400.0), (10.0, 20.0), (500.0, 400.0),   # on a bound
          (11.0, 200.0), (499.0, 399.0), (250.0, 200.0),                                                  # inside
          (9.0, 200.0), (250.0, 401.0)]                                                                   # outside
    pos = np.array([[(u - cam["cx"]) / cam["fx"], (v - cam["cy"]) / cam["fy"], 1.0] for u, v in uv])
    nml = pos / np.linalg.norm(pos, axis=1, keepdims=True)
    lms = dict(pos_w=pos, mean_normal=nml, min_valid_dist=np.full(len(uv), 0.5, np.float32), max_valid_dist=np.full(len(uv), 2.0, np.float32))
    on = np.array([True] * 6 + [False] * 5)
    inside = np.array([False] * 6 + [True] * 3 + [False] * 2)
    return cam, bounds, lms, on, inside
