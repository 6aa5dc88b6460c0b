"""CPU checks of the fisheye and radial-division restatement (tests/camera_models_oracle.c): fisheye undistortion bit-identical to
cv2.fisheye.undistortPoints called as camera::fisheye calls it (float32 K and D, R = None, P = K), radial division against numpy, both
compute_image_bounds against an assembly of the reference code, the strict / inclusive bound rules, and the ctypes layout of
b200_camera_intrinsics_t.  No GPU needed."""
import ctypes as C
import math
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import camera_models_oracle as CM  # noqa: E402

try:
    import cv2
except ImportError:  # the cv2 comparisons are skipped, the rest runs
    cv2 = None
needs_cv2 = pytest.mark.skipif(cv2 is None, reason="OpenCV (cv2) is not installed")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TUM_VI, AIST = CM.TUM_VI, CM.AIST


def _K32(cam):
    return np.array([[cam["fx"], 0, cam["cx"]], [0, cam["fy"], cam["cy"]], [0, 0, 1]], np.float32)


def _D32(cam):
    return np.array([cam.get(k, 0.0) for k in ("k1", "k2", "k3", "k4")], np.float32)


def cv_fisheye(cam, xy):
    """camera::fisheye::undistort_keypoints' call (fisheye.cc:295): cv_cam_matrix_ and cv_dist_params_ are CV_32F."""
    xy = np.ascontiguousarray(xy, np.float32).reshape(-1, 1, 2)
    K = _K32(cam)
    return cv2.fisheye.undistortPoints(xy, K, _D32(cam), R=None, P=K).reshape(-1, 2)


def _grid(cols, rows):
    u, v = np.meshgrid(np.arange(int(cols), dtype=np.float32), np.arange(int(rows), dtype=np.float32))
    return np.stack([u.ravel(), v.ravel()], 1)


def _random_fisheye(rng):
    cols, rows = int(rng.integers(320, 961)), int(rng.integers(240, 721))
    f = rng.uniform(0.25, 0.8) * cols
    return dict(model="fisheye", fx=f, fy=f * rng.uniform(0.98, 1.02), cx=cols / 2 + rng.normal(0, 8), cy=rows / 2 + rng.normal(0, 8),
                k1=rng.normal(0, 0.05), k2=rng.normal(0, 0.02), k3=rng.normal(0, 0.01), k4=rng.normal(0, 0.005), cols=float(cols), rows=float(rows))


def _fisheye_points(cam, rng, n_random=20000):
    pts = [_grid(cam["cols"], cam["rows"])]
    pts.append(np.stack([rng.uniform(-0.5, cam["cols"] + 0.5, n_random), rng.uniform(-0.5, cam["rows"] + 0.5, n_random)], 1).astype(np.float32))
    cx, cy = np.float32(cam["cx"]), np.float32(cam["cy"])
    # at the principal point (theta_d = 0 <= eps) and one float step away from it
    pts.append(np.array([[cx, cy], [np.nextafter(cx, np.float32(1e9)), cy], [cx, np.nextafter(cy, np.float32(-1e9))]], np.float32))
    # far outside: theta_d beyond pi / 2 (clipped)
    r = 3.0 * max(cam["fx"], cam["fy"])
    ang = rng.uniform(0, 2 * np.pi, 500)
    pts.append(np.stack([cx + r * np.cos(ang), cy + r * np.sin(ang)], 1).astype(np.float32))
    return np.concatenate(pts)


def _same_bits(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


@needs_cv2
@pytest.mark.parametrize("name", ["tum_vi", "aist"] + [f"random{i}" for i in range(20)])
def test_fisheye_oracle_is_bit_identical_to_cv2(name):
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    cam = {"tum_vi": TUM_VI, "aist": AIST}.get(name) or _random_fisheye(np.random.default_rng(1000 + int(name[6:])))
    xy = _fisheye_points(cam, rng)
    got, want = CM.undistort_points(cam, xy), cv_fisheye(cam, xy)
    bad = np.nonzero(~np.all(got.view(np.uint32) == want.view(np.uint32), axis=1))[0]
    assert len(bad) == 0, (len(bad), xy[bad[:5]], got[bad[:5]], want[bad[:5]])
    pp = len(xy) - 503  # the principal point maps to (cx, cy) of the float K
    assert got[pp, 0] == np.float32(cam["cx"]) and got[pp, 1] == np.float32(cam["cy"])


@needs_cv2
def test_tum_vi_needs_the_float_intrinsics():
    """camera::fisheye hands OpenCV float K and D: with double K and D most TUM-VI keypoints come out different."""
    xy = _fisheye_points(TUM_VI, np.random.default_rng(3), 0)[:20000]
    K64 = np.array([[TUM_VI["fx"], 0, TUM_VI["cx"]], [0, TUM_VI["fy"], TUM_VI["cy"]], [0, 0, 1]])
    D64 = np.array([TUM_VI[k] for k in ("k1", "k2", "k3", "k4")])
    d64 = cv2.fisheye.undistortPoints(xy.reshape(-1, 1, 2), K64, D64, R=None, P=K64).reshape(-1, 2)
    got = CM.undistort_points(TUM_VI, xy)
    assert (got != d64).any(axis=1).sum() > 1000


def _newton_flags(cam, xy):
    """numpy restatement of the Newton loop's outcome: (converged, flipped) per point."""
    f = lambda k: np.float64(np.float32(cam[k]))
    k = [f(n) for n in ("k1", "k2", "k3", "k4")]
    pw = np.stack([(xy[:, 0].astype(np.float64) - f("cx")) / f("fx"), (xy[:, 1].astype(np.float64) - f("cy")) / f("fy")], 1)
    td = np.minimum(np.maximum(-np.pi / 2, np.sqrt(pw[:, 0] * pw[:, 0] + pw[:, 1] * pw[:, 1])), np.pi / 2)
    th = td.copy()
    conv = ~(np.abs(td) > 1e-8)
    active = ~conv
    with np.errstate(all="ignore"):
        for _ in range(10):
            t2 = th * th
            t4, t6, t8 = t2 * t2, t2 * t2 * t2, t2 * t2 * t2 * t2
            a, b, c, d = k[0] * t2, k[1] * t4, k[2] * t6, k[3] * t8
            fix = (th * (1 + a + b + c + d) - td) / (1 + 3 * a + 5 * b + 7 * c + 9 * d)
            th = np.where(active, th - fix, th)
            done = active & (np.abs(fix) < 1e-8)
            conv |= done
            active &= ~done
    flipped = ((td < 0) & (th > 0)) | ((td > 0) & (th < 0))
    return conv, flipped


@needs_cv2
def test_fisheye_sentinel_for_non_converged_and_flipped_points():
    rng = np.random.default_rng(7)
    xy = rng.uniform(-200, 700, (200000, 2)).astype(np.float32)
    n_nc = n_fl = 0
    for d in ((-0.5, 0.1, 0.0, 0.0), (0.3, -0.4, 0.2, -0.1)):
        cam = dict(TUM_VI, k1=d[0], k2=d[1], k3=d[2], k4=d[3])
        got, want = CM.undistort_points(cam, xy), cv_fisheye(cam, xy)
        assert _same_bits(got, want)
        conv, flipped = _newton_flags(cam, xy)
        sentinel = (got == CM.SENTINEL).all(axis=1)
        assert np.array_equal(sentinel, ~conv | flipped)
        n_nc += int((~conv).sum())
        n_fl += int((conv & flipped).sum())
    assert n_nc > 0 and n_fl > 0, (n_nc, n_fl)


@pytest.mark.parametrize("d", [0.0, -0.05, -0.2, 0.1])
def test_radial_division_matches_the_closed_form(d):
    cam = dict(model="radial_division", fx=612.3, fy=611.7, cx=641.2, cy=361.9, distortion=d, cols=1280.0, rows=720.0)
    rng = np.random.default_rng(11)
    xy = np.concatenate([_grid(1280, 720)[::7], rng.uniform(-50, 1330, (20000, 2))]).astype(np.float32)
    px = (xy[:, 0].astype(np.float64) - cam["cx"]) / cam["fx"]
    py = (xy[:, 1].astype(np.float64) - cam["cy"]) / cam["fy"]
    und = 1.0 + d * (px * px + py * py)
    want = np.stack([(px / und * cam["fx"] + cam["cx"]), (py / und * cam["fy"] + cam["cy"])], 1).astype(np.float32)
    assert _same_bits(CM.undistort_points(cam, xy), want)


def _ref_fisheye_bounds(cam):
    """fisheye::compute_image_bounds (fisheye.cc:68-135) assembled from cv2 and float32 numpy."""
    f32 = np.float32
    cx, cy, fx, fy = cam["cx"], cam["cy"], cam["fx"], cam["fy"]
    cols, rows = f32(cam["cols"]), f32(cam["rows"])
    theta_d = math.sqrt(((0.0 - cx) / fx) ** 2 + ((0.0 - cy) / fy) ** 2)
    if theta_d > math.pi / 2:
        u = cv_fisheye(cam, [[cx, 0.0], [cols, cy], [0.0, cy], [cx, rows]])
        dtx, dty = f32(fx / math.tan(5.0 * math.pi / 180.0)), f32(fy / math.tan(5.0 * math.pi / 180.0))
        mnx, mxx, mny, mxy = f32(-float(dtx) + cx), f32(float(dtx) + cx), f32(-float(dty) + cy), f32(float(dty) + cy)
        a, b, c, d = u[2, 0], u[1, 0], u[0, 1], u[3, 1]
        return "wide", (mnx if (a < mnx or float(a) > cx) else a, mxx if (b > mxx or float(b) < cx) else b,
                        mny if (c < mny or float(c) > cy) else c, mxy if (d > mxy or float(d) < cy) else d)
    u = cv_fisheye(cam, [[0, 0], [cols, 0], [0, rows], [cols, rows]])
    return "normal", (min(u[0, 0], u[2, 0]), max(u[1, 0], u[3, 0]), min(u[0, 1], u[1, 1]), max(u[2, 1], u[3, 1]))


@needs_cv2
def test_image_bounds_fisheye_both_branches():
    kind, want = _ref_fisheye_bounds(TUM_VI)
    assert kind == "wide"
    assert _same_bits(CM.image_bounds(TUM_VI), want)
    kind, want = _ref_fisheye_bounds(AIST)
    assert kind == "normal"
    assert _same_bits(CM.image_bounds(AIST), want)
    assert _same_bits(CM.image_bounds(dict(AIST, k1=0.0, k2=0.0, k3=0.0, k4=0.0)), (0.0, 960.0, 0.0, 540.0))


def test_image_bounds_radial_division():
    cam = dict(model="radial_division", fx=612.3, fy=611.7, cx=641.2, cy=361.9, distortion=-0.15, cols=1280.0, rows=720.0)
    c = np.array([[0, 0], [1280, 0], [0, 720], [1280, 720]], np.float64)
    px, py = (c[:, 0] - cam["cx"]) / cam["fx"], (c[:, 1] - cam["cy"]) / cam["fy"]
    und = 1.0 + cam["distortion"] * (px * px + py * py)
    u = np.stack([px / und * cam["fx"] + cam["cx"], py / und * cam["fy"] + cam["cy"]], 1).astype(np.float32)
    want = (min(u[0, 0], u[2, 0]), max(u[1, 0], u[3, 0]), min(u[0, 1], u[1, 1]), max(u[2, 1], u[3, 1]))
    assert _same_bits(CM.image_bounds(cam), want)
    assert _same_bits(CM.image_bounds(dict(cam, distortion=0.0)), (0.0, 1280.0, 0.0, 720.0))


def test_bound_rules_strict_for_fisheye_inclusive_for_radial_division():
    cam, bounds, lms, on, inside = CM.on_bound_landmarks()
    fish = CM.can_observe(dict(cam, model="fisheye"), np.eye(4), lms, img_bounds=bounds)
    rad = CM.can_observe(dict(cam, model="radial_division"), np.eye(4), lms, img_bounds=bounds)
    assert np.array_equal(fish["observable"], inside)
    assert np.array_equal(rad["observable"], inside | on)
    # fisheye follows the perspective rule of the oracle
    from oracle import pyoracle as O
    persp = O.can_observe(dict(cam, model="perspective"), np.eye(4), lms, img_bounds=bounds)
    for k in ("observable", "reproj", "x_right", "pred_scale_level"):
        assert np.array_equal(fish[k], persp[k]), k


def test_camera_intrinsics_layout_and_model_codes(tmp_path):
    from stella_vslam_b200 import _lib, tracking
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    fields = [f for f, _ in _lib.CameraIntrinsics._fields_]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200vslam.h"\nint main(void) {\n'
                   + "".join(f'  printf("%zu\\n", offsetof(b200_camera_intrinsics_t, {f}));\n' for f in fields)
                   + '  printf("%zu\\n", sizeof(b200_camera_intrinsics_t));\n  return 0;\n}\n')
    subprocess.check_call(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert got == [getattr(_lib.CameraIntrinsics, f).offset for f in fields] + [C.sizeof(_lib.CameraIntrinsics)]
    # the fields that existed before keep their offsets; k4 and distortion follow rows
    assert [getattr(_lib.CameraIntrinsics, f).offset for f in fields] == [0, 8, 16, 24, 32, 40, 48, 56, 64, 72, 80, 88, 96, 104]
    assert C.sizeof(_lib.CameraIntrinsics) == 112
    base = dict(fx=1.0, fy=2.0, cx=3.0, cy=4.0, k1=5.0, k2=6.0, p1=7.0, p2=8.0, k3=9.0, k4=10.0, distortion=11.0, cols=12.0, rows=13.0)
    for model, code in ((None, 0), ("perspective", 0), ("equirectangular", 1), ("fisheye", 2), ("radial_division", 3)):
        cam = dict(base) if model is None else dict(base, model=model)
        ci = tracking.camera_intrinsics(cam)
        assert ci.model == code
        assert [ci.fx, ci.k3, ci.cols, ci.rows, ci.k4, ci.distortion] == [1.0, 9.0, 12.0, 13.0, 10.0, 11.0]
    with pytest.raises(ValueError):
        tracking.camera_intrinsics(dict(base, model="omnidirectional"))
