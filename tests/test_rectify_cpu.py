"""util::stereo_rectifier without a GPU: the CPU restatement (tests/rectify_oracle.c) against OpenCV itself, and the Python mirror's YAML
parsing and constructor errors (util/stereo_rectifier.cc:16-89).

Maps: the EuRoC and TUM-VI calibrations, and a fisheye rotation with rays behind the camera, are bit-identical to cv2.  On random
calibrations a few pixels in a million differ by one float ulp where the ray is almost parallel to the image plane, or by less than
1e-9 pixel where the double result cancels to almost zero (u near 0); OpenCV's vectorised map code rounds those intermediate steps
differently.  The fixed-point form that remap uses is identical there too, so every rectified frame is.  Remap is bit-identical
everywhere."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import rectify_oracle as R
from golden.natural import load_images
from stella_vslam_b200 import _lib, feature
from workloads import synth

cv2 = pytest.importorskip("cv2")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _same(a, b):
    """Bit equality of float maps; infinities compare by sign, as np.array_equal does."""
    return np.array_equal(a, b)


def _cv_map(model, K, D, Rm, Kr, cols, rows):
    f = cv2.initUndistortRectifyMap if model == "perspective" else cv2.fisheye.initUndistortRectifyMap
    return f(np.asarray(K, np.float64).reshape(3, 3), np.asarray(D, np.float64), np.asarray(Rm, np.float64).reshape(3, 3),
             np.asarray(Kr, np.float64).reshape(3, 3), (cols, rows), cv2.CV_32FC1)


def _calib_map(cal, eye, ours=True):
    args = (cal["K"][eye], cal["D"][eye], cal["R"][eye], cal["K_rect"])
    if ours:
        return R.rect_map(cal["model"], cal["cols"], cal["rows"], *args)
    return _cv_map(cal["model"], *args, cal["cols"], cal["rows"])


@pytest.mark.parametrize("name", ["euroc", "tum_vi"])
@pytest.mark.parametrize("eye", [0, 1])
def test_calibration_maps_bit_identical_to_cv2(name, eye):
    cal = {"euroc": synth.EUROC_STEREO, "tum_vi": synth.TUM_VI_STEREO}[name]
    mx, my = _calib_map(cal, eye)
    cx, cy = _calib_map(cal, eye, ours=False)
    assert _same(mx, cx) and _same(my, cy)


def random_calibration(seed, cols, rows, model, n_dist):
    rng = np.random.default_rng(seed)
    f = rng.uniform(300, 900)
    K = np.array([[f, 0, cols / 2 + rng.uniform(-30, 30)], [0, f * rng.uniform(0.98, 1.02), rows / 2 + rng.uniform(-30, 30)], [0, 0, 1]])
    Rm = cv2.Rodrigues(rng.normal(0, 0.05, 3))[0]
    Kr = np.array([[f * (0.9 if model == "perspective" else 0.4), 0, cols / 2], [0, f * (0.9 if model == "perspective" else 0.4), rows / 2], [0, 0, 1]])
    sig = [0.2, 0.05, 1e-3, 1e-3, 0.01, 0.1, 0.02, 0.01] if model == "perspective" else [0.05, 0.01, 0.005, 0.001]
    return K, rng.normal(0, sig[:n_dist]), Rm, Kr


@pytest.mark.parametrize("size", [(1241, 376), (1920, 1080)])
@pytest.mark.parametrize("model,n_dist", [("perspective", 4), ("perspective", 5), ("perspective", 8), ("fisheye", 4)])
@pytest.mark.parametrize("seed", [1, 2])
def test_random_calibration_maps_match_cv2(size, model, n_dist, seed):
    cols, rows = size
    K, D, Rm, Kr = random_calibration(seed, cols, rows, model, n_dist)
    mx, my = R.rect_map(model, cols, rows, K, D, Rm, Kr)
    cx, cy = _cv_map(model, K, D, Rm, Kr, cols, rows)
    for ours, ref in ((mx, cx), (my, cy)):
        diff = ours != ref
        assert diff.sum() <= 6, int(diff.sum())
        # one float ulp, or a cancellation residue of at most 1e-9 pixel next to zero
        assert (np.abs(ours[diff] - ref[diff]) <= np.maximum(np.spacing(np.abs(ref[diff])), 1e-9)).all()
    a, b = R.fixed_point(mx, my), R.fixed_point(cx, cy)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_fisheye_rays_behind_the_camera():
    cal = synth.TUM_VI_STEREO
    Rm = cv2.Rodrigues(np.array([0.0, 1.9, 0.0]))[0]
    mx, my = R.rect_map("fisheye", 512, 512, cal["K"][0], cal["D"][0], Rm, cal["K_rect"])
    cx, cy = _cv_map("fisheye", cal["K"][0], cal["D"][0], Rm, cal["K_rect"], 512, 512)
    assert _same(mx, cx) and _same(my, cy)
    assert np.isneginf(mx).sum() > 10000 and np.isposinf(mx).sum() > 10000
    sxy, _ = R.fixed_point(mx, my)
    assert (sxy[~np.isfinite(mx)] == -32768).all()     # cvRound gives INT_MIN for both infinities: every tap lies outside


def test_unsupported_coefficient_counts():
    cal = synth.EUROC_STEREO
    for n in (12, 14, 3):
        with pytest.raises(ValueError):
            R.rect_map("perspective", 752, 480, cal["K"][0], np.zeros(n), cal["R"][0], cal["K_rect"])
    with pytest.raises(ValueError):
        R.rect_map("fisheye", 512, 512, cal["K"][0], np.zeros(5), cal["R"][0], cal["K_rect"])


def test_weight_table_sums_to_32768():
    tab, bad = R.weights()
    assert bad == 0 and (tab.sum(1) == 32768).all()
    fy, fx = np.divmod(np.arange(1024), 32)
    assert np.array_equal(tab[:, 0], (32 - fy) * (32 - fx) * 32) and np.array_equal(tab[:, 3], fy * fx * 32)


def _image(rng, rows, cols, c):
    img = rng.integers(0, 256, (rows, cols) + (() if c == 1 else (c,)), dtype=np.uint8)
    return cv2.GaussianBlur(img, (5, 5), 1.0) if min(rows, cols) >= 5 else img


SIZES = [(752, 480), (512, 512), (1920, 1080), (1, 1), (3, 5)]


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("channels", [1, 3, 4])
def test_remap_bit_identical_to_cv2(size, channels):
    cols, rows = size
    rng = np.random.default_rng(cols * 7 + channels)
    img = _image(rng, rows, cols, channels)
    mx = rng.uniform(-3, cols + 2, (rows, cols)).astype(np.float32)
    my = rng.uniform(-3, rows + 2, (rows, cols)).astype(np.float32)
    assert np.array_equal(R.remap(img, mx, my), cv2.remap(img, mx, my, cv2.INTER_LINEAR))


@pytest.mark.parametrize("name", ["euroc", "tum_vi"])
@pytest.mark.parametrize("channels", [1, 3, 4])
def test_rectify_bit_identical_to_cv2(name, channels):
    cal = {"euroc": synth.EUROC_STEREO, "tum_vi": synth.TUM_VI_STEREO}[name]
    rng = np.random.default_rng(5 + channels)
    for eye in range(2):
        img = _image(rng, cal["rows"], cal["cols"], channels)
        mx, my = _calib_map(cal, eye)
        assert np.array_equal(R.remap(img, mx, my), cv2.remap(img, mx, my, cv2.INTER_LINEAR))


def test_rectify_natural_euroc_frame(golden_dir):
    img = load_images(golden_dir)["euroc_752x480"]
    mx, my = _calib_map(synth.EUROC_STEREO, 0)
    assert np.array_equal(R.remap(img, mx, my), cv2.remap(img, mx, my, cv2.INTER_LINEAR))


BORDER_VALUES = np.array([0, 1, 2.5, 3.25, 6.5, 7, 7.5, 7.99, 8, 8.5, -0.5, -0.75, -1, -1.00001, -2,
                          1 / 64, 3 / 64, 5 / 64, 7 / 64, 2 + 1 / 64, 2 + 3 / 64, -1 / 64, -3 / 64,  # map * 32 exactly at a half
                          3e4, 65535.9, -65535.9, 1e12, -1e12], np.float32)


def border_maps():
    """Every pairing of BORDER_VALUES as (x, y): windows fully inside; partly outside on each side; fully outside; integer
    coordinates; map * 32 exactly at a half (half-even rounding); and +-1e12."""
    gx, gy = np.meshgrid(BORDER_VALUES, BORDER_VALUES)
    return gx.astype(np.float32), gy.astype(np.float32)


@pytest.mark.parametrize("channels", [1, 3, 4])
def test_remap_border_cases(channels):
    rng = np.random.default_rng(11)
    img = rng.integers(1, 256, (8, 8) + (() if channels == 1 else (channels,)), dtype=np.uint8)   # no zero pixel: a 0 is a border read
    gx, gy = border_maps()
    # an 8 x 8 source sampled through 28 x 28 maps: the output has the maps' size
    assert np.array_equal(R.remap(img, gx, gy), cv2.remap(img, gx, gy, cv2.INTER_LINEAR))
    out = R.remap(img, gx, gy)
    i8 = list(BORDER_VALUES).index(8.0)
    assert (out[:, i8] == 0).all() and (out[i8, :] == 0).all()    # x = 8 or y = 8: the window starts past the last pixel


def test_half_even_rounding_of_the_fraction():
    sxy, frac = R.fixed_point(np.array([1 / 64, 3 / 64, -1 / 64], np.float32), np.zeros(3, np.float32))
    assert list(frac) == [0, 2, 0] and list(sxy[:, 0]) == [0, 0, 0]     # 0.5 -> 0, 1.5 -> 2, -0.5 -> -0


# --- Python mirror: YAML parsing and the constructor's errors (no device needed: they are raised before the handle is made) ---------

EUROC_CAMERA = dict(name="EuRoC stereo", setup="stereo", model="perspective", fx=435.2046959714599, fy=435.2046959714599,
                    cx=367.4517211914062, cy=252.2008514404297, cols=752, rows=480)


def euroc_rectifier_node():
    cal = synth.EUROC_STEREO
    return dict(K_left=list(cal["K"][0]), D_left=list(cal["D"][0]), R_left=list(cal["R"][0]), K_right=list(cal["K"][1]),
                D_right=list(cal["D"][1]), R_right=list(cal["R"][1]))


def test_parse_yaml_euroc():
    a = feature.stereo_rectifier.parse_yaml(EUROC_CAMERA, euroc_rectifier_node())
    assert a["model"] == "perspective" and (a["cols"], a["rows"]) == (752, 480)
    # cv_cam_matrix_ is CV_32F: the rectified intrinsics reach the map builder rounded to float
    assert a["K_rect"][0, 0] == float(np.float32(EUROC_CAMERA["fx"])) != EUROC_CAMERA["fx"]
    assert a["K_rect"][1, 2] == float(np.float32(EUROC_CAMERA["cy"])) and a["K_rect"][2, 2] == 1.0 and a["K_rect"][0, 1] == 0.0
    assert np.array_equal(a["R_right"], np.asarray(synth.EUROC_STEREO["R"][1]).reshape(3, 3))   # row-major
    assert a["D_left"].shape == (5,) and a["K_left"][0, 2] == 367.215


def test_parse_yaml_fisheye_model_key():
    node = dict(euroc_rectifier_node(), model="fisheye", D_left=[0.1, 0.2, 0.3, 0.4])
    assert feature.stereo_rectifier.parse_yaml(EUROC_CAMERA, node)["model"] == "fisheye"
    assert feature.stereo_rectifier.load_model_type({}) == "perspective"


@pytest.mark.parametrize("camera,node,msg", [
    (dict(EUROC_CAMERA, setup="monocular"), {}, "'setup' must be set to 'stereo'"),
    (dict(EUROC_CAMERA, model="fisheye"), {}, "'model' must be set to 'perspective'"),
    (EUROC_CAMERA, {"model": "radial_division"}, "Invalid camera model: radial_division"),
    (EUROC_CAMERA, {"model": "equirectangular"}, "Invalid model type for stereo rectification: perspective"),
])
def test_constructor_errors(camera, node, msg):
    with pytest.raises(RuntimeError, match=msg):
        feature.stereo_rectifier.parse_yaml(camera, dict(euroc_rectifier_node(), **node))


def test_model_string_checked_before_setup():
    # load_model_type runs in the member initialiser list, before the setup test (stereo_rectifier.cc:17)
    with pytest.raises(RuntimeError, match="Invalid camera model"):
        feature.stereo_rectifier.parse_yaml(dict(EUROC_CAMERA, setup="monocular"), dict(euroc_rectifier_node(), model="bogus"))


def test_thin_prism_and_tilt_models_rejected():
    a = feature.stereo_rectifier.parse_yaml(EUROC_CAMERA, euroc_rectifier_node())
    for n in (12, 14):
        with pytest.raises(RuntimeError, match="thin-prism and tilt"):
            feature.stereo_rectifier(**dict(a, D_left=np.zeros(n)))


def test_params_struct_layout(tmp_path):
    T = _lib.RectifierParams
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "b200vslam.h"', "int main(void) {",
             'printf("%zu\\n", sizeof(b200_rectifier_params_t));']
    lines += [f'printf("%zu\\n", offsetof(b200_rectifier_params_t, {f}));' for f, _ in T._fields_]
    (tmp_path / "p.c").write_text("\n".join(lines + ["return 0; }"]))
    subprocess.check_call(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(tmp_path / "p.c"), "-o", str(tmp_path / "p")])
    got = [int(v) for v in subprocess.check_output([str(tmp_path / "p")], text=True).split()]
    assert got == [C.sizeof(T)] + [getattr(T, f).offset for f, _ in T._fields_]


@pytest.mark.parametrize("name", ["euroc", "tum_vi"])
def test_raw_stereo_pair_rectifies_back(name):
    cal = {"euroc": synth.EUROC_STEREO, "tum_vi": synth.TUM_VI_STEREO}[name]
    raw_l, raw_r = synth.make_raw_stereo_pair(cal, seed=3)
    want_l, want_r = synth.make_stereo_pair(cal["cols"], cal["rows"], seed=3)
    got_l, got_r = R.rectify_pair(cal, raw_l, raw_r)
    h, w = cal["rows"], cal["cols"]
    core = (slice(h // 4, 3 * h // 4), slice(w // 4, 3 * w // 4))
    for got, want in ((got_l, want_l), (got_r, want_r)):
        assert np.abs(got[core].astype(int) - want[core]).mean() < 12
