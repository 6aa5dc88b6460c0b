"""The C++ mirror of the RGB-D frame step and the depth-seeded landmarks (include/b200vslam.hpp: feature::orb_extractor::rgbd_depths,
module::depth_landmarks) drives the same problems as the Python mirror and gets the same results, bit for bit."""
import subprocess

import numpy as np
import pytest

import cbuild

TUM_RGBD = dict(model=0, fx=517.306408, fy=516.469215, cx=318.643040, cy=255.313989, k1=0.262383, k2=-0.953104, p1=-0.005358, p2=0.002628,
                k3=1.163314, cols=640.0, rows=480.0, k4=0.0, distortion=0.0)


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return cbuild.cpp_mirror("rgbd_api_test", tmp_path_factory.mktemp("rgbd_api"))


def test_cpp_mirror_builds_and_reports_usage(exe):
    assert subprocess.run([exe], capture_output=True).returncode == 2


def _hex(a):
    a = np.ascontiguousarray(a)
    w = a.dtype.itemsize if a.dtype.fields is None else 4
    return " ".join(b.tobytes().hex() for b in np.frombuffer(a.tobytes(), np.uint8).reshape(-1, w))


def _parse(lines):
    return {ln.split(" ", 1)[0]: (ln.split(" ", 1)[1] if " " in ln else "") for ln in lines}


@pytest.mark.gpu
def test_cpp_rgbd_depths_match_python(exe, tmp_path):
    from stella_vslam_b200 import feature
    from workloads import synth
    n, w, h = 3, 640, 480
    frames = [synth.make_rgbd_frames(w, h, seed=40 + s) for s in range(n)]
    gray, d16 = np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames])
    path = tmp_path / "rgbd.bin"
    with open(path, "wb") as f:
        f.write(np.array([n, w, h], np.int32).tobytes() + gray.tobytes() + d16.tobytes())
        f.write(np.array([TUM_RGBD["model"]], np.int32).tobytes())
        f.write(np.array([TUM_RGBD[k] for k in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2", "k3", "cols", "rows", "k4", "distortion")] + [40.0, 5000.0],
                         np.float64).tobytes())
    lines = subprocess.check_output([exe, "rgbd", str(path)], text=True).splitlines()
    ex = feature.orb_extractor(feature.orb_params(), 800, max_batch=n)
    ex.extract_batch(gray)
    cam = dict(TUM_RGBD, model="perspective")
    want = ex.rgbd_depths(cam, d16, 5000.0, 40.0)
    for fr in range(n):
        block = _parse(lines[5 * fr:5 * fr + 5])
        assert block["frame"] == f"{fr} {len(want[fr]['depths'])}"
        assert block["undist"] == _hex(want[fr]["undist_keypts"])
        for k in ("bearings", "depths", "x_right"):
            assert block[k] == _hex(want[fr][k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1])
def test_cpp_depth_landmarks_match_python(exe, tmp_path, mode):
    from stella_vslam_b200 import mapping
    rng = np.random.default_rng(mode)
    n = 1800
    depth = rng.uniform(0.3, 9.0, n).astype(np.float32)
    depth[rng.random(n) < 0.3] = -1
    x, y = rng.uniform(0, 640, n).astype(np.float32), rng.uniform(0, 480, n).astype(np.float32)
    octave = rng.integers(0, 8, n).astype(np.int32)
    has_lm = (rng.random(n) < 0.1).astype(np.uint8)
    pose = np.eye(4)
    pose[:3, 3] = [0.3, -0.2, 1.5]
    sf = np.cumprod(np.concatenate([[np.float32(1.0)], np.full(7, np.float32(1.2))])).astype(np.float32)
    inv_last = np.float32(np.float32(1.0) / sf[-1])
    prm = (1.0 / 517.306408, 1.0 / 516.469215, 318.643040, 255.313989, 3.0)
    path = tmp_path / "lm.bin"
    with open(path, "wb") as f:
        f.write(np.array([mode, n], np.int32).tobytes() + x.tobytes() + y.tobytes() + depth.tobytes() + octave.tobytes() + has_lm.tobytes())
        f.write(pose.astype(np.float64).tobytes() + np.array(prm, np.float64).tobytes() + sf.tobytes() + inv_last.tobytes())
    got = _parse(subprocess.check_output([exe, "landmarks", str(path)], text=True).splitlines())
    want = mapping.depth_landmarks([dict(mode=mode, pose_wc=pose, fx_inv=prm[0], fy_inv=prm[1], cx=prm[2], cy=prm[3], depth_thr=prm[4], x=x, y=y,
                                         octave=octave, depth=depth, has_landmark=has_lm, scale_factors=sf, inv_scale_factor_last=inv_last)])[0]
    assert got["created"] == str(len(want["idx"])) and len(want["idx"]) > 100
    for k in ("idx", "pos_w", "mean_normal", "min_valid_dist", "max_valid_dist"):
        assert got[k] == _hex(want[k]), k
