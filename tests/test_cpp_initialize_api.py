"""The C++ mirror of initialize::perspective / bearing_vector (include/b200vslam.hpp, b200::initialize) drives the same frame pairs as
the Python mirror (stella_vslam_b200.initialize) and gets the same outcome, pose, points and flags, bit for bit."""
import os
import subprocess

import numpy as np
import pytest

import cbuild
import initialize_oracle as O


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return cbuild.cpp_mirror("initialize_api_test", tmp_path_factory.mktemp("initialize_api"))


def test_cpp_mirror_compiles(exe):
    assert os.access(exe, os.X_OK)


CASES = {
    "euroc_F": lambda: O.perspective_problem(seed=500, n=800),
    "planar_H": lambda: O.plane_problem(seed=0),
    "pure_rotation_decompose": lambda: O.plane_problem(seed=3, inlier_frac=0.2, tilt=0.6, t_norm=0.0),
    "fisheye_F": lambda: O.perspective_problem(seed=504, n=800, model="fisheye"),
    "equirect_E": lambda: O.equirect_problem(seed=1),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_cpp_initializer_matches_python(exe, tmp_path, case):
    from stella_vslam_b200 import _lib, initialize as I
    p = CASES[case]()
    ci = _lib.camera_intrinsics(p["cam_ref"])
    cam = [ci.model, ci.fx, ci.fy, ci.cx, ci.cy, ci.k1, ci.k2, ci.p1, ci.p2, ci.k3, ci.cols, ci.rows, ci.k4, ci.distortion]
    ur, uc = np.asarray(p["undist_ref"], np.float32), np.asarray(p["undist_cur"], np.float32)
    path = tmp_path / "problem.bin"
    with open(path, "wb") as f:
        f.write(np.array(cam, np.float64).tobytes())
        f.write(np.array(p.get("bounds_ref", (0, 0, 0, 0)), np.float32).tobytes())
        f.write(np.array([len(ur), len(uc)], np.int32).tobytes())
        for a, t in ((ur, np.float32), (p["bearings_ref"], np.float64), (uc, np.float32), (p["bearings_cur"], np.float64),
                     (p["ref_matches_with_cur"], np.int32)):
            f.write(np.ascontiguousarray(a, t).tobytes())
    lines = subprocess.check_output([exe, str(path)], text=True).splitlines()
    bearing = p["cam_ref"].get("model") == "equirectangular"
    ref = dict(camera=p["cam_ref"], img_bounds=p.get("bounds_ref", (0, 0, 0, 0)), undist_keypts=ur, bearings=p["bearings_ref"])
    cur = dict(camera=p["cam_cur"], img_bounds=p.get("bounds_cur", (0, 0, 0, 0)), undist_keypts=uc, bearings=p["bearings_cur"])
    ini = (I.bearing_vector if bearing else I.perspective)(ref, use_fixed_seed=True)
    ok = ini.initialize(cur, p["ref_matches_with_cur"])
    r = ini.last_result_
    model = {None: 0, "H": 1, "F": 2, "E": 3}[r["model"]]
    assert lines[0] == f"succeeded {int(ok)} status {ini.status()} stage {r['stage']} model {model}"
    assert np.array_equal(np.array(lines[1].split()[1:], np.float64), ini.get_rotation_ref_to_cur().reshape(9))
    assert np.array_equal(np.array(lines[2].split()[1:], np.float64), ini.get_translation_ref_to_cur())
    pts = np.array(lines[3].split()[1:], np.float64)
    assert np.array_equal(pts, ini.get_triangulated_pts().reshape(-1))
    assert (lines[4].split() + [""])[1] == "".join("1" if v else "0" for v in ini.get_triangulated_flags())
    if case != "pure_rotation_decompose":
        assert ok
    else:
        assert r["stage"] == I.STAGE_DECOMPOSE and np.array_equal(ini.get_rotation_ref_to_cur(), np.eye(3))
