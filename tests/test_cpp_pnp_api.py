"""The C++ mirror of solve::pnp_solver (include/b200vslam.hpp, b200::solve) drives the same problems as the Python mirror
(stella_vslam_b200.solve) and gets the same minimal sets, the same RANSAC results and the same compute_pose."""
import subprocess

import numpy as np
import pytest

import cbuild
from workloads import synth


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return cbuild.cpp_mirror("pnp_api_test", tmp_path_factory.mktemp("pnp_api"))


@pytest.mark.parametrize("n,seed", [(4, ()), (300, ()), (1000, (3, 1, 4, 1, 5))])
def test_cpp_sampler_matches_python(exe, n, seed):
    from stella_vslam_b200 import solve
    out = subprocess.check_output([exe, "sampler", str(n), "30"] + [str(w) for w in seed], text=True)
    cpp = np.array(out.split(), np.int64).reshape(30, 4)
    np.testing.assert_array_equal(cpp, solve.draw_min_sets(n, 30, solve.mt19937(seed or None)))


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["perspective", "equirect"])
def test_cpp_solver_matches_python(exe, tmp_path, model):
    from stella_vslam_b200 import solve
    pr = synth.make_pnp_problem(80, 400, 0.5, model)
    path = tmp_path / "problem.bin"
    with open(path, "wb") as f:
        f.write(np.array([400, len(pr["scale_factors"])], np.int32).tobytes())
        f.write(np.ascontiguousarray(pr["bearings"], np.float64).tobytes())
        f.write(np.ascontiguousarray(pr["points"], np.float64).tobytes())
        f.write(np.asarray(pr["octaves"], np.int32).tobytes())
        f.write(np.asarray(pr["scale_factors"], np.float32).tobytes())
    lines = subprocess.check_output([exe, "ransac", str(path)], text=True).splitlines()
    s = solve.pnp_solver(pr["bearings"], pr["octaves"], pr["points"], pr["scale_factors"], use_fixed_seed=True)
    for k, recompute in enumerate((True, False)):
        s.find_via_ransac(30, recompute)
        valid, pose, flags = lines[3 * k:3 * k + 3]
        assert valid == f"valid {int(s.solution_is_valid())}" and s.solution_is_valid()
        vals = np.array(pose.split()[1:], np.float64)
        assert np.array_equal(vals[:9], s.get_best_rotation().reshape(9)) and np.array_equal(vals[9:], s.get_best_translation())
        assert flags.split()[1] == "".join("1" if v else "0" for v in s.get_inlier_flags())
    err, R, t = solve.pnp_solver.compute_pose(pr["bearings"][:50], pr["points"][:50], np.zeros((3, 3)), np.zeros(3), 10)
    vals = np.array(lines[6].split()[1:], np.float64)
    assert vals[0] == err and np.array_equal(vals[1:10], R.reshape(9)) and np.array_equal(vals[10:], t)
