"""The C++ mirror of solve::essential_solver (include/b200vslam.hpp, b200::solve) drives the same problems as the Python mirror
(stella_vslam_b200.solve) and gets the same minimal sets and the same RANSAC results, bit for bit."""
import subprocess

import numpy as np
import pytest

import cbuild
from workloads import synth


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return cbuild.cpp_mirror("essential_api_test", tmp_path_factory.mktemp("essential_api"))


@pytest.mark.parametrize("set_size", [5, 8])
@pytest.mark.parametrize("n,seed", [(8, ()), (500, ()), (1500, (3, 1, 4, 1, 5))])
def test_cpp_sampler_matches_python(exe, set_size, n, seed):
    from stella_vslam_b200 import solve
    out = subprocess.check_output([exe, "sampler", str(set_size), str(n), "30"] + [str(w) for w in seed], text=True)
    cpp = np.array(out.split(), np.int64).reshape(30, set_size)
    np.testing.assert_array_equal(cpp, solve.draw_min_sets(n, 30, solve.mt19937(seed or None), set_size=set_size))


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["perspective", "equirect"])
def test_cpp_solver_matches_python(exe, tmp_path, model):
    from stella_vslam_b200 import solve
    p = synth.make_essential_problem(31, 400, 0.5, model)
    rng = np.random.default_rng(1)
    n1, n2 = 430, 420
    b1, b2 = rng.standard_normal((n1, 3)), rng.standard_normal((n2, 3))
    i1, i2 = rng.permutation(n1)[:400], rng.permutation(n2)[:400]
    b1[i1], b2[i2] = p["bearings_1"], p["bearings_2"]
    matches = np.stack([i1, i2], 1).astype(np.int32)
    path = tmp_path / "problem.bin"
    with open(path, "wb") as f:
        f.write(np.array([n1, n2, len(matches)], np.int32).tobytes())
        f.write(np.ascontiguousarray(b1, np.float64).tobytes())
        f.write(np.ascontiguousarray(b2, np.float64).tobytes())
        f.write(np.ascontiguousarray(matches).tobytes())
    lines = subprocess.check_output([exe, "ransac", str(path)], text=True).splitlines()
    s = solve.essential_solver(b1, b2, matches, use_fixed_seed=True)
    for k, recompute in enumerate((True, False)):
        s.find_via_ransac(200, recompute)
        valid, cost, E, flags = lines[4 * k:4 * k + 4]
        assert valid == f"valid {int(s.solution_is_valid())} status 0" and s.solution_is_valid()
        assert np.float32(float(cost.split()[1])).tobytes() == s.get_best_cost().tobytes()
        assert np.array_equal(np.array(E.split()[1:], np.float64), s.get_best_E_21().reshape(9))
        assert flags.split()[1] == "".join("1" if v else "0" for v in s.get_inlier_matches())
