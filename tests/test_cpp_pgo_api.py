"""The C++ mirror of optimize::graph_optimizer (include/b200vslam.hpp, b200::optimize::graph_optimizer) runs the same graph as the
Python mirror (stella_vslam_b200.optimize) and gets bit-identical estimates, poses and corrected landmarks."""
import os
import subprocess

import numpy as np
import pytest

import cbuild
from workloads import synth


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return cbuild.cpp_mirror("pgo_api_test", tmp_path_factory.mktemp("pgo_api"))


def test_cpp_mirror_compiles(exe):
    assert os.path.exists(exe)


@pytest.mark.gpu
@pytest.mark.parametrize("fix_scale", [False, True])
def test_cpp_graph_optimizer_matches_python(exe, tmp_path, fix_scale):
    from stella_vslam_b200 import optimize
    g = synth.make_pose_graph(200, seed=21, fix_scale=fix_scale)
    path = tmp_path / "graph.bin"
    with open(path, "wb") as f:
        f.write(np.array([len(g["estimate"]), len(g["e_v1"]), len(g["points"]), int(fix_scale)], np.int32).tobytes())
        f.write(np.ascontiguousarray(g["estimate"], np.float64).tobytes())
        f.write(np.ascontiguousarray(g["fixed"], np.uint8).tobytes())
        f.write(np.ascontiguousarray(g["e_v1"], np.int32).tobytes())
        f.write(np.ascontiguousarray(g["e_v2"], np.int32).tobytes())
        f.write(np.ascontiguousarray(g["e_meas"], np.float64).tobytes())
        f.write(np.ascontiguousarray(g["points"], np.float64).tobytes())
        f.write(np.ascontiguousarray(g["point_ref"], np.int32).tobytes())
    lines = subprocess.check_output([exe, str(path)], text=True).splitlines()
    got = optimize.graph_optimizer(fix_scale=fix_scale).optimize(g)
    nv, npt = len(g["estimate"]), len(g["points"])
    est = np.array([ln.split() for ln in lines[:nv]], np.float64)
    pose = np.array(lines[nv:nv + 16 * nv], np.float64).reshape(nv, 4, 4)
    pts = np.array(lines[nv + 16 * nv:nv + 16 * nv + 3 * npt], np.float64).reshape(npt, 3)
    assert np.array_equal(est, got["estimate"]) and np.array_equal(pose, got["pose_cw"]) and np.array_equal(pts, got["points"])
    assert lines[-1] == f"iterations {got['iterations']}"
