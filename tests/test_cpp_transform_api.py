"""The C++ mirror of optimize::transform_optimizer (include/b200vslam.hpp, b200::optimize::transform_optimizer) runs the same loop
candidate as the Python mirror (stella_vslam_b200.optimize) and gets a bit-identical Sim3, the same keep flags and inlier count."""
import os
import subprocess

import numpy as np
import pytest

import cbuild
from workloads import synth


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return cbuild.cpp_mirror("transform_api_test", tmp_path_factory.mktemp("transform_api"))


def test_cpp_mirror_compiles(exe):
    assert os.path.exists(exe)


@pytest.mark.gpu
@pytest.mark.parametrize("models,fix_scale", [(("perspective", "perspective"), False), (("equirect", "perspective"), True)])
def test_cpp_transform_optimizer_matches_python(exe, tmp_path, models, fix_scale):
    from stella_vslam_b200 import optimize
    pr = synth.make_sim3_pair(31, 250, models=models, fix_scale=fix_scale, outlier_frac=0.2)
    n = len(pr["obs_1"])
    path = tmp_path / "pair.bin"
    with open(path, "wb") as f:
        f.write(np.array([n, int(fix_scale)], np.int32).tobytes())
        for k in ("sim3_12", "rot_1w", "trans_1w", "rot_2w", "trans_2w"):
            f.write(np.ascontiguousarray(pr[k], np.float64).tobytes())
        for c in (pr["cam_1"], pr["cam_2"]):
            f.write(np.int32(c["model"]).tobytes())
            f.write(np.array([c[k] for k in ("fx", "fy", "cx", "cy", "fxb", "cols", "rows")], np.float64).tobytes())
        for k, dt in (("obs_1", np.float32), ("inv_sigma_sq_1", np.float32), ("pos_w_2", np.float64), ("obs_2", np.float32),
                      ("inv_sigma_sq_2", np.float32), ("pos_w_1", np.float64)):
            f.write(np.ascontiguousarray(pr[k], dt).tobytes())
    lines = subprocess.check_output([exe, str(path)], text=True).splitlines()
    got = optimize.transform_optimizer(fix_scale).optimize(pr)
    assert np.array_equal(np.array(lines[0].split(), np.float64), got["sim3_12"])
    assert np.array_equal(np.array(lines[1:1 + n], np.uint8), got["keep"])
    assert lines[-1] == f"inliers {got['num_inliers']}"
