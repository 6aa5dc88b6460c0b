"""The C++ mirror (include/b200vslam.hpp) compiles against the C ABI alone and honours the no-fallback contract."""
import subprocess
import sys

import pytest

import cbuild


def test_cpp_mirror_compiles_and_fails_loudly_without_gpu(tmp_path):
    exe = cbuild.cpp_mirror("host_api_test", tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "sm_90a" in r.stdout


@pytest.mark.gpu
def test_cpp_mirror_runs_on_gpu(tmp_path):
    exe = cbuild.cpp_mirror("host_api_test", tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "keypoints" in r.stdout and "self matches" in r.stdout and "projection matches" in r.stdout and "stereo matches" in r.stdout and "tracking matches" in r.stdout
