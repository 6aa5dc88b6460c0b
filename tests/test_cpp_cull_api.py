"""The C++ mirror of keyframe culling (include/b200vslam.hpp: b200::module::local_map_cleaner) drives the same problems as the Python
mirror and gets the same results, and makes the reference's early return without a call."""
import subprocess

import numpy as np
import pytest

import cbuild


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return cbuild.cpp_mirror("cull_api_test", tmp_path_factory.mktemp("cull_api"))


def test_cpp_mirror_builds_and_reports_usage(exe):
    assert subprocess.run([exe], capture_output=True).returncode == 2


def _write(path, problems):
    with open(path, "wb") as f:
        f.write(np.array([len(problems)], np.int32).tobytes())
        for pr in problems:
            f.write(np.array([pr["cur_id"]], np.uint32).tobytes() + np.array([len(pr["covisibilities"])], np.int32).tobytes())
            for cv in pr["covisibilities"]:
                kl = np.asarray(cv["kp_landmark"], np.int32)
                f.write(np.array([cv["id"]], np.uint32).tobytes() + np.array([int(cv["is_root"]), len(kl), int(cv["depth"] is not None)], np.int32).tobytes())
                f.write(np.array([cv["depth_thr"]], np.float64).tobytes() + kl.tobytes())
                if cv["depth"] is not None:
                    f.write(np.asarray(cv["depth"], np.float32).tobytes())
            off = np.asarray(pr["obs_offsets"], np.int32)
            f.write(np.array([len(off) - 1], np.int32).tobytes() + off.tobytes())
            f.write(np.asarray(pr["obs_rank"], np.int32).tobytes() + np.asarray(pr["obs_octave"], np.int32).tobytes())
            f.write(np.asarray(pr["obs_weight"], np.uint8).tobytes())


def _run(exe, path, thr, top_n):
    out, k = [], -1
    for ln in subprocess.check_output([exe, str(path), repr(thr), str(top_n)], text=True).splitlines():
        w = ln.split()
        if w[0] == "problem":
            out.append(dict(n_removed=int(w[2]), ranks=[]))
        else:
            out[-1]["ranks"].append(tuple(int(v) for v in w[2:]))
    return out


@pytest.mark.gpu
def test_cpp_cull_matches_python(exe, tmp_path):
    from stella_vslam_b200 import mapping
    from workloads import synth
    rng = np.random.default_rng(5)
    problems = [synth.gather_cull_problem(synth.make_cull_map(rng, n_keypoints=int(rng.integers(200, 1200)), stereo_frac=0.5)) for _ in range(6)]
    path = tmp_path / "cull.bin"
    _write(path, problems)
    got = _run(exe, path, 0.9, 30)
    want = mapping.remove_redundant_keyframes(problems)
    assert sum(w["n_removed"] for w in want) > 0
    for g, w in zip(got, want):
        assert g["n_removed"] == w["n_removed"]
        assert g["ranks"] == list(zip(w["skipped"].tolist(), w["n_valid"].tolist(), w["n_redundant"].tolist(), w["removed"].tolist()))
    for thr, top_n in ((-0.5, 30), (0.9, 0)):  # the early return: no call, nothing removed, the outputs stay as given
        assert all(g["n_removed"] == 0 and all(r == (0, 0, 0, 0) for r in g["ranks"]) for g in _run(exe, path, thr, top_n))
