"""The C++ mirror of robust-match tracking (include/b200vslam.hpp: tracking::frame_tracker::robust_match_based_track) drives the same frames
as the Python mirror (stella_vslam_b200.tracking.frame_tracker) and gets the same results, bit for bit."""
import subprocess

import numpy as np
import pytest

import cbuild

KITTI = dict(model="perspective", fx=718.856, fy=718.856, cx=607.1928, cy=185.2157, fxb=386.1448, cols=1241.0, rows=376.0, setup="stereo")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return cbuild.cpp_mirror("robust_track_api_test", tmp_path_factory.mktemp("robust_track_api"))


def test_cpp_mirror_builds_and_reports_usage(exe):
    assert subprocess.run([exe], capture_output=True).returncode == 2


def _hex(a):
    a = np.ascontiguousarray(a)
    return " ".join(b.tobytes().hex() for b in np.frombuffer(a.tobytes(), np.uint8).reshape(-1, a.dtype.itemsize))


@pytest.mark.gpu
def test_cpp_robust_track_matches_python(exe, tmp_path):
    from stella_vslam_b200 import feature, solve, tracking
    from workloads import synth
    n, w, h = 3, 1241, 376
    gray = np.stack([synth.make_frame(w, h, seed=50 + i) for i in range(n)])
    ex = feature.orb_extractor(feature.orb_params(), 800, max_batch=n)
    kps, descs = ex.extract_batch(gray)
    seed = list(range(1, 11))
    frames = [dict(synth.make_robust_frame(kps[0], descs[0], KITTI, seed=70, stereo=True), frame=0),
              dict(synth.make_robust_frame(kps[2], descs[2], KITTI, seed=71, stereo=True), frame=2, engine=solve.mt19937(seed)),
              dict(synth.make_robust_frame(kps[1], descs[1], KITTI, seed=72, stereo=True, kf_keypoints=4), frame=1)]
    tr = tracking.frame_tracker(ex, KITTI, use_fixed_seed=True)
    want = tr.robust_match_based_track(frames)
    path = tmp_path / "robust.bin"
    with open(path, "wb") as f:
        f.write(np.array([n, w, h], np.int32).tobytes() + gray.tobytes())
        f.write(np.array([0, 0], np.int32).tobytes())
        f.write(np.array([KITTI[k] for k in ("fx", "fy", "cx", "cy", "fxb", "cols", "rows")], np.float64).tobytes())
        f.write(np.array([tr.num_matches_thr], np.uint32).tobytes())
        for fr in frames:
            kf = fr["keyframe"]
            f.write(np.array([fr["frame"], len(fr["kp_x_right"]), len(kf["desc"])], np.int32).tobytes())
            f.write(np.ascontiguousarray(fr["last_pose_cw"], np.float64).tobytes() + np.ascontiguousarray(fr["kp_x_right"], np.float32).tobytes())
            f.write(np.ascontiguousarray(kf["desc"], np.uint8).tobytes() + np.ascontiguousarray(kf["angle"], np.float32).tobytes())
            f.write(np.ascontiguousarray(kf["bearings"], np.float64).tobytes() + np.ascontiguousarray(kf["valid"], np.uint8).tobytes())
            f.write(np.ascontiguousarray(kf["pos_w"], np.float64).tobytes())
            seeded = "engine" in fr
            f.write(np.array([int(seeded)], np.int32).tobytes() + (np.array(seed, np.uint32).tobytes() if seeded else b""))
    lines = subprocess.check_output([exe, "track", str(path)], text=True).splitlines()
    for i, g in enumerate(want):
        head, kp, pose = lines[3 * i:3 * i + 3]
        assert head == (f"frame {g['n_keypoints']} {g['n_matches']} {int(g['essential_valid'])} {g['n_inliers']} {int(g['applied'])} {g['status']} "
                        f"{g['n_valid']} {int(g['tracked'])}")
        if g["applied"]:
            assert kp == ("kp " + _hex(g["kp_landmark"])).rstrip()
            assert pose == "pose " + _hex(g["pose_cw"].reshape(16))
    assert lines[3 * n] == "chain_ms_positive 1"
    assert want[0]["tracked"] and want[1]["tracked"] and not want[2]["applied"]
