"""The device local BA, global BA and pose optimiser on windows shaped like real tracking (tests/ba_windows.py): several cameras
per window, mostly 2-observation landmarks, 1-observation landmarks in free keyframes, landmarks seen by 64 / 65 / every keyframe,
points behind a camera, near / far / polar / seam points, an empty and a backward-looking free keyframe.  Each result is checked
against the oracle (test_lba_gpu.check_same: identical iterations and flags, 1e-5 on poses and points) AND directly against the
numpy restatement (reported chi2 == numpy's cost of the device state to 1e-9, flags == numpy's chi-square and depth tests), so a
bug the oracle and the kernel share cannot hide."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ba_windows as W  # noqa: E402
from oracle import pyoracle as O  # noqa: E402
from test_ba_windows_cpu import POSE_FRAMES, pose_pins  # noqa: E402
from test_global_ba import _check as check_global  # noqa: E402
from test_lba_gpu import check_same  # noqa: E402
from test_pose_opt_gpu import _same as same_pose  # noqa: E402

pytestmark = pytest.mark.gpu

NAMES = list(W.WINDOWS) + list(W.LONG_WINDOWS)


@pytest.fixture(scope="module")
def windows():
    return {n: W.window(n) for n in NAMES}


@pytest.fixture(scope="module")
def optimize():
    from stella_vslam_b200 import optimize
    return optimize


@pytest.mark.parametrize("name", NAMES)
def test_local_ba_vs_oracle_and_numpy(windows, optimize, name):
    pr = windows[name]
    E = len(pr["e_pose"])
    every = np.ones(E, bool)
    wp = W.WindowProblem(pr)
    got = optimize.local_bundle_adjuster().optimize(pr)
    check_same(got, O.lba_solve(pr), pr)
    # round 1 alone on the device: its robust chi2 is numpy's Huber cost of its state, its flags numpy's chi-square + depth test
    r5 = optimize.local_bundle_adjuster(5, 0).optimize(pr)
    for st in (r5, got):
        W.assert_clear_of_thresholds(pr, st["pose_cw"], st["points"])
    assert abs(wp.robust_cost(r5["pose_cw"], r5["points"], every) - r5["chi2"][0]) <= 1e-9 * r5["chi2"][0]
    assert r5["chi2"][0] == got["chi2"][0]
    chi5, pc5 = wp.edge_chi2(r5["pose_cw"], r5["points"], every)
    active = ~wp.outlier_test(r5["pose_cw"], r5["points"])
    assert np.array_equal(~active, r5["outliers"].astype(bool))
    assert np.all(~active[pr["behind"]]) and np.all(pc5[pr["behind"], 2] < 0)           # the depth test fired
    assert (chi5[pr["behind"]] <= W.thresholds(pr)[pr["behind"]]).sum() >= 3             # ... and decided alone
    assert not active[pr["e_pose"] == pr["outlier_kf"]].any()
    # the full protocol: round-2 chi2 over the edges left active, flags from the chi2 of each edge's last activation
    chi_f, _ = wp.edge_chi2(got["pose_cw"], got["points"], every)
    assert abs(chi_f[active].sum() - got["chi2"][1]) <= 1e-9 * got["chi2"][1]
    want = wp.outlier_test(got["pose_cw"], got["points"], chi=np.where(active, chi_f, chi5))
    assert np.array_equal(want, got["outliers"].astype(bool))
    assert np.allclose(got["pose_cw"][pr["empty_kf"]], pr["pose_cw"][pr["empty_kf"]], rtol=0, atol=1e-12)


def test_batch_of_all_windows_equals_single_calls(windows, optimize):
    ba = optimize.local_bundle_adjuster()
    prs = [windows[n] for n in NAMES]
    got = ba.optimize_batch(prs)
    for g, pr in zip(got, prs):
        one = ba.optimize(pr)
        assert np.array_equal(one["pose_cw"], g["pose_cw"]) and np.array_equal(one["points"], g["points"])
        assert np.array_equal(one["outliers"], g["outliers"]) and one["iterations"] == g["iterations"] and one["chi2"] == g["chi2"]


@pytest.mark.parametrize("name", ["three_cams", "two_view_mono"])
def test_global_ba(windows, optimize, name):
    pr = windows[name]
    wp = W.WindowProblem(pr)
    got = optimize.global_bundle_adjuster(10).optimize(pr)
    check_global(got, O.global_ba_solve(pr, 10), pr)
    assert abs(wp.robust_cost(got["pose_cw"], got["points"], np.ones(len(pr["e_pose"]), bool)) - got["chi2"]) <= 1e-9 * got["chi2"]


# ---- pose optimiser ---------------------------------------------------------------------------------------------------------
SIZES = [(5, dict(cam="kitti", stereo_frac=0.5, outlier_frac=0.0)),
         (6, dict(cam="euroc", cam_index=1, n_cams=2, n_behind=1, outlier_frac=0.0)),
         (255, dict(cam="kitti", stereo_frac=0.6, n_behind=6, n_far=4, cam_index=2, n_cams=3)),
         (256, dict(cam="equirect", n_pole=8, n_seam=8, cam_index=1, n_cams=2)),
         (257, dict(cam="euroc", n_near=3, n_behind=5)),
         (4097, dict(cam="kitti", stereo_frac=0.7, n_behind=20, n_far=20, cam_index=1, n_cams=3)),
         (20000, dict(cam="equirect", n_pole=40, n_seam=40, n_behind=30, cam_index=2, n_cams=3))]   # a 3840x1920 frame's keypoints


@pytest.mark.parametrize("n,spec", SIZES, ids=[str(n) for n, _ in SIZES])
def test_pose_optimizer_sizes_vs_oracle_and_numpy(optimize, n, spec):
    pr = W.make_frame(seed=n, n_obs=n, **spec)
    dev = lambda p, a, b, c: optimize.pose_optimizer(a, b, c).optimize(p)
    got = dev(pr, 2, 2, 10)
    same_pose(got, O.pose_optimize(pr))
    pose_pins(pr, got, (2, 2, 10), dev)


@pytest.mark.parametrize("name", list(POSE_FRAMES))
def test_pose_optimizer_frames_vs_oracle_and_numpy(optimize, name):
    pr = W.make_frame(**POSE_FRAMES[name])
    dev = lambda p, a, b, c: optimize.pose_optimizer(a, b, c).optimize(p)
    for cfg in ((2, 2, 10), (4, 0, 10), (0, 3, 10)):
        got = dev(pr, *cfg)
        same_pose(got, O.pose_optimize(pr, *cfg))
        pose_pins(pr, got, cfg, dev)


def test_pose_optimizer_uses_the_problems_own_camera(optimize):
    # the same frame with its camera at index 0, or at index 2 behind two decoys with other intrinsics: the same result, bit for bit
    a = W.make_frame(**dict(POSE_FRAMES["mixed"], cam_index=0, n_cams=1))
    b = W.make_frame(**dict(POSE_FRAMES["mixed"], cam_index=2, n_cams=3))
    po = optimize.pose_optimizer()
    ga, gb = po.optimize(a), po.optimize(b)
    assert ga[0] == gb[0] and np.array_equal(ga[1], gb[1]) and np.array_equal(ga[2], gb[2])
    same_pose(gb, O.pose_optimize(b))


def test_pose_optimizer_refuses_a_frame_with_several_cameras(optimize):
    from stella_vslam_b200 import _lib
    good = W.make_frame(**POSE_FRAMES["stereo"])
    mixed = W.make_frame(**dict(POSE_FRAMES["stereo"], cam_index=1, n_cams=2))
    mixed["e_cam"] = mixed["e_cam"].copy()
    mixed["e_cam"][len(mixed["e_cam"]) // 2] = 0
    po = optimize.pose_optimizer()
    with pytest.raises(RuntimeError, match="one camera"):
        po.optimize(mixed)
    # in a batch, one such frame refuses the whole call and nothing is written
    packed = [optimize.pack_problem(p) for p in (good, mixed)]
    arr = (optimize.LbaProblem * 2)(*[pk[0] for pk in packed])
    pose = np.full((2, 4, 4), 7.0)
    flags = np.full(sum(len(p["e_pose"]) for p in (good, mixed)), 9, np.uint8)
    valid = np.full(2, 123, np.uint32)
    rc = po._L.b200_pose_optimize(po._h, 2, arr, 2, 2, 10, pose.ctypes.data_as(C.c_void_p),
                                  flags.ctypes.data_as(C.c_void_p), valid.ctypes.data_as(C.c_void_p))
    assert rc == _lib.ERR_INVALID
    assert np.all(pose == 7.0) and np.all(flags == 9) and np.all(valid == 123)
    same_pose(po.optimize(good), O.pose_optimize(good))          # the handle is still usable
