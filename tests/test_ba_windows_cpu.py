"""Pins the local-BA and pose-optimiser oracles (oracle/lba_oracle.c) on windows shaped like real tracking (tests/ba_windows.py):
several cameras per window, mostly 2-observation landmarks, points behind a camera, near / far / polar / seam points, an empty and
a backward-looking free keyframe.  As in test_lba_scipy.py, an independent numpy restatement with a camera per edge decides:
  1. the chi2 the oracle reports equals numpy's cost of the state it returns;
  2. the outlier flags equal numpy's chi-square and depth tests;
  3. the end state is within the gain threshold of scipy.optimize.least_squares' optimum of the same cost.
The pose optimiser gets the same pin: its flags and n_valid are the chi-square test at the returned pose (threshold by x_right; the
reference has no depth test there, so points behind the camera simply have to agree), and with num_trials > 0 the returned pose is
within 1e-3 relative cost of scipy's plain least-squares optimum over the edges its last trial optimised."""
import os
import sys

import numpy as np
import pytest
from scipy.optimize import least_squares
from scipy.sparse import lil_matrix
from scipy.spatial.transform import Rotation as R

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ba_windows as W  # noqa: E402
from oracle import pyoracle as O  # noqa: E402

KITTI_FXB = W.CAMS["kitti"]["fxb"]
SCIPY = dict(method="trf", xtol=1e-14, ftol=1e-14, gtol=1e-10, max_nfev=60)


def test_windows_have_the_shapes_of_real_tracking():
    single = 0
    for name in list(W.WINDOWS) + list(W.LONG_WINDOWS):
        pr = W.window(name)
        K, L = len(pr["pose_cw"]), len(pr["points"])
        deg = np.bincount(pr["e_point"], minlength=L)
        assert deg.min() >= 1 and (deg == 2).mean() > 0.4 and (deg == 1).any(), name
        single += (deg[pr["e_point"][pr["pose_fixed"][pr["e_pose"]] == 0]] == 1).sum()   # 1-observation landmarks in free keyframes
        # a camera per keyframe: e_cam is the keyframe's camera, and every camera of the window is used
        assert np.array_equal(pr["e_cam"], pr["e_pose"] % len(pr["cams"])) and len(np.unique(pr["e_cam"])) == len(pr["cams"])
        stereo_cam = [i for i, c in enumerate(pr["cams"]) if c["fxb"] > 0]
        if stereo_cam:   # mono edges inside stereo keyframes, and sub-pixel disparities of the far points
            m = np.isin(pr["e_cam"], stereo_cam)
            assert (pr["e_obs"][m, 2] < 0).sum() > 10 and (pr["e_obs"][m, 2] >= 0).sum() > 10
            far = np.isin(pr["e_point"], np.nonzero(pr["kinds"] == "far")[0]) & (pr["e_obs"][:, 2] >= 0)
            T, P = pr["gt_pose_cw"][pr["e_pose"][far]], pr["gt_points"][pr["e_point"][far]]
            z = np.einsum("ej,ej->e", T[:, 2, :3], P) + T[:, 2, 3]
            assert far.any() and np.all(KITTI_FXB / z < 1.0)
        free = pr["pose_fixed"] == 0
        assert free[pr["empty_kf"]] and not (pr["e_pose"] == pr["empty_kf"]).any()
        assert free[pr["outlier_kf"]] and (pr["e_pose"] == pr["outlier_kf"]).sum() >= 10
        assert len(pr["behind"]) >= 4 and {"near", "far"} <= set(pr["kinds"])
        if any(c["model"] == 1 for c in pr["cams"]):
            assert {"pole", "seam"} <= set(pr["kinds"])
            # the seam landmarks are observed within a few pixels of u = 0 or u = cols (their one observation)
            seam = np.isin(pr["e_point"], np.nonzero(pr["kinds"] == "seam")[0])
            u = pr["e_obs"][seam, 0]
            assert seam.sum() >= 4 and np.all(np.minimum(np.abs(u), np.abs(W.CAMS["equirect"]["cols"] - u)) < 16), u
    assert single >= 20
    deep = np.bincount(W.window("deep_degrees")["e_point"])
    assert {64, 65} <= set(deep) and (W.window("deep_degrees")["pose_fixed"] == 0).sum() > 65


def _scipy_optimum(wp, x0, sel, robust):
    def fun(x):
        T, P = wp.unpack(x)
        chi, _ = wp.edge_chi2(T, P, sel)
        return np.sqrt((wp.huber(chi, sel) if robust else chi) + 1e-300)   # one residual per edge; per-edge Huber width
    # each residual depends on its keyframe's 6 and its landmark's 3 parameters: finite differences over column groups
    pr, col = wp.pr, {int(k): i for i, k in enumerate(wp.free_k)}
    S = lil_matrix((int(sel.sum()), len(x0)), dtype=np.int8)
    for r, e in enumerate(np.nonzero(sel)[0]):
        k, b = int(pr["e_pose"][e]), 6 * len(wp.free_k) + 3 * int(pr["e_point"][e])
        if k in col:
            S[r, 6 * col[k]:6 * col[k] + 6] = 1
        S[r, b:b + 3] = 1
    return 2.0 * least_squares(fun, x0, jac_sparsity=S, **SCIPY).cost


@pytest.mark.parametrize("name", list(W.WINDOWS))
def test_local_ba_oracle_pins(name):
    pr = W.window(name)
    E = len(pr["e_pose"])
    every = np.ones(E, bool)
    wp = W.WindowProblem(pr)
    # ---- first round alone: reported robust chi2 == numpy's Huber cost of the returned state; that state is scipy's Huber optimum
    r1 = O.lba_solve(pr, iters1=40, iters2=0)
    chi1 = wp.robust_cost(r1["pose_cw"], r1["points"], every)
    assert abs(chi1 - r1["chi2"][0]) <= 1e-9 * r1["chi2"][0]
    opt1 = _scipy_optimum(wp, wp.pack(r1["pose_cw"], r1["points"]), every, True)
    assert opt1 <= r1["chi2"][0] * (1 + 1e-12) and r1["chi2"][0] - opt1 <= 2e-3 * opt1, (r1["chi2"][0], opt1)
    # ---- the protocol: round 1 (5 iterations), outliers, round 2 on the rest
    r5 = O.lba_solve(pr, iters1=5, iters2=0)
    ref = O.lba_solve(pr, iters1=5, iters2=10)
    for st in (r5, ref):
        W.assert_clear_of_thresholds(pr, st["pose_cw"], st["points"])
    chi5, pc5 = wp.edge_chi2(r5["pose_cw"], r5["points"], every)
    active = ~wp.outlier_test(r5["pose_cw"], r5["points"])
    assert np.array_equal(~active, r5["outliers"].astype(bool))
    # the depth test is decisive: points behind their camera pass the chi-square test, and every edge of the backward keyframe
    # is rejected after round 1
    b = pr["behind"]
    assert np.all(pc5[b, 2] < 0) and np.all(~active[b])
    bk = pr["e_pose"] == pr["outlier_kf"]
    assert not active[bk].any() and (chi5[bk] <= W.thresholds(pr)[bk]).mean() > 0.5
    assert (chi5[b] <= W.thresholds(pr)[b]).sum() >= 3
    # final flags: chi2 of the last activation (round 2 for active edges, round 1 for the others) and the depth at the end state
    chi_f, _ = wp.edge_chi2(ref["pose_cw"], ref["points"], every)
    want = wp.outlier_test(ref["pose_cw"], ref["points"], chi=np.where(active, chi_f, chi5))
    assert np.array_equal(want, ref["outliers"].astype(bool)) and ref["n_outliers"] == want.sum()
    assert abs(chi_f[active].sum() - ref["chi2"][1]) <= 1e-9 * ref["chi2"][1]
    opt2 = _scipy_optimum(wp, wp.pack(ref["pose_cw"], ref["points"]), active, False)
    assert opt2 <= ref["chi2"][1] * (1 + 1e-12) and ref["chi2"][1] - opt2 <= 5e-3 * opt2, (ref["chi2"][1], opt2)
    # a keyframe with no active edge does not move: the empty one never, the backward one not in round 2
    assert np.allclose(ref["pose_cw"][pr["empty_kf"]], pr["pose_cw"][pr["empty_kf"]], rtol=0, atol=1e-12)
    assert np.allclose(ref["pose_cw"][pr["outlier_kf"]], r5["pose_cw"][pr["outlier_kf"]], rtol=0, atol=1e-12)


# ---- pose optimiser ---------------------------------------------------------------------------------------------------------
POSE_FRAMES = {
    "mono": dict(seed=1, n_obs=400, cam="euroc", n_near=5, n_far=5),
    "stereo": dict(seed=2, n_obs=400, cam="kitti", stereo_frac=1.0, n_far=8),
    "mixed": dict(seed=3, n_obs=500, cam="kitti", stereo_frac=0.6, n_behind=8, n_near=4, n_far=6),
    "equirect": dict(seed=4, n_obs=600, cam="equirect", n_pole=10, n_seam=10, n_behind=6),
    "behind_cam1": dict(seed=5, n_obs=300, cam="euroc", n_behind=12, cam_index=1, n_cams=3),
}


def pose_chi2(pr, pose):
    wp = W.WindowProblem(pr)
    return wp.edge_chi2(np.asarray(pose)[None], pr["points"], np.ones(len(pr["e_pose"]), bool))


def pose_pins(pr, result, cfg=(2, 2, 10), optimize=O.pose_optimize):
    """The numpy / scipy pins of one pose-optimiser result (shared with the device tests): flags and n_valid are the chi-square test
    at the returned pose; with num_trials > 0 the pose is the plain least-squares optimum over the edges its last trial optimised
    (the inliers of the run one trial shorter), within the 1e-3 gain threshold the trials stop on."""
    n_valid, pose, flags = result
    chi, pc = pose_chi2(pr, pose)
    thr = W.thresholds(pr)
    assert np.min(np.abs(chi - thr) / thr) > W.MARGIN
    assert np.array_equal(flags, chi > thr) and n_valid == (~flags).sum()
    if not cfg[1] or n_valid < 5:
        return
    inl = ~optimize(pr, cfg[0], cfg[1] - 1, cfg[2])[2]

    def fun(xi):
        T = np.array(pose, np.float64)
        dR = R.from_rotvec(xi[:3]).as_matrix()
        T[:3, :3], T[:3, 3] = dR @ T[:3, :3], dR @ T[:3, 3] + xi[3:]
        c, _ = W.WindowProblem(pr).edge_chi2(T[None], pr["points"], inl)
        return np.sqrt(c + 1e-300)
    got = chi[inl].sum()
    opt = 2.0 * least_squares(fun, np.zeros(6), **SCIPY).cost
    assert opt <= got * (1 + 1e-12) and got - opt <= 1e-3 * opt, (got, opt)


@pytest.mark.parametrize("name", list(POSE_FRAMES))
def test_pose_optimizer_oracle_pins(name):
    pr = W.make_frame(**POSE_FRAMES[name])
    n, pose, flags = O.pose_optimize(pr)
    pose_pins(pr, (n, pose, flags))
    assert flags[pr["gt_outlier"]].mean() > 0.9
    _, pc = pose_chi2(pr, pose)
    if len(pr["behind"]):      # no depth test: points behind the camera that fit stay inliers
        assert np.all(pc[pr["behind"], 2] < 0) and (~flags[pr["behind"]]).mean() > 0.5
    # the other protocols: robust trials only (the Huber state is not a plain least-squares optimum: flags / n_valid only), and
    # plain trials only
    for cfg in ((4, 0, 10), (0, 3, 10)):
        pose_pins(pr, O.pose_optimize(pr, *cfg), cfg)


def test_pose_optimizer_oracle_honours_the_problem_camera():
    # the same frame with its camera at index 0 or at index 2 among decoys gives the same result
    a = W.make_frame(**dict(POSE_FRAMES["mixed"], cam_index=0, n_cams=1))
    b = W.make_frame(**dict(POSE_FRAMES["mixed"], cam_index=2, n_cams=3))
    ra, rb = O.pose_optimize(a), O.pose_optimize(b)
    assert ra[0] == rb[0] and np.array_equal(ra[1], rb[1]) and np.array_equal(ra[2], rb[2])
