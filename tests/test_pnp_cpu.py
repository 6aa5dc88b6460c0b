"""solve::pnp_solver on the CPU: the restated Eigen pieces against numpy, EPnP against the true pose and cv2, the RANSAC rules on
hand-built inputs and max_cos_errors_ against util::cos."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pnp_oracle as O  # noqa: E402

from workloads import synth  # noqa: E402


def _psd(rng, n, rank=None):
    A = rng.standard_normal((n, rank or n))
    return A @ A.T


@pytest.mark.parametrize("n", [3, 12])
def test_svd_square_against_numpy(n):
    rng = np.random.default_rng(n)
    for trial in range(20):
        A = rng.standard_normal((n, n)) if trial % 2 else _psd(rng, n)
        U, V, sv, nz = O.svd_square(A)
        Un, svn, _ = np.linalg.svd(A)
        assert nz == n
        np.testing.assert_allclose(sv, svn, rtol=0, atol=1e-13 * svn[0])
        for j in range(n):  # U's columns up to sign (the singular values are distinct here)
            s = np.sign(U[:, j] @ Un[:, j])
            np.testing.assert_allclose(U[:, j] * s, Un[:, j], atol=1e-11)
        np.testing.assert_allclose(U @ np.diag(sv) @ V.T, A, atol=1e-12 * svn[0])


@pytest.mark.parametrize("k", [3, 4, 5])
def test_preconditioned_svd_solve_against_lstsq(k):
    rng = np.random.default_rng(10 + k)
    for trial in range(20):
        A, b = rng.standard_normal((6, k)) * 10.0 ** rng.uniform(-3, 3), rng.standard_normal(6)
        x, rank, sv = O.svd_solve_6xk(A, b)
        assert rank == k
        np.testing.assert_allclose(sv, np.linalg.svd(A)[1], rtol=1e-13)
        np.testing.assert_allclose(x, np.linalg.lstsq(A, b, rcond=None)[0], rtol=1e-10, atol=1e-12 * np.abs(x).max())


@pytest.mark.parametrize("k", [3, 4, 5])
def test_preconditioned_svd_solve_rank_deficient(k):
    """A repeated column: rank() drops the zero singular value and solve() returns the minimum-norm least-squares solution."""
    rng = np.random.default_rng(20 + k)
    A = rng.standard_normal((6, k))
    A[:, -1] = A[:, 0]
    b = rng.standard_normal(6)
    x, rank, sv = O.svd_solve_6xk(A, b)
    assert rank == k - 1
    np.testing.assert_allclose(x, np.linalg.lstsq(A, b, rcond=None)[0], atol=1e-12)
    x0, rank0, _ = O.svd_solve_6xk(np.zeros((6, k)), b)
    assert rank0 == 0 and not x0.any()


def test_householder_qr_solve_against_lstsq():
    rng = np.random.default_rng(3)
    for _ in range(20):
        A, b = rng.standard_normal((6, 4)), rng.standard_normal(6)
        np.testing.assert_allclose(O.householder_qr_solve(A, b), np.linalg.lstsq(A, b, rcond=None)[0], rtol=1e-11, atol=1e-13)


def _noise_free(seed, n, model="perspective"):
    pr = synth.make_pnp_problem(seed, n, 1.0, model)
    pc = pr["points"] @ pr["gt_rot_cw"].T + pr["gt_trans_cw"]
    return pc / np.linalg.norm(pc, axis=1, keepdims=True), pr["points"], pr["gt_rot_cw"], pr["gt_trans_cw"]


@pytest.mark.parametrize("model", ["perspective", "equirect"])
def test_epnp_recovers_the_true_pose(model):
    for seed, n in [(1, 6), (2, 20), (3, 300), (4, 1000)]:
        b, p, R, t = _noise_free(seed, n, model)
        Re, te, err, wrote = O.compute_pose(b, p, 10)
        assert wrote and err < 1e-12
        np.testing.assert_allclose(Re, R, atol=1e-9)
        np.testing.assert_allclose(te, t, atol=1e-9)


def test_epnp_minimal_sets():
    """On 4 points the N-candidate that reaches a zero reprojection error recovers the pose; most minimal sets do.  Four points
    spread over tens of metres condition the solve worse than n points, so the bound is 1e-7 here."""
    b, p, R, t = _noise_free(5, 400)
    rng = np.random.default_rng(0)
    good = 0
    for _ in range(100):
        idx = rng.choice(len(b), 4, replace=False)
        Re, te, err, wrote = O.compute_pose(b[idx], p[idx], 10)
        assert wrote
        if err < 1e-14:
            np.testing.assert_allclose(Re, R, atol=1e-7)
            np.testing.assert_allclose(te, t, atol=1e-7 * max(1.0, np.abs(t).max()))
            good += 1
    assert good >= 60


def test_epnp_against_cv2():
    cv2 = pytest.importorskip("cv2")
    K = np.array([[synth.KITTI["fx"], 0, synth.KITTI["cx"]], [0, synth.KITTI["fy"], synth.KITTI["cy"]], [0, 0, 1.0]])
    for seed, n in [(6, 6), (7, 50), (8, 500)]:
        b, p, R, t = _noise_free(seed, n)
        uv = (b[:, :2] / b[:, 2:]) * [K[0, 0], K[1, 1]] + [K[0, 2], K[1, 2]]
        ok, rvec, tvec = cv2.solvePnP(p, uv, K, None, flags=cv2.SOLVEPNP_EPNP)
        assert ok
        Re, te, err, wrote = O.compute_pose(b, p, 10)
        np.testing.assert_allclose(Re, cv2.Rodrigues(rvec)[0], atol=1e-6)
        np.testing.assert_allclose(te, tvec.ravel(), atol=1e-5)


def test_coplanar_points_take_the_pseudo_inverse_branch():
    pr = synth.make_pnp_problem(9, 200, 1.0, "perspective", case="coplanar")
    assert np.ptp(pr["points"][:, 2]) == 0.0
    pc = pr["points"] @ pr["gt_rot_cw"].T + pr["gt_trans_cw"]
    b = pc / np.linalg.norm(pc, axis=1, keepdims=True)
    Re, te, err, wrote = O.compute_pose(b, pr["points"], 10)
    assert wrote and err < 1e-10
    np.testing.assert_allclose(Re, pr["gt_rot_cw"], atol=1e-7)


def _prob(pr, **kw):
    d = dict(bearings=pr["bearings"], points=pr["points"], octaves=pr["octaves"], scale_factors=pr["scale_factors"])
    d.update(kw)
    return d


def _inlier_sets(pr, k, seed=0):
    rng = np.random.default_rng(seed)
    idx = np.flatnonzero(pr["gt_inlier"])
    return np.stack([rng.choice(idx, 4, replace=False) for _ in range(k)]).astype(np.int32)


def test_ransac_strict_inlier_count():
    """num_inliers > min_num_inliers is strict: exactly 10 inliers and min_num_inliers = 10 is no solution."""
    pr = synth.make_pnp_problem(11, 60, 0.0, "perspective", case="min_inliers")
    ms = _inlier_sets(pr, 30)
    r10 = O.pnp_ransac(_prob(pr, min_num_inliers=10), ms)
    assert not r10["valid"] and r10["best_iter"] == -1 and not r10["inlier_flags"].any()
    r9 = O.pnp_ransac(_prob(pr, min_num_inliers=9), ms)
    assert r9["valid"] and r9["num_inliers"] == 10
    np.testing.assert_array_equal(r9["inlier_flags"], pr["gt_inlier"])


def test_ransac_first_of_equal_costs_wins():
    """Duplicated minimal sets give equal costs; min_cost > cost is strict, so the first of them wins."""
    pr = synth.make_pnp_problem(12, 200, 0.6)
    s = _inlier_sets(pr, 1)[0]
    r = O.pnp_ransac(_prob(pr), np.stack([s, s, s]))
    assert r["valid"] and r["best_iter"] == 0


def test_ransac_hypothesis_without_pose_is_rejected():
    """A minimal set with a bearing of z = 0 (equirectangular) gives NaN reprojection errors: compute_pose writes nothing, and the
    hypothesis cannot win (the reference rescores the previous pose, hypothesis 0 reads uninitialised memory)."""
    pr = synth.make_pnp_problem(13, 200, 0.6, "equirect")
    s = _inlier_sets(pr, 2)
    pr["bearings"] = pr["bearings"].copy()
    bad = int(np.flatnonzero(~pr["gt_inlier"])[0])
    pr["bearings"][bad] = [1.0, 0.0, 0.0]
    nan_set = np.array([bad, s[0][1], s[0][2], s[0][3]], np.int32)
    _, _, err, wrote = O.compute_pose(pr["bearings"][nan_set], pr["points"][nan_set], 10)
    assert not wrote and not err < np.finfo(float).max
    r = O.pnp_ransac(_prob(pr), np.stack([nan_set, s[1], nan_set]))
    assert r["valid"] and r["best_iter"] == 1
    r0 = O.pnp_ransac(_prob(pr), np.stack([nan_set]))
    assert not r0["valid"]


def test_ransac_recompute():
    pr = synth.make_pnp_problem(14, 300, 0.5, "perspective")
    ms = _inlier_sets(pr, 30)
    off = O.pnp_ransac(_prob(pr, recompute=False), ms)
    on = O.pnp_ransac(_prob(pr, recompute=True), ms)
    assert off["valid"] and on["valid"]
    for k in ("best_iter", "num_inliers", "min_cost"):
        assert off[k] == on[k]
    np.testing.assert_array_equal(off["inlier_flags"], on["inlier_flags"])  # the flags stay those of the best hypothesis
    f = off["inlier_flags"]
    R, t, _, _ = O.compute_pose(pr["bearings"][f], pr["points"][f], 10)
    np.testing.assert_array_equal(on["rot_cw"], R)
    np.testing.assert_array_equal(on["trans_cw"], t)
    assert not np.array_equal(on["rot_cw"], off["rot_cw"])
    np.testing.assert_allclose(on["rot_cw"], pr["gt_rot_cw"], atol=1e-3)


def test_ransac_early_return_draws_nothing():
    """n < 4 or n < min_num_inliers: find_via_ransac returns before touching the engine."""
    from stella_vslam_b200 import solve
    pr = synth.make_pnp_problem(15, 8, 1.0)
    s = solve.pnp_solver(pr["bearings"], pr["octaves"], pr["points"], pr["scale_factors"], use_fixed_seed=True)
    before = bytes(s.random_engine_)
    s.find_via_ransac(30, False)
    assert not s.solution_is_valid() and bytes(s.random_engine_) == before
    assert not O.pnp_ransac(_prob(pr), np.zeros((0, 4)))["valid"]


def test_max_cos_errors_use_util_cos():
    from oracle import pyoracle
    sf = synth.make_pnp_problem(0, 8)["scale_factors"]
    mine = O.max_cos_errors(sf, np.arange(8))
    ref = np.array([pyoracle.lib().orc_util_cos(float(np.float32(np.float64(s) * (np.pi / 180.0)))) for s in sf], np.float32)
    np.testing.assert_array_equal(mine, ref)
    assert np.all(np.abs(mine - np.cos(np.deg2rad(sf.astype(np.float64)))) < 1e-3)


@pytest.mark.parametrize("model", ["perspective", "equirect"])
def test_no_inlier_decision_near_its_threshold(model):
    """The workloads keep every inlier decision of the winning pose at least 1e-12 from its threshold, so numpy-side checks decide
    the same way as the restatement."""
    from stella_vslam_b200 import solve
    for seed in range(4):
        pr = synth.make_pnp_problem(100 + seed, 500, 0.5, model)
        ms = solve.draw_min_sets(500, 30)
        r = O.pnp_ransac(_prob(pr, recompute=False), ms)
        assert r["valid"]
        pc = pr["points"] @ r["rot_cw"].T + r["trans_cw"]
        cosang = np.sum(pc * pr["bearings"], 1) / np.linalg.norm(pc, axis=1)
        mc = O.max_cos_errors(pr["scale_factors"], pr["octaves"]).astype(np.float64)
        assert np.min(np.abs(cosang - mc)) > 1e-12
        np.testing.assert_array_equal(r["inlier_flags"], cosang > mc)
