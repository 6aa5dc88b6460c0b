"""optimize::transform_optimizer without a GPU: the oracle's forward / backward reprojection edges against a numpy restatement, its
numeric Jacobian against an independent difference, its LM against scipy.optimize.least_squares, the noise-free recovery, the round-1
early return, gather_mutual_edges' skip rules, and the ctypes mirror of b200_transform_problem_t."""
import os

import numpy as np
import pytest
import scipy.linalg as sl
import scipy.optimize as so

import transform_oracle as O
import transform_reference as TR
import test_abi_layout as ABI
from workloads import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = [("perspective", "perspective"), ("equirect", "equirect"), ("perspective", "equirect")]


def _edges(pr):
    """(side, camera-frame point, camera, observation, inv_sigma_sq) of every edge, edge_12 then edge_21 per pair."""
    out = []
    for i in range(len(pr["obs_1"])):
        out.append((0, pr["rot_2w"] @ pr["pos_w_2"][i] + pr["trans_2w"], pr["cam_1"], pr["obs_1"][i], pr["inv_sigma_sq_1"][i]))
        out.append((1, pr["rot_1w"] @ pr["pos_w_1"][i] + pr["trans_1w"], pr["cam_2"], pr["obs_2"][i], pr["inv_sigma_sq_2"][i]))
    return out


@pytest.mark.parametrize("models", MODELS)
def test_edge_errors_match_numpy(models):
    pr = synth.make_sim3_pair(3, 40, models=models, outlier_frac=0.2)
    M = TR.mat(pr["sim3_12"])
    for side, pc, cam, obs, w in _edges(pr):
        e, chi = O.transform_edge(pr["sim3_12"], side, pc, cam, obs, w)
        want = TR.np_error(M, side, pc, cam, obs)
        np.testing.assert_allclose(e, want, rtol=0, atol=1e-9 * max(1.0, np.abs(TR.project(cam, pc)).max()))
        assert chi == pytest.approx(float(w) * (e @ e), rel=1e-14)


@pytest.mark.parametrize("models", MODELS)
@pytest.mark.parametrize("fix_scale", [False, True])
def test_numeric_jacobian_matches_independent_difference(models, fix_scale):
    pr = synth.make_sim3_pair(4, 12, models=models, fix_scale=fix_scale, outlier_frac=0.0)
    S = pr["sim3_12"]
    for side, pc, cam, obs, w in _edges(pr):
        J = O.transform_jacobian(S, side, pc, cam, obs, w, fix_scale)
        Jr = np.zeros((2, 7))
        for d in range(6 if fix_scale else 7):
            du = np.zeros(7)
            du[d] = 1e-6
            fp = TR.np_error(sl.expm(TR.hat(du)) @ TR.mat(S), side, pc, cam, obs)
            fm = TR.np_error(sl.expm(TR.hat(-du)) @ TR.mat(S), side, pc, cam, obs)
            Jr[:, d] = (fp - fm) / 2e-6
        np.testing.assert_allclose(J, Jr, rtol=0, atol=2e-4 * max(1.0, np.abs(Jr).max()))
        if fix_scale:
            assert np.array_equal(J[:, 6], np.zeros(2))


@pytest.mark.parametrize("models", MODELS)
def test_lm_optimum_matches_least_squares(models):
    # small noise, no outliers: every edge stays inside the Huber zone, so both rounds minimise the plain weighted least squares
    pr = synth.make_sim3_pair(5, 60, models=models, outlier_frac=0.0, pixel_sigma=0.2)
    ref = O.transform_optimize(pr, 10.0, num_iter=50)
    assert ref["n_outliers_round1"] == 0 and ref["num_inliers"] == 60
    S0 = TR.mat(pr["sim3_12"])
    edges = _edges(pr)

    def resid(u):
        M = sl.expm(TR.hat(u)) @ S0
        return np.concatenate([np.sqrt(float(w)) * TR.np_error(M, side, pc, cam, obs) for side, pc, cam, obs, w in edges])

    sol = so.least_squares(resid, np.zeros(7), xtol=1e-15, ftol=1e-15, gtol=1e-15, method="lm")
    assert 2 * sol.cost < 10.0 * len(edges) * 0.1          # well inside the Huber zone on average
    assert max(float(w) * (r @ r) for (_, _, _, _, w), r in zip(edges, resid(sol.x).reshape(-1, 2))) < 10.0
    want = sl.expm(TR.hat(sol.x)) @ S0
    np.testing.assert_allclose(TR.mat(ref["sim3_12"]), want, rtol=0, atol=1e-6 * max(1.0, np.abs(want).max()))


def _noise_free(pr):
    """Points back-projected from the (float) observations through the true Sim3, so every edge's error at the truth is rounding."""
    pr = dict(pr)
    gt = TR.mat(pr["gt_sim3_12"])
    for side, obs_key, pos_key, cam_key, R_key, t_key, M in ((0, "obs_1", "pos_w_2", "cam_1", "rot_2w", "trans_2w", np.linalg.inv(gt)),
                                                             (1, "obs_2", "pos_w_1", "cam_2", "rot_1w", "trans_1w", gt)):
        cam = pr[cam_key]
        assert cam["model"] == 0
        R, t = pr[R_key], pr[t_key]
        pts = []
        for o, pw in zip(pr[obs_key].astype(np.float64), pr[pos_key]):
            # depth of the point in the frame whose camera observes it, then the ray through the observation
            z = (np.linalg.inv(M) @ np.append(R @ pw + t, 1.0))[2]
            p_obs = np.array([(o[0] - cam["cx"]) / cam["fx"] * z, (o[1] - cam["cy"]) / cam["fy"] * z, z])
            pc = (M @ np.append(p_obs, 1.0))[:3]
            pts.append(R.T @ (pc - t))
        pr[pos_key] = np.array(pts)
    return pr


@pytest.mark.parametrize("fix_scale", [False, True])
def test_noise_free_recovers_truth(fix_scale):
    pr = _noise_free(synth.make_sim3_pair(6, 80, fix_scale=fix_scale, outlier_frac=0.0, pixel_sigma=0.0))
    r = O.transform_optimize(pr, 10.0, num_iter=20)
    assert r["num_inliers"] == 80
    gt = pr["gt_sim3_12"]
    q = r["sim3_12"][:4] * np.sign(r["sim3_12"][3] * gt[3])
    np.testing.assert_allclose(q, gt[:4], rtol=0, atol=1e-9)
    np.testing.assert_allclose(r["sim3_12"][4:], gt[4:], rtol=0, atol=1e-9 * max(1.0, np.abs(gt[4:7]).max()))
    if fix_scale:
        assert r["sim3_12"][7] == pr["sim3_12"][7]


def test_round1_early_return_keeps_input_and_flags():
    pr = synth.make_sim3_pair(7, 14, outlier_frac=0.0, pixel_sigma=0.5)
    bad = np.arange(14) < 6                                      # 6 gross outliers leave 8 < 10 survivors
    pr["obs_1"] = pr["obs_1"].copy()
    pr["obs_1"][bad] += 200.0
    r = O.transform_optimize(pr)
    assert r["num_inliers"] == 0 and r["iterations"] == [5, 0] and r["trials"][1] == 0
    assert np.array_equal(r["sim3_12"], pr["sim3_12"])
    assert np.array_equal(r["keep"], (~bad).astype(np.uint8)) and r["n_outliers_round1"] == 6


def test_zero_matches_returns_zero():
    pr = synth.make_sim3_pair(8, 10)
    for k in ("obs_1", "inv_sigma_sq_1", "pos_w_2", "obs_2", "inv_sigma_sq_2", "pos_w_1"):
        pr[k] = pr[k][:0]
    r = O.transform_optimize(pr)
    assert r["num_inliers"] == 0 and r["iterations"] == [0, 0] and np.array_equal(r["sim3_12"], pr["sim3_12"])


def _keyframes():
    cam = dict(model=0, fx=500.0, fy=500.0, cx=320.0, cy=240.0, fxb=0.0, cols=640.0, rows=480.0)
    lm = lambda i, obs, erased=False: dict(pos_w=np.array([0.1 * i, -0.05 * i, 5.0 + i]), will_be_erased=erased, observations=obs)
    kf1 = dict(id=1, rot_cw=np.eye(3), trans_cw=np.zeros(3), camera=cam, undist_keypts=np.arange(16, dtype=np.float32).reshape(8, 2),
               octaves=np.array([0, 1, 2, 3, 0, 1, 2, 3]), inv_level_sigma_sq=[1.0, 0.5, 0.25, 0.125])
    kf2 = dict(id=2, rot_cw=np.eye(3), trans_cw=np.array([0.3, 0, 0]), camera=cam,
               undist_keypts=100 + np.arange(16, dtype=np.float32).reshape(8, 2), octaves=np.array([3, 2, 1, 0, 3, 2, 1, 0]),
               inv_level_sigma_sq=[1.0, 0.5, 0.25, 0.125])
    kf1["landmarks"] = [lm(0, {1: 0}), None, lm(2, {1: 2}), lm(3, {1: 3}, erased=True), lm(4, {1: 4}), lm(5, {1: 5}), lm(6, {1: 6}), lm(7, {1: 7})]
    matched = [lm(10, {2: 5}),              # kept: idx2 5
               lm(11, {2: 1}),              # keyframe 1 has no landmark at idx1 1
               None,                        # no match
               lm(13, {2: 3}),              # lm_1 will be erased
               lm(14, {2: 4}, erased=True),  # lm_2 will be erased
               lm(15, {3: 0}),              # lm_2 not observed in keyframe 2
               lm(16, {2: -1}),             # negative index
               lm(17, {2: 7})]              # kept: idx2 7
    return kf1, kf2, matched


def test_gather_mutual_edges_skip_rules():
    from stella_vslam_b200.optimize import gather_mutual_edges
    kf1, kf2, matched = _keyframes()
    pr, idx1 = gather_mutual_edges(kf1, kf2, matched)
    assert list(idx1) == [0, 7] and pr["n_matches"] == 2
    np.testing.assert_array_equal(pr["obs_1"], kf1["undist_keypts"][[0, 7]])
    np.testing.assert_array_equal(pr["obs_2"], kf2["undist_keypts"][[5, 7]])
    np.testing.assert_array_equal(pr["inv_sigma_sq_1"], np.float32([1.0, 0.125]))
    np.testing.assert_array_equal(pr["inv_sigma_sq_2"], np.float32([0.25, 1.0]))
    np.testing.assert_array_equal(pr["pos_w_1"], np.array([kf1["landmarks"][0]["pos_w"], kf1["landmarks"][7]["pos_w"]]))
    np.testing.assert_array_equal(pr["pos_w_2"], np.array([matched[0]["pos_w"], matched[7]["pos_w"]]))


def test_ctypes_mirror_matches_the_header(tmp_path):
    from stella_vslam_b200 import optimize
    ABI._check(tmp_path, os.path.join(ROOT, "include"), "b200vslam.h", {"b200_transform_problem_t": optimize.TransformProblem})
