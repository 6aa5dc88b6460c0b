"""GPU parity: b200_pnp_ransac / b200_epnp_compute_pose (solve::pnp_solver) against the CPU restatement, bit for bit, and the
relocalisation chain PnP -> pose optimisation on a synthetic lost frame."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pnp_oracle as O  # noqa: E402

from workloads import synth  # noqa: E402

pytestmark = pytest.mark.gpu


def _problem(seed, n, model, recompute, case=None, inlier_frac=None, max_num_iter=30):
    from stella_vslam_b200 import solve
    rng = np.random.default_rng(seed)
    frac = rng.uniform(0.2, 0.8) if inlier_frac is None else inlier_frac
    pr = synth.make_pnp_problem(seed, n, frac, model, case=case)
    d = dict(bearings=pr["bearings"], points=pr["points"], octaves=pr["octaves"], scale_factors=pr["scale_factors"], recompute=recompute,
             min_num_inliers=10, gauss_newton_num_iter=10)
    d["min_sets"] = solve.draw_min_sets(n, max_num_iter, solve.mt19937((seed,))) if n >= 4 else np.zeros((0, 4), np.int32)
    return d


def _assert_same(dev, ref, n, min_num_inliers):
    assert dev["status"] == ref["status"] == 0
    assert dev["valid"] == ref["valid"]
    assert dev["best_iter"] == ref["best_iter"]
    assert dev["num_inliers"] == ref["num_inliers"]
    assert dev["min_cost"] == ref["min_cost"]
    if n < 4 or n < min_num_inliers:  # returned before drawing: the flags are not touched
        assert dev["inlier_flags"] is None
        return
    np.testing.assert_array_equal(dev["inlier_flags"], ref["inlier_flags"])
    if ref["valid"]:
        assert np.array_equal(dev["rot_cw"], ref["rot_cw"]) and np.array_equal(dev["trans_cw"], ref["trans_cw"])


def _check_batch(problems):
    from stella_vslam_b200 import solve
    dev = solve.pnp_ransac_batch(problems)
    for d, pr in zip(dev, problems):
        _assert_same(d, O.pnp_ransac(pr, pr["min_sets"]), len(pr["bearings"]), pr["min_num_inliers"])
    return dev


@pytest.mark.parametrize("model", ["perspective", "equirect"])
@pytest.mark.parametrize("recompute", [False, True])
def test_single_problem_bit_identical(model, recompute):
    dev = _check_batch([_problem(1, 300, model, recompute)])
    assert dev[0]["valid"]


@pytest.mark.parametrize("case", ["coplanar", "min_inliers"])
def test_special_cases(case):
    probs = [_problem(2, 200, m, rc, case=case, inlier_frac=0.0 if case == "min_inliers" else 0.6) for m in ("perspective", "equirect")
             for rc in (False, True)]
    for p in probs:  # min_inliers: 10 true inliers with the default min_num_inliers 10 -> never valid; 9 -> may be
        p2 = dict(p, min_num_inliers=9)
        _check_batch([p, p2])


def test_small_and_degenerate_sizes():
    probs = [_problem(3 + n, n, "perspective", True) for n in (0, 2, 3, 4, 9, 10, 11)]
    probs += [dict(_problem(20, 4, "equirect", False), min_num_inliers=2), dict(_problem(21, 6, "perspective", True), min_num_inliers=3)]
    probs += [dict(_problem(22, 50, "perspective", True), min_sets=np.zeros((0, 4), np.int32))]  # max_num_iter 0: all flags false
    dev = _check_batch(probs)
    assert not dev[-1]["valid"] and not dev[-1]["inlier_flags"].any()


def test_batch_of_1024_bit_identical():
    rng = np.random.default_rng(7)
    ns = rng.integers(4, 2001, 1024)
    ns[:4] = [4, 2000, 10, 11]
    probs = [_problem(1000 + i, int(n), "equirect" if i % 3 == 0 else "perspective", bool(i % 2)) for i, n in enumerate(ns)]
    dev = _check_batch(probs)
    assert sum(d["valid"] for d in dev) > 900


def test_duplicated_minimal_sets_first_wins():
    p = _problem(30, 400, "perspective", False)
    p["min_sets"] = np.repeat(p["min_sets"][:3], 4, axis=0)
    dev = _check_batch([p])[0]
    assert dev["valid"] and dev["best_iter"] % 4 == 0


def test_hypotheses_without_pose_bit_identical():
    """A bearing with z = 0 makes every reprojection error of a minimal set that contains it NaN: compute_pose writes no pose and the
    hypothesis is rejected, at index 0 (where the reference reads uninitialised memory) and later."""
    probs = []
    for seed, model, recompute in [(90, "equirect", False), (91, "equirect", True), (92, "perspective", False)]:
        p = _problem(seed, 300, model, recompute)
        p["bearings"] = np.array(p["bearings"], copy=True)
        bad = 7
        p["bearings"][bad] = [1.0, 0.0, 0.0]
        ms = np.array(p["min_sets"], copy=True)
        for it in (0, 5, 6, 29):
            ms[it] = [bad] + [v for v in ms[it] if v != bad][:3] if bad in ms[it] else [bad, *ms[it][1:]]
        p["min_sets"] = ms
        _, _, _, wrote = O.compute_pose(p["bearings"][ms[0]], p["points"][ms[0]], 10)
        assert not wrote
        probs.append(p)
    only_bad = dict(probs[0], min_sets=probs[0]["min_sets"][[0, 5]])  # no hypothesis writes a pose: invalid
    dev = _check_batch(probs + [only_bad])
    assert all(d["best_iter"] not in (0, 5, 6, 29) for d in dev[:3]) and not dev[-1]["valid"]


def test_compute_pose_bit_identical():
    from stella_vslam_b200 import solve
    probs = []
    for i, (n, model) in enumerate([(4, "perspective"), (5, "equirect"), (6, "perspective"), (300, "perspective"), (2000, "equirect"),
                                    (1, "perspective"), (40, "perspective")]):
        pr = synth.make_pnp_problem(40 + i, n, 0.7, model)
        probs.append(dict(bearings=pr["bearings"], points=pr["points"], num_iter=5 if i % 2 else 10, rot_cw=np.eye(3) * 2, trans_cw=np.ones(3)))
    bad = synth.make_pnp_problem(50, 5, 1.0, "equirect")
    bad["bearings"][0] = [1.0, 0.0, 0.0]  # NaN reprojection errors: nothing written, the given pose stays
    probs.append(dict(bearings=bad["bearings"], points=bad["points"], num_iter=10, rot_cw=np.eye(3) * 3, trans_cw=np.ones(3) * 5))
    dev = solve.compute_pose_batch(probs)
    for d, p in zip(dev, probs):
        R, t, err, wrote = O.compute_pose(p["bearings"], p["points"], p["num_iter"], p["rot_cw"], p["trans_cw"])
        assert d["status"] == 0 and d["wrote"] == wrote
        assert np.array_equal(d["rot_cw"], R) and np.array_equal(d["trans_cw"], t)
        assert d["reproj_error"] == err or (np.isnan(err) and np.isnan(d["reproj_error"]))
    assert not dev[-1]["wrote"] and np.array_equal(dev[-1]["rot_cw"], np.eye(3) * 3)


def test_solver_class_matches_restatement():
    from stella_vslam_b200 import solve
    pr = synth.make_pnp_problem(60, 500, 0.4, "perspective")
    s = solve.pnp_solver(pr["bearings"], pr["octaves"], pr["points"], pr["scale_factors"], use_fixed_seed=True)
    s.find_via_ransac(30, True)
    s.find_via_ransac(30, False)  # the second call continues the engine
    sets = solve.draw_min_sets(500, 60)[30:]
    ref = O.pnp_ransac(dict(bearings=pr["bearings"], points=pr["points"], octaves=pr["octaves"], scale_factors=pr["scale_factors"],
                            recompute=False), sets)
    assert s.solution_is_valid() == ref["valid"] is True
    assert np.array_equal(s.get_best_rotation(), ref["rot_cw"]) and np.array_equal(s.get_best_translation(), ref["trans_cw"])
    assert s.get_inlier_flags() == list(ref["inlier_flags"])
    np.testing.assert_allclose(s.get_best_rotation(), pr["gt_rot_cw"], atol=5e-2)  # a minimal-set pose: no recompute


def test_invalid_input_writes_nothing():
    from stella_vslam_b200 import _lib, solve
    base = _problem(70, 100, "perspective", True)
    for bad in (dict(octaves=np.full(100, 8, np.int32)), dict(min_sets=np.full((30, 4), 100, np.int32)),
                dict(min_sets=np.full((30, 4), -1, np.int32))):
        keep = []
        S, fl = solve._pack(dict(base, **bad), keep)
        fl[:] = 7
        S.valid, S.best_iter = 5, 5
        arr = (solve.PnpProblem * 1)(S)
        rc = solve._L().b200_pnp_ransac(solve._handle(0), 1, arr)
        assert rc == _lib.ERR_INVALID
        assert arr[0].valid == 5 and arr[0].best_iter == 5 and np.all(fl == 7)
    arr = (solve.EpnpProblem * 1)()
    arr[0].n = 0
    assert solve._L().b200_epnp_compute_pose(solve._handle(0), 1, arr) == _lib.ERR_INVALID
    assert solve._L().b200_pnp_ransac(solve._handle(0), -1, None) == _lib.ERR_INVALID


def test_relocalisation_chain_recovers_the_pose():
    """A lost frame: PnP (find_via_ransac(30, false) as the relocalizer runs it) on its 2D-3D matches, then pose_optimizer on the
    matches PnP kept, from the PnP pose.  The result is the true pose within the pose optimiser's accuracy."""
    from stella_vslam_b200 import optimize, solve
    fr = synth.make_pose_problem(seed=5, n_obs=800, model="mono", outlier_frac=0.2)
    cam = fr["cams"][0]
    xy = fr["e_obs"][:, :2].astype(np.float64)
    b = np.stack([(xy[:, 0] - cam["cx"]) / cam["fx"], (xy[:, 1] - cam["cy"]) / cam["fy"], np.ones(len(xy))], 1)
    b /= np.linalg.norm(b, axis=1, keepdims=True)
    sf = np.cumprod(np.concatenate([[np.float32(1.0)], np.full(7, np.float32(1.2))])).astype(np.float32)
    octave = np.rint(np.log(1.0 / np.sqrt(fr["e_inv_sigma_sq"].astype(np.float64))) / np.log(1.2)).astype(np.int32)  # 1 / sf^2
    assert octave.min() >= 0 and octave.max() <= 7
    s = solve.pnp_solver(b, octave, fr["points"], sf, use_fixed_seed=True)
    s.find_via_ransac(30, False)
    assert s.solution_is_valid()
    keep = np.array(s.get_inlier_flags())
    sub = dict(fr)
    sub["pose_cw"] = s.get_best_cam_pose()[None]
    for k in ("e_pose", "e_point", "e_cam", "e_obs", "e_inv_sigma_sq", "e_delta"):
        sub[k] = fr[k][keep]
    n_valid, pose, _ = optimize.pose_optimizer().optimize(sub)
    gt = fr["gt_pose_cw"]
    assert n_valid > 0.5 * keep.sum()
    dR = pose[:3, :3] @ gt[:3, :3].T
    assert np.arccos(np.clip((np.trace(dR) - 1) / 2, -1, 1)) < np.deg2rad(0.2)
    assert np.linalg.norm(pose[:3, 3] - gt[:3, 3]) < 0.05
