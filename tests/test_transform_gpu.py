"""optimize::transform_optimizer on the GPU (b200_transform_optimize) against the CPU oracle (tests/transform_oracle.c): perspective,
equirectangular and mixed pairs, with and without fix_scale, with gross outliers; batch independence, run-to-run identity on a handle
shared with the pose optimiser and PnP, the 0 / 9 / 10-pair boundaries and rejected input."""
import numpy as np
import pytest

import transform_oracle as O
from workloads import synth

CHI_SQ = 10.0
CASES = [(m, fs, of, seed) for seed, (m, of) in enumerate([(("perspective", "perspective"), 0.1), (("equirect", "equirect"), 0.2),
                                                          (("perspective", "equirect"), 0.3), (("equirect", "perspective"), 0.15)])
         for fs in (False, True)]


def _compare(got, ref, pr, num_iter=10, sim3_tol=1e-6):
    """The device result against the oracle's: Sim3 1e-6 relative (1e-5 after a stagnated round), chi2 1e-6, flags and counts equal; iterations where neither side's
    round ended in a failed LM step (after one, the trial sequences depend on the last bits of chi2).  lambda_init of round 1 with
    perspective cameras only is linearised at the caller's Sim3 with correctly rounded operations and agrees to 1e-9.  With an
    equirectangular camera (atan2, asin) and in round 2 (after five LM steps through exp's sin and cos) CUDA's libm and glibc differ by
    an ulp, which the 1e-9 central difference amplifies about 5e8 times: 1e-6 there."""
    g, r = got["sim3_12"], ref["sim3_12"]
    # a round that stagnated (an LM step failed on either side) stops wherever the last bits of chi2 stopped it: 1e-5 there
    stalled = any(ref["failed_at"][k] >= 0 or got["iterations"][k] < (5, num_iter)[k] for k in range(2) if ref["iterations"][k] > 0)
    tol = 1e-5 if stalled else sim3_tol
    np.testing.assert_allclose(g[:4] * np.sign(g[3] * r[3]), r[:4], rtol=0, atol=tol)
    np.testing.assert_allclose(g[4:7], r[4:7], rtol=0, atol=tol * max(1.0, np.abs(r[4:7]).max()))
    assert abs(g[7] - r[7]) <= tol * abs(r[7])
    for k in range(2):
        assert abs(got["chi2"][k] - ref["chi2"][k]) <= 1e-6 * max(1.0, abs(ref["chi2"][k])), (k, got["chi2"], ref["chi2"])
        tol = 1e-9 if k == 0 and pr["cam_1"]["model"] == 0 and pr["cam_2"]["model"] == 0 else 1e-6
        assert abs(got["lambda_init"][k] - ref["lambda_init"][k]) <= tol * abs(ref["lambda_init"][k]), (k, got["lambda_init"], ref["lambda_init"])
        if ref["failed_at"][k] < 0 and got["iterations"][k] == (5, num_iter)[k]:
            assert got["iterations"][k] == ref["iterations"][k], (k, got["iterations"], ref["iterations"])
    assert got["n_outliers_round1"] == ref["n_outliers_round1"]
    assert np.array_equal(got["keep"], ref["keep"]) and got["num_inliers"] == ref["num_inliers"]


@pytest.mark.gpu
@pytest.mark.parametrize("models,fix_scale,outlier_frac,seed", CASES)
def test_vs_oracle(models, fix_scale, outlier_frac, seed):
    from stella_vslam_b200 import optimize
    pr = synth.make_sim3_pair(100 + seed, 300, models=models, fix_scale=fix_scale, outlier_frac=outlier_frac)
    got = optimize.transform_optimizer(fix_scale).optimize(pr, CHI_SQ)
    ref = O.transform_optimize(pr, CHI_SQ, 10)
    _compare(got, ref, pr)
    assert got["num_inliers"] >= 0.6 * 300 and not (got["keep"].astype(bool) & pr["gt_outlier"]).any()
    if fix_scale:
        assert got["sim3_12"][7] == pr["sim3_12"][7]


def _mixed_batch(n_problems, seed=0):
    rng = np.random.default_rng(seed)
    models = [("perspective", "perspective"), ("equirect", "equirect"), ("perspective", "equirect"), ("equirect", "perspective")]
    return [synth.make_sim3_pair(int(rng.integers(1 << 30)), int(rng.integers(20, 1001)), models=models[k % 4], fix_scale=False,
                                 outlier_frac=float(rng.uniform(0.1, 0.3))) for k in range(n_problems)]


def _same(a, b):
    for k in ("sim3_12", "keep", "chi2", "lambda_init"):
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k
    for k in ("num_inliers", "n_outliers_round1", "iterations", "trials"):
        assert a[k] == b[k], k


@pytest.mark.gpu
def test_batch_equals_single_and_runs_are_identical():
    from stella_vslam_b200 import optimize
    probs = _mixed_batch(1024)
    opt = optimize.transform_optimizer(False)
    batch = opt.optimize_batch(probs, CHI_SQ)
    again = opt.optimize_batch(probs, CHI_SQ)
    for a, b in zip(batch, again):
        _same(a, b)
    for pr, b in zip(probs, batch):
        _same(opt.optimize(pr, CHI_SQ), b)


@pytest.mark.gpu
def test_small_mixed_batch_vs_oracle():
    from stella_vslam_b200 import optimize
    probs = _mixed_batch(8, seed=3)
    # ten iterations leave some of these free-scale problems short of convergence (the scale still moves by ~1e-6 per iteration),
    # and the ~1e-8 Jacobian noise of the equirectangular edges then shifts where they stop: 1e-5 on the Sim3 here
    for pr, got in zip(probs, optimize.transform_optimizer(False).optimize_batch(probs, CHI_SQ)):
        _compare(got, O.transform_optimize(pr, CHI_SQ, 10), pr, sim3_tol=1e-5)


@pytest.mark.gpu
def test_handle_shared_with_pose_optimizer_and_pnp():
    from stella_vslam_b200 import optimize, solve
    probs = _mixed_batch(16, seed=5)
    r1 = optimize.transform_optimizer(False).optimize_batch(probs, CHI_SQ)     # a fresh handle
    h = solve._handle(0)                                                      # a handle after a pose optimisation and a PnP RANSAC
    L = optimize._bind()
    pp = synth.make_pose_problem(1, n_obs=400, model="stereo")
    P, keep = optimize.pack_problem(pp)
    assert L.b200_pose_optimize(h, 1, optimize.C.byref(P), 2, 2, 10, optimize.ptr(np.zeros((1, 4, 4))), optimize.ptr(np.zeros(400, np.uint8)),
                                optimize.ptr(np.zeros(1, np.uint32))) == 0
    pnp = synth.make_pnp_problem(80, 300, 0.5, "perspective")
    solve.pnp_solver(pnp["bearings"], pnp["octaves"], pnp["points"], pnp["scale_factors"], use_fixed_seed=True).find_via_ransac(30, True)
    packed = [optimize.pack_transform_problem(pr, False) for pr in probs]
    arr = (optimize.TransformProblem * len(packed))(*[pk[0] for pk in packed])
    assert L.b200_transform_optimize(h, len(packed), arr, CHI_SQ, 10) == 0
    for i, pk in enumerate(packed):
        _same(optimize._transform_result(arr[i], pk[1]), r1[i])


@pytest.mark.gpu
@pytest.mark.parametrize("n", [0, 9, 10])
@pytest.mark.parametrize("fix_scale", [False, True])
def test_match_count_boundaries(n, fix_scale):
    from stella_vslam_b200 import optimize
    pr = synth.make_sim3_pair(40 + n, max(n, 1), fix_scale=fix_scale, outlier_frac=0.0, pixel_sigma=0.5)
    for k in ("obs_1", "inv_sigma_sq_1", "pos_w_2", "obs_2", "inv_sigma_sq_2", "pos_w_1"):
        pr[k] = pr[k][:n]
    got = optimize.transform_optimizer(fix_scale).optimize(pr, CHI_SQ)
    ref = O.transform_optimize(pr, CHI_SQ, 10)
    _compare(got, ref, pr)
    if n < 10:
        assert got["num_inliers"] == 0 and got["iterations"][1] == 0 and np.array_equal(got["sim3_12"], pr["sim3_12"])
    else:
        assert got["num_inliers"] == 10 and got["iterations"][1] > 0


@pytest.mark.gpu
def test_invalid_input_writes_nothing():
    from stella_vslam_b200 import _lib, optimize
    good = synth.make_sim3_pair(9, 30)
    bad = []
    s = good["sim3_12"].copy(); s[7] = 0.0; bad.append(dict(good, sim3_12=s))
    s = good["sim3_12"].copy(); s[:4] *= 3.0; bad.append(dict(good, sim3_12=s))
    s = good["sim3_12"].copy(); s[5] = np.nan; bad.append(dict(good, sim3_12=s))
    bad.append(dict(good, cam_1=dict(good["cam_1"], model=2)))
    w = good["inv_sigma_sq_2"].copy(); w[3] = 0.0; bad.append(dict(good, inv_sigma_sq_2=w))
    p = good["pos_w_1"].copy(); p[2, 1] = np.inf; bad.append(dict(good, pos_w_1=p))
    o = good["obs_1"].copy(); o[4, 0] = np.nan; bad.append(dict(good, obs_1=o))
    R = good["rot_2w"].copy(); R[1, 1] = np.nan; bad.append(dict(good, rot_2w=R))
    opt = optimize.transform_optimizer(False)
    for pr in bad:
        packed = [optimize.pack_transform_problem(good, False), optimize.pack_transform_problem(pr, False)]
        arr = (optimize.TransformProblem * 2)(*[pk[0] for pk in packed])
        for i, pk in enumerate(packed):
            pk[1]["keep"][...] = 7
            arr[i].keep = pk[1]["keep"].ctypes.data
            arr[i].num_inliers = 12345
        assert opt._L.b200_transform_optimize(opt._h, 2, arr, CHI_SQ, 10) == _lib.ERR_INVALID
        for i, pk in enumerate(packed):
            assert (pk[1]["keep"] == 7).all() and arr[i].num_inliers == 12345
    arr = (optimize.TransformProblem * 1)(optimize.pack_transform_problem(good, False)[0])
    assert opt._L.b200_transform_optimize(opt._h, 1, arr, 0.0, 10) == _lib.ERR_INVALID
    assert opt._L.b200_transform_optimize(opt._h, 1, arr, CHI_SQ, -1) == _lib.ERR_INVALID
    assert opt._L.b200_transform_optimize(opt._h, -1, arr, CHI_SQ, 10) == _lib.ERR_INVALID
