"""The method of tests/test_transform_precision_gpu.py pinned without a GPU: the reference system of tests/transform_reference.py
against the CPU oracle (tests/transform_oracle.c), its step readback, and the oracle's own steps judged by the GPU file's harness.

Measured (this file, on the GPU file's cases):
  - edge errors: the reference and the oracle agree to 1e-12 of the projection's magnitude;
  - Jacobian, per column group (rotation, translation, scale) as a fraction of the group's largest entry in the problem: the stencil
    at 1e-4 agrees with 3e-4 and 3e-5 to 1.8e-9 or better (the scale column at 3e-5; 7e-11 elsewhere).  g2o's delta-1e-9 difference (the oracle's, and the kernel's) is off by
    rotation 1.5e-7 .. 3e-7, translation 8e-7 .. 1.5e-6 and scale 7e-6 .. 3.5e-5 at units 1, and rotation 1.5e-7 .. 3e-7,
    translation 1.1e-9 .. 1.7e-9 and scale 7e-6 .. 3.5e-5 with every translation times 1e-3 (the translation columns grow by 1000,
    their noise does not);
  - step readback: Newton on pgo_oracle.exp recovers x to 4 u (1 + |t|) for theta from 1e-9 to 1e-1 and sigma on both sides of
    g2o's 1e-5 switch; g2o's log alone is off by 1.7e-7 relative at theta = 1e-3;
  - the oracle's round-2 steps (the control of the GPU file): omega_orc 2e-11 .. 2e-9 on the first steps at units 1e-3 and
    4e-9 .. 6e-8 at units 1, growing to 1e-6 .. 7e-4 on the later, converged steps at units 1 where the step is as small as the
    Jacobian noise; forward error at most 0.6 kappa_bound omega_orc.  Over all cases, 132 steps have omega_orc <= 1e-6;
  - the reference LM of round 1 ends within 1e-7 (tangent) of the oracle's round-1 state on outlier-free problems at units 1e-3,
    with the same iteration and trial counts."""
import numpy as np
import pytest
import scipy.linalg as sl
import scipy.optimize as so

import test_transform_precision_gpu as G
import transform_oracle as O
import transform_reference as R
from workloads import synth

MODELS = list(G.MODELS)


def _group_errors(A, J):
    """max |A - J| per column group (rotation, translation, scale) over the group's largest |J| in the problem."""
    out = []
    for g in (slice(0, 3), slice(3, 6), slice(6, 7)):
        out.append(float(np.abs(A[..., g] - J[..., g]).max() / np.abs(J[..., g]).max()))
    return out


@pytest.mark.parametrize("models", MODELS)
def test_edge_errors_match_oracle(models):
    pr = synth.make_sim3_pair(3, 60, models=G.MODELS[models], outlier_frac=0.3)
    S = pr["sim3_12"]
    e = R.errors(pr, R.mat(S))
    pcs = R.camera_points(pr)
    w = R.weights(pr)
    for i in range(len(pcs[0])):
        for s, (cam, obs) in enumerate(((pr["cam_1"], pr["obs_1"][i]), (pr["cam_2"], pr["obs_2"][i]))):
            eo, chi = O.transform_edge(S, s, pcs[s][i], cam, obs, w[i, s])
            assert np.abs(eo - e[i, s]).max() <= 1e-12 * np.abs(R.project(cam, pcs[s][i])).max()
            assert chi == pytest.approx(w[i, s] * (e[i, s] @ e[i, s]), rel=1e-12)


@pytest.mark.parametrize("f", G.UNITS)
@pytest.mark.parametrize("models", MODELS)
def test_jacobian_against_stencils_and_oracle(models, f):
    pr = R.scaled(synth.make_sim3_pair(3, 200, models=G.MODELS[models], outlier_frac=0.3), f)
    seam, pole = R.guard(pr, pr["sim3_12"])
    pr = R._subset(pr, ~(seam | pole))
    S = pr["sim3_12"]
    J = R.jacobian(pr, S)
    for d in (3e-4, 3e-5):
        assert max(_group_errors(R.jacobian(pr, S, delta=d), J)) <= 5e-9
    noise = _group_errors(R.oracle_jacobian(pr, S), J)
    print(f"{models} units {f:g}: oracle Jacobian noise rotation {noise[0]:.1e} translation {noise[1]:.1e} scale {noise[2]:.1e}")
    assert noise[0] <= 2e-6 and noise[2] <= 1e-4
    assert noise[1] <= (1e-4 if f == 1.0 else 1e-8)
    Jf = R.jacobian(pr, S, fix_scale=True)
    assert np.array_equal(Jf[..., 6], np.zeros_like(Jf[..., 6])) and np.array_equal(Jf[..., :6], J[..., :6])


@pytest.mark.parametrize("sigma", [0.0, 3e-6, 3e-5, -2e-2])
@pytest.mark.parametrize("theta", [1e-9, 1e-7, 3e-6, 2e-5, 1e-3, 4e-3, 1e-1])
def test_step_readback_round_trip(theta, sigma):
    rng = np.random.default_rng(int(1e6 * theta) + 7)
    S0 = synth.make_sim3_pair(5, 10)["sim3_12"]
    for t_scale in (1.0, 1e-3):
        g = np.array(S0)
        g[4:7] *= t_scale
        axis = rng.standard_normal(3)
        x = np.concatenate([theta * axis / np.linalg.norm(axis), theta * t_scale * rng.standard_normal(3), [sigma]])
        S1 = R.oplus(g, x)                                        # rounded to 8 doubles
        xr = R.read_step(g, S1)
        # g2o's (e^sigma - 1) / sigma loses u / |sigma| relative above its 1e-5 switch: the exp itself is that noisy
        tol = 4 * R.U * (1 + np.abs(g[4:7]).max()) + (np.abs(x[3:6]).max() * R.U / abs(sigma) if abs(sigma) >= 1e-5 else 0.0)
        assert np.abs(xr - x).max() <= tol, (np.abs(xr - x), tol)
        if sigma == 0.0:
            xf = R.read_step(g, S1, fix_scale=True)
            assert xf[6] == 0.0 and np.abs(xf - x).max() <= tol


def test_log_only_readback_fails_in_the_small_angle_branch():
    g = synth.make_sim3_pair(5, 10)["sim3_12"]
    x = np.array([1e-3, 0.0, 0.0, 1e-3, 0.0, 0.0, 0.0])
    S1 = R.oplus(g, x)
    assert np.abs(R.read_step(g, S1) - x).max() <= 4 * R.U * (1 + np.abs(g[4:7]).max())
    bad = np.abs(R.read_step(g, S1, log_only=True) - x).max() / 1e-3
    assert 1e-7 < bad < 1e-6, bad                                 # theta^2 / 6 = 1.7e-7


def test_oracle_steps_are_the_control():
    """The oracle's round-2 steps judged by the GPU file's harness on every case: the forward error is bounded by kappa_bound omega,
    the reported chi2 equals the reference's, and enough steps are sharp for the GPU file to judge."""
    sharp = 0
    for name in G.NAMES:
        for f in G.UNITS:
            pr = G.case(name, f)
            runs = G.oracle_runs(pr, range(G.K + 1))
            steps, skipped = G.round2_steps(pr, runs)
            for st in steps:
                J = st["J"]
                if name != "near_optimum":
                    assert J["forward"] <= G.FWD_C * J["kappa_bound"] * max(J["omega"], J["floor"]), (name, f, st["k"])
                assert abs(runs[st["k"]]["chi2"][1] / st["chi2"] - 1) <= G.CHI_TOL
                sharp += J["omega"] <= G.SHARP
            print(f"{name} units {f:g}: omega_orc {['%.1e' % s['J']['omega'] for s in steps]} skipped {skipped}")
            if f < 1.0 and name != "near_optimum":
                assert steps and steps[0]["J"]["omega"] <= G.SHARP, name
    print("sharp steps", sharp)
    assert sharp >= 120


@pytest.mark.parametrize("name", ["pp_clean", "ee_clean", "n10"])
def test_reference_round1_against_oracle(name):
    pr = G.case(name, 1e-3)
    ref = R.lm_round(pr, pr["sim3_12"], 5, None, pr["fix_scale"], G.CHI_SQ)
    orc = O.transform_optimize(pr, G.CHI_SQ, 0)
    assert not ref["failed"] and (orc["iterations"][0], orc["trials"][0]) == (ref["iterations"], ref["trials"])
    assert R.tangent_distance(orc["sim3_12"], ref["S"]) <= 1e-7
    assert abs(orc["lambda_init"][0] / ref["lambda_init"] - 1) <= 1e-8


@pytest.mark.parametrize("models", MODELS)
def test_gauss_newton_optimum_against_least_squares(models):
    # small noise and no outliers: every edge stays inside the Huber zone, so the robust cost is the plain weighted least squares
    pr = R.scaled(synth.make_sim3_pair(5, 80, models=G.MODELS[models], outlier_frac=0.0, pixel_sigma=0.2), 1e-3)
    S, chi = R.gauss_newton(pr, pr["sim3_12"])
    assert (R.edge_chi2(pr, S) < R.huber_delta(G.CHI_SQ) ** 2).all()
    M0 = R.mat(pr["gt_sim3_12"])
    sw = np.sqrt(R.weights(pr))[..., None]

    def resid(u):
        return (sw * R.errors(pr, sl.expm(R.hat(u)) @ M0)).ravel()

    sol = so.least_squares(resid, np.zeros(7), xtol=1e-15, ftol=1e-15, gtol=1e-15, method="lm")
    want = sl.expm(R.hat(sol.x)) @ M0
    got = R.mat(S)
    assert np.abs(got[:3, :3] - want[:3, :3]).max() <= 1e-8
    assert np.abs(got[:3, 3] - want[:3, 3]).max() <= 1e-8 * R.length_scale(pr)
    assert chi == pytest.approx(2 * sol.cost, rel=1e-9)


def test_cases_keep_off_the_seam_and_poles():
    for name in G.NAMES:
        for f in G.UNITS:
            pr = G.case(name, f)
            for S in (pr["sim3_12"], pr["gt_sim3_12"]):
                seam, pole = R.guard(pr, S, pr["fix_scale"])
                assert not seam.any() and not pole.any(), name
    # the seam and pole case keeps most of its 200 points near the seam and the poles
    assert len(G.case("seam_pole", 1.0)["obs_1"]) >= 380
