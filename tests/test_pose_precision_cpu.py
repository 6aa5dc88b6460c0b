"""The method of tests/test_pose_precision_gpu.py, pinned without a GPU: the reference of tests/pose_reference.py judges the CPU oracle's
pose optimiser one LM step at a time.  The oracle solves its own 6x6 system exactly, so its step must sit at the readback floor
against the reference system at lambda_init = 1e-5 max diag(H_ref); the lambda of steps 2..5 must be the one the reference's rho
predicts; a round re-posed as a problem of its own must take the round's step; and the problem rebuilt from a tracking chain's outputs
must be the one the chain solved.  Otherwise the reference, not the device, would be what the GPU file judges."""
import numpy as np
import pytest

import ba_windows as BW
import lba_reference as R
import pose_reference as P
from oracle import pyoracle as O

# Without Huber a gross outlier can make the first trial fail (rho < 0, lambda doubled and the trial repeated), so the frames of
# the Huber-off cases carry none: in the protocol, the rounds without Huber come after the outliers have been classified out.
FRAMES = {
    "mono": lambda out=0.1: BW.make_frame(1, 300, "kitti", outlier_frac=out),
    "stereo": lambda out=0.1: BW.make_frame(2, 300, "kitti", stereo_frac=1.0, outlier_frac=out),
    "mixed": lambda out=0.3: BW.make_frame(3, 400, "kitti", stereo_frac=0.5, outlier_frac=out),
    # seam points lie 4-10 px (0.4-0.9 deg) from the +-pi seam: a start within 0.2 deg keeps them on their side
    "equirect_pole_seam": lambda out=0.1: BW.make_frame(4, 300, "equirect", n_pole=8, n_seam=8, outlier_frac=out, rot_deg=0.2, trans_m=0.02),
    "behind": lambda out=0.1: BW.make_frame(5, 300, "kitti", stereo_frac=0.5, n_behind=8, n_near=3, n_far=5, outlier_frac=out),
    "decoy_cams": lambda out=0.1: BW.make_frame(6, 300, "euroc", n_cams=3, cam_index=2, outlier_frac=out),
    # every point 0.3 m away: lambda_init's maximum is a translation entry of diag(H)
    "near_points": lambda out=0.1: BW.make_frame(9, 300, "kitti", n_near=300, outlier_frac=out, rot_deg=0.2, trans_m=0.005),
}


# The oracle solves its own system exactly, but forms it in float64 by its own formulas: on perspective frames its step sits within
# 4x the readback floor; the equirectangular Jacobians near a pole differ from the reference's by tens of ulps (measured up to 6.3x
# the floor), which the floor does not model.  A wrong lambda or a wrong H moves omega by orders of magnitude more.
FLOOR_C = 16


def _at_floor(J):
    assert J["omega"] <= FLOOR_C * max(J["floor"], P.ROUNDOFF), (J["omega"], J["floor"])
    assert J["forward"] <= J["kappa_bound"] * J["omega"], (J["forward"], J["kappa_bound"], J["omega"])


@pytest.mark.parametrize("huber", [True, False])
@pytest.mark.parametrize("name", list(FRAMES))
def test_oracle_first_step_at_readback_floor(name, huber):
    pr = FRAMES[name]() if huber else FRAMES[name](0.0)
    n, pose, flags = O.pose_optimize(pr, 1, 0, 1) if huber else O.pose_optimize(pr, 0, 1, 1)
    S = P.system(pr, robust=huber)
    lam = P.lambda_init(S)
    J = P.judge(S, lam, pose)
    print(f"{name} huber {huber}: omega {J['omega']:.2e} floor {J['floor']:.2e} kappa_bound {J['kappa_bound']:.2e} forward {J['forward']:.2e}")
    _at_floor(J)
    lam_next, rho = P.replay_lambda(S, lam, pose, pr)
    assert lam_next is not None and rho > 0
    P.check_flags(pr, pose, flags)
    assert n == (~flags).sum()


@pytest.mark.parametrize("name", ["mixed", "equirect_pole_seam"])
def test_replayed_lambda_of_later_steps(name):
    """Steps 2..5 of the first round, each judged at the lambda the reference's rho predicts from the step before: a wrong lambda would
    put the oracle's step far above the floor.  A gain-threshold stop shows as two equal states; nothing is judged beyond it."""
    pr = FRAMES[name]()
    prev = pr["pose_cw"][0]
    lam = None
    judged = 0
    for k in range(1, 6):
        _, pose, _ = O.pose_optimize(pr, 1, 0, k)
        if k > 1 and np.array_equal(pose, prev):
            break
        S = P.system(pr, prev)
        lam = P.lambda_init(S) if lam is None else lam
        J = P.judge(S, lam, pose)
        print(f"{name} step {k} lambda {lam:.3e}: omega {J['omega']:.2e} floor {J['floor']:.2e}")
        _at_floor(J)
        lam, rho = P.replay_lambda(S, lam, pose, pr)
        assert lam is not None, (k, rho)                         # the trial was accepted
        prev = pose
        judged += 1
    assert judged >= 3


def test_small_angle_readback():
    """exp_oplus / log_step across g2o's small-angle branch (theta < 1e-5): a step read back from the state it produced is the step,
    on both sides of the branch, the rotation's small error of the truncated series included."""
    rng = np.random.default_rng(0)
    T = BW.make_frame(7, 10)["pose_cw"][0]
    for th in (1e-7, 1e-6, 9.9e-6, 1.01e-5, 1e-3):
        d = np.concatenate([th * rng.standard_normal(3) / np.sqrt(3), 1e-3 * rng.standard_normal(3)])
        d[:3] *= th / np.linalg.norm(d[:3])
        back = R.log_step(R.exp_oplus(T, d), T)
        # I + O + O^2 / 2 normalised is a rotation by theta (1 - theta^2 / 6): the readback sees it, to the series' own error
        tol = 1e-12 + (th * th / 6 if th < 1e-5 else 0.0)
        assert np.abs(back - d).max() <= tol * np.abs(d).max() + 1e-16, (th, back - d)


@pytest.mark.parametrize("rnd", [2, 3, 4])
def test_reposed_round_takes_the_rounds_step(rnd):
    """Round rnd of the (2, 2) protocol with one iteration per round: the inliers of round rnd - 1 at its pose, as a problem of their
    own, take the same step as the continuing run, and the continuing run's flags follow the reference rule (outliers come back)."""
    pr = BW.make_frame(8, 600, "kitti", stereo_frac=0.5, outlier_frac=0.3, rot_deg=3.0, trans_m=0.3)
    _, pose0, flags0 = O.pose_optimize(pr, *P.protocol_prefix(rnd - 1, 2, 2), 1)
    P.check_flags(pr, pose0, flags0)
    _, pose1, flags1 = O.pose_optimize(pr, *P.protocol_prefix(rnd, 2, 2), 1)
    P.check_flags(pr, pose1, flags1)
    huber = P.robust_in_round(rnd - 1, 2, 2)
    assert huber == (rnd <= 2)
    rp = P.reposed(pr, pose0, flags0)
    _, pose_r, flags_r = O.pose_optimize(rp, 1, 0, 1) if huber else O.pose_optimize(rp, 0, 1, 1)
    S = P.system(rp, robust=huber)
    lam = P.lambda_init(S)
    Jc, Jr = P.judge(S, lam, pose1), P.judge(S, lam, pose_r)
    print(f"round {rnd}: {len(rp['e_pose'])} inliers, omega continuing {Jc['omega']:.2e} re-posed {Jr['omega']:.2e} floor {Jr['floor']:.2e}")
    _at_floor(Jr)
    # the continuing run steps from its quaternion, not from the matrix it exported: the same step to the rounding of that state
    assert R.rel(Jc["x"], Jr["x"]) <= 1e-9, R.rel(Jc["x"], Jr["x"])
    assert np.array_equal(flags_r, flags1[~flags0])


def _orb_frame(stereo_cam, seed):
    from stella_vslam_b200 import feature
    from workloads import synth
    img = synth.make_frame(1241, 376, seed=seed)
    r = O.orb_extract(img, min_area=800)
    prm = feature.orb_params()
    fr = synth.make_tracking_frame(r["kps"], r["desc"], stereo_cam, prm.scale_factors_, seed=seed + 20, stereo=True)
    return r, fr, prm


def test_chain_rebuild_reproduces_track_local_map():
    """A KITTI stereo frame where a fifth of the keypoints have no x_right: the problem rebuilt from O.track_local_map's outputs gives
    its pose bit for bit and its outlier flags, and the 2D edges carry the stereo frame's 3D delta."""
    cam = dict(model="perspective", fx=718.856, fy=718.856, cx=607.1928, cy=185.2157, fxb=386.1448, cols=1241.0, rows=376.0, setup="stereo")
    r, fr, prm = _orb_frame(cam, 50)
    ref = O.track_local_map(cam, r["kps"], r["desc"], fr, prm.scale_factors_, prm.inv_level_sigma_sq_, prm.log_scale_factor_, monocular=False)
    und, _ = O.undistort_keypoints(cam, r["kps"])
    pp = P.chain_problem(cam, und, ref["kp_landmark"], fr["landmarks"]["pos_w"], fr["kp_x_right"], prm.inv_level_sigma_sq_, fr["pose_cw"])
    no_xr = pp["e_obs"][:, 2] < 0
    assert 0.1 * len(no_xr) < no_xr.sum() < 0.5 * len(no_xr)
    assert (pp["e_delta"] == P.DELTA_3D).all() and P.DELTA_3D != P.DELTA_2D
    n, pose, flags = O.pose_optimize(pp)
    assert np.array_equal(pose, ref["pose_cw"]) and n == ref["n_valid"]
    assert np.array_equal(flags, ref["kp_outlier"][pp["kp_index"]]) and not ref["kp_outlier"][ref["kp_landmark"] < 0].any()
    P.check_flags(pp, pose, flags)
    # the delta matters on this frame: some 2D edges sit between the two thresholds at the start, where the two deltas weigh them apart
    e2, _, _ = P.edge_chi2(pp, pp["pose_cw"])
    assert ((e2 > P.DELTA_2D ** 2) & no_xr).any()
    # and so one step with the per-edge (mono) delta is not the chain's step
    S = P.system(pp, robust=True)
    _, pose1, _ = O.pose_optimize(pp, 1, 0, 1)
    alt = dict(pp, e_delta=np.where(no_xr, P.DELTA_2D, P.DELTA_3D).astype(np.float32))
    _, pose_alt, _ = O.pose_optimize(alt, 1, 0, 1)
    lam = P.lambda_init(S)
    J, Ja = P.judge(S, lam, pose1), P.judge(S, lam, pose_alt)
    assert J["omega"] <= 4 * max(J["floor"], P.ROUNDOFF) < Ja["omega"] / 100, (J["omega"], Ja["omega"])
