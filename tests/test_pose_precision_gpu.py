"""Each LM step of the device's pose optimiser (pose_optimize_kernel, through b200_pose_optimize and through every tracking chain's
stage C) judged against the high-precision reference of tests/pose_reference.py, with the CPU oracle's step as the control
(tests/test_pose_precision_cpu.py pins the method without a GPU).

test_pose_opt_gpu.py and the chain tests compare the pose after 2 + 2 rounds of 10 iterations with the oracle's to 1e-5; LM converges to
the point b fixes, so a normal matrix without the Huber weight, a stereo row missing from H, a wrong lambda_init or a lost CTA partial
only makes worse steps towards the same pose.  Here one step is judged at the level of one 6x6 solve.  Per case:
  - the normwise backward error of the step read back from the output pose against H_ref + lambda I is at most
    2 max(omega_orc, omega_floor, 4 u): omega_orc is the oracle's step judged the same way, omega_floor the rounding of the states;
  - the forward error against the exact step is at most kappa_bound * omega;
  - the outlier flags equal the reference classification on every edge whose chi2 is clear of its threshold by 1e-9 (relative).
lambda is the reference's: lambda_init = 1e-5 max diag(H_ref) for a first step (LM's doubling replayed if the reference rejects a
trial), for the later steps of a round the lambda the reference's rho predicts from the step before.

Measured on an H100 80GB HBM3: see DESIGN.md section 4 for the values of omega_dev, omega_orc, omega_floor and kappa_bound."""
import numpy as np
import pytest

import ba_windows as BW
import camera_models_oracle as CMO
import lba_reference as R
import pose_reference as P
from oracle import pyoracle as O

pytestmark = pytest.mark.gpu

FWD_C = 1.0


def _judge(tag, S, lam, dev_pose, S_orc, lam_orc, orc_pose):
    J = P.judge(S, lam, dev_pose)
    Jo = P.judge(S_orc, lam_orc, orc_pose, x_exact=J["x_exact"] if S_orc is S and lam_orc == lam else None)
    ratio = J["forward"] / (J["kappa_bound"] * J["omega"]) if J["omega"] > 0 else 0.0
    print(f"{tag}: omega_dev {J['omega']:.2e} omega_orc {Jo['omega']:.2e} floor {J['floor']:.2e} | kappa_bound {J['kappa_bound']:.2e} "
          f"forward {J['forward']:.2e} (forward / kappa omega {ratio:.1e})")
    assert J["omega"] <= 2 * max(Jo["omega"], J["floor"], P.ROUNDOFF), (tag, J["omega"], Jo["omega"], J["floor"])
    assert J["forward"] <= FWD_C * J["kappa_bound"] * J["omega"], (tag, J["forward"], J["kappa_bound"], J["omega"])
    return J


def _one_step(tag, pr, huber, dev):
    """Judge the device's result dev = (n_valid, pose, flags) of a (1, 0, 1) / (0, 1, 1) call on pr."""
    n_valid, pose, flags = dev
    _, orc_pose, _ = O.pose_optimize(pr, 1, 0, 1) if huber else O.pose_optimize(pr, 0, 1, 1)
    S = P.system(pr, robust=huber)
    lam, trials = P.first_trial_lambda(S, pr)
    J = _judge(f"{tag} ({len(pr['e_pose'])} edges, huber {huber}, trial {trials})", S, lam, pose, S, lam, orc_pose)
    P.check_flags(pr, pose, flags)
    assert n_valid == (~np.asarray(flags, bool)).sum()
    return J, trials


def _opt(a, b, k):
    from stella_vslam_b200 import optimize
    return optimize.pose_optimizer(a, b, k)


# ---------------------------------------------------------------------------------------------------------------------
# b200_pose_optimize
# ---------------------------------------------------------------------------------------------------------------------
SIZES = (5, 6, 31, 32, 33, 255, 256, 257, 512, 513, 2000, 20000)    # warps, one edge more than threads, multiples of kPoseThreads


def _sized(n):
    return BW.make_frame(1000 + n, n, "kitti", stereo_frac=0.5, outlier_frac=0.1)


def _converged(pr):
    """pr started 1e-6 rad from the optimum of its Huber-free cost: the step takes the small-angle branch of exp."""
    _, opt, _ = O.pose_optimize(pr, 0, 1, 50)
    d = np.zeros(6)
    d[:3] = 1e-6 * np.array([0.6, -0.48, 0.64])
    return dict(pr, pose_cw=R.exp_oplus(opt, d)[None])


REGIMES = {
    "huber_outliers30": (lambda: BW.make_frame(201, 2000, "kitti", stereo_frac=0.5, outlier_frac=0.3), True),
    "huber_clean": (lambda: BW.make_frame(202, 2000, "kitti", stereo_frac=0.5, outlier_frac=0.0), True),
    "no_huber": (lambda: BW.make_frame(203, 2000, "kitti", stereo_frac=0.5, outlier_frac=0.0), False),
    "large_error": (lambda: BW.make_frame(204, 2000, "kitti", stereo_frac=0.5, outlier_frac=0.1, rot_deg=5.0, trans_m=0.5), True),
    "near_optimum": (lambda: _converged(BW.make_frame(205, 2000, "kitti", stereo_frac=0.5, outlier_frac=0.0)), False),
    "mono_euroc_decoys": (lambda: BW.make_frame(206, 1500, "euroc", n_cams=3, cam_index=2, outlier_frac=0.2), True),
    "equirect_pole_seam": (lambda: BW.make_frame(207, 1500, "equirect", n_pole=8, n_seam=8, rot_deg=0.2, trans_m=0.02), True),
    "behind_near_far": (lambda: BW.make_frame(208, 1500, "kitti", stereo_frac=0.5, n_behind=10, n_near=4, n_far=8), True),
    # every point 0.3 m away: the largest diagonal entry of H is a translation one (elsewhere it is a rotation one)
    "near_points": (lambda: BW.make_frame(209, 1000, "kitti", n_near=1000, rot_deg=0.2, trans_m=0.005), True),
}


@pytest.mark.parametrize("n", SIZES)
def test_first_step_sizes(n):
    pr = _sized(n)
    _, trials = _one_step(f"n {n}", pr, True, _opt(1, 0, 1).optimize(pr))
    assert trials == 1


@pytest.mark.parametrize("name", list(REGIMES))
def test_first_step_regimes(name):
    make, huber = REGIMES[name]
    pr = make()
    dev = _opt(1, 0, 1).optimize(pr) if huber else _opt(0, 1, 1).optimize(pr)
    J, trials = _one_step(name, pr, huber, dev)
    assert trials == 1
    if name == "near_optimum":
        assert 0 < np.linalg.norm(J["x_exact"][:3]) < 1e-5 and 0 < np.linalg.norm(J["x"][:3]) < 1e-5
    if name == "near_points":
        d = np.abs(np.asarray(P.system(pr)["H"].diagonal(), np.float64))
        assert d[3:].max() > 2 * d[:3].max()
    if name == "huber_outliers30":
        e2, _, _ = P.edge_chi2(pr, pr["pose_cw"])
        assert (e2 > np.asarray(pr["e_delta"], np.float64) ** 2).mean() > 0.25        # many edges in Huber's linear branch


LATER = {
    "mixed": lambda: BW.make_frame(3, 400, "kitti", stereo_frac=0.5, outlier_frac=0.3),
    "large_stereo": lambda: BW.make_frame(211, 3000, "kitti", stereo_frac=0.7, outlier_frac=0.1, rot_deg=3.0, trans_m=0.3),
}


@pytest.mark.parametrize("name", list(LATER))
def test_later_steps(name):
    """Steps 1..5 of round 1: step k is the difference between the each_iter = k - 1 and k runs (the device is run-to-run
    deterministic), at the lambda the reference's rho predicts from the device's step k - 1; the oracle's control likewise.  A
    gain-threshold stop shows as two equal states."""
    pr = LATER[name]()
    prev_dev = prev_orc = pr["pose_cw"][0]
    lam = lam_orc = None
    judged = 0
    for k in range(1, 6):
        _, dev, _ = _opt(1, 0, k).optimize(pr)
        _, orc, _ = O.pose_optimize(pr, 1, 0, k)
        if k > 1 and np.array_equal(dev, prev_dev):
            break
        S, S_orc = P.system(pr, prev_dev), P.system(pr, prev_orc)
        if lam is None:
            lam, lam_orc = P.lambda_init(S), P.lambda_init(S_orc)
        _judge(f"{name} step {k} lambda {lam:.3e}", S, lam, dev, S_orc, lam_orc, orc)
        lam, rho = P.replay_lambda(S, lam, dev, pr)
        assert lam is not None, (k, rho)                             # every replayed trial was accepted
        lam_orc, _ = P.replay_lambda(S_orc, lam_orc, orc, pr)
        prev_dev, prev_orc = dev, orc
        judged += 1
    assert judged >= 3


ROUNDS = {
    "mixed600": lambda: BW.make_frame(8, 600, "kitti", stereo_frac=0.5, outlier_frac=0.3, rot_deg=3.0, trans_m=0.3),
    "stereo3000": lambda: BW.make_frame(212, 3000, "kitti", stereo_frac=0.8, outlier_frac=0.2),
}


def _reposed_rounds(pr):
    """[(round, huber, re-posed problem)] for rounds 2..4 of the default (2, 2, 10) protocol, from the device's own earlier rounds."""
    out = []
    for rnd in (2, 3, 4):
        _, pose, flags = _opt(*P.protocol_prefix(rnd - 1, 2, 2), 10).optimize(pr)
        P.check_flags(pr, pose, flags)
        out.append((rnd, P.robust_in_round(rnd - 1, 2, 2), P.reposed(pr, pose, flags)))
    return out


@pytest.mark.parametrize("name", list(ROUNDS))
def test_first_step_of_later_rounds(name):
    pr = ROUNDS[name]()
    for rnd, huber, rp in _reposed_rounds(pr):
        assert huber == (rnd <= 2)                                   # round 3 is the first without Huber
        dev = _opt(1, 0, 1).optimize(rp) if huber else _opt(0, 1, 1).optimize(rp)
        _one_step(f"{name} round {rnd}", rp, huber, dev)


def test_ragged_batch():
    """Every problem above in ONE b200_pose_optimize call, Huber on: each judged on its own and bit-identical to its single call."""
    probs = [(f"n {n}", _sized(n)) for n in SIZES] + [(k, m()) for k, (m, _) in REGIMES.items()]
    probs += [(f"{k} round {r}", rp) for k, m in ROUNDS.items() for r, _, rp in _reposed_rounds(m())]
    probs.insert(3, ("four edges", BW.make_frame(7, 4)))
    po = _opt(1, 0, 1)
    got = po.optimize_batch([p for _, p in probs])
    for (tag, pr), g in zip(probs, got):
        one = po.optimize(pr)
        assert g[0] == one[0] and np.array_equal(g[1], one[1]) and np.array_equal(g[2], one[2]), tag
        if len(pr["e_pose"]) < 5:
            assert g[0] == 0 and np.array_equal(g[1], pr["pose_cw"][0])
            continue
        _one_step(f"batch {tag}", pr, True, g)


# ---------------------------------------------------------------------------------------------------------------------
# the tracking chains
# ---------------------------------------------------------------------------------------------------------------------
KITTI = dict(model="perspective", fx=718.856, fy=718.856, cx=607.1928, cy=185.2157, fxb=386.1448, cols=1241.0, rows=376.0)
RADIAL = dict(model="radial_division", fx=612.3, fy=611.7, cx=480.5, cy=270.2, distortion=-0.15, fxb=0.0, cols=960.0, rows=540.0)
EQUI = dict(model="equirectangular", cols=1920.0, rows=960.0, fxb=0.0, setup="monocular")
TRIALS = [(1, 0), (0, 1)]


@pytest.fixture(scope="module")
def mods():
    from stella_vslam_b200 import feature, tracking
    from workloads import synth
    return feature, tracking, synth


def _extract(feature, synth, w, h, seeds, n=800):
    ex = feature.orb_extractor(feature.orb_params(), n, max_batch=len(seeds))
    kps, descs = ex.extract_batch(np.stack([synth.make_frame(w, h, seed=s) for s in seeds]))
    return ex, kps, descs


def _chain_step(tag, cam, und, kp_lm, pos_w, xr, isig, start, dev_pose, trials):
    """Judge a chain's pose against the problem rebuilt from its matches; returns the rebuilt problem (None below 5 edges)."""
    pp = P.chain_problem(cam, und, kp_lm, pos_w, xr, isig, start)
    if len(pp["e_pose"]) < 5:
        assert np.array_equal(dev_pose, np.asarray(start).reshape(4, 4)), tag
        return None
    huber = trials[0] != 0
    _, orc, _ = O.pose_optimize(pp, *trials, 1)
    S = P.system(pp, robust=huber)
    lam, n_trials = P.first_trial_lambda(S, pp)
    _judge(f"{tag} ({len(pp['e_pose'])} edges, trials {trials}, trial {n_trials})", S, lam, dev_pose, S, lam, orc)
    if huber and xr is not None:
        # the setup's delta matters here: 2D edges (no x_right) above the mono threshold weigh differently under the mono delta
        no_xr = pp["e_obs"][:, 2] < 0
        e2, _, _ = P.edge_chi2(pp, pp["pose_cw"])
        assert no_xr.any() and (no_xr & (e2 > float(P.DELTA_2D) ** 2)).any(), tag
    return pp


@pytest.mark.parametrize("trials", TRIALS)
@pytest.mark.parametrize("case", ["kitti_stereo", "equirect"])
def test_local_map_chain_step(mods, case, trials):
    feature, tracking, synth = mods
    if case == "kitti_stereo":
        ex, kps, descs = _extract(feature, synth, 1241, 376, (50, 51, 52))
        cam = dict(KITTI, setup="stereo")
        frames = [dict(synth.make_tracking_frame(kps[i], descs[i], cam, ex.orb_params_.scale_factors_, seed=70 + i, stereo=True), frame=i)
                  for i in range(3)]
    else:
        ex, kps, descs = _extract(feature, synth, 1920, 960, (40, 41), n=2500)
        cam = EQUI
        frames = [dict(synth.make_tracking_frame(kps[i], descs[i], cam, ex.orb_params_.scale_factors_, seed=45 + i, pixel_sigma=0.7), frame=i)
                  for i in range(2)]
    tr = tracking.local_map_tracker(ex, cam, num_trials_robust=trials[0], num_trials=trials[1], num_each_iter=1)
    got = tr.track(frames)
    isig = ex.orb_params_.inv_level_sigma_sq_
    for fr, g in zip(frames, got):
        und, _ = O.undistort_keypoints(cam, kps[fr["frame"]])
        pp = _chain_step(f"local map {case} frame {fr['frame']}", cam, und, g["kp_landmark"], fr["landmarks"]["pos_w"], fr.get("kp_x_right"),
                         isig, fr["pose_cw"], g["pose_cw"], trials)
        assert not g["kp_outlier"][g["kp_landmark"] < 0].any()
        if pp is not None:
            P.check_flags(pp, g["pose_cw"], g["kp_outlier"][pp["kp_index"]])
            assert g["n_valid"] == len(pp["e_pose"]) - g["kp_outlier"].sum()


def _frame_tracker_case(mods, chain, case):
    """(camera, extractor, kps, descs, frames, monocular, tracker kwargs, oracle kwargs)"""
    feature, tracking, synth = mods
    if case == "kitti_stereo":
        ex, kps, descs = _extract(feature, synth, 1241, 376, (50, 51, 52))
        cam = dict(KITTI, setup="stereo")
        mk = dict(motion=lambda i: synth.make_motion_frame(kps[i], descs[i], cam, ex.orb_params_.scale_factors_, seed=70 + i, stereo=True),
                  robust=lambda i: synth.make_robust_frame(kps[i], descs[i], cam, seed=70 + i, stereo=True),
                  bow=lambda i: synth.make_bow_frame(kps[i], descs[i], cam, seed=70 + i, stereo=True))[chain]
        frames = [dict(mk(i), frame=i) for i in range(3)]
        return cam, ex, kps, descs, frames, False, dict(margin=10.0, use_fixed_seed=True)
    if case == "radial_division":
        ex, kps, descs = _extract(feature, synth, 960, 540, (500, 501))
        und = [CMO.undistort_keypoints(RADIAL, k)[0] for k in kps]
        frames = [dict(synth.make_motion_frame(und[i], descs[i], RADIAL, ex.orb_params_.scale_factors_, seed=510 + i), frame=i) for i in range(2)]
        return RADIAL, ex, kps, descs, frames, True, dict(grid=(64, 48))
    # "gated": the second frame's matches stay below num_matches_thr; its pose must come back bit-unchanged
    ex, kps, descs = _extract(feature, synth, 640, 376, (11, 11))
    cam = dict(KITTI, cols=640.0, cx=320.0, setup="monocular")
    sf = ex.orb_params_.scale_factors_
    frames = [dict(synth.make_motion_frame(kps[0], descs[0], cam, sf, seed=1), frame=0),
              dict(synth.make_motion_frame(kps[1], descs[1], cam, sf, seed=5, shift_px=200.0, landmark_frac=0.05), frame=1)]
    return cam, ex, kps, descs, frames, True, dict(margin=10.0)


FT_CASES = [("motion", "kitti_stereo"), ("motion", "radial_division"), ("motion", "gated"), ("robust", "kitti_stereo"), ("bow", "kitti_stereo")]


@pytest.mark.parametrize("trials", TRIALS)
@pytest.mark.parametrize("chain,case", FT_CASES)
def test_frame_tracker_chain_step(mods, chain, case, trials):
    """frame_tracker's chains return the landmarks after discard_outliers: the matches are the oracle composition's (its pose stage
    replaced by one that discards nothing; the chain tests pin the chain's matches to it), and the chain's landmarks must be exactly
    those matches minus the reference's outliers at the chain's pose."""
    import bow_track_oracle as BT
    import motion_track_oracle as MT
    import robust_track_oracle as RT
    feature, tracking, synth = mods
    cam, ex, kps, descs, frames, mono, kw = _frame_tracker_case(mods, chain, case)
    tr = tracking.frame_tracker(ex, cam, num_trials_robust=trials[0], num_trials=trials[1], num_each_iter=1, **kw)
    got = dict(motion=tr.motion_based_track, robust=tr.robust_match_based_track, bow=tr.bow_match_based_track)[chain](frames)
    prm = ex.orb_params_
    isig = prm.inv_level_sigma_sq_
    judged = 0
    for fr, g in zip(frames, got):
        i = fr["frame"]
        seen = []

        def keep_all(pp, *_):
            seen.append(pp)
            return len(pp["e_pose"]), np.asarray(pp["pose_cw"], np.float64).reshape(4, 4).copy(), np.zeros(len(pp["e_pose"]), bool)

        if chain == "motion":
            ref = MT.motion_based_track(cam, kps[i], descs[i], fr, prm.scale_factors_, isig, margin=tr._prm.margin, num_matches_thr=tr.num_matches_thr,
                                        true_baseline=tr.true_baseline, monocular=mono, img_bounds=tuple(tr._prm.img_bounds),
                                        grid=(tr._prm.grid_cols, tr._prm.grid_rows), pose_fn=keep_all)
            pos_w, start = fr["table"]["pos_w"], fr["pose_cw"]
        elif chain == "robust":
            ref = RT.robust_match_based_track(cam, kps[i], descs[i], fr, isig, num_matches_thr=tr.num_matches_thr, monocular=mono, pose_fn=keep_all)
            pos_w, start = fr["keyframe"]["pos_w"], fr["last_pose_cw"]
        else:
            ref = BT.bow_match_based_track(cam, kps[i], descs[i], fr, isig, num_matches_thr=tr.num_matches_thr, monocular=mono, pose_fn=keep_all)
            pos_w, start = fr["keyframe"]["pos_w"], fr["last_pose_cw"]
        tag = f"{chain} {case} frame {i}"
        if not seen:                                                 # gated / not applied / fewer than 5 edges: no step
            if case == "gated":
                assert i == 1 and not g["tracked"]
            if g["pose_cw"] is not None:
                assert np.array_equal(g["pose_cw"], np.asarray(start).reshape(4, 4)), tag
            continue
        und, _ = CMO.undistort_keypoints(cam, kps[i])
        pre = ref["kp_landmark"]
        pp = _chain_step(tag, cam, und, pre, pos_w, fr.get("kp_x_right"), isig, start, g["pose_cw"], trials)
        for k in ("points", "e_obs", "e_inv_sigma_sq", "e_delta"):
            assert np.array_equal(pp[k], seen[0][k]), (tag, k)
        # discard_outliers: the chain's landmarks are the matches minus the reference classification at its pose
        clear = P.decision_margins(pp, g["pose_cw"]) > P.MARGIN
        assert (~clear).sum() <= 3
        want = P.classify(pp, g["pose_cw"])
        dropped = g["kp_landmark"][pp["kp_index"]] < 0
        assert np.array_equal(dropped[clear], want[clear]), tag
        assert np.array_equal(g["kp_landmark"][pp["kp_index"]][~dropped], pre[pp["kp_index"]][~dropped])
        assert ((g["kp_landmark"] >= 0) <= (pre >= 0)).all()
        judged += 1
    assert judged >= 1
