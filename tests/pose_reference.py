"""High-precision reference of one LM step of the motion-only pose optimiser (test infrastructure).

optimize::pose_optimizer_g2o solves, per frame, a 6-unknown damped system: one free pose, every landmark fixed, one edge per keypoint
that carries a landmark.  Its edges are the pose blocks of the three reprojection edges, so the system is tests/lba_reference.py's
with the frame's pose free and every landmark fixed; this module adds what differs from bundle adjustment:

  - the classification between rounds (pose_optimizer_g2o.cc:133-167): EVERY edge, active or not, is re-tested at the round's pose
    (an outlier can come back), against (double)5.99146f without x_right and (double)7.81473f with it; there is no depth test.  The
    Huber kernel is on from the first round when num_trials_robust != 0 and is dropped after round num_trials_robust only when
    num_trials != 0 (:123-127, :164);
  - the rebuild of the problem a tracking chain solved from the chain's outputs: one edge per keypoint with a landmark, in keypoint
    order, at the undistorted keypoint, inv_level_sigma_sq[octave], x_right (or -1), and ONE Huber delta for the whole frame, chosen
    by the camera's setup (:84-88): sqrt(5.99146f) for a monocular frame, sqrt(7.81473f) for stereo and RGB-D -- also on the 2D
    edges of keypoints that have no x_right."""
import math

import numpy as np

import lba_reference as R

THR_2D, THR_3D = R.THR_2D, R.THR_3D
DELTA_2D = np.float32(np.sqrt(np.float32(5.99146)))     # std::sqrt(chi_sq_2D) in float
DELTA_3D = np.float32(np.sqrt(np.float32(7.81473)))
MARGIN = 1e-9                                          # relative distance from a threshold below which a decision is not judged


def frame_problem(pr):
    """pr with its single pose free and every landmark fixed, whatever the flags it came with."""
    return dict(pr, pose_fixed=np.zeros(1, np.uint8), point_fixed=np.ones(len(pr["points"]), np.uint8))


def system(pr, pose_cw=None, level=None, robust=True):
    """lba_reference.system of the frame at pose_cw (default: its own) over the edges with level 0 (default: all), Huber on every
    active edge when robust: the 6x6 H and b in longdouble, chi2 by math.fsum."""
    E = len(pr["e_pose"])
    level = np.zeros(E, bool) if level is None else np.asarray(level).astype(bool)
    return R.system(frame_problem(pr), pose_cw, pr["points"], level, np.full(E, bool(robust)))


def lambda_init(S):
    return R.lambda_init(S)


def chi2(S, pr, pose_cw):
    """The system's cost (its level and Huber switch) at pose_cw, by math.fsum."""
    return R.chi2(frame_problem(pr), np.asarray(pose_cw, np.float64).reshape(1, 4, 4), pr["points"], S["level"], S["robust"])


def robust_in_round(r, num_trials_robust, num_trials):
    """Is the Huber kernel on in round r (0-based) of a (num_trials_robust, num_trials) protocol?"""
    return num_trials_robust != 0 and (num_trials == 0 or r < num_trials_robust)


def protocol_prefix(r, num_trials_robust, num_trials):
    """(num_trials_robust', num_trials') whose r rounds are the first r rounds of (num_trials_robust, num_trials), Huber switch included."""
    a = min(r, num_trials_robust)
    return a, r - a


def edge_chi2(pr, pose_cw):
    """(chi2 (E,), threshold (E,), pc (E, 3)) of every edge at pose_cw, the threshold chosen by x_right."""
    pose = np.asarray(pose_cw, np.float64).reshape(1, 4, 4)
    err, pc = R.residuals(pr, pose, pr["points"])
    e2, _, _ = R.edge_costs(pr, err, np.zeros(len(err), bool))
    thr = np.where(np.asarray(pr["e_obs"], np.float32)[:, 2] < 0, THR_2D, THR_3D)
    return e2, thr, pc


def classify(pr, pose_cw):
    """The outlier flags of pose_optimizer_g2o.cc:133-167 at pose_cw: chi2 above the threshold of the edge; every edge, no depth test."""
    e2, thr, _ = edge_chi2(pr, pose_cw)
    return thr < e2


def decision_margins(pr, pose_cw):
    """Per edge, the relative distance of its classification from a flip: |chi2 - thr| / thr, and for an equirectangular point behind
    the camera also |x_c| / |p_c| (atan2 changes branch at the +-pi seam)."""
    e2, thr, pc = edge_chi2(pr, pose_cw)
    m = np.abs(e2 - thr) / thr
    equi = np.array([pr["cams"][c]["model"] == 1 for c in np.asarray(pr["e_cam"])], bool)
    seam = equi & (pc[:, 2] < 0)
    if seam.any():
        m[seam] = np.minimum(m[seam], np.abs(pc[seam, 0]) / np.linalg.norm(pc[seam], axis=1))
    return m


def check_flags(pr, pose_cw, flags, max_skipped=0.01):
    """flags equal the reference classification at pose_cw on every edge whose decision is clear by MARGIN; at most max_skipped of the
    edges (and at most 3) may be that close.  Returns the number of skipped edges."""
    clear = decision_margins(pr, pose_cw) > MARGIN
    skipped = int((~clear).sum())
    assert skipped <= max(3, max_skipped * len(clear)), skipped
    want = classify(pr, pose_cw)
    bad = np.nonzero(clear & (np.asarray(flags, bool) != want))[0]
    assert len(bad) == 0, (bad[:10], len(bad))
    return skipped


def reposed(pr, pose_cw, flags):
    """The problem of the next round as a problem of its own: the inliers of the last classification, at the pose it was made at."""
    keep = ~np.asarray(flags, bool)
    ne = int(keep.sum())
    out = dict(pr, pose_cw=np.asarray(pose_cw, np.float64).reshape(1, 4, 4), points=np.asarray(pr["points"])[np.asarray(pr["e_point"])[keep]],
               point_fixed=np.ones(ne, np.uint8), e_pose=np.zeros(ne, np.int32), e_point=np.arange(ne, dtype=np.int32),
               e_cam=np.asarray(pr["e_cam"])[keep], e_obs=np.asarray(pr["e_obs"])[keep], e_inv_sigma_sq=np.asarray(pr["e_inv_sigma_sq"])[keep],
               e_delta=np.asarray(pr["e_delta"])[keep])
    for k in ("e_robust", "e_can_be_outlier"):
        out[k] = None
    return out


# ---------------------------------------------------------------------------------------------------------------------
# problems rebuilt from a tracking chain's outputs
# ---------------------------------------------------------------------------------------------------------------------
_MODELS = {"perspective": 0, "equirectangular": 1, "fisheye": 2, "radial_division": 3}


def chain_problem(camera, und, kp_landmark, pos_w, kp_x_right, inv_level_sigma_sq, pose_cw):
    """The pose problem a chain solves for one frame: und the frame's undistorted keypoints (x, y, octave), kp_landmark its landmark
    per keypoint (-1: none), pos_w the landmark positions, kp_x_right None on a monocular frame.  Fisheye and radial-division frames
    use the perspective edges on undistorted keypoints; the Huber delta follows camera["setup"], not the edge."""
    kl = np.asarray(kp_landmark, np.int64)
    idx = np.nonzero(kl >= 0)[0]
    ne = len(idx)
    g = lambda k: float(camera.get(k, 0.0))
    model = _MODELS[camera.get("model", "perspective")]
    cam = dict(model=1 if model == 1 else 0, fx=g("fx"), fy=g("fy"), cx=g("cx"), cy=g("cy"), fxb=g("fxb"), cols=g("cols"), rows=g("rows"))
    xr = np.full(ne, -1.0, np.float32) if kp_x_right is None else np.asarray(kp_x_right, np.float32)[idx]
    delta = DELTA_2D if camera.get("setup", "monocular") == "monocular" else DELTA_3D
    oct_ = np.asarray(und["octave"], np.int64)[idx]
    return dict(pose_cw=np.asarray(pose_cw, np.float64).reshape(1, 4, 4), pose_fixed=np.zeros(1, np.uint8),
                points=np.asarray(pos_w, np.float64).reshape(-1, 3)[kl[idx]], point_fixed=np.ones(ne, np.uint8),
                e_pose=np.zeros(ne, np.int32), e_point=np.arange(ne, dtype=np.int32), e_cam=np.zeros(ne, np.uint8),
                e_obs=np.stack([np.asarray(und["x"], np.float32)[idx], np.asarray(und["y"], np.float32)[idx], xr], 1).astype(np.float32),
                e_inv_sigma_sq=np.asarray(inv_level_sigma_sq, np.float32)[oct_], e_delta=np.full(ne, delta, np.float32), e_robust=None,
                e_can_be_outlier=None, cams=[cam], kp_index=idx)


# ---------------------------------------------------------------------------------------------------------------------
# judging one step
# ---------------------------------------------------------------------------------------------------------------------
ROUNDOFF = 4 * 2.0 ** -53


def held_floor(S, lam, x_exact, A):
    """Backward error of the exact step applied to the state as an implementation holds it -- the normalised quaternion of the matrix
    it was handed, or of its own last step, which it exported as that matrix -- and read back against the matrix.  Once the steps are
    small (the later steps of a round, a start near the optimum) this rounding of the start state, not that of the output, is what
    the readback allows.  That rounding is one realisation; the floor is the larger of it and the bound of a start state off by one
    unit roundoff (of 1 + |t|) in every tangent coordinate, which moves the read step by as much."""
    T = S["pose_cw"][0]
    Tq = T.copy()
    Tq[:3, :3] = R._rot(R._quat(T[:3, :3]))
    x = R.log_step(R.exp_oplus(Tq, x_exact), T)
    one = R.backward_error(A, x.astype(R.LD), S["b"])
    a_inf = float(abs(A).sum(axis=1).max())
    delta = 2.0 ** -53 * (1.0 + np.abs(T[:3, 3]).max())
    bound = a_inf * delta / (a_inf * float(np.abs(x_exact).max()) + float(np.abs(np.asarray(S["b"], np.float64)).max()))
    return max(one, bound)


def judge(S, lam, pose_out, x_exact=None):
    """lba_reference.judge of the step from the system's pose to pose_out, with the readback floor: the larger of the output state's
    rounding (lba_reference.floor) and the held state's (held_floor)."""
    J = R.judge(S, lam, np.asarray(pose_out, np.float64).reshape(1, 4, 4), S["points"], x_exact=x_exact)
    J["floor"] = max(R.floor(S, lam, J["x_exact"], J["A"])[0], held_floor(S, lam, J["x_exact"], J["A"]))
    return J


def first_trial_lambda(S, pr, lam=None):
    """(lambda, trials): the damping of the first trial OptimizationAlgorithmLevenberg accepts from the system's state, starting at lam
    (default lambda_init), with the reference's exact steps and chi2 -- lambda *= ni, ni *= 2 after each rejection, at most 10 trials."""
    lam = lambda_init(S) if lam is None else lam
    ni = 2.0
    for trial in range(1, 11):
        x = R.exact_step(R.damped(S["H"], lam), S["b"])
        pose, _ = R.apply_step(S, x)
        if R.predicted_lambda(S, lam, x, chi2(S, pr, pose[0])) is not None:
            return lam, trial
        lam *= ni
        ni *= 2.0
    raise AssertionError("no trial accepted")


def replay_lambda(S, lam, pose_out, pr):
    """(lambda after the step to pose_out, rho): OptimizationAlgorithmLevenberg's update of an accepted first trial, from the
    reference chi2 at both poses; lambda None when the trial would have been rejected."""
    x = R.read_step(S, np.asarray(pose_out, np.float64).reshape(1, 4, 4), S["points"])
    chi_new = chi2(S, pr, pose_out)
    scale = math.fsum(x * (lam * x + np.asarray(S["b"], np.float64))) + 1e-3
    return R.predicted_lambda(S, lam, x, chi_new), (S["chi2"] - chi_new) / scale
