"""High-precision reference of one local / global bundle-adjustment LM step (test infrastructure).

The damped system g2o's Levenberg-Marquardt solves for optimize::local_bundle_adjuster_g2o and optimize::global_bundle_adjuster,
restated in numpy independently of oracle/lba_oracle.c and of the device's Schur route:

  - residuals e = obs - proj(R p + t) of the three edge models (perspective mono, perspective stereo with the x_right row,
    equirectangular), each with its own camera (e_cam), and their analytic Jacobians in g2o's parametrisation: a keyframe
    updates as T <- exp([omega, upsilon]) T (SE3Quat::exp, rotation first), a landmark as p <- p + delta;
  - H = sum_e J_e^T (w_e rho'_e) J_e and b = -sum_e J_e^T (w_e rho'_e) e_e over the active edges (constructQuadraticForm with
    RobustKernelHuber: the information scaled by rho' only), for the FULL system -- free keyframes with an active edge first, then
    the landmarks with an active edge -- assembled in np.longdouble, entry by entry in edge order, as a scipy.sparse matrix.
    Nothing is reduced: a Schur complement, landmark inverse or blocked Cholesky of the implementation under test is not shared.
    A landmark or keyframe whose edges are all inactive is not in the system (g2o's initializeOptimization keeps only vertices
    with an active edge; the oracle keeps them, with H = 0, b = 0, so its step there is 0 -- the same thing).

An implementation's step is read back from its output state (per keyframe log(T_new T_old^-1) through the same V matrix and
small-angle branch as g2o's exp, per landmark p_new - p_old) and judged by its normwise backward error against H + lambda I, and
per keyframe block row.  The readback floor is the backward error of the reference's own exact step after it has been applied
to the input state in float64 and read back the same way: the rounding of an output state allows no less."""
import math

import numpy as np
import scipy.sparse as sp

from sparse_lm import backward_error, damped, exact_step, factor, kappa_bound, rel  # noqa: F401

THR_2D, THR_3D = float(np.float32(5.99146)), float(np.float32(7.81473))   # constexpr float chi_sq_2D / chi_sq_3D
LD = np.longdouble


# ---------------------------------------------------------------------------------------------------------------------
# SE(3) in g2o's conventions
# ---------------------------------------------------------------------------------------------------------------------
def _skew(w):
    return np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])


def _rv(om):
    """SE3Quat::exp's R and V for the rotation part om (small-angle branch below 1e-5)."""
    th = float(np.linalg.norm(om))
    O = _skew(om)
    O2 = O @ O
    if th < 1e-5:
        a, b, c, d = 1.0, 0.5, 0.5, 1.0 / 6.0
    else:
        a, b = math.sin(th) / th, (1 - math.cos(th)) / (th * th)
        c, d = b, (th - math.sin(th)) / (th ** 3)
    return np.eye(3) + a * O + b * O2, np.eye(3) + c * O + d * O2


def _quat(R):
    """Unit quaternion (x, y, z, w), w >= 0, of a rotation matrix (Eigen's branch on the trace)."""
    t = R[0, 0] + R[1, 1] + R[2, 2]
    q = np.zeros(4)
    if t > 0:
        s = math.sqrt(t + 1.0)
        q[3] = 0.5 * s
        s = 0.5 / s
        q[:3] = [(R[2, 1] - R[1, 2]) * s, (R[0, 2] - R[2, 0]) * s, (R[1, 0] - R[0, 1]) * s]
    else:
        i = int(np.argmax([R[0, 0], R[1, 1], R[2, 2]]))
        j, k = (i + 1) % 3, (i + 2) % 3
        s = math.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0)
        q[i] = 0.5 * s
        s = 0.5 / s
        q[3] = (R[k, j] - R[j, k]) * s
        q[j] = (R[j, i] + R[i, j]) * s
        q[k] = (R[k, i] + R[i, k]) * s
    q = -q if q[3] < 0 else q
    return q / np.linalg.norm(q)


def _rot(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def exp_oplus(T, d):
    """exp(d) T for a 4x4 T and d = [omega, upsilon], the rotation of exp(d) taken through a normalised quaternion as g2o does."""
    R, V = _rv(np.asarray(d[:3], np.float64))
    R = _rot(_quat(R))
    out = np.eye(4)
    out[:3, :3] = R @ T[:3, :3]
    out[:3, 3] = R @ T[:3, 3] + V @ np.asarray(d[3:], np.float64)
    return out


def log_step(T_new, T_old):
    """d with exp(d) T_old = T_new: omega from the quaternion of R_new R_old^T, upsilon = V(omega)^-1 (t_new - R_d t_old)."""
    Rd = T_new[:3, :3] @ T_old[:3, :3].T
    td = T_new[:3, 3] - Rd @ T_old[:3, 3]
    q = _quat(Rd)
    s = np.linalg.norm(q[:3])
    om = np.zeros(3) if s == 0 else 2.0 * math.atan2(s, q[3]) * q[:3] / s
    _, V = _rv(om)
    return np.concatenate([om, np.linalg.solve(V, td)])


# ---------------------------------------------------------------------------------------------------------------------
# the three edge models
# ---------------------------------------------------------------------------------------------------------------------
def _cam_arrays(pr):
    e_cam = np.asarray(pr["e_cam"], np.int64)
    f = lambda k: np.array([float(c[k]) for c in pr["cams"]])[e_cam]
    return {k: f(k) for k in ("model", "fx", "fy", "cx", "cy", "fxb", "cols", "rows")}


def camera_points(pr, pose_cw, points):
    T = np.asarray(pose_cw, np.float64).reshape(-1, 4, 4)
    P = np.asarray(points, np.float64).reshape(-1, 3)
    ep, el = np.asarray(pr["e_pose"]), np.asarray(pr["e_point"])
    return np.einsum("eij,ej->ei", T[ep, :3, :3], P[el]) + T[ep, :3, 3], T, P


def residuals(pr, pose_cw, points):
    """(err (E,3), pc (E,3)): e = obs - proj, the third row the stereo x_right row (0 on mono and equirectangular edges)."""
    pc, _, _ = camera_points(pr, pose_cw, points)
    c = _cam_arrays(pr)
    obs = np.asarray(pr["e_obs"], np.float32).astype(np.float64)
    x, y, z = pc[:, 0], pc[:, 1], pc[:, 2]
    equi = c["model"] == 1
    err = np.zeros((len(pc), 3))
    with np.errstate(divide="ignore", invalid="ignore"):
        u = np.where(equi, c["cols"] * (0.5 + np.arctan2(x, z) / (2 * np.pi)), c["fx"] * x / z + c["cx"])
        L = np.sqrt(x * x + y * y + z * z)
        v = np.where(equi, c["rows"] * (0.5 + np.arcsin(y / L) / np.pi), c["fy"] * y / z + c["cy"])
        ur = u - c["fxb"] / z
    err[:, 0] = obs[:, 0] - u
    err[:, 1] = obs[:, 1] - v
    err[:, 2] = np.where(~equi & (obs[:, 2] >= 0), obs[:, 2] - ur, 0.0)
    return err, pc


def jacobians(pr, pose_cw, points):
    """(Jp (E,3,6), Jl (E,3,3)): d err / d [omega, upsilon] of exp(.) T and d err / d p, by the chain rule through
    d proj / d pc, d pc / d [omega, upsilon] = [-[pc]x, I] and d pc / d p = R."""
    pc, T, _ = camera_points(pr, pose_cw, points)
    c = _cam_arrays(pr)
    obs2 = np.asarray(pr["e_obs"], np.float32)[:, 2]
    x, y, z = pc[:, 0], pc[:, 1], pc[:, 2]
    E = len(pc)
    equi = c["model"] == 1
    D = np.zeros((E, 3, 3))            # d proj / d pc
    with np.errstate(divide="ignore", invalid="ignore"):
        D[:, 0] = np.stack([c["fx"] / z, 0 * z, -c["fx"] * x / (z * z)], 1)
        D[:, 1] = np.stack([0 * z, c["fy"] / z, -c["fy"] * y / (z * z)], 1)
        D[:, 2] = D[:, 0] + np.stack([0 * z, 0 * z, c["fxb"] / (z * z)], 1)
        r2 = x * x + z * z
        L = np.sqrt(r2 + y * y)
        De = np.zeros((E, 3, 3))
        De[:, 0] = (c["cols"] / (2 * np.pi))[:, None] * np.stack([z, 0 * z, -x], 1) / r2[:, None]
        ey = np.zeros((E, 3))
        ey[:, 1] = 1.0
        De[:, 1] = (c["rows"] / np.pi)[:, None] * (ey * L[:, None] - y[:, None] * pc / L[:, None]) / (L * np.sqrt(r2))[:, None]
    D = np.where(equi[:, None, None], De, D)
    D[(equi | (obs2 < 0)), 2] = 0.0
    D = -D                             # err = obs - proj
    dpose = np.zeros((E, 3, 6))
    dpose[:, :, :3] = -np.stack([np.stack([0 * x, -z, y], 1), np.stack([z, 0 * x, -x], 1), np.stack([-y, x, 0 * x], 1)], 1)
    dpose[:, :, 3:] = np.eye(3)
    R = T[np.asarray(pr["e_pose"]), :3, :3]
    return D @ dpose, D @ R


def edge_costs(pr, err, robust):
    """(chi2_e = w |e|^2, robust cost, weight w rho') per edge (RobustKernelHuber at delta = e_delta)."""
    w = np.asarray(pr["e_inv_sigma_sq"], np.float32).astype(np.float64)
    d = np.asarray(pr["e_delta"], np.float32).astype(np.float64)
    e2 = w * (err * err).sum(1)
    over = robust & (e2 > d * d)
    with np.errstate(invalid="ignore", divide="ignore"):
        cost = np.where(over, 2 * np.sqrt(e2) * d - d * d, e2)
        rho1 = np.where(over, d / np.sqrt(e2), 1.0)
    return e2, cost, w * rho1


def first_round_masks(pr):
    E = len(pr["e_pose"])
    rob = np.ones(E, bool) if pr.get("e_robust") is None else np.asarray(pr["e_robust"]).astype(bool)
    return np.zeros(E, bool), rob


def second_round_masks(pr, pose_cw, points):
    """local_bundle_adjuster_g2o.cc:317-348 at the state after the first round: an edge leaves (level 1) when its chi2 exceeds the
    chi-square threshold of its dimension or its perspective depth is not positive; every edge that can be an outlier drops Huber."""
    err, pc = residuals(pr, pose_cw, points)
    level, rob = first_round_masks(pr)
    e2, _, _ = edge_costs(pr, err, np.zeros(len(err), bool))
    obs2 = np.asarray(pr["e_obs"], np.float32)[:, 2]
    thr = np.where(obs2 < 0, THR_2D, THR_3D)
    persp = _cam_arrays(pr)["model"] != 1
    can = np.ones(len(err), bool) if pr.get("e_can_be_outlier") is None else np.asarray(pr["e_can_be_outlier"]).astype(bool)
    level = can & ((thr < e2) | (persp & ~(pc[:, 2] > 0)))
    return level, rob & ~can


def chi2(pr, pose_cw, points, level, robust):
    err, _ = residuals(pr, pose_cw, points)
    _, cost, _ = edge_costs(pr, err, robust)
    return math.fsum(cost[~level])


# ---------------------------------------------------------------------------------------------------------------------
# the full damped system
# ---------------------------------------------------------------------------------------------------------------------
def system(pr, pose_cw=None, points=None, level=None, robust=None):
    """dict(H (csr, longdouble), b (longdouble), chi2 (math.fsum), pose_col (K: first unknown of the keyframe, -1 outside),
    pt_col (L), n_pose (6 x free keyframes in the system), level, robust, pose_cw, points) at the state (default: the problem's)
    over the edges with level 0 (default: all), Huber where robust (default: the problem's e_robust)."""
    pose_cw = np.asarray(pr["pose_cw"] if pose_cw is None else pose_cw, np.float64).reshape(-1, 4, 4)
    points = np.asarray(pr["points"] if points is None else points, np.float64).reshape(-1, 3)
    l0, r0 = first_round_masks(pr)
    level = l0 if level is None else np.asarray(level).astype(bool)
    robust = r0 if robust is None else np.asarray(robust).astype(bool)
    K, L = len(pose_cw), len(points)
    ep, el = np.asarray(pr["e_pose"], np.int64), np.asarray(pr["e_point"], np.int64)
    act = ~level
    pfree = ~np.asarray(pr["pose_fixed"]).astype(bool)
    lfree = np.ones(L, bool) if pr.get("point_fixed") is None else ~np.asarray(pr["point_fixed"]).astype(bool)
    p_in = np.zeros(K, bool)
    p_in[ep[act]] = True
    p_in &= pfree
    l_in = np.zeros(L, bool)
    l_in[el[act]] = True
    l_in &= lfree
    pose_col = np.where(p_in, 6 * (np.cumsum(p_in) - 1), -1)
    n_pose = 6 * int(p_in.sum())
    pt_col = np.where(l_in, n_pose + 3 * (np.cumsum(l_in) - 1), -1)
    n = n_pose + 3 * int(l_in.sum())
    err, _ = residuals(pr, pose_cw, points)
    Jp, Jl = jacobians(pr, pose_cw, points)
    _, cost, ww = edge_costs(pr, err, robust)
    idx = np.nonzero(act)[0]
    # per edge: 9 unknowns (6 pose, 3 landmark), columns -1 where the vertex is not in the system
    J = np.concatenate([Jp[idx], Jl[idx]], 2).astype(LD)                                   # (m, 3, 9)
    cols = np.concatenate([pose_col[ep[idx]][:, None] + np.arange(6), pt_col[el[idx]][:, None] + np.arange(3)], 1)
    cols[:, :6] = np.where(pose_col[ep[idx]][:, None] >= 0, cols[:, :6], -1)
    cols[:, 6:] = np.where(pt_col[el[idx]][:, None] >= 0, cols[:, 6:], -1)
    w = ww[idx].astype(LD)
    blk = np.einsum("e,eda,edc->eac", w, J, J)                                               # (m, 9, 9) in longdouble
    g = -np.einsum("e,eda,ed->ea", w, J, err[idx].astype(LD))
    rr = np.broadcast_to(cols[:, :, None], blk.shape)
    cc = np.broadcast_to(cols[:, None, :], blk.shape)
    keep = (rr >= 0) & (cc >= 0)
    H = sp.coo_matrix((blk[keep], (rr[keep], cc[keep])), shape=(n, n)).tocsr()
    b = np.zeros(n, LD)
    kb = cols >= 0
    np.add.at(b, cols[kb], g[kb])
    return dict(H=H, b=b, chi2=math.fsum(cost[act]), pose_col=pose_col, pt_col=pt_col, n_pose=n_pose, level=level, robust=robust,
                pose_cw=pose_cw, points=points)


def lambda_init(S):
    """computeLambdaInit: tau * max |H_jj| over the free vertices, tau = 1e-5."""
    return float(1e-5 * np.abs(S["H"].diagonal()).max())


def read_step(S, pose_out, points_out):
    """The step an implementation took from the system's state to (pose_out, points_out), in the system's unknown order (float64)."""
    x = np.zeros(S["H"].shape[0])
    pose_out = np.asarray(pose_out, np.float64).reshape(-1, 4, 4)
    points_out = np.asarray(points_out, np.float64).reshape(-1, 3)
    for k in np.nonzero(S["pose_col"] >= 0)[0]:
        x[S["pose_col"][k]:S["pose_col"][k] + 6] = log_step(pose_out[k], S["pose_cw"][k])
    m = S["pt_col"] >= 0
    x[(S["pt_col"][m][:, None] + np.arange(3)).ravel()] = (points_out[m] - S["points"][m]).ravel()
    return x


def apply_step(S, x):
    """The state x moves the system's state to, in float64 (the keyframes through exp as g2o applies it)."""
    pose = S["pose_cw"].copy()
    pts = S["points"].copy()
    for k in np.nonzero(S["pose_col"] >= 0)[0]:
        pose[k] = exp_oplus(pose[k], x[S["pose_col"][k]:S["pose_col"][k] + 6])
    m = S["pt_col"] >= 0
    pts[m] += np.asarray(x, np.float64)[(S["pt_col"][m][:, None] + np.arange(3))]
    return pose, pts


def keyframe_backward_error(A, x, b, n_pose):
    """Largest backward error of one keyframe's 6 block rows: ||(A x - b)_k||_inf / (||A_k||_inf ||x||_inf + ||b_k||_inf)."""
    if n_pose == 0:
        return 0.0
    r = np.abs(A[:n_pose] @ x - b[:n_pose]).reshape(-1, 6).max(1)
    a = np.asarray(abs(A[:n_pose]).sum(axis=1)).ravel().reshape(-1, 6).max(1)
    bb = np.abs(b[:n_pose]).reshape(-1, 6).max(1)
    return float((r / (a * np.abs(x).max() + bb)).max())


def judge(S, lam, pose_out, points_out, lu=None, x_exact=None):
    """dict(x, omega, omega_kf, forward, x_exact, A, kappa_bound) of the step to (pose_out, points_out) at damping lam."""
    A = damped(S["H"], lam)
    b = S["b"]
    if x_exact is None:
        x_exact = exact_step(A, b, lu)
    x = read_step(S, pose_out, points_out)
    xl = x.astype(LD)
    return dict(x=x, omega=backward_error(A, xl, b), omega_kf=keyframe_backward_error(A, xl, b, S["n_pose"]), forward=rel(x, x_exact),
                x_exact=x_exact, A=A, kappa_bound=kappa_bound(A, lam))


def floor(S, lam, x_exact, A=None):
    """(omega, omega_kf) of the reference's exact step after it has been applied to the state in float64 and read back."""
    A = damped(S["H"], lam) if A is None else A
    pose, pts = apply_step(S, x_exact)
    x = read_step(S, pose, pts).astype(LD)
    return backward_error(A, x, S["b"]), keyframe_backward_error(A, x, S["b"], S["n_pose"])


def predicted_lambda(S, lam, x, chi2_new):
    """The lambda after an accepted first trial (OptimizationAlgorithmLevenberg::solve): rho = (chi2_old - chi2_new) /
    (x^T (lam x + b) + 1e-3), lam * max(1/3, min(2/3, 1 - (2 rho - 1)^3)); None when rho <= 0 (the trial would be rejected)."""
    b = np.asarray(S["b"], np.float64)
    scale = math.fsum(x * (lam * x + b)) + 1e-3
    rho = (S["chi2"] - chi2_new) / scale
    if not rho > 0:
        return None
    return lam * max(1.0 / 3.0, min(2.0 / 3.0, 1.0 - (2 * rho - 1) ** 3))


def check_step(S, lam, lam_reported, chi2_reported, lam_final, pose_out, points_out, pr, lu=None, x_exact=None):
    """The assertions both files make on one step; returns the judge dict with the floor added."""
    if lam_reported is not None:
        assert abs(lam_reported - lambda_init(S)) <= 1e-12 * lam_reported, (lam_reported, lambda_init(S))
    J = judge(S, lam, pose_out, points_out, lu, x_exact)
    J["floor"], J["floor_kf"] = floor(S, lam, J["x_exact"], J["A"])
    chi_new = chi2(pr, pose_out, points_out, S["level"], S["robust"])
    assert abs(chi2_reported - chi_new) <= 1e-11 * chi_new, (chi2_reported, chi_new)
    pred = predicted_lambda(S, lam, J["x"], chi_new)
    assert pred is not None and abs(lam_final - pred) <= 1e-8 * pred, (lam_final, pred)
    fixed = np.asarray(pr["pose_fixed"]).astype(bool)
    assert np.array_equal(np.asarray(pose_out)[fixed], np.asarray(pr["pose_cw"])[fixed])
    out = (S["pt_col"] < 0)
    assert np.array_equal(np.asarray(points_out)[out], np.asarray(S["points"])[out])
    return J


# ---------------------------------------------------------------------------------------------------------------------
# maps for global BA
# ---------------------------------------------------------------------------------------------------------------------
def revisit_map(K, L, m, seed, model="stereo"):
    """synth.make_ba_problem's map of K keyframes (one fixed) whose last m keyframes return to the places of the first m: keyframe
    K - m + i takes keyframe i's true pose (perturbed as the others are) and observes, with fresh noise, every landmark keyframe i
    observes, in place of its own observations.  The reduced system then couples the newest keyframes with the oldest: not banded."""
    from workloads import synth
    pr = synth.make_ba_problem(K, 1, L, seed=seed, model=model)
    rng = np.random.default_rng(seed + 1000)
    gt, gp = pr["gt_pose_cw"].copy(), pr["gt_points"]
    pose0 = pr["pose_cw"].copy()
    keep = pr["e_pose"] < K - m
    e_pose, e_point = list(pr["e_pose"][keep]), list(pr["e_point"][keep])
    e_obs, e_isq = list(pr["e_obs"][keep]), list(pr["e_inv_sigma_sq"][keep])
    cam = pr["cams"][0]
    for i in range(m):
        k = K - m + i
        gt[k] = gt[i]
        dR = np.linalg.qr(np.eye(3) + np.deg2rad(0.5) * _skew(rng.standard_normal(3) / np.sqrt(3)))[0]
        dR = dR * np.sign(np.diag(dR))[None, :]
        c = -gt[i, :3, :3].T @ gt[i, :3, 3] + 0.05 * rng.standard_normal(3) / np.sqrt(3)
        pose0[k, :3, :3] = dR @ gt[i, :3, :3]
        pose0[k, :3, 3] = -pose0[k, :3, :3] @ c
        for e in np.nonzero(pr["e_pose"] == i)[0]:
            l = int(pr["e_point"][e])
            pc = gt[k, :3, :3] @ gp[l] + gt[k, :3, 3]
            sig = 1.0 / math.sqrt(float(pr["e_inv_sigma_sq"][e]))
            if cam["model"] == 1:
                uv = np.array([cam["cols"] * (0.5 + math.atan2(pc[0], pc[2]) / (2 * np.pi)),
                               cam["rows"] * (0.5 + math.asin(pc[1] / np.linalg.norm(pc)) / np.pi)])
            else:
                uv = np.array([cam["fx"] * pc[0] / pc[2] + cam["cx"], cam["fy"] * pc[1] / pc[2] + cam["cy"]])
            nz = sig * rng.standard_normal(3)
            xr = -1.0 if pr["e_obs"][e, 2] < 0 else max(-1.0, uv[0] - cam["fxb"] / pc[2] + nz[2])
            e_pose.append(k); e_point.append(l); e_obs.append((uv[0] + nz[0], uv[1] + nz[1], xr)); e_isq.append(pr["e_inv_sigma_sq"][e])
    e_point = np.array(e_point, np.int64)
    used = np.unique(e_point)
    E = len(e_pose)
    return dict(pr, pose_cw=pose0, points=pr["points"][used], e_pose=np.array(e_pose, np.int32),
                e_point=np.searchsorted(used, e_point).astype(np.int32), e_cam=np.zeros(E, np.uint8),
                e_obs=np.array(e_obs, np.float32).reshape(E, 3), e_inv_sigma_sq=np.array(e_isq, np.float32),
                e_delta=np.full(E, pr["e_delta"][0], np.float32), gt_pose_cw=gt, gt_points=gp[used])


def gross_landmarks(pr, n, seed):
    """pr with every observation of n random landmarks moved by 20 px in x and y: after the first round all their edges fail the
    chi-square test, so in the second round those landmarks have no active edge and leave the system."""
    rng = np.random.default_rng(seed)
    pick = rng.choice(len(pr["points"]), n, replace=False)
    obs = np.array(pr["e_obs"], np.float32)
    m = np.isin(pr["e_point"], pick)
    obs[m, 0] += np.float32(20.0)
    obs[m, 1] += np.float32(20.0)
    obs[m & (obs[:, 2] >= 0), 2] += np.float32(20.0)
    return dict(pr, e_obs=obs)
