"""High-precision reference of one LM step of loop detection's Sim3 refinement (test infrastructure).

optimize::transform_optimizer solves, per loop candidate, a 7-unknown damped system: one Sim3_12 vertex, a forward edge_12 and a
backward edge_21 per matched pair, Huber delta sqrt(chi_sq) computed in float.  This module restates that system in vectorised numpy,
independently of tests/transform_oracle.c and of the kernel:

  - the edges: obs (float32 widened to double) - cam_project(S.map(pc)) for edge_12 and S^-1 for edge_21, perspective and
    equirectangular, Omega = inv_sigma_sq I, the Sim3 as its 4x4 matrix [s R | t];
  - the Jacobian by a fourth-order central stencil at delta 1e-4 (translation: 1e-4 of the scene's median depth) through
    Sim3(u) * S, the update applied as the exact matrix
    exponential of the 4x4 twist (u[6] = 0 under fix_scale) -- not g2o's delta-1e-9 difference, which the kernel and the oracle share
    and which is the noise this reference is there to see past;
  - the robust system over an active set, H = sum w rho'(chi2) J^T J and b = -sum w rho'(chi2) J^T e in longdouble, its robust chi2
    by math.fsum and the number of edges beyond the Huber delta;
  - the step an implementation took, read back from its states before and after by Newton on the exp it applied (pgo_oracle.exp,
    g2o's Sim3(update), I + Omega + Omega^2 below theta = 1e-5 included), and the backward error the rounding of those states allows;
  - round 1 of the protocol replayed with exact solves, and the Gauss-Newton optimum over an active set;
  - guards that keep equirectangular edges' stencils off the seam and away from the poles."""
import math

import numpy as np
import scipy.linalg as sl
import scipy.sparse as sp

import pgo_oracle as PO
from sparse_lm import backward_error, damped, exact_step, kappa_bound, rel  # noqa: F401

LD = np.longdouble
DELTA = 1e-4
U = 2.0 ** -53
ROUNDOFF = 4 * U
STENCIL = ((-1.0, 2), (8.0, 1), (-8.0, -1), (1.0, -2))       # (weight, multiple of delta) of f'(0) = sum / (12 delta)
# An equirectangular edge whose polar distance (pi/2 - |phi|) falls under POLE_GUARD rad at any stencil state is flagged: the
# derivatives of asin grow like 1/distance^k there, so the fourth-order stencil at 3e-4 (the coarsest the tests compare) would err by
# (3e-4 / distance)^4 / 30, 2e-11 at 0.02 rad.
POLE_GUARD = 0.02


# ---------------------------------------------------------------------------------------------------------------------
# one edge (also used per edge by tests/test_transform_cpu.py)
# ---------------------------------------------------------------------------------------------------------------------
def hat(u):
    """The 4x4 twist of a Sim3 update (omega, upsilon, sigma): expm(hat(u)) is g2o's Sim3(u) as a matrix."""
    w, v, s = u[:3], u[3:6], u[6]
    M = np.zeros((4, 4))
    M[:3, :3] = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]) + s * np.eye(3)
    M[:3, 3] = v
    return M


def mat(g):
    """4x4 similarity [s R | t] of a Sim3 8-vector."""
    x, y, z, w = g[:4]
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    M = np.eye(4)
    M[:3, :3] = g[7] * R
    M[:3, 3] = g[4:7]
    return M


def project(cam, p):
    """cam_project of one point or of (..., 3) points."""
    p = np.asarray(p, np.float64)
    if cam["model"] == 1:
        th, ph = np.arctan2(p[..., 0], p[..., 2]), -np.arcsin(p[..., 1] / np.linalg.norm(p, axis=-1))
        return np.stack([cam["cols"] * (0.5 + th / (2 * np.pi)), cam["rows"] * (0.5 - ph / np.pi)], -1)
    return np.stack([cam["fx"] * p[..., 0] / p[..., 2] + cam["cx"], cam["fy"] * p[..., 1] / p[..., 2] + cam["cy"]], -1)


def np_error(M12, side, pc, cam, obs):
    """forward_reproj_edge / backward_reproj_edge::computeError with the Sim3 as a 4x4 matrix."""
    M = M12 if side == 0 else np.linalg.inv(M12)
    return np.asarray(obs, np.float32).astype(np.float64) - project(cam, (M @ np.append(pc, 1.0))[:3])


# ---------------------------------------------------------------------------------------------------------------------
# every edge of a problem
# ---------------------------------------------------------------------------------------------------------------------
def camera_points(pr):
    """(pc12, pc21): the camera-frame points of edge_12 (keyframe 2's frame, observed by camera 1) and edge_21 (keyframe 1's)."""
    pw2, pw1 = np.asarray(pr["pos_w_2"], np.float64).reshape(-1, 3), np.asarray(pr["pos_w_1"], np.float64).reshape(-1, 3)
    return pw2 @ np.asarray(pr["rot_2w"]).T + pr["trans_2w"], pw1 @ np.asarray(pr["rot_1w"]).T + pr["trans_1w"]


def weights(pr):
    """(n, 2) inv_sigma_sq of edge_12 and edge_21, float32 widened."""
    return np.stack([np.asarray(pr["inv_sigma_sq_1"], np.float32), np.asarray(pr["inv_sigma_sq_2"], np.float32)], 1).astype(np.float64)


def _points_at(pr, M, pcs=None):
    """(n, 2, 3): the points mapped by M (edge_12) and M^-1 (edge_21)."""
    pc12, pc21 = camera_points(pr) if pcs is None else pcs
    Mi = np.linalg.inv(M)
    return np.stack([pc12 @ M[:3, :3].T + M[:3, 3], pc21 @ Mi[:3, :3].T + Mi[:3, 3]], 1)


def errors(pr, M, pcs=None):
    """(n, 2, 2) errors of edge_12 and edge_21 at the Sim3 matrix M."""
    p = _points_at(pr, M, pcs)
    u = np.stack([project(pr["cam_1"], p[:, 0]), project(pr["cam_2"], p[:, 1])], 1)
    obs = np.stack([np.asarray(pr["obs_1"], np.float32), np.asarray(pr["obs_2"], np.float32)], 1).astype(np.float64)
    return obs - u


def edge_chi2(pr, S):
    """(n, 2) chi2 of both edges of every pair at the Sim3 8-vector S."""
    e = errors(pr, mat(S))
    return weights(pr) * (e * e).sum(-1)


def huber_delta(chi_sq):
    """transform_optimizer.cc:23: std::sqrt of the float chi_sq, in float, widened."""
    return float(np.sqrt(np.float32(chi_sq)))


def rho(chi, delta):
    return np.where(chi <= delta * delta, chi, 2 * np.sqrt(chi) * delta - delta * delta)


def rho_prime(chi, delta):
    return np.where(chi <= delta * delta, 1.0, delta / np.sqrt(np.maximum(chi, 1e-300)))


def robust_chi2(pr, S, active, chi_sq):
    """math.fsum of rho over both edges of the active pairs at S."""
    return math.fsum(rho(edge_chi2(pr, S)[np.asarray(active, bool)], huber_delta(chi_sq)).ravel())


def length_scale(pr):
    """The scene's length unit: the median distance of edge_12's points from keyframe 2's camera."""
    return float(np.median(np.linalg.norm(camera_points(pr)[0], axis=1)))


def _steps(pr, delta, length=None):
    """The stencil step of each update coordinate: delta for rotation and scale, delta times the scene's length unit for translation,
    so that the stencil sees the same relative perturbation whatever the units."""
    h = np.full(7, float(delta))
    h[3:6] *= length_scale(pr) if length is None else length
    return h


def _stencil_states(S, fix_scale, h):
    """[(d, weight, M)] of the perturbed states expm(hat(k h_d e_d)) mat(S) of the stencil."""
    M0 = mat(S)
    out = []
    for d in range(6 if fix_scale else 7):
        for c, k in STENCIL:
            u = np.zeros(7)
            u[d] = k * h[d]
            out.append((d, c, sl.expm(hat(u)) @ M0))
    return out


def jacobian(pr, S, fix_scale=False, delta=DELTA, length=None):
    """(n, 2, 2, 7): d error / d update of both edges of every pair, the fourth-order stencil at `delta` (translation: delta times
    length_scale) (column 6 zero under fix_scale).  The 28 perturbed states are shared by every edge."""
    pcs = camera_points(pr)
    h = _steps(pr, delta, length)
    J = np.zeros((len(pcs[0]), 2, 2, 7))
    for d, c, M in _stencil_states(S, fix_scale, h):
        J[..., d] += c * errors(pr, M, pcs) / (12 * h[d])
    return J


def oracle_jacobian(pr, S, fix_scale=False):
    """(n, 2, 2, 7) g2o's delta-1e-9 central difference, per edge from tests/transform_oracle.c."""
    import transform_oracle as TO
    pcs = camera_points(pr)
    w = weights(pr)
    obs = (np.asarray(pr["obs_1"], np.float32), np.asarray(pr["obs_2"], np.float32))
    cams = (pr["cam_1"], pr["cam_2"])
    J = np.zeros((len(pcs[0]), 2, 2, 7))
    for i in range(len(pcs[0])):
        for s in range(2):
            J[i, s] = TO.transform_jacobian(S, s, pcs[s][i], cams[s], obs[s][i], w[i, s], fix_scale)
    return J


def system(pr, S, active=None, fix_scale=False, chi_sq=10.0, delta=DELTA):
    """The robust system at S over the active pairs (default: all): dict(H (7x7 longdouble), b, chi2 (math.fsum of rho),
    n_beyond (active edges with chi2 > delta^2), S, active, fix_scale, chi_sq)."""
    n = len(pr["obs_1"])
    act = np.ones(n, bool) if active is None else np.asarray(active, bool)
    hd = huber_delta(chi_sq)
    e = errors(pr, mat(S))[act]
    chi = (weights(pr)[act] * (e * e).sum(-1))
    J = jacobian(_subset(pr, act), S, fix_scale, delta, length_scale(pr))
    ww = (weights(pr)[act] * rho_prime(chi, hd)).astype(LD)                       # (m, 2)
    JL = J.astype(LD)
    H = np.einsum("is,iska,iskb->ab", ww, JL, JL)
    b = -np.einsum("is,iska,isk->a", ww, JL, e.astype(LD))
    return dict(H=H, b=b, chi2=math.fsum(rho(chi, hd).ravel()), n_beyond=int((chi > hd * hd).sum()), S=np.asarray(S, np.float64),
                active=act, fix_scale=bool(fix_scale), chi_sq=chi_sq)


def _subset(pr, act):
    out = dict(pr)
    for k in ("obs_1", "inv_sigma_sq_1", "pos_w_2", "obs_2", "inv_sigma_sq_2", "pos_w_1"):
        out[k] = np.asarray(pr[k])[act]
    return out


def lambda_init(Sys):
    """computeLambdaInit: 1e-5 max |H_jj|."""
    return float(1e-5 * np.abs(np.diagonal(Sys["H"])).max())


def damped_matrix(Sys, lam):
    return damped(sp.csc_matrix(Sys["H"]), lam)


def solve(Sys, lam):
    """(H + lam I)^-1 b, exact to the float64 rounding of the result."""
    return exact_step(damped_matrix(Sys, lam), Sys["b"])


# ---------------------------------------------------------------------------------------------------------------------
# steps
# ---------------------------------------------------------------------------------------------------------------------
def _full(x, fix_scale):
    u = np.zeros(7)
    u[:len(x)] = x
    if fix_scale:
        u[6] = 0.0
    return u


def oplus(S0, x, fix_scale=False):
    """transform_vertex::oplusImpl: Sim3(x) * S0, x[6] zeroed under fix_scale, as the device evaluates it."""
    return PO.mul(PO.exp(_full(x, fix_scale)), S0)


def read_step(S0, S1, fix_scale=False, log_only=False):
    """The x with oplus(S0, x) == S1: Newton on pgo_oracle.exp, from g2o's log of S1 S0^-1, on the 12 entries of [s R | t] (the
    quaternions' sign does not matter).  log_only: g2o's log alone, whose first-order branch below theta ~ 4.5e-3 is off by about
    theta^2 / 6 relative."""
    x = PO.log(PO.mul(np.asarray(S1, np.float64), PO.inverse(S0)))
    if fix_scale:
        x[6] = 0.0
    if log_only:
        return x
    m = 6 if fix_scale else 7
    T = mat(S1)[:3].ravel()
    best = None
    for _ in range(12):
        r = T - mat(oplus(S0, x, fix_scale))[:3].ravel()
        nr = np.abs(r).max()
        if best is not None and nr >= best[0]:
            break
        best = (nr, x.copy())
        Jg = np.zeros((12, m))
        for d in range(m):
            h = 1e-7 * max(1.0, abs(x[d]))
            xp, xm = x.copy(), x.copy()
            xp[d] += h
            xm[d] -= h
            Jg[:, d] = (mat(oplus(S0, xp, fix_scale))[:3].ravel() - mat(oplus(S0, xm, fix_scale))[:3].ravel()) / (2 * h)
        x = x.copy()
        x[:m] += np.linalg.lstsq(Jg, r, rcond=None)[0]
        if nr == 0.0:
            break
    return best[1]


def judge(Sys, lam, S1):
    """dict(x, omega, forward, x_exact, A, kappa_bound, floor) of the step from the system's state to S1 at damping lam."""
    A = damped_matrix(Sys, lam)
    x_exact = exact_step(A, Sys["b"])
    x = read_step(Sys["S"], S1, Sys["fix_scale"])
    return dict(x=x, omega=backward_error(A, x.astype(LD), Sys["b"]), forward=rel(x, x_exact), x_exact=x_exact, A=A,
                kappa_bound=kappa_bound(A, lam), floor=floor(Sys, x_exact, A, S1))


def floor(Sys, x_exact, A, S1=None):
    """The backward error the rounding of the 8 exported doubles of the states before and after allows: the exact step applied to
    the start state in float64 and read back (one realisation), or the bound of both states off by one unit roundoff of (1 + |t|)
    in every tangent coordinate, whichever is larger."""
    S0 = Sys["S"]
    b = Sys["b"]
    x = read_step(S0, oplus(S0, x_exact, Sys["fix_scale"]), Sys["fix_scale"])
    one = backward_error(A, x.astype(LD), b)
    a_inf = float(abs(A).sum(axis=1).max())
    t = max(np.abs(S0[4:7]).max(), 0.0 if S1 is None else np.abs(np.asarray(S1)[4:7]).max())
    delta = 2 * U * (1.0 + t)
    bound = a_inf * delta / (a_inf * float(np.abs(x_exact).max()) + float(np.abs(np.asarray(b, np.float64)).max()))
    return max(one, bound)


def gain_ratio(Sys, lam, x, chi_new):
    """OptimizationAlgorithmLevenberg's rho: (chi2_old - chi2_new) / (x^T (lam x + b) + 1e-3)."""
    b = np.asarray(Sys["b"], np.float64)
    return (Sys["chi2"] - chi_new) / (math.fsum(x * (lam * x + b)) + 1e-3)


def lambda_factor(r):
    """The factor an accepted trial multiplies lambda by: max(1/3, min(2/3, 1 - (2 rho - 1)^3))."""
    return max(1.0 / 3.0, min(2.0 / 3.0, 1.0 - (2 * r - 1) ** 3))


# rho below RHO_LO gives the factor 2/3, above RHO_HI 1/3; between them the factor moves with rho
RHO_LO, RHO_HI = (1 + (1 / 3) ** (1 / 3)) / 2, (1 + (2 / 3) ** (1 / 3)) / 2


def on_clamp(r, margin=1e-3):
    """Is rho on the 1/3 or 2/3 clamp of lambda_factor with relative margin?"""
    return (0 < r and r * (1 + margin) < RHO_LO) or r > RHO_HI * (1 + margin)


def lm_round(pr, S, iters=5, active=None, fix_scale=False, chi_sq=10.0):
    """OptimizationAlgorithmLevenberg for `iters` iterations from S over the active pairs (default: all) with the reference's exact
    solves and chi2: tau 1e-5, g2o's rho rule with computeScale's +1e-3, at most 10 trials, a failed step ends the round.  Returns
    dict(S, last: the last trial state, iterations, trials, lambda_init, chi2, failed, states: S after each iteration)."""
    cur = np.asarray(S, np.float64).copy()
    last = cur
    lam, ni, trials, failed, states, chi = None, 2.0, 0, False, [], None
    it = 0
    for it in range(1, iters + 1):
        Sys = system(pr, cur, active, fix_scale, chi_sq)
        chi = Sys["chi2"]
        if lam is None:
            lam = lam0 = lambda_init(Sys)
        q = 0
        while True:
            x = solve(Sys, lam)
            last = oplus(cur, x, fix_scale)
            tchi = robust_chi2(pr, last, Sys["active"], chi_sq)
            trials += 1
            r = gain_ratio(Sys, lam, x, tchi)
            if r > 0 and math.isfinite(tchi):
                lam *= lambda_factor(r)
                ni = 2.0
                cur, chi = last, tchi
            else:
                lam *= ni
                ni *= 2.0
            q += 1
            if not (r < 0 and q < 10):
                break
        states.append(cur)
        if q == 10 or r == 0:
            failed = True
            break
    return dict(S=cur, last=last, iterations=it if iters > 0 else 0, trials=trials, lambda_init=lam0 if iters > 0 else 0.0, chi2=chi,
                failed=failed, states=states)


def gauss_newton(pr, S, active=None, fix_scale=False, chi_sq=10.0, tol=1e-13, max_iter=20):
    """Undamped Gauss-Newton on the reference system from S over the active pairs until the step's largest entry is under tol (or
    max_iter steps).  Under fix_scale the zero scale column gets a unit pivot.  Returns (S, chi2)."""
    S = np.asarray(S, np.float64).copy()
    for _ in range(max_iter):
        Sys = system(pr, S, active, fix_scale, chi_sq)
        H = Sys["H"].copy()
        if fix_scale:
            H[6, 6] = 1.0
        x = exact_step(sp.csc_matrix(H), Sys["b"])
        S = oplus(S, x, fix_scale)
        if np.abs(x).max() <= tol:
            break
    return S, system(pr, S, active, fix_scale, chi_sq)["chi2"]


def tangent_distance(Sa, Sb, fix_scale=False):
    """||x||_inf of the step from Sb to Sa."""
    return float(np.abs(read_step(Sb, Sa, fix_scale)).max())


# ---------------------------------------------------------------------------------------------------------------------
# equirectangular guards and the units device
# ---------------------------------------------------------------------------------------------------------------------
def guard(pr, S, fix_scale=False, delta=3e-4):
    """(seam, pole): per pair, does any equirectangular edge's stencil at `delta` (the coarsest the tests use) jump by more than
    cols / 2 (crosses the +-pi seam), or come within POLE_GUARD rad of a pole?"""
    pcs = camera_points(pr)
    n = len(pcs[0])
    seam, pole = np.zeros(n, bool), np.zeros(n, bool)
    cams = (pr["cam_1"], pr["cam_2"])
    if all(c["model"] != 1 for c in cams):
        return seam, pole
    p0 = _points_at(pr, mat(S), pcs)
    for _, _, M in _stencil_states(S, fix_scale, _steps(pr, delta)) + [(None, None, mat(S))]:
        p = _points_at(pr, M, pcs)
        for s in range(2):
            if cams[s]["model"] != 1:
                continue
            th0, th = np.arctan2(p0[:, s, 0], p0[:, s, 2]), np.arctan2(p[:, s, 0], p[:, s, 2])
            seam |= np.abs(th - th0) * cams[s]["cols"] / (2 * np.pi) > cams[s]["cols"] / 2
            pole |= np.pi / 2 - np.abs(np.arcsin(p[:, s, 1] / np.linalg.norm(p[:, s], axis=1))) < POLE_GUARD
    return seam, pole


def scaled(pr, f):
    """The problem with every translation multiplied by f: points, both keyframe translations and the Sim3's t (initial and true).
    Projections do not change; the translation columns of J grow by 1/f, so their delta-1e-9 noise falls by f."""
    out = dict(pr)
    for k in ("pos_w_1", "pos_w_2", "trans_1w", "trans_2w"):
        out[k] = np.asarray(pr[k], np.float64) * f
    for k in ("sim3_12", "gt_sim3_12"):
        if k in pr:
            g = np.array(pr[k], np.float64)
            g[4:7] *= f
            out[k] = g
    return out
