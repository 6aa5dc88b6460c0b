"""High-precision reference of one pose-graph LM step (test infrastructure).

The linear system g2o's Levenberg-Marquardt solves for optimize::graph_optimizer, H x = b with H = J^T J and b = -J^T e over the free
vertices, built in float64 from an accurate Jacobian instead of g2o's central difference at delta 1e-9: a fourth-order central stencil
at delta 1e-4 on the oracle's edge error (tests/pgo_oracle.c, orc_graph_linearize), assembled as a scipy.sparse matrix in the free-vertex
order of b200_pgo_envelope (reverse Cuthill-McKee).  An implementation's step is read back from its output estimate, a solve is judged
by its normwise backward error against this system, and its forward error against the system's exact solution (splu plus one step of
iterative refinement) is bounded through the condition number."""
import math

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spl

import pgo_oracle as O
from sparse_lm import backward_error, damped, exact_step, factor, kappa_bound, rel  # noqa: F401

DELTA, STENCIL = 1e-4, 4


def scaled(graph, f):
    """The graph with every translation (estimates, measurements, landmarks) multiplied by f: the same topology, order and envelope,
    and the same rotation and scale parts of every error; only the translation parts of the errors scale by f."""
    est = np.array(graph["estimate"], np.float64).reshape(-1, 8)
    meas = np.array(graph["e_meas"], np.float64).reshape(-1, 8)
    est[:, 4:7] *= f
    meas[:, 4:7] *= f
    pts = np.asarray(graph.get("points", np.zeros((0, 3))), np.float64) * f
    return dict(graph, estimate=est, e_meas=meas, points=pts)


# g2o's Sim3 log switches to first-order formulas for |sigma| < 1e-5 and rotation angles under about 4.5e-3; a stencil that straddles
# either switch differentiates a different function than g2o's delta-1e-9 difference does.  The loops keep their residuals near zero
# (dead-reckoned estimates, measurements taken from them), and the chains and grids below carry noise in the translations only, with
# fixed scale, so every rotation and scale residual stays on one side of both switches.
def chain_graph(nf, seed, reach=3):
    """A fixed root and nf free keyframes 1 m apart along a gently turning track, each joined to the `reach` keyframes before it, with
    fixed scale.  The estimates drift in translation (dead reckoning); the measurements are the true relative Sim3s with 1e-2 m noise.
    7 nf mod 32 sets how many padding rows the last 32x32 tile of the envelope has."""
    rng = np.random.default_rng(seed)
    true = [O.exp(np.array([0.0, 0.01 * i, 0.0, 0.0, 0.0, -float(i), 0.0])) for i in range(nf + 1)]
    drift, est = np.zeros(7), []
    for i in range(nf + 1):
        est.append(O.mul(O.exp(drift), true[i]))
        drift[3:6] += 1e-2 * rng.standard_normal(3)
    e1, e2, meas = [], [], []
    for i in range(1, nf + 1):
        for j in range(max(0, i - reach), i):
            noise = np.zeros(7)
            noise[3:6] = 1e-2 * rng.standard_normal(3)
            e1.append(i)
            e2.append(j)
            meas.append(O.mul(O.exp(noise), O.mul(true[j], O.inverse(true[i]))))
    fixed = np.zeros(nf + 1, np.uint8)
    fixed[0] = 1
    return dict(estimate=np.array(est), fixed=fixed, e_v1=np.array(e1, np.int32), e_v2=np.array(e2, np.int32), e_meas=np.array(meas),
                fix_scale=True, points=np.zeros((0, 3)), point_ref=np.zeros(0, np.int32))


def noisy(graph, seed, sigma=1e-2):
    """The graph with fixed scale and every measurement's translation moved by Gaussian noise (sigma per component)."""
    rng = np.random.default_rng(seed)
    meas = np.array(graph["e_meas"], np.float64).reshape(-1, 8).copy()
    meas[:, 4:7] += sigma * rng.standard_normal((len(meas), 3))
    return dict(graph, e_meas=meas, fix_scale=True)


def positions(graph):
    """vertex -> position in the free-vertex order (-1 for a fixed vertex), and the order itself."""
    order = O.rcm(graph)[0]
    pos = -np.ones(len(graph["estimate"]), np.int64)
    pos[order] = np.arange(len(order))
    return pos, order


def jacobian_matrix(graph, J, pos):
    """The (7 m) x (7 nf) sparse Jacobian of the per-edge blocks J (m,2,7,7)."""
    ne = len(J)
    cols_v = np.stack([pos[np.asarray(graph["e_v1"])], pos[np.asarray(graph["e_v2"])]], 1)         # (m, 2)
    e, s, r, d = np.meshgrid(np.arange(ne), np.arange(2), np.arange(7), np.arange(7), indexing="ij")
    keep = cols_v[e, s] >= 0
    rows = (7 * e + r)[keep]
    cols = (7 * cols_v[e, s] + d)[keep]
    return sp.csr_matrix((J[keep], (rows, cols)), shape=(7 * ne, 7 * int((pos >= 0).sum())))


def system(graph, delta=DELTA, stencil=STENCIL):
    """dict(H (csc), b, chi2 (math.fsum of e^T e), err, J (m,2,7,7), pos, order) at the graph's estimate."""
    pos, order = positions(graph)
    err, J = O.graph_linearize(graph, delta, stencil)
    Jm = jacobian_matrix(graph, J, pos)
    H = (Jm.T @ Jm).tocsc()
    b = -(Jm.T @ err.ravel())
    return dict(H=H, b=b, chi2=math.fsum((err * err).ravel()), err=err, J=J, pos=pos, order=order)


def block_error(J, Jref):
    """Max over the 7x7 blocks of max |J - Jref| / max |Jref| (blocks of fixed vertices, all zero, skipped)."""
    Jr = Jref.reshape(-1, 49)
    J = J.reshape(-1, 49)
    m = np.abs(Jr).max(1)
    nz = m > 0
    return float((np.abs(J - Jr).max(1)[nz] / m[nz]).max())


def step(graph, est_out, order, near=None):
    """The LM step an implementation took, per free vertex x_v = log(est_out_v est_v^-1) (oplus is left multiplication by exp(x)),
    in position order.  log returns rotations of at most pi, and a first LM step can turn a vertex further (the drifted 4 000-keyframe
    loop with fixed scale, the noisy grids).  exp(x) is the same Sim3 for omega + 2 pi k omega / |omega|, with upsilon solved again
    through that rotation's V matrix; with `near` (a step in the same order) each vertex takes the k in {-1, 0, 1} whose rotation is
    nearest near's."""
    est = np.asarray(graph["estimate"], np.float64).reshape(-1, 8)
    x = np.zeros(7 * len(order))
    for p, v in enumerate(order):
        D = O.mul(est_out[v], O.inverse(est[v]))
        u = O.log(D)
        th = np.linalg.norm(u[:3])
        if near is not None and th > 0.0:
            want = near[7 * p:7 * p + 3]
            cands = [u[:3] * (1 + 2 * np.pi * k / th) for k in (-1, 0, 1)]
            w = min(cands, key=lambda c: np.linalg.norm(c - want))
            if w is not cands[1]:
                V = np.stack([O.exp(np.concatenate([w, np.eye(3)[i], u[6:]]))[4:7] for i in range(3)], 1)
                u = np.concatenate([w, np.linalg.solve(V, D[4:7]), u[6:]])
        x[7 * p:7 * p + 7] = u
    return x


def kappa(A):
    """2-norm condition number of the SPD matrix A by eigsh (largest, and smallest by shift-invert at 0): for small graphs."""
    hi = spl.eigsh(A, k=1, which="LA", return_eigenvectors=False, tol=1e-6)[0]
    lo = spl.eigsh(A, k=1, sigma=0, which="LM", return_eigenvectors=False, tol=1e-6)[0]
    return float(hi / lo)


def gauss_newton(graph, est=None, tol=1e-10, max_iter=12):
    """Gauss-Newton on the reference system from `est` (default: the graph's estimate) until the step's largest entry is under tol
    times max(1, largest |t|) -- rounding of edge_error keeps it above about 5e-11 -- or max_iter steps.  Undamped steps diverge from
    the drifted estimates at the graphs' own units, so there it starts from a converged LM estimate.  Returns (estimate, chi2)."""
    est = np.array(graph["estimate"] if est is None else est, np.float64).reshape(-1, 8).copy()
    for _ in range(max_iter):
        S = system(dict(graph, estimate=est))
        d = S["H"].diagonal()
        x = exact_step((S["H"] + sp.diags((d == 0).astype(np.float64))).tocsc(), S["b"])  # fixed scale: unit pivot on the zero column
        for p, v in enumerate(S["order"]):
            est[v] = O.mul(O.exp(x[7 * p:7 * p + 7]), est[v])
        if np.abs(x).max() <= tol * max(1.0, np.abs(est[:, 4:7]).max()):
            break
    return est, system(dict(graph, estimate=est))["chi2"]


# The graphs the precision tests solve: the drifted loops of tests/test_pgo_gpu.py's large-graph cases (500 to 4 000 keyframes, free
# and fixed scale), its 2.5-lap revisit graph, chains whose 7 nf mod 32 is 0, 1 and 31 (no padding row, 31 and 1 padding rows in the
# last tile), and noisy grids: 96 x 40 (small enough for the CPU oracle) and 96 x 576 (noise 1e-3), whose envelope is within 0.1 % of
# B200_PGO_MAX_ENVELOPE_DOUBLES -- the longest active-row lists and the largest update grids the entry point accepts.
CASES = {
    "loop500": lambda: _synth().make_pose_graph(500, seed=3),
    "loop2000": lambda: _synth().make_pose_graph(2000, seed=5),
    "loop4000_fixed_scale": lambda: _synth().make_pose_graph(4000, seed=6, fix_scale=True),
    "loop4000": lambda: _synth().make_pose_graph(4000, seed=7),
    "revisit1200": lambda: _synth().make_pose_graph(1200, seed=8, laps=2.5),
    "chain_pad0": lambda: chain_graph(320, seed=1),
    "chain_pad31": lambda: chain_graph(311, seed=2),
    "chain_pad1": lambda: chain_graph(297, seed=3),
    "grid96x40": lambda: noisy(_grid(96, 40), seed=4),
    "grid96x576": lambda: noisy(_grid(96, 576), seed=5, sigma=1e-3),
}


def _synth():
    from workloads import synth
    return synth


def _grid(w, h):
    from test_pgo_gpu import _grid_graph
    return _grid_graph(w, h)
