"""Global-BA maps at the scale of the panel-by-panel Cholesky (test infrastructure): a vectorised generator of multi-lap maps, whose
reduced system couples every keyframe with the keyframes that revisit its place, and an exact LM step for systems of up to 24 000
keyframe unknowns.

synth.make_ba_problem lays its keyframes on an open arc: no landmark is seen by keyframes more than a few dozen apart, so the reduced
matrix is a narrow band and every far tile of the trailing update subtracts zero.  Global BA runs after a loop closure, where the
keyframes of later laps observe the landmarks of the first.  `multi_lap_map` drives `laps` laps of a closed loop; keyframe i and the
keyframes K/laps and 2 K/laps later stand at the same place (with pose jitter) and observe the same landmarks with fresh noise.

`exact_step` solves H + lambda I of lba_reference.system through the Schur complement formed in float64 from the reference's
longdouble entries and factored densely by LAPACK, then refines against the full longdouble residual, which does not use the Schur
route.  sparse_lm.exact_step factors the full system with SuperLU instead; with far couplings its fill is the dense reduced block,
which takes hours at 24 000 unknowns."""
import math

import numpy as np
import scipy.linalg as sla
import scipy.sparse as sp
from scipy.sparse.csgraph import reverse_cuthill_mckee

import lba_reference as R
from workloads.synth import KITTI

U = 2.0 ** -53


def _rodrigues(w):
    """Rotation matrices (n, 3, 3) of the rotation vectors w (n, 3)."""
    th = np.linalg.norm(w, axis=1)
    k = w / np.where(th > 0, th, 1.0)[:, None]
    Kx = np.zeros((len(w), 3, 3))
    Kx[:, 0, 1], Kx[:, 0, 2], Kx[:, 1, 2] = -k[:, 2], k[:, 1], -k[:, 0]
    Kx = Kx - Kx.transpose(0, 2, 1)
    s, c = np.sin(th)[:, None, None], (1 - np.cos(th))[:, None, None]
    return np.eye(3) + s * Kx + c * Kx @ Kx


def _rot_y(a):
    c, s = np.cos(a), np.sin(a)
    out = np.zeros((len(a), 3, 3))
    out[:, 0, 0], out[:, 0, 2], out[:, 1, 1], out[:, 2, 0], out[:, 2, 2] = c, s, 1.0, -s, c
    return out


def _project(cam, pc):
    """(uv (n, 2), visible (n,)) of camera-frame points, with synth.make_ba_problem's visibility rules."""
    if cam["model"] == 1:
        L = np.linalg.norm(pc, axis=1)
        uv = np.stack([cam["cols"] * (0.5 + np.arctan2(pc[:, 0], pc[:, 2]) / (2 * np.pi)),
                       cam["rows"] * (0.5 + np.arcsin(pc[:, 1] / L) / np.pi)], 1)
        return uv, L > 2.0
    z = pc[:, 2]
    with np.errstate(divide="ignore", invalid="ignore"):
        uv = np.stack([cam["fx"] * pc[:, 0] / z + cam["cx"], cam["fy"] * pc[:, 1] / z + cam["cy"]], 1)
    vis = (z > 3.0) & (z < 80.0) & (uv[:, 0] > 0) & (uv[:, 0] < cam["cols"]) & (uv[:, 1] > 0) & (uv[:, 1] < cam["rows"])
    return uv, vis


def multi_lap_map(K, L, seed, model="stereo", laps=3, n_fixed=1, min_obs=3, max_obs=8, spacing=1.0, outlier_frac=0.05,
                  pixel_sigma=1.0):
    """K keyframes (the first n_fixed fixed: the spanning root, two for the monocular gauge) driving `laps` laps of a closed loop of
    P = ceil(K / laps) places `spacing` m apart, looking along the direction of travel; keyframe i stands at place i mod P.  About L
    landmarks, each placed 5..60 m in front of one place; on every lap it is observed by min_obs..max_obs consecutive keyframes at or
    behind that place (the loop wraps), each with its own level noise, stereo x_right (85 %) and gross outliers.  Landmarks left
    with fewer than two visible observations are dropped.  The layout, the noise model and the perturbation of the initial state are
    synth.make_ba_problem's, gt_* included."""
    rng = np.random.default_rng(seed)
    P = -(-K // laps)
    equirect = model == "equirect"
    cam = dict(model=1 if equirect else 0, fx=KITTI["fx"], fy=KITTI["fy"], cx=KITTI["cx"], cy=KITTI["cy"], fxb=KITTI["fxb"],
               cols=3840.0 if equirect else float(KITTI["cols"]), rows=1920.0 if equirect else float(KITTI["rows"]))
    radius = P * spacing / (2 * np.pi)
    place = np.arange(K) % P
    th = 2 * np.pi * place / P
    centers = np.stack([radius * np.sin(th), 0.3 * np.sin(place * spacing / 15.0), -radius * np.cos(th)], 1)
    centers[P:] += 0.1 * rng.standard_normal((K - P, 3)) / np.sqrt(3)       # a revisit stands near, not on, the first lap's spot
    # camera z along the direction of travel (cos th, 0, sin th), x outwards
    Rwc = _rot_y(np.pi / 2 - th + 0.02 * rng.standard_normal(K)) @ _rodrigues(0.01 * rng.standard_normal((K, 3)))
    gt_pose = np.zeros((K, 4, 4))
    gt_pose[:, :3, :3] = Rwc.transpose(0, 2, 1)
    gt_pose[:, :3, 3] = -np.einsum("kij,kj->ki", gt_pose[:, :3, :3], centers)
    gt_pose[:, 3, 3] = 1.0
    inv_sigma = (np.float32(1.0) / np.cumprod(np.concatenate([[np.float32(1.0)], np.full(7, np.float32(1.2))])).astype(np.float32) ** 2
                 ).astype(np.float32)
    sigma_lvl = 1.0 / np.sqrt(inv_sigma.astype(np.float64))
    # landmarks: back-projected from the first lap's keyframe at their place, as make_ba_problem samples them
    owner = rng.integers(0, P, L)
    depth = rng.uniform(5, 60, L)
    u = rng.uniform(0.05, 0.95, L) * (KITTI["cols"] if not equirect else 1241)
    v = rng.uniform(0.05, 0.95, L) * (KITTI["rows"] if not equirect else 376)
    pc = np.stack([(u - KITTI["cx"]) / KITTI["fx"] * depth, (v - KITTI["cy"]) / KITTI["fy"] * depth, depth], 1)
    To = gt_pose[owner]
    pts = np.einsum("lji,lj->li", To[:, :3, :3], pc - To[:, :3, 3])
    # observations: per lap, n consecutive keyframes starting 0..2 places behind the owner
    e_pose, e_point = [], []
    for lap in range(laps):
        n = rng.integers(min_obs, max_obs + 1, L)
        s0 = rng.integers(0, 3, L)
        lm = np.repeat(np.arange(L), n)
        j = s0[lm] + np.arange(len(lm)) - np.repeat(np.cumsum(n) - n, n)
        kf = lap * P + (owner[lm] - j) % P
        keep = kf < K
        e_pose.append(kf[keep])
        e_point.append(lm[keep])
    e_pose, e_point = np.concatenate(e_pose), np.concatenate(e_point)
    T = gt_pose[e_pose]
    pce = np.einsum("eij,ej->ei", T[:, :3, :3], pts[e_point]) + T[:, :3, 3]
    uv, vis = _project(cam, pce)
    e_pose, e_point, uv, pce = e_pose[vis], e_point[vis], uv[vis], pce[vis]
    deg = np.bincount(e_point, minlength=L)
    keep = deg[e_point] >= 2
    e_pose, e_point, uv, pce = e_pose[keep], e_point[keep], uv[keep], pce[keep]
    used = np.unique(e_point)
    e_point = np.searchsorted(used, e_point)
    order = np.lexsort((e_pose, e_point))                                    # landmark by landmark, keyframes ascending
    e_pose, e_point, uv, pce = e_pose[order], e_point[order], uv[order], pce[order]
    E = len(e_pose)
    lvl = rng.integers(0, 8, E)
    noise = pixel_sigma * sigma_lvl[lvl][:, None] * rng.standard_normal((E, 3))
    x, y = uv[:, 0] + noise[:, 0], uv[:, 1] + noise[:, 1]
    xr = np.full(E, -1.0)
    if model == "stereo":
        has = rng.random(E) < 0.85
        xr = np.where(has, uv[:, 0] - cam["fxb"] / pce[:, 2] + noise[:, 2], -1.0)
        xr[xr < 0] = -1.0
    out = rng.random(E) < outlier_frac
    x = x + out * rng.choice([-1.0, 1.0], E) * rng.uniform(15, 30, E)
    y = y + out * rng.choice([-1.0, 1.0], E) * rng.uniform(15, 30, E)
    chi = np.float32(np.sqrt(np.float32(5.99146))) if model != "stereo" else np.float32(np.sqrt(np.float32(7.81473)))
    pose_fixed = np.zeros(K, np.uint8)
    pose_fixed[:n_fixed] = 1
    pose0 = gt_pose.copy()
    free = np.nonzero(pose_fixed == 0)[0]
    Rn = _rodrigues(np.deg2rad(0.5) * rng.standard_normal((len(free), 3)) / np.sqrt(3)) @ gt_pose[free, :3, :3]
    cn = centers[free] + 0.05 * rng.standard_normal((len(free), 3)) / np.sqrt(3)
    pose0[free, :3, :3] = Rn
    pose0[free, :3, 3] = -np.einsum("kij,kj->ki", Rn, cn)
    pts = pts[used]
    pts0 = pts + 0.01 * depth[used][:, None] * rng.standard_normal((len(used), 3))
    return dict(pose_cw=pose0, pose_fixed=pose_fixed, points=pts0, point_fixed=None, e_pose=e_pose.astype(np.int32),
                e_point=e_point.astype(np.int32), e_cam=np.zeros(E, np.uint8), e_obs=np.stack([x, y, xr], 1).astype(np.float32),
                e_inv_sigma_sq=inv_sigma[lvl], e_delta=np.full(E, chi, np.float32), e_robust=None, e_can_be_outlier=None, cams=[cam],
                gt_pose_cw=gt_pose, gt_points=pts, laps=laps, places=P)


# the maps of tests/test_gba_scale_gpu.py: name -> (keyframes, landmarks, seed, model, fixed keyframes); about 15 landmarks per
# keyframe, n = 6 x free keyframes unknowns in the reduced system
MAPS = {
    "free500": (501, 7500, 501, "stereo", 1),            # n = 3 000; the CPU oracle runs as the control
    "free1000": (1001, 15000, 1001, "stereo", 1),        # n = 6 000: full last panel
    "free2047": (2048, 30700, 2047, "stereo", 1),        # n = 12 282: partial last panel (18 columns)
    "free3333": (3334, 50000, 3333, "stereo", 1),        # n = 19 998: trailing-update tile ids past 10.6 million, partial panel
    "free4000": (4001, 60000, 4000, "stereo", 1),        # n = 24 000: the limit; full panel; trailing-update grid past 65 535 CTAs
    "mono998": (1000, 15000, 998, "mono", 2),            # two fixed keyframes fix the monocular gauge; n = 5 988: partial panel
    "equirect1001": (1002, 15000, 1001, "equirect", 1),  # n = 6 006: partial panel (6 columns)
}


def named_map(name):
    K, L, seed, model, n_fixed = MAPS[name]
    return multi_lap_map(K, L, seed, model=model, n_fixed=n_fixed)


def huber_margin(pr, pose_cw, points):
    """Smallest relative distance |w |e|^2 - delta^2| / delta^2 of any edge's Huber decision from its threshold at a state."""
    err, _ = R.residuals(pr, pose_cw, points)
    e2, _, _ = R.edge_costs(pr, err, np.zeros(len(err), bool))
    d2 = np.asarray(pr["e_delta"], np.float32).astype(np.float64) ** 2
    return float(np.min(np.abs(e2 - d2) / d2))


def keyframe_blocks(pr):
    """The reduced system's nonzero keyframe blocks: (i, j) column pairs of free keyframes, i <= j, that share a landmark."""
    fixed = np.asarray(pr["pose_fixed"]).astype(bool)
    col = np.where(fixed, -1, np.cumsum(~fixed) - 1)[pr["e_pose"]]
    m = col >= 0
    Kf = int((~fixed).sum())
    inc = sp.csr_matrix((np.ones(m.sum()), (col[m], np.asarray(pr["e_point"])[m])), shape=(Kf, len(pr["points"])))
    co = sp.triu(inc @ inc.T).tocoo()
    return co.row, co.col, Kf


# ---------------------------------------------------------------------------------------------------------------------
# the exact step through a dense Schur complement
# ---------------------------------------------------------------------------------------------------------------------
class SchurSolver:
    """x = (H + lambda I)^-1 r for the system of lba_reference.system, in float64, through the keyframe Schur complement
    S = App - Apl All^-1 Alp, factored by LAPACK's banded Cholesky (scipy.linalg.cholesky_banded) after a reverse Cuthill-McKee
    reordering.  On a multi-lap map that ordering interleaves the laps place by place, so the band is a few hundred unknowns wide
    where the keyframe order's is the whole matrix: at n = 24 000 the factorisation takes a few seconds instead of the minutes a
    dense one (scipy.linalg.cho_factor) takes on 8 cores.  The band is measured from S's pattern, so any map is factored exactly."""

    def __init__(self, S, lam):
        A = R.damped(S["H"], lam)
        self.A, self.b, self.np_ = A, S["b"], S["n_pose"]
        A64 = A.astype(np.float64).tocsr()
        n, npo = A64.shape[0], self.np_
        Apl = A64[:npo, npo:].tocsr()
        All = A64[npo:, npo:].tocoo()
        nl = (n - npo) // 3
        D = np.zeros((nl, 3, 3))
        D[All.row // 3, All.row % 3, All.col % 3] = All.data                 # landmark blocks: block diagonal
        self.Dinv = sp.bsr_matrix((np.linalg.inv(D), np.arange(nl), np.arange(nl + 1)), shape=(n - npo, n - npo)).tocsr()
        self.Apl, self.W = Apl, (Apl @ self.Dinv).tocsr()
        Sr = (A64[:npo, :npo] - self.W @ Apl.T).tocsr()
        self.perm = reverse_cuthill_mckee(Sr, symmetric_mode=True)
        Sp = Sr[self.perm][:, self.perm].tocoo()
        low = Sp.row >= Sp.col                                                # (the lower triangle, as cho_factor(lower=True) reads)
        self.band = int((Sp.row - Sp.col)[low].max())
        ab = np.zeros((self.band + 1, npo))
        ab[(Sp.row - Sp.col)[low], Sp.col[low]] = Sp.data[low]
        self.chol = sla.cholesky_banded(ab, lower=True, overwrite_ab=True, check_finite=False)

    def solve(self, r):
        r = np.asarray(r, np.float64)
        rp, rl = r[:self.np_], r[self.np_:]
        xp = np.empty(self.np_)
        xp[self.perm] = sla.cho_solve_banded((self.chol, True), (rp - self.W @ rl)[self.perm], check_finite=False)
        return np.concatenate([xp, self.Dinv @ (rl - self.Apl.T @ xp)])


def exact_step(S, lam, min_refine=1, max_refine=4, target=U):
    """(x, omegas): the Schur solve of (H + lambda I) x = b refined against the full longdouble residual -- at least min_refine
    times (sparse_lm.exact_step refines once), then until its normwise backward error is at most `target` or after max_refine
    refinement steps; omegas[k] is the backward error after k refinements."""
    sv = SchurSolver(S, lam)
    a_inf, b_inf = abs(sv.A).sum(axis=1).max(), np.abs(S["b"]).max()
    x = sv.solve(S["b"])
    omegas = []
    for k in range(max_refine + 1):
        r = S["b"] - sv.A @ x.astype(R.LD)                                    # (sparse_lm.backward_error, without a second product)
        omegas.append(float(np.abs(r).max() / (a_inf * np.abs(x).max() + b_inf)))
        if (k >= min_refine and omegas[-1] <= target) or k == max_refine:
            break
        x = x + sv.solve(r)
    return x, omegas


class LandmarksFirstLU:
    """Sparse LU (SuperLU) of A with the landmark unknowns eliminated first and no fill-reducing reordering: the same factorisation
    family as sparse_lm.factor, which on multi-lap maps orders so badly that 3 000 keyframe unknowns take minutes.  Passed as `lu` to
    sparse_lm.exact_step."""

    def __init__(self, A, n_pose):
        import scipy.sparse.linalg as spl
        n = A.shape[0]
        self.perm = np.concatenate([np.arange(n_pose, n), np.arange(n_pose)])
        Ap = A.astype(np.float64).tocsr()[self.perm][:, self.perm].tocsc()
        self.lu = spl.splu(Ap, permc_spec="NATURAL", diag_pivot_thresh=0.0, options=dict(SymmetricMode=True))

    def solve(self, r):
        x = np.empty(len(self.perm))
        x[self.perm] = self.lu.solve(np.asarray(r, np.float64)[self.perm])
        return x
