"""Local-BA windows and pose-optimiser frames shaped like real tracking, in the flattened layout of synth.make_ba_problem /
synth.make_pose_problem (the C ABI's b200_lba_problem_t), plus an independent numpy restatement of their residuals.

workloads/synth builds one kind of window: one camera, every landmark seen 4..8 times, every point well in front of every camera.
Real monocular windows are different, and these generators mix what the synthetic ones never have:
  - the observation counts of a real window: mostly landmarks fresh from two-view triangulation (2 observations), some with a
    single observation (a rank-2 landmark block in a free keyframe: only lambda makes it invertible), a few long-lived ones seen
    by every keyframe, and, in a long window, degrees 64 and 65 (one 64-bit keyframe mask word and the next);
  - several cameras in one window, one per keyframe (KITTI stereo, EuRoC-like mono, equirectangular), so e_cam varies per edge
    and mono edges (x_right < 0) sit inside stereo keyframes;
  - points behind one observing camera (observed where the projection puts them, so the chi-square test passes and only the
    depth test can reject them), points at 0.3 m and at 1-2 km (sub-pixel stereo disparity), equirectangular points a few
    degrees from a pole and a few pixels from the +-pi seam;
  - a free keyframe with no observation at all and one that looks backwards, so that the depth test rejects every one of its
    observations after the first round.

`decision_margins` measures how far every accept/reject decision of a state lies from its threshold; the tests require 1e-9
(relative) so that FMA contraction on the device or 1-ulp libm differences cannot flip one."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_lba_scipy import Problem  # noqa: E402
from workloads.synth import KITTI  # noqa: E402

CAMS = {
    "kitti": dict(model=0, fx=KITTI["fx"], fy=KITTI["fy"], cx=KITTI["cx"], cy=KITTI["cy"], fxb=KITTI["fxb"], cols=float(KITTI["cols"]),
                  rows=float(KITTI["rows"])),
    # EuRoC MAV cam0 (example/euroc/EuRoC_mono.yaml): mono, different intrinsics and image size
    "euroc": dict(model=0, fx=458.654, fy=457.296, cx=367.215, cy=248.375, fxb=0.0, cols=752.0, rows=480.0),
    "equirect": dict(model=1, fx=0.0, fy=0.0, cx=0.0, cy=0.0, fxb=0.0, cols=3840.0, rows=1920.0),
}
THR_2D, THR_3D = float(np.float32(5.99146)), float(np.float32(7.81473))   # constexpr float chi_sq_2D / chi_sq_3D
INV_SIGMA_SQ = (np.float32(1.0) / np.cumprod(np.concatenate([[np.float32(1.0)], np.full(7, np.float32(1.2))])).astype(np.float32) ** 2
                ).astype(np.float32)
MARGIN = 1e-9


def _rodrigues(w):
    """Rotation matrix of the rotation vector w."""
    th = np.linalg.norm(w)
    if th < 1e-12:
        return np.eye(3)
    k = w / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def project(cam, pc):
    """Pixel coordinates (n, 2) of camera-frame points under one camera (no visibility test)."""
    if cam["model"] == 1:
        th = np.arctan2(pc[:, 0], pc[:, 2])
        ph = -np.arcsin(pc[:, 1] / np.linalg.norm(pc, axis=1))
        return np.stack([cam["cols"] * (0.5 + th / (2 * np.pi)), cam["rows"] * (0.5 - ph / np.pi)], 1)
    return np.stack([cam["fx"] * pc[:, 0] / pc[:, 2] + cam["cx"], cam["fy"] * pc[:, 1] / pc[:, 2] + cam["cy"]], 1)


def thresholds(pr):
    """Chi-square threshold of every edge, chosen by x_right like the reference (mono / equirectangular: 2D, stereo: 3D)."""
    return np.where(pr["e_obs"][:, 2] >= 0, THR_3D, THR_2D)


class WindowProblem(Problem):
    """test_lba_scipy.Problem with a camera per edge (e_cam into cams)."""

    def edge_chi2(self, T, P, sel):
        pr = self.pr
        ep, el, obs = pr["e_pose"][sel], pr["e_point"][sel], pr["e_obs"][sel].astype(np.float64)
        cams = np.asarray(pr["e_cam"])[sel]
        pc = np.einsum("eij,ej->ei", T[ep, :3, :3], P[el]) + T[ep, :3, 3]
        e = np.zeros((len(ep), 3))
        for ci, cam in enumerate(pr["cams"]):
            m = cams == ci
            if not m.any():
                continue
            uv = project(cam, pc[m])
            e[m, 0], e[m, 1] = obs[m, 0] - uv[:, 0], obs[m, 1] - uv[:, 1]
            if cam["model"] != 1:
                xr = obs[m, 2] - (uv[:, 0] - cam["fxb"] / pc[m, 2])
                e[m, 2] = np.where(obs[m, 2] >= 0, xr, 0.0)
        return (e * e).sum(1) * pr["e_inv_sigma_sq"][sel].astype(np.float64), pc

    def robust_cost(self, T, P, sel):
        chi, _ = self.edge_chi2(T, P, sel)
        rob = np.ones(len(chi), bool) if self.pr.get("e_robust") is None else np.asarray(self.pr["e_robust"])[sel].astype(bool)
        return np.where(rob, self.huber(chi, sel), chi).sum()

    def outlier_test(self, T, P, chi=None):
        """(chi2 > threshold) | (non-positive depth, perspective edges only) for every edge; chi: the chi2 to test (default: at T, P)."""
        every = np.ones(len(self.pr["e_pose"]), bool)
        c, pc = self.edge_chi2(T, P, every)
        chi = c if chi is None else chi
        persp = np.array([self.pr["cams"][i]["model"] != 1 for i in self.pr["e_cam"]], bool)
        o = (chi > thresholds(self.pr)) | (persp & (pc[:, 2] <= 0))
        if self.pr.get("e_can_be_outlier") is not None:
            o &= np.asarray(self.pr["e_can_be_outlier"]).astype(bool)
        return o


def decision_margins(pr, T, P, depth_test=True):
    """Smallest relative distance of any decision at state (T, P) from its threshold: chi2 against the chi-square threshold, the depth
    of perspective edges against 0 (depth_test), and x_c against 0 for equirectangular edges behind the camera (the sign flip of
    atan2 at the +-pi seam).  Returns a dict name -> margin."""
    wp = WindowProblem(pr)
    every = np.ones(len(pr["e_pose"]), bool)
    chi, pc = wp.edge_chi2(T, P, every)
    thr = thresholds(pr)
    equi = np.array([pr["cams"][i]["model"] == 1 for i in pr["e_cam"]], bool)
    L = np.linalg.norm(pc, axis=1)
    out = dict(chi2=float(np.min(np.abs(chi - thr) / thr)) if len(chi) else np.inf)
    if depth_test and (~equi).any():
        out["depth"] = float(np.min(np.abs(pc[~equi, 2]) / L[~equi]))
    seam = equi & (pc[:, 2] < 0)
    if seam.any():
        out["seam"] = float(np.min(np.abs(pc[seam, 0]) / L[seam]))
    return out


def assert_clear_of_thresholds(pr, T, P, depth_test=True):
    m = decision_margins(pr, T, P, depth_test)
    assert min(m.values()) > MARGIN, m


# ---------------------------------------------------------------------------------------------------------------------
# local-BA windows
# ---------------------------------------------------------------------------------------------------------------------
def _visible(cam, pc):
    if cam["model"] == 1:
        return np.linalg.norm(pc, axis=1) > 0.2
    z = pc[:, 2]
    with np.errstate(divide="ignore", invalid="ignore"):
        uv = project(cam, pc)
    return (z > 0.2) & (uv[:, 0] > 8) & (uv[:, 0] < cam["cols"] - 8) & (uv[:, 1] > 8) & (uv[:, 1] < cam["rows"] - 8)


def make_window(seed, n_kf=10, n_fixed=2, n_points=200, cams=("kitti", "euroc", "equirect"), degrees=None, deep_degrees=(),
                n_near=4, n_far=6, n_behind=6, n_pole=4, n_seam=4, empty_kf=True, outlier_kf=True, outlier_frac=0.04, spacing=0.6):
    """One local-BA window.  Keyframes move forward along +z, `spacing` m apart, camera i % len(cams) on keyframe i (oldest n_fixed
    keyframes fixed).  degrees: {observation count: probability} of the ordinary landmarks ("all" = every keyframe that sees it);
    deep_degrees: extra far landmarks observed by exactly that many keyframes.  The returned dict has synth.make_ba_problem's keys
    plus `behind` (edges whose point lies behind their camera), `empty_kf` / `outlier_kf` (keyframe ids or -1) and `kinds` (per landmark)."""
    rng = np.random.default_rng(seed)
    cam_list = [CAMS[c] for c in cams]
    K = n_kf
    cam_of = np.arange(K) % len(cams)
    if degrees is None:
        degrees = {1: 0.10, 2: 0.62, 3: 0.12, 4: 0.06, 6: 0.05, "all": 0.05}
    free = np.arange(n_fixed, K)
    empty = int(free[len(free) // 2]) if empty_kf else -1          # a free keyframe that observes nothing
    bad_kf = -1      # a free keyframe looking backwards: every landmark it observes lies behind it, so the depth test rejects them all
    if outlier_kf:
        bad_kf = int([k for k in free[::-1] if k != empty and cam_list[cam_of[k]]["model"] == 0][0])
    centers = np.stack([0.2 * np.sin(0.7 * np.arange(K)), 0.05 * np.cos(1.3 * np.arange(K)), spacing * np.arange(K)], 1)
    gt = np.zeros((K, 4, 4))
    for k in range(K):
        Rcw = _rodrigues(0.02 * rng.standard_normal(3)).T
        if k == bad_kf:
            Rcw = np.diag([-1.0, 1.0, -1.0]) @ Rcw
        gt[k, :3, :3], gt[k, :3, 3], gt[k, 3, 3] = Rcw, -Rcw @ centers[k], 1.0

    def to_world(k, pc):
        return (pc - gt[k, :3, 3]) @ gt[k, :3, :3]          # R^T (pc - t)

    def cam_pts(k, pw):
        return pw @ gt[k, :3, :3].T + gt[k, :3, 3]

    def in_frustum(k, depth, n):
        # a direction inside keyframe k's image (KITTI-like field of view for the equirectangular keyframes, so every landmark is
        # a candidate for its perspective neighbours)
        cam = cam_list[cam_of[k]] if cam_list[cam_of[k]]["model"] == 0 else CAMS["kitti"]
        u, v = rng.uniform(0.1, 0.9, n) * cam["cols"], rng.uniform(0.1, 0.9, n) * cam["rows"]
        return np.stack([(u - cam["cx"]) / cam["fx"] * depth, (v - cam["cy"]) / cam["fy"] * depth, depth], 1)

    pts, want, kinds = [], [], []
    anchor = {}                                               # landmark -> the keyframe it was placed for (observed first)
    keys = list(degrees)
    probs = np.array([degrees[k] for k in keys], np.float64)
    for _ in range(n_points):
        k0 = int(rng.integers(0, K))
        d = float(rng.uniform(3.0, 40.0))
        pts.append(to_world(k0, in_frustum(k0, np.array([d]), 1))[0])
        want.append(keys[rng.choice(len(keys), p=probs / probs.sum())])
        kinds.append("ordinary")
    for _ in range(n_near):                                   # 0.3 m in front of a keyframe
        k0 = int(rng.integers(1, K))
        pc = np.array([rng.uniform(-0.02, 0.02), rng.uniform(-0.02, 0.02), 0.3])
        pts.append(to_world(k0, pc)); want.append(2); kinds.append("near")
    for _ in range(n_far):                                    # 1-2 km: sub-pixel stereo disparity
        k0 = int(rng.integers(0, K))
        pts.append(to_world(k0, in_frustum(k0, np.array([rng.uniform(1000, 2000)]), 1)[0]))
        want.append("all" if rng.random() < 0.5 else 2); kinds.append("far")
    for dd in deep_degrees:                                   # long-lived: exactly dd observers
        pts.append(to_world(0, np.array([rng.uniform(-2, 2), rng.uniform(-1, 1), spacing * K + rng.uniform(30, 60)])))
        want.append(dd); kinds.append("deep")
    equi_kf = [k for k in range(K) if cam_list[cam_of[k]]["model"] == 1 and k != empty]
    for i in range(n_pole if equi_kf else 0):                 # 2-4 degrees from a pole
        k0 = equi_kf[int(rng.integers(0, len(equi_kf)))]
        el, az = np.deg2rad(rng.uniform(86, 88)), rng.uniform(-np.pi, np.pi)
        dirn = np.array([np.cos(el) * np.sin(az), (1 if i % 2 else -1) * np.sin(el), np.cos(el) * np.cos(az)])
        anchor[len(pts)] = k0
        pts.append(to_world(k0, dirn * rng.uniform(6, 15))); want.append(2); kinds.append("pole")
    for i in range(n_seam if equi_kf else 0):                 # 4-10 px from the +-pi seam, on either side
        k0 = equi_kf[int(rng.integers(0, len(equi_kf)))]
        th = (np.pi - rng.uniform(4, 10) * 2 * np.pi / CAMS["equirect"]["cols"]) * (1 if i % 2 else -1)
        ph = rng.uniform(-0.3, 0.3)
        dirn = np.array([np.cos(ph) * np.sin(th), -np.sin(ph), np.cos(ph) * np.cos(th)])
        anchor[len(pts)] = k0
        pts.append(to_world(k0, dirn * rng.uniform(8, 20))); want.append(1); kinds.append("seam")
    pts = np.array(pts)
    L = len(pts)
    proj = [cam_pts(k, pts) for k in range(K)]
    vis = np.stack([_visible(cam_list[cam_of[k]], proj[k]) for k in range(K)], 1)      # (L, K)
    e_pose, e_point, e_obs, e_isq, e_cam = [], [], [], [], []

    def add_edge(k, l, noise_px=1.0, stereo_ok=True):
        cam = cam_list[cam_of[k]]
        pc = proj[k][l]
        uv = project(cam, pc[None])[0]
        lvl = int(rng.integers(0, 8))
        sig = noise_px / np.sqrt(float(INV_SIGMA_SQ[lvl]))
        x, y = uv + sig * rng.standard_normal(2)
        xr = -1.0
        if stereo_ok and cam["fxb"] > 0 and pc[2] > 0 and rng.random() < 0.7:
            xr = uv[0] - cam["fxb"] / pc[2] + sig * rng.standard_normal()
            xr = xr if xr >= 0 else -1.0
        e_pose.append(k); e_point.append(l); e_obs.append((x, y, xr)); e_isq.append(INV_SIGMA_SQ[lvl]); e_cam.append(cam_of[k])

    vis[:, empty if empty >= 0 else []] = False
    if bad_kf >= 0:      # observed where the projection puts the points behind it (x / z and y / z do not change sign)
        vis[:, bad_kf] = _visible(cam_list[cam_of[bad_kf]], -proj[bad_kf])
    for l in range(L):
        seen = np.nonzero(vis[l])[0]
        if len(seen) == 0:
            continue
        # nearest keyframes first, from a random one that sees the landmark (long-lived landmarks: from the newest keyframe back)
        k0 = seen[int(rng.integers(0, len(seen)))] if kinds[l] != "deep" else seen[-1]
        if vis[l, anchor.get(l, 0)] and l in anchor:    # polar / seam points: seen where they were placed
            k0 = anchor[l]
        order = seen[np.argsort(np.abs(seen - k0), kind="stable")]
        n = len(order) if want[l] == "all" else min(int(want[l]), len(order))
        chosen = list(order[:n])
        if bad_kf in chosen and n - 1 < 2:      # the outlier keyframe's landmarks have two good observations that pin them
            chosen = [k for k in order if k != bad_kf][:2]
            chosen += [bad_kf] if len(chosen) == 2 else []
        for k in chosen:
            add_edge(k, l)
    # points behind a camera: a landmark between two keyframes, seen normally from behind it and, from a free perspective keyframe
    # it lies behind, exactly where that keyframe's projection puts it (chi2 small, depth negative: only the depth test rejects it)
    behind = []
    persp_free = [k for k in free if cam_list[cam_of[k]]["model"] == 0 and k not in (empty, bad_kf)]
    for _ in range(n_behind if persp_free else 0):
        kb = persp_free[int(rng.integers(0, len(persp_free)))]
        ka = [k for k in range(K) if centers[k, 2] <= centers[kb, 2] - 2.5 * spacing]
        if not ka:
            continue
        ka = ka[-1]
        gap = centers[kb, 2] - centers[ka, 2]
        pc_a = np.array([rng.uniform(-0.3, 0.3), rng.uniform(-0.2, 0.2), rng.uniform(0.3, 0.6) * gap])
        pw = to_world(ka, pc_a)
        pts = np.vstack([pts, pw])
        l = len(pts) - 1
        for k in range(K):
            proj[k] = np.vstack([proj[k], cam_pts(k, pw[None])])
        kinds.append("behind")
        front = [k for k in range(K) if k not in (empty, bad_kf) and _visible(cam_list[cam_of[k]], proj[k][l:l + 1])[0]]
        for k in sorted(front, key=lambda k: abs(k - ka))[:2]:
            add_edge(k, l)
        assert proj[kb][l, 2] < -0.3
        behind.append(len(e_pose))
        add_edge(kb, l, noise_px=0.3, stereo_ok=False)
    L = len(pts)
    e_pose, e_point = np.array(e_pose, np.int32), np.array(e_point, np.int32)
    e_obs, e_isq, e_cam = np.array(e_obs, np.float64), np.array(e_isq, np.float32), np.array(e_cam, np.uint8)
    E = len(e_pose)
    gross = (rng.random(E) < outlier_frac) & (e_pose != bad_kf)
    gross[behind] = False
    gross &= ~np.isin(e_point, [l for l, kind in enumerate(kinds) if kind == "seam"])   # seam edges stay near the seam
    e_obs[gross, 0] += rng.choice([-1, 1], gross.sum()) * rng.uniform(15, 30, gross.sum())
    e_obs[gross, 1] += rng.choice([-1, 1], gross.sum()) * rng.uniform(15, 30, gross.sum())
    used = np.unique(e_point)                                      # landmarks nobody observes are not part of a window
    pts, kinds = pts[used], np.asarray(kinds)[used]
    e_point = np.searchsorted(used, e_point).astype(np.int32)
    L = len(pts)
    behind = np.array(behind, np.int64)
    e_obs = e_obs.astype(np.float32)
    delta = np.where(e_obs[:, 2] >= 0, np.float32(np.sqrt(np.float32(7.81473))), np.float32(np.sqrt(np.float32(5.99146)))).astype(np.float32)
    pose_fixed = np.zeros(K, np.uint8)
    pose_fixed[:n_fixed] = 1
    pose0 = gt.copy()
    for k in range(n_fixed, K):                                # 0.3 deg about the centre, 3 cm of centre noise
        dR = _rodrigues(np.deg2rad(0.3) * rng.standard_normal(3) / np.sqrt(3))
        Rn = dR @ gt[k, :3, :3]
        pose0[k, :3, :3], pose0[k, :3, 3] = Rn, -Rn @ (centers[k] + 0.03 * rng.standard_normal(3) / np.sqrt(3))
    depth = np.linalg.norm(pts[:, None, :] - centers[None], axis=2).min(1)   # to the nearest keyframe
    # 0.3 % of the depth; a tenth of that for the polar and seam points, whose azimuth moves by radians per metre
    scale = np.where(np.isin(kinds, ("pole", "seam")), 0.0003, 0.003)
    pts0 = pts + (scale * depth)[:, None] * rng.standard_normal((L, 3))
    return dict(pose_cw=pose0, pose_fixed=pose_fixed, points=pts0, point_fixed=None, e_pose=e_pose, e_point=e_point, e_cam=e_cam,
                e_obs=e_obs, e_inv_sigma_sq=e_isq, e_delta=delta, e_robust=None, e_can_be_outlier=None, cams=[dict(c) for c in cam_list],
                gt_pose_cw=gt, gt_points=pts, behind=behind, empty_kf=empty, outlier_kf=bad_kf, kinds=kinds)


# the window kinds every test runs on (small enough for scipy on the CPU; the long one only against the oracle)
WINDOWS = {
    "three_cams": dict(seed=1, n_kf=9, n_points=70),
    "kitti_euroc": dict(seed=2, n_kf=8, n_points=70, cams=("kitti", "euroc"), n_pole=0, n_seam=0),
    "equirect_persp": dict(seed=3, n_kf=8, n_points=70, cams=("equirect", "kitti"), n_pole=6, n_seam=6),
    "two_view_mono": dict(seed=4, n_kf=10, n_points=90, cams=("euroc",), degrees={1: 0.15, 2: 0.8, 3: 0.05}, n_far=4, n_pole=0, n_seam=0),
}
LONG_WINDOWS = {
    # 70 free keyframes: landmarks seen by 64, 65 and 70 of them straddle the first 64-bit keyframe mask word
    "deep_degrees": dict(seed=5, n_kf=72, n_points=900, cams=("kitti", "euroc"), spacing=0.25, deep_degrees=(64, 64, 65, 65, 69, "all"),
                         n_pole=0, n_seam=0),
}


def window(name):
    spec = dict(WINDOWS, **LONG_WINDOWS)[name]
    return make_window(**spec)


# ---------------------------------------------------------------------------------------------------------------------
# pose-optimiser frames
# ---------------------------------------------------------------------------------------------------------------------
def make_frame(seed, n_obs, cam="kitti", stereo_frac=0.0, cam_index=0, n_cams=1, n_behind=0, n_near=0, n_far=0, n_pole=0, n_seam=0,
               outlier_frac=0.1, rot_deg=1.0, trans_m=0.1):
    """One frame for the pose optimiser: ONE free pose, its n_obs observed landmarks (fixed) and one edge per observation, with the
    camera at index cam_index of a list of n_cams (the others are decoys with different intrinsics) and e_cam = cam_index throughout.
    stereo_frac: share of edges with an x_right (KITTI).  n_behind: points behind the camera, observed where the projection puts them
    (the pose optimiser has no depth test: they must simply agree).  n_pole / n_seam: equirectangular points near a pole / the seam."""
    rng = np.random.default_rng(seed)
    c = CAMS[cam]
    Rcw = _rodrigues(0.3 * rng.standard_normal(3))
    tcw = rng.normal(0, 2.0, 3)
    gt = np.eye(4)
    gt[:3, :3], gt[:3, 3] = Rcw, tcw
    n_special = n_behind + n_near + n_far + n_pole + n_seam
    n_plain = n_obs - n_special
    assert n_plain >= 0
    if c["model"] == 1:
        d = rng.standard_normal((n_plain, 3))
        pc = d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(2, 40, n_plain)[:, None]
    else:
        depth = rng.uniform(2, 60, n_plain)
        u, v = rng.uniform(10, c["cols"] - 10, n_plain), rng.uniform(10, c["rows"] - 10, n_plain)
        pc = np.stack([(u - c["cx"]) / c["fx"] * depth, (v - c["cy"]) / c["fy"] * depth, depth], 1)
    extra = []
    for depth_rng, n, sign in (((0.5, 3.0), n_behind, -1.0), ((0.3, 0.3), n_near, 1.0), ((1000, 2000), n_far, 1.0)):
        if n:
            depth = rng.uniform(*depth_rng, n)
            ref = c if c["model"] == 0 else CAMS["kitti"]
            u, v = rng.uniform(10, ref["cols"] - 10, n), rng.uniform(10, ref["rows"] - 10, n)
            extra.append(np.stack([(u - ref["cx"]) / ref["fx"] * depth, (v - ref["cy"]) / ref["fy"] * depth, depth], 1) * sign)
    for i in range(n_pole):
        el, az = np.deg2rad(rng.uniform(86, 88)), rng.uniform(-np.pi, np.pi)
        extra.append(np.array([[np.cos(el) * np.sin(az), (1 if i % 2 else -1) * np.sin(el), np.cos(el) * np.cos(az)]]) * rng.uniform(3, 20))
    for i in range(n_seam):
        th = (np.pi - rng.uniform(4, 10) * 2 * np.pi / c["cols"]) * (1 if i % 2 else -1)
        ph = rng.uniform(-0.5, 0.5)
        extra.append(np.array([[np.cos(ph) * np.sin(th), -np.sin(ph), np.cos(ph) * np.cos(th)]]) * rng.uniform(3, 20))
    pc = np.concatenate([pc] + extra) if extra else pc
    perm = rng.permutation(n_obs)
    pc = pc[perm]
    behind = np.nonzero((perm >= n_plain) & (perm < n_plain + n_behind))[0]
    pw = (pc - tcw) @ Rcw
    lvl = rng.integers(0, 8, n_obs)
    sig = 1.0 / np.sqrt(INV_SIGMA_SQ[lvl].astype(np.float64))
    uv = project(c, pc)
    xr = np.full(n_obs, -1.0)
    if stereo_frac > 0:
        has = (rng.random(n_obs) < stereo_frac) & (pc[:, 2] > 0)
        xr[has] = (uv[:, 0] - c["fxb"] / pc[:, 2] + sig * rng.standard_normal(n_obs))[has]
        xr[xr < 0] = -1.0
    x, y = uv[:, 0] + sig * rng.standard_normal(n_obs), uv[:, 1] + sig * rng.standard_normal(n_obs)
    bad = rng.random(n_obs) < outlier_frac
    bad[behind] = False
    x[bad] += rng.choice([-1, 1], bad.sum()) * rng.uniform(10, 60, bad.sum())
    y[bad] += rng.choice([-1, 1], bad.sum()) * rng.uniform(10, 60, bad.sum())
    dR = _rodrigues(np.deg2rad(rot_deg) * rng.standard_normal(3) / np.sqrt(3))
    pose0 = np.eye(4)
    pose0[:3, :3] = dR @ Rcw
    pose0[:3, 3] = dR @ tcw + trans_m * rng.standard_normal(3) / np.sqrt(3)
    isq = INV_SIGMA_SQ[lvl]
    delta = np.where(xr >= 0, np.float32(np.sqrt(np.float32(7.81473))), np.float32(np.sqrt(np.float32(5.99146)))).astype(np.float32)
    decoys = [CAMS[k] for k in ("euroc", "kitti", "equirect") if k != cam]
    cams = [dict(decoys[i % len(decoys)]) for i in range(n_cams)]
    cams[cam_index] = dict(c)
    return dict(pose_cw=pose0[None], pose_fixed=np.zeros(1, np.uint8), points=pw, point_fixed=np.ones(n_obs, np.uint8),
                e_pose=np.zeros(n_obs, np.int32), e_point=np.arange(n_obs, dtype=np.int32), e_cam=np.full(n_obs, cam_index, np.uint8),
                e_obs=np.stack([x, y, xr], 1).astype(np.float32), e_inv_sigma_sq=isq, e_delta=delta, e_robust=None, e_can_be_outlier=None,
                cams=cams, gt_pose_cw=gt, gt_outlier=bad, behind=behind)
