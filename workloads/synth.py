"""Seeded synthetic inputs (numpy only) shaped like BASELINE.json's configs: textured frames with corners,
descriptor sets with planted near-duplicates, and local-BA problems (K poses, L landmarks, E observations).

No dataset exists in the container or on the GPU box (SURVEY.md section 8d), so every bench/test input comes from here.
"""
import numpy as np


def _value_noise(rng, h, w, cell):
    gh, gw = h // cell + 2, w // cell + 2
    g = rng.random((gh, gw)).astype(np.float32)
    ys = np.arange(h, dtype=np.float32) / cell
    xs = np.arange(w, dtype=np.float32) / cell
    y0, x0 = ys.astype(np.int32), xs.astype(np.int32)
    fy, fx = (ys - y0)[:, None], (xs - x0)[None, :]
    a = g[y0][:, x0]
    b = g[y0][:, x0 + 1]
    c = g[y0 + 1][:, x0]
    d = g[y0 + 1][:, x0 + 1]
    return (a * (1 - fx) + b * fx) * (1 - fy) + (c * (1 - fx) + d * fx) * fy


_PAD = 64


def _make_pattern(w, h, seed, n_shapes=None):
    """Padded float32 scene (h+2*PAD, w+2*PAD): 4 octaves of value noise + random filled rectangles/discs."""
    rng = np.random.default_rng(seed)
    H, W = h + 2 * _PAD, w + 2 * _PAD
    img = np.zeros((H, W), np.float32)
    for cell, amp in ((96, 80.0), (32, 45.0), (11, 30.0), (4, 26.0)):
        img += amp * _value_noise(rng, H, W, cell)
    if n_shapes is None:
        n_shapes = max(40, int(400 * (w * h) / (1920 * 1080)))
    for _ in range(n_shapes):
        cx, cy = int(rng.integers(0, W)), int(rng.integers(0, H))
        s = int(rng.integers(6, 48))
        g = float(rng.integers(0, 256))
        y0, y1, x0, x1 = max(cy - s, 0), min(cy + s, H), max(cx - s, 0), min(cx + s, W)
        if rng.random() < 0.6:
            img[y0:y1, x0:x1] = g
        else:
            yy, xx = np.mgrid[y0:y1, x0:x1]
            m = (yy - cy) ** 2 + (xx - cx) ** 2 <= s * s
            img[y0:y1, x0:x1][m] = g
    return img


def _render(pattern, w, h, seed, shift, noise_sigma):
    dx, dy = int(shift[0]), int(shift[1])
    dx, dy = max(-_PAD, min(_PAD, dx)), max(-_PAD, min(_PAD, dy))
    view = pattern[_PAD + dy:_PAD + dy + h, _PAD + dx:_PAD + dx + w]
    nrng = np.random.default_rng(seed * 7919 + 17 * (dx + 101) + (dy + 103))
    view = view + noise_sigma * nrng.standard_normal(view.shape, dtype=np.float32)
    p = np.pad(view, 1, mode="edge")
    box = sum(p[i:i + h, j:j + w] for i in range(3) for j in range(3)) / np.float32(9.0)
    return np.clip(np.rint(box), 0, 255).astype(np.uint8)


def make_frame(w=1920, h=1080, seed=1234, shift=(0, 0), n_shapes=None, noise_sigma=2.0):
    """u8 HxW frame: 4 octaves of value noise + random filled rectangles/discs + iid noise, then a 3x3 box blur.

    `shift` translates the underlying pattern (pixels), so consecutive frames of a stream overlap and match.
    """
    return _render(_make_pattern(w, h, seed, n_shapes), w, h, seed, shift, noise_sigma)


def make_stream(n_frames, w=1920, h=1080, stream=0, max_step=8):
    """Frames of one synthetic stream: the pattern follows a seeded 2-D random walk (<= max_step px per frame)."""
    rng = np.random.default_rng(99 + stream)
    pattern = _make_pattern(w, h, 1234 + stream)
    pos = np.zeros(2, np.int64)
    frames = []
    for _ in range(n_frames):
        frames.append(_render(pattern, w, h, 1234 + stream, (int(pos[0]), int(pos[1])), 2.0))
        pos = np.clip(pos + rng.integers(-max_step, max_step + 1, 2), -60, 60)
    return frames


def make_descriptor_pair(n1=2000, n2=2000, seed=7, dup_frac=0.6, max_flips=40):
    """Two descriptor sets + angles: dup_frac of set 2 are rows of set 1 with k in [0,max_flips] bit flips."""
    rng = np.random.default_rng(seed)
    d1 = rng.integers(0, 256, (n1, 32), dtype=np.uint8)
    d2 = rng.integers(0, 256, (n2, 32), dtype=np.uint8)
    a1 = (rng.random(n1) * 360).astype(np.float32)
    a2 = (rng.random(n2) * 360).astype(np.float32)
    n_dup = int(dup_frac * n2)
    src = rng.integers(0, n1, n_dup)
    dst = rng.permutation(n2)[:n_dup]
    for s, t in zip(src, dst):
        row = d1[s].copy()
        k = int(rng.integers(0, max_flips + 1))
        bits = rng.choice(256, size=k, replace=False)
        for b in bits:
            row[b >> 3] ^= np.uint8(1 << (b & 7))
        d2[t] = row
        a2[t] = np.float32((a1[s] + rng.normal(0, 8)) % 360)
    valid2 = (rng.random(n2) < 0.9).astype(np.uint8)
    return d1, a1, d2, a2, valid2


# ---------------------------------------------------------------------------------------------------------------------
# local-BA problems (SURVEY.md section 8d): K keyframes on an arc, L landmarks in the frustum union, E observations
# ---------------------------------------------------------------------------------------------------------------------
KITTI = dict(fx=718.856, fy=718.856, cx=607.1928, cy=185.2157, fxb=386.1448, cols=1241, rows=376)  # example/kitti/KITTI_stereo_00-02.yaml


def _rot_y(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


def _rodrigues(w):
    th = np.linalg.norm(w)
    if th < 1e-12:
        return np.eye(3)
    k = w / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def make_ba_problem(n_poses=50, n_fixed=10, n_points=10000, seed=0, model="stereo", outlier_frac=0.05, pixel_sigma=1.0,
                    min_obs=4, max_obs=8, arc_m=200.0, perturb=True):
    """Synthetic local-BA problem in the flattened layout of the C ABI.

    model: "mono" | "stereo" (perspective, KITTI intrinsics) | "equirect" (3840x1920).
    Returns dict(pose_cw (K,4,4), pose_fixed (K,), points (L,3), e_pose, e_point, e_cam, e_obs (E,3) f32,
                 e_inv_sigma_sq f32, e_delta f32, cams (list of dict), gt_pose_cw, gt_points).
    """
    rng = np.random.default_rng(seed)
    K, L = n_poses, n_points
    equirect = model == "equirect"
    cam = dict(model=1 if equirect else 0, fx=KITTI["fx"], fy=KITTI["fy"], cx=KITTI["cx"], cy=KITTI["cy"], fxb=KITTI["fxb"],
               cols=3840.0 if equirect else float(KITTI["cols"]), rows=1920.0 if equirect else float(KITTI["rows"]))
    # keyframes on a gentle arc, looking along the direction of travel
    s = np.linspace(0, arc_m, K)
    radius = 4 * arc_m
    ang = s / radius
    centers = np.stack([radius * np.sin(ang), 0.3 * np.sin(s / 15.0), radius * (1 - np.cos(ang))], 1)
    gt_pose = np.zeros((K, 4, 4))
    for k in range(K):
        Rwc = _rot_y(ang[k] + 0.02 * rng.standard_normal()) @ _rodrigues(0.01 * rng.standard_normal(3))
        Rcw = Rwc.T
        gt_pose[k, :3, :3] = Rcw
        gt_pose[k, :3, 3] = -Rcw @ centers[k]
        gt_pose[k, 3, 3] = 1
    sf = np.float32(1.0)
    inv_sigma = [np.float32(1.0)]
    for _ in range(1, 8):
        sf = np.float32(1.2) * sf
        inv_sigma.append(np.float32(1.0) / (sf * sf))
    inv_sigma = np.array(inv_sigma, np.float32)
    sigma_lvl = 1.0 / np.sqrt(inv_sigma.astype(np.float64))

    def project(Tcw, pw):
        pc = pw @ Tcw[:3, :3].T + Tcw[:3, 3]
        if equirect:
            th = np.arctan2(pc[:, 0], pc[:, 2])
            ph = -np.arcsin(pc[:, 1] / np.linalg.norm(pc, axis=1))
            uv = np.stack([cam["cols"] * (0.5 + th / (2 * np.pi)), cam["rows"] * (0.5 - ph / np.pi)], 1)
            vis = np.linalg.norm(pc, axis=1) > 2.0
            return uv, pc, vis
        z = pc[:, 2]
        uv = np.stack([cam["fx"] * pc[:, 0] / z + cam["cx"], cam["fy"] * pc[:, 1] / z + cam["cy"]], 1)
        vis = (z > 3.0) & (z < 80.0) & (uv[:, 0] > 0) & (uv[:, 0] < cam["cols"]) & (uv[:, 1] > 0) & (uv[:, 1] < cam["rows"])
        return uv, pc, vis

    # landmarks: sampled in front of random keyframes at 5..60 m
    pts = np.zeros((L, 3))
    owner = rng.integers(0, K, L)
    depth = rng.uniform(5, 60, L)
    u = rng.uniform(0.05, 0.95, L) * (KITTI["cols"] if not equirect else 1241)
    v = rng.uniform(0.05, 0.95, L) * (KITTI["rows"] if not equirect else 376)
    for l in range(L):
        Tcw = gt_pose[owner[l]]
        pc = np.array([(u[l] - KITTI["cx"]) / KITTI["fx"] * depth[l], (v[l] - KITTI["cy"]) / KITTI["fy"] * depth[l], depth[l]])
        pts[l] = Tcw[:3, :3].T @ (pc - Tcw[:3, 3])
    e_pose, e_point, e_obs, e_isq = [], [], [], []
    order = np.argsort(np.abs(np.arange(K)[None, :] - owner[:, None]), axis=1)  # nearest keyframes first
    proj = [project(gt_pose[k], pts) for k in range(K)]
    for l in range(L):
        want = int(rng.integers(min_obs, max_obs + 1))
        got = 0
        for k in order[l]:
            uv, pc, vis = proj[k]
            if not vis[l]:
                continue
            lvl = int(rng.integers(0, 8))
            noise = pixel_sigma * sigma_lvl[lvl] * rng.standard_normal(3)
            x, y = uv[l, 0] + noise[0], uv[l, 1] + noise[1]
            xr = -1.0
            if model == "stereo" and rng.random() < 0.85:
                xr = uv[l, 0] - cam["fxb"] / pc[l, 2] + noise[2]
                if xr < 0:
                    xr = -1.0
            if rng.random() < outlier_frac:
                x += rng.choice([-1, 1]) * rng.uniform(15, 30)
                y += rng.choice([-1, 1]) * rng.uniform(15, 30)
            e_pose.append(k)
            e_point.append(l)
            e_obs.append((x, y, xr))
            e_isq.append(inv_sigma[lvl])
            got += 1
            if got >= want:
                break
    E = len(e_pose)
    chi = np.float32(np.sqrt(np.float32(5.99146))) if model != "stereo" else np.float32(np.sqrt(np.float32(7.81473)))
    pose_fixed = np.zeros(K, np.uint8)
    pose_fixed[:n_fixed] = 1   # the oldest keyframes play the "fixed" role (observers outside the local window)
    pose0, pts0 = gt_pose.copy(), pts.copy()
    if perturb:
        for k in range(K):
            if pose_fixed[k]:
                continue
            dR = _rodrigues(np.deg2rad(0.5) * rng.standard_normal(3) / np.sqrt(3))
            Rn = dR @ gt_pose[k, :3, :3]                     # 0.5 deg about the camera centre, 5 cm of centre noise
            cn = centers[k] + 0.05 * rng.standard_normal(3) / np.sqrt(3)
            pose0[k, :3, :3] = Rn
            pose0[k, :3, 3] = -Rn @ cn
        pts0 = pts + 0.01 * depth[:, None] * rng.standard_normal((L, 3))
    return dict(pose_cw=pose0, pose_fixed=pose_fixed, points=pts0, point_fixed=None, e_pose=np.array(e_pose, np.int32),
                e_point=np.array(e_point, np.int32), e_cam=np.zeros(E, np.uint8), e_obs=np.array(e_obs, np.float32).reshape(E, 3),
                e_inv_sigma_sq=np.array(e_isq, np.float32), e_delta=np.full(E, chi, np.float32), e_robust=None,
                e_can_be_outlier=None, cams=[cam], gt_pose_cw=gt_pose, gt_points=pts)


def make_pose_problem(seed=0, n_obs=1500, model="stereo", outlier_frac=0.1, pixel_sigma=1.0, rot_deg=1.0, trans_m=0.15):
    """One frame for optimize::pose_optimizer in the flattened layout of b200_lba_problem_t: ONE free pose (perturbed), the
    `n_obs` landmarks it observes (fixed, exact) and one edge per observation with level-dependent noise and gross outliers."""
    rng = np.random.default_rng(seed)
    equirect = model == "equirect"
    cam = dict(model=1 if equirect else 0, fx=KITTI["fx"], fy=KITTI["fy"], cx=KITTI["cx"], cy=KITTI["cy"], fxb=KITTI["fxb"],
               cols=3840.0 if equirect else float(KITTI["cols"]), rows=1920.0 if equirect else float(KITTI["rows"]))
    Rcw = _rot_y(0.3 * rng.standard_normal()) @ _rodrigues(0.05 * rng.standard_normal(3))
    tcw = rng.normal(0, 2.0, 3)
    gt = np.eye(4)
    gt[:3, :3], gt[:3, 3] = Rcw, tcw
    depth = rng.uniform(4, 60, n_obs)
    if equirect:
        d = rng.standard_normal((n_obs, 3))
        pc = d / np.linalg.norm(d, axis=1, keepdims=True) * depth[:, None]
    else:
        u, v = rng.uniform(20, cam["cols"] - 20, n_obs), rng.uniform(20, cam["rows"] - 20, n_obs)
        pc = np.stack([(u - cam["cx"]) / cam["fx"] * depth, (v - cam["cy"]) / cam["fy"] * depth, depth], 1)
    pw = (pc - tcw) @ Rcw                                # Rcw^T (pc - tcw)
    inv_sigma = (np.float32(1.0) / np.cumprod(np.concatenate([[np.float32(1.0)], np.full(7, np.float32(1.2))])).astype(np.float32) ** 2).astype(np.float32)
    lvl = rng.integers(0, 8, n_obs)
    sig = pixel_sigma / np.sqrt(inv_sigma[lvl].astype(np.float64))
    if equirect:
        th, ph = np.arctan2(pc[:, 0], pc[:, 2]), -np.arcsin(pc[:, 1] / np.linalg.norm(pc, axis=1))
        x, y = cam["cols"] * (0.5 + th / (2 * np.pi)), cam["rows"] * (0.5 - ph / np.pi)
    else:
        x, y = cam["fx"] * pc[:, 0] / pc[:, 2] + cam["cx"], cam["fy"] * pc[:, 1] / pc[:, 2] + cam["cy"]
    xr = np.full(n_obs, -1.0)
    if model == "stereo":
        has = rng.random(n_obs) < 0.8
        xr[has] = (x - cam["fxb"] / pc[:, 2] + sig * rng.standard_normal(n_obs))[has]
        xr[xr < 0] = -1.0
    x, y = x + sig * rng.standard_normal(n_obs), y + sig * rng.standard_normal(n_obs)
    bad = rng.random(n_obs) < outlier_frac
    x[bad] += rng.choice([-1, 1], bad.sum()) * rng.uniform(10, 60, bad.sum())
    y[bad] += rng.choice([-1, 1], bad.sum()) * rng.uniform(10, 60, bad.sum())
    dR = _rodrigues(np.deg2rad(rot_deg) * rng.standard_normal(3) / np.sqrt(3))
    pose0 = np.eye(4)
    pose0[:3, :3] = dR @ Rcw
    pose0[:3, 3] = dR @ tcw + trans_m * rng.standard_normal(3) / np.sqrt(3)
    chi = np.float32(np.sqrt(np.float32(7.81473))) if model == "stereo" else np.float32(np.sqrt(np.float32(5.99146)))  # setup-type dependent, :99-101
    return dict(pose_cw=pose0[None], pose_fixed=np.zeros(1, np.uint8), points=pw, point_fixed=np.ones(n_obs, np.uint8),
                e_pose=np.zeros(n_obs, np.int32), e_point=np.arange(n_obs, dtype=np.int32), e_cam=np.zeros(n_obs, np.uint8),
                e_obs=np.stack([x, y, xr], 1).astype(np.float32), e_inv_sigma_sq=inv_sigma[lvl], e_delta=np.full(n_obs, chi, np.float32),
                e_robust=None, e_can_be_outlier=None, cams=[cam], gt_pose_cw=gt, gt_outlier=bad)


def make_guided_problem(seed, n_train=2000, n_queries=1500, mode=0, stereo=False, width=640, height=480, margin=5.0, num_levels=8,
                        scale_factor=1.2):
    """A synthetic problem for the grid-guided projection matchers (match.projection): a frame with `n_train` keypoints and
    `n_queries` landmarks that reproject near some of them.  Built to exercise every gate: several landmarks compete for one
    keypoint (the sequential occupancy matters), near-duplicate descriptors sit next to each other (ratio test), octaves fall
    outside the level window, some keypoints are pre-occupied, some landmarks are invalid, undistorted bounds are fractional and
    a few keypoints / reprojections fall outside them."""
    rng = np.random.default_rng(seed)
    sf = np.float32(1.0) * np.cumprod(np.concatenate([[np.float32(1.0)], np.full(num_levels - 1, np.float32(scale_factor))])).astype(np.float32)
    bounds = (np.float32(-11.37), np.float32(width + 9.21), np.float32(-7.9), np.float32(height + 6.53))
    # keypoints: uniform background + tight clusters
    n_cl = n_train // 3
    centers = rng.uniform([0, 0], [width, height], (max(n_cl // 12, 1), 2))
    pts = np.concatenate([rng.uniform([bounds[0] - 3, bounds[2] - 3], [bounds[1] + 3, bounds[3] + 3], (n_train - n_cl, 2)),
                          centers[rng.integers(0, len(centers), n_cl)] + rng.normal(0, 4.0, (n_cl, 2))])
    pts = pts[rng.permutation(n_train)].astype(np.float32)
    octave = rng.choice(num_levels, n_train, p=np.array([.3, .22, .16, .12, .08, .06, .04, .02])).astype(np.uint8)
    angle = rng.uniform(0, 360, n_train).astype(np.float32)
    desc = rng.integers(0, 256, (n_train, 32), dtype=np.uint8)
    # near-duplicate descriptors between spatial neighbours (sorted by x so duplicates are usually inside one window)
    order = np.argsort(pts[:, 0], kind="stable")
    for a, b in zip(order[0:n_train - 1:7], order[1:n_train:7]):
        noise = rng.integers(0, 256, 32, dtype=np.uint8) & rng.integers(0, 256, 32, dtype=np.uint8) & rng.integers(0, 256, 32, dtype=np.uint8) \
            & rng.integers(0, 256, 32, dtype=np.uint8)
        desc[b] = desc[a] ^ noise
        if rng.random() < 0.5:
            octave[b] = octave[a]
    src = rng.integers(0, n_train, n_queries)
    src[1::5] = src[0:n_queries - 1:5][:len(src[1::5])]          # two landmarks on one keypoint
    strength = rng.integers(1, 6, n_queries)                     # AND of k random bytes: ~ 256 / 2^k flipped bits
    q_desc = desc[src].copy()
    for k in range(1, 6):  # per-landmark noise level
        sel = strength == k
        fl = rng.integers(0, 256, (sel.sum(), 32), dtype=np.uint8)
        for _ in range(k):
            fl &= rng.integers(0, 256, (sel.sum(), 32), dtype=np.uint8)
        q_desc[sel] ^= fl
    level = np.clip(octave[src].astype(np.int64) + rng.integers(-2, 3, n_queries), 0, num_levels - 1)
    q_xy = pts[src].astype(np.float64) + rng.normal(0, 2.5, (n_queries, 2))
    far = rng.random(n_queries) < 0.03
    q_xy[far] += rng.normal(0, 400, (far.sum(), 2))
    q_margin = (np.float32(margin) * sf[level]).astype(np.float32)
    lo, hi = np.maximum(0, level - 1), np.minimum(num_levels - 1, level + 1)
    unchecked = rng.random(n_queries) < 0.05
    lo[unchecked], hi[unchecked] = -1, -1
    prob = dict(t_x=pts[:, 0].copy(), t_y=pts[:, 1].copy(), t_octave=octave, t_angle=angle, t_desc=desc,
                t_occupied=(rng.random(n_train) < 0.08).astype(np.uint8), bounds=bounds, grid=(64, 48), scale_factors=sf,
                q_desc=q_desc, q_x=q_xy[:, 0].astype(np.float32), q_y=q_xy[:, 1].astype(np.float32), q_margin=q_margin,
                q_min_level=lo.astype(np.int8), q_max_level=hi.astype(np.int8),
                q_angle=((angle[src] + rng.normal(0, 18, n_queries)) % 360).astype(np.float32),
                q_valid=(rng.random(n_queries) > 0.1).astype(np.uint8),
                q_reproj=q_xy.copy(), inv_level_sigma_sq=(np.float32(1.0) / (sf * sf)).astype(np.float32),
                do_reprojection_matching=(mode == 3))
    if mode == 4:  # area::match_in_consistent_area: level-0 keypoints only, one integer margin
        prob.update(q_min_level=np.zeros(n_queries, np.int8), q_max_level=np.zeros(n_queries, np.int8),
                    q_margin=np.full(n_queries, np.float32(int(margin * 4))), q_valid=(level == 0).astype(np.uint8))
    if stereo:
        xr = (pts[:, 0] - rng.uniform(2, 60, n_train)).astype(np.float32)
        xr[rng.random(n_train) < 0.3] = -1.0                    # no stereo match for this keypoint
        prob["t_x_right"] = xr
        prob["q_x_right"] = (xr[src] + rng.normal(0, q_margin * 0.6)).astype(np.float32)
    return prob


def make_keyframe_pair(seed, n1=2000, n2=2000, stereo=False, n_nodes=150, num_levels=8, scale_factor=1.2, bearing_noise=1.5e-3):
    """Two keyframes looking at the same synthetic points, for the all-pairs matchers with greedy state (bow_tree::*,
    robust::match_for_triangulation).  Returns (keyfrm_1, keyfrm_2, geometry): dicts with desc, angle, octave, bearings (unit,
    f64), node (BoW node id), no_landmark / has_landmark (u8), stereo (u8 | None), scale_factors; geometry holds E_12 with
    bearing_1 . (E_12 bearing_2) = 0 for true correspondences, the epipole of keyframe 1 in keyframe 2, the pair list (perm1[k],
    perm2[k]) and its mask `wrong` of the correspondences moved off their epipolar plane.
    Corresponding keypoints share descriptors up to noise of varied strength; some rows have two look-alike candidates (ratio
    test), some correspondences violate the epipolar constraint, some sit next to the epipole."""
    rng = np.random.default_rng(seed)
    sf = np.cumprod(np.concatenate([[np.float32(1.0)], np.full(num_levels - 1, np.float32(scale_factor))])).astype(np.float32)
    n_common = int(0.7 * min(n1, n2))
    # relative pose: x1 = R_12 x2 + t_12  (mostly forward motion, so the epipole lies inside the image)
    R_12 = _rodrigues(rng.normal(0, 0.03, 3))
    t_12 = np.array([0.15, -0.05, 0.6]) + rng.normal(0, 0.02, 3)
    tx = np.array([[0, -t_12[2], t_12[1]], [t_12[2], 0, -t_12[0]], [-t_12[1], t_12[0], 0]])
    E_12 = tx @ R_12
    pts2 = np.stack([rng.uniform(-4, 4, n_common), rng.uniform(-3, 3, n_common), rng.uniform(4, 30, n_common)], 1)
    near_epipole = rng.random(n_common) < 0.04           # along the baseline as seen from camera 2
    c1_in_2 = -R_12.T @ t_12
    pts2[near_epipole] = c1_in_2 * rng.uniform(8, 30, (near_epipole.sum(), 1)) + rng.normal(0, 0.15, (near_epipole.sum(), 3))
    pts1 = pts2 @ R_12.T + t_12

    def unit(v):
        return v / np.linalg.norm(v, axis=1, keepdims=True)

    def side(n, pts, perm):
        b = unit(np.stack([rng.uniform(-0.8, 0.8, n), rng.uniform(-0.6, 0.6, n), np.ones(n)], 1))
        b[perm] = unit(unit(pts) + rng.normal(0, bearing_noise, pts.shape))
        return b

    perm1, perm2 = rng.permutation(n1)[:n_common], rng.permutation(n2)[:n_common]
    bearings1, bearings2 = side(n1, pts1, perm1), side(n2, pts2, perm2)
    wrong = rng.random(n_common) < 0.1                   # correspondences that break the epipolar constraint
    bearings2[perm2[wrong]] = unit(bearings2[perm2[wrong]] + rng.normal(0, 0.05, (wrong.sum(), 3)))
    desc1 = rng.integers(0, 256, (n1, 32), dtype=np.uint8)
    desc2 = rng.integers(0, 256, (n2, 32), dtype=np.uint8)
    strength = rng.integers(2, 6, n_common)
    fl = np.full((n_common, 32), 255, np.uint8)
    for k in range(6):
        r = rng.integers(0, 256, (n_common, 32), dtype=np.uint8)
        fl = np.where((strength > k)[:, None], fl & r, fl)
    desc2[perm2] = desc1[perm1] ^ fl
    octave1 = rng.choice(num_levels, n1, p=np.array([.3, .22, .16, .12, .08, .06, .04, .02])).astype(np.uint8)
    octave2 = octave1[rng.integers(0, n1, n2)]
    octave2[perm2] = octave1[perm1]
    angle1 = rng.uniform(0, 360, n1).astype(np.float32)
    angle2 = rng.uniform(0, 360, n2).astype(np.float32)
    angle2[perm2] = (angle1[perm1] + rng.normal(0, 14, n_common)) % 360
    node1, node2 = rng.integers(0, n_nodes, n1).astype(np.int32), rng.integers(0, n_nodes, n2).astype(np.int32)
    same_node = rng.random(n_common) < 0.9
    node2[perm2[same_node]] = node1[perm1[same_node]]
    # look-alikes: a second candidate in the same node with a similar descriptor and the same bearing (passes every gate)
    free2 = np.setdiff1d(np.arange(n2), perm2)
    for k, j in zip(rng.permutation(n_common)[:len(free2) // 2], free2):
        noise = rng.integers(0, 256, 32, dtype=np.uint8) & rng.integers(0, 256, 32, dtype=np.uint8) & rng.integers(0, 256, 32, dtype=np.uint8) \
            & rng.integers(0, 256, 32, dtype=np.uint8)
        desc2[j] = desc2[perm2[k]] ^ noise
        bearings2[j], angle2[j], node2[j] = bearings2[perm2[k]], angle2[perm2[k]], node2[perm2[k]]
    has_lm1, has_lm2 = (rng.random(n1) < 0.5).astype(np.uint8), (rng.random(n2) < 0.5).astype(np.uint8)

    def kf(desc, angle, octave, bearings, node, has_lm, n):
        return dict(desc=desc, angle=angle, octave=octave, bearings=np.ascontiguousarray(bearings), node=node, has_landmark=has_lm,
                    no_landmark=(1 - has_lm).astype(np.uint8), stereo=(rng.random(n) < 0.4).astype(np.uint8) if stereo else None, scale_factors=sf)

    geometry = dict(E_12=E_12, epiplane_in_keyfrm_2=c1_in_2 / np.linalg.norm(c1_in_2), valid_epiplane=True, perm1=perm1, perm2=perm2,
                    wrong=wrong)
    return kf(desc1, angle1, octave1, bearings1, node1, has_lm1, n1), kf(desc2, angle2, octave2, bearings2, node2, has_lm2, n2), geometry


def make_stereo_pair(w=752, h=480, seed=77, disparities=(9, 23, 41), noise_sigma=2.0):
    """(left, right) rectified frames: the right view shows the same pattern moved left by a disparity that differs per
    horizontal band, with independent sensor noise, so match::stereo finds sub-pixel disparities around those values."""
    pattern = _make_pattern(w, h, seed)
    left = _render(pattern, w, h, seed, (0, 0), noise_sigma)
    right = np.empty_like(left)
    bands = np.linspace(0, h, len(disparities) + 1).astype(int)
    for k, d in enumerate(disparities):
        right[bands[k]:bands[k + 1]] = _render(pattern, w, h, seed + 1, (int(d), 0), noise_sigma)[bands[k]:bands[k + 1]]
    return left, right


# Stereo rectification calibrations (StereoRectifier blocks of example/euroc/EuRoC_stereo.yaml and example/tum_vi/TUM_VI_stereo.yaml):
# K, D, R per eye (left, right), row-major; K_rect is the rectified Camera block's matrix, fxb its focal_x_baseline.
EUROC_STEREO = dict(
    model="perspective", cols=752, rows=480, fxb=47.90639384423901,
    K_rect=(435.2046959714599, 0.0, 367.4517211914062, 0.0, 435.2046959714599, 252.2008514404297, 0.0, 0.0, 1.0),
    K=((458.654, 0.0, 367.215, 0.0, 457.296, 248.375, 0.0, 0.0, 1.0), (457.587, 0.0, 379.999, 0.0, 456.134, 255.238, 0.0, 0.0, 1.0)),
    D=((-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05, 0.0), (-0.28368365, 0.07451284, -0.00010473, -3.555907e-05, 0.0)),
    R=((0.999966347530033, -0.001422739138722922, 0.008079580483432283, 0.001365741834644127, 0.9999741760894847, 0.007055629199258132,
        -0.008089410156878961, -0.007044357138835809, 0.9999424675829176),
       (0.9999633526194376, -0.003625811871560086, 0.007755443660172947, 0.003680398547259526, 0.9999684752771629, -0.007035845251224894,
        -0.007729688520722713, 0.007064130529506649, 0.999945173484644)))
TUM_VI_STEREO = dict(
    model="fisheye", cols=512, rows=512, fxb=6.242596912726197,
    K_rect=(61.75453410721205, 0.0, 240.22941720459062, 0.0, 61.75453410721205, 255.73235402091632, 0.0, 0.0, 1.0),
    K=((190.97847715128717, 0.0, 254.93170605935475, 0.0, 190.9733070521226, 256.8974428996504, 0.0, 0.0, 1.0),
       (190.44236969414825, 0.0, 252.59949716835982, 0.0, 190.4344384721956, 254.91723064636983, 0.0, 0.0, 1.0)),
    D=((0.0034823894022493434, 0.0007150348452162257, -0.0020532361418706202, 0.00020293673591811182),
       (0.0034003170790442797, 0.001766278153469831, -0.00266312569781606, 0.0003299517423931039)),
    R=((0.9997641946925044, 0.01925271884177015, 0.010044293307535757, -0.01901185247371587, 0.9995418997803748, -0.02354867403818772,
        -0.010493068014919314, 0.02335216051329943, 0.99967223234568),
       (0.9997411981023351, 0.01955199401713946, 0.011629976219300583, -0.019819377433695273, 0.9995311538731381, 0.02333805294307984,
        -0.011168218078479885, -0.023562511898925578, 0.9996599816627474)))


def _rect_forward(calib, eye, j, i):
    """The rectification map of one eye at fractional rectified pixels (j, i): where the raw view sees that rectified pixel."""
    K, D = np.asarray(calib["K"][eye], np.float64).reshape(3, 3), np.asarray(calib["D"][eye], np.float64)
    iR = np.linalg.inv(np.asarray(calib["K_rect"], np.float64).reshape(3, 3) @ np.asarray(calib["R"][eye], np.float64).reshape(3, 3))
    _x, _y, _w = (iR[r, 0] * j + iR[r, 1] * i + iR[r, 2] for r in range(3))
    x, y = _x / _w, _y / _w
    if calib["model"] == "fisheye":
        r = np.sqrt(x * x + y * y)
        th = np.arctan(r)
        th2 = th * th
        s = np.where(r > 0, th * (1 + D[0] * th2 + D[1] * th2 ** 2 + D[2] * th2 ** 3 + D[3] * th2 ** 4) / np.maximum(r, 1e-300), 1.0)
        xd, yd = x * s, y * s
    else:
        k = np.concatenate([D, np.zeros(8)])[:8]
        r2 = x * x + y * y
        kr = (1 + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2) / (1 + ((k[7] * r2 + k[6]) * r2 + k[5]) * r2)
        xd = x * kr + 2 * k[2] * x * y + k[3] * (r2 + 2 * x * x)
        yd = y * kr + k[2] * (r2 + 2 * y * y) + 2 * k[3] * x * y
    return K[0, 0] * xd + K[0, 2], K[1, 1] * yd + K[1, 2]


def make_raw_stereo_pair(calib, seed=77, disparities=(9, 23, 41), noise_sigma=2.0):
    """(left, right) RAW views of a rig with calibration `calib` (EUROC_STEREO / TUM_VI_STEREO layout): make_stereo_pair's rectified
    frames seen through the distortion and rotation of each eye, so that rectifying them gives back approximately the rectified pair.
    Each raw pixel samples the rectified frame (bilinearly) at an approximate inverse of the rectification map, found by a few
    fixed-point iterations; the inverse only has to be good enough for the stereo matcher to find the bands' disparities."""
    w, h = calib["cols"], calib["rows"]
    rect = make_stereo_pair(w, h, seed=seed, disparities=disparities, noise_sigma=noise_sigma)
    v, u = np.mgrid[0:h, 0:w].astype(np.float64)
    out = []
    for eye in range(2):
        j, i = u.copy(), v.copy()
        for _ in range(8):
            fu, fv = _rect_forward(calib, eye, j, i)
            ok = np.isfinite(fu) & np.isfinite(fv)
            j = np.where(ok, j + (u - fu), j)
            i = np.where(ok, i + (v - fv), i)
            j, i = np.clip(j, -w, 2 * w), np.clip(i, -h, 2 * h)
        img = rect[eye].astype(np.float64)
        j0, i0 = np.floor(j).astype(np.int64), np.floor(i).astype(np.int64)
        a, b = j - j0, i - i0

        def px(y, x):
            return img[np.clip(y, 0, h - 1), np.clip(x, 0, w - 1)]

        s = (1 - b) * ((1 - a) * px(i0, j0) + a * px(i0, j0 + 1)) + b * ((1 - a) * px(i0 + 1, j0) + a * px(i0 + 1, j0 + 1))
        out.append(np.clip(np.rint(s), 0, 255).astype(np.uint8))
    return tuple(out)


def make_tracking_frame(kps, desc, camera, scale_factors, seed=0, stereo=False, landmark_frac=0.7, clutter_frac=0.3, pre_matched_frac=0.15,
                        pixel_sigma=1.0, rot_deg=0.5, trans_m=0.05, max_flips=30):
    """A local map for one extracted frame (track_local_map workload): most keypoints get a landmark at a random depth (descriptor = the
    keypoint's with a few flipped bits, position off by ~pixel_sigma pixels), plus clutter landmarks (random descriptors; some behind the
    camera or outside the image), a few landmarks the frame already carries (kp_landmark, skipped by the search) and a few without
    observations.  The pose handed to the tracker is the true pose perturbed by rot_deg / trans_m.  Perspective and equirectangular
    cameras (the keypoints are taken as undistorted)."""
    rng = np.random.default_rng(seed)
    n_kp = len(kps)
    sf = np.asarray(scale_factors, np.float64)
    fx, fy, cx, cy = camera.get("fx", 1.0), camera.get("fy", 1.0), camera.get("cx", 0.0), camera.get("cy", 0.0)
    Rcw = _rot_y(0.2 * rng.standard_normal()) @ _rodrigues(0.05 * rng.standard_normal(3))
    tcw = rng.normal(0, 1.0, 3)
    center = -Rcw.T @ tcw
    pick = np.nonzero(rng.random(n_kp) < landmark_frac)[0]
    z = rng.uniform(4, 40, len(pick))
    u = kps["x"][pick].astype(np.float64) + pixel_sigma * rng.standard_normal(len(pick))
    v = kps["y"][pick].astype(np.float64) + pixel_sigma * rng.standard_normal(len(pick))
    equirect = camera.get("model", "perspective") == "equirectangular"

    def back_project(uu, vv, depth):
        if equirect:                                                 # camera/equirectangular.cc:42-49: pixel -> bearing
            lon, lat = (uu / camera["cols"] - 0.5) * 2 * np.pi, -(vv / camera["rows"] - 0.5) * np.pi
            b = np.stack([np.cos(lat) * np.sin(lon), -np.sin(lat), np.cos(lat) * np.cos(lon)], 1)
            return b * depth[:, None]
        return np.stack([(uu - cx) / fx * depth, (vv - cy) / fy * depth, depth], 1)

    pc = back_project(u, v, z)
    n_cl = int(clutter_frac * len(pick))
    zc = rng.uniform(4, 60, n_cl) if equirect else rng.uniform(-10, 60, n_cl)   # (perspective: some behind the camera)
    uc, vc = rng.uniform(-200, camera["cols"] + 200, n_cl), rng.uniform(-100, camera["rows"] + 100, n_cl)
    if equirect:
        uc, vc = np.clip(uc, 0, camera["cols"] - 1), np.clip(vc, 0, camera["rows"] - 1)
    pcc = back_project(uc, vc, zc)
    pc_all = np.concatenate([pc, pcc])
    pw = (pc_all - tcw) @ Rcw
    n_lm = len(pw)
    ldesc = rng.integers(0, 256, (n_lm, 32), dtype=np.uint8)
    for j, k in enumerate(pick):
        row = desc[k].copy()
        for b in rng.choice(256, int(rng.integers(0, max_flips + 1)), replace=False):
            row[b >> 3] ^= np.uint8(1 << (b & 7))
        ldesc[j] = row
    octave = np.concatenate([kps["octave"][pick].astype(np.int64), rng.integers(0, len(sf), n_cl)])
    dist = np.linalg.norm(pw - center, axis=1)
    max_valid = (dist * sf[octave]).astype(np.float32)              # landmark::update_mean_normal_and_obs_scale_variance (landmark.cc:256-311)
    min_valid = (max_valid / np.float32(sf[-1])).astype(np.float32)
    normal = (pw - center) / np.maximum(dist, 1e-9)[:, None] + 0.2 * rng.standard_normal((n_lm, 3))
    normal /= np.linalg.norm(normal, axis=1, keepdims=True)
    flip = rng.random(n_lm) < 0.03                                   # seen from behind: fails the viewing-angle test
    normal[flip] *= -1
    kp_of = np.concatenate([pick, np.full(n_cl, -1)])
    perm = rng.permutation(n_lm)                                     # the reference's local_landmarks_ order is arbitrary
    pw, ldesc, max_valid, min_valid, normal, kp_of = pw[perm], ldesc[perm], max_valid[perm], min_valid[perm], normal[perm], kp_of[perm]
    has_obs = (rng.random(n_lm) > 0.04).astype(np.uint8)
    skip = np.zeros(n_lm, np.uint8)
    kp_landmark = np.full(n_kp, -1, np.int32)
    for l in np.nonzero((kp_of >= 0) & (rng.random(n_lm) < pre_matched_frac))[0]:   # carried over from the motion-model step
        kp_landmark[kp_of[l]] = l
        skip[l] = 1
    skip[rng.random(n_lm) < 0.02] = 1                                # will_be_erased / temporal-ratio skips
    kp_x_right = None
    if stereo:
        kp_x_right = np.full(n_kp, -1.0, np.float32)
        zk = np.full(n_kp, np.nan)
        zk[pick] = z
        ok = ~np.isnan(zk) & (rng.random(n_kp) < 0.8)
        kp_x_right[ok] = (kps["x"][ok] - camera["fxb"] / zk[ok] + 0.5 * rng.standard_normal(ok.sum())).astype(np.float32)
    dR = _rodrigues(np.deg2rad(rot_deg) * rng.standard_normal(3) / np.sqrt(3))
    pose = np.eye(4)
    pose[:3, :3] = dR @ Rcw
    pose[:3, 3] = dR @ tcw + trans_m * rng.standard_normal(3) / np.sqrt(3)
    gt = np.eye(4)
    gt[:3, :3], gt[:3, 3] = Rcw, tcw
    return dict(pose_cw=pose, gt_pose_cw=gt, kp_landmark=kp_landmark, kp_x_right=kp_x_right,
                landmarks=dict(pos_w=pw, mean_normal=normal, min_valid_dist=min_valid, max_valid_dist=max_valid, desc=ldesc, skip=skip,
                               has_observation=has_obs))



def make_motion_frame(kps, desc, camera, scale_factors, seed=0, stereo=False, motion="forward", true_baseline=None, landmark_frac=0.7,
                      clutter_frac=0.2, rotated_frac=0.05, no_obs_frac=0.05, pixel_sigma=0.7, shift_px=0.0, rot_deg=0.2, trans_m=0.02, max_flips=25):
    """The last-frame table of frame_tracker::motion_based_track for one extracted frame (keypoints taken as undistorted).  Most keypoints
    get an entry whose landmark lies at a random depth along the keypoint's ray under a true pose (descriptor = the keypoint's with a few
    flipped bits, octave = the keypoint's, angle within a few degrees of it), plus `rotated_frac` entries turned 40-180 degrees (rejected by
    the 30-degree orientation gate), clutter entries (random descriptors and positions) and `no_obs_frac` entries without observations,
    in a shuffled (last-frame keypoint) order.  The predicted pose is the true pose turned about the camera's y axis so that reprojections
    move by about `shift_px` pixels (between margin and 2 * margin: the first search falls short and the second succeeds; beyond 2 * margin
    both fail), then perturbed by rot_deg / trans_m.  The last pose sees the current camera centre moved by twice true_baseline along its
    optical axis ("forward"), against it ("backward") or sideways.  Perspective-family and equirectangular cameras."""
    rng = np.random.default_rng(seed)
    n_kp = len(kps)
    sf = np.asarray(scale_factors, np.float64)
    equirect = camera.get("model", "perspective") == "equirectangular"
    fx, fy, cx, cy = camera.get("fx", 1.0), camera.get("fy", 1.0), camera.get("cx", 0.0), camera.get("cy", 0.0)
    if true_baseline is None:
        true_baseline = camera.get("fxb", 0.0) / fx if fx else 0.0
    Rcw = _rot_y(0.2 * rng.standard_normal()) @ _rodrigues(0.05 * rng.standard_normal(3))
    tcw = rng.normal(0, 1.0, 3)

    def back_project(uu, vv, depth):
        if equirect:                                                 # camera/equirectangular.cc:42-49: pixel -> bearing
            lon, lat = (uu / camera["cols"] - 0.5) * 2 * np.pi, -(vv / camera["rows"] - 0.5) * np.pi
            return np.stack([np.cos(lat) * np.sin(lon), -np.sin(lat), np.cos(lat) * np.cos(lon)], 1) * depth[:, None]
        return np.stack([(uu - cx) / fx * depth, (vv - cy) / fy * depth, depth], 1)

    pick = np.nonzero(rng.random(n_kp) < landmark_frac)[0]
    z = rng.uniform(4, 40, len(pick))
    u = kps["x"][pick].astype(np.float64) + pixel_sigma * rng.standard_normal(len(pick))
    v = kps["y"][pick].astype(np.float64) + pixel_sigma * rng.standard_normal(len(pick))
    n_cl = int(clutter_frac * len(pick))
    zc = rng.uniform(4, 60, n_cl) if equirect else rng.uniform(-10, 60, n_cl)
    uc, vc = rng.uniform(-200, camera["cols"] + 200, n_cl), rng.uniform(-100, camera["rows"] + 100, n_cl)
    if equirect:
        uc, vc = np.clip(uc, 0, camera["cols"] - 1), np.clip(vc, 0, camera["rows"] - 1)
    pc = np.concatenate([back_project(u, v, z), back_project(uc, vc, zc)])
    pw = (pc - tcw) @ Rcw
    n_lm = len(pw)
    ldesc = rng.integers(0, 256, (n_lm, 32), dtype=np.uint8)
    for j, k in enumerate(pick):
        row = desc[k].copy()
        for b in rng.choice(256, int(rng.integers(0, max_flips + 1)), replace=False):
            row[b >> 3] ^= np.uint8(1 << (b & 7))
        ldesc[j] = row
    octave = np.concatenate([kps["octave"][pick].astype(np.int64), rng.integers(0, len(sf), n_cl)]).astype(np.uint8)
    angle = np.concatenate([kps["angle"][pick].astype(np.float64) + rng.uniform(-8, 8, len(pick)), rng.uniform(0, 360, n_cl)])
    turned = rng.random(n_lm) < rotated_frac
    angle[turned] += rng.uniform(40, 180, turned.sum()) * rng.choice([-1, 1], turned.sum())
    angle = np.mod(angle, 360.0).astype(np.float32)
    has_obs = (rng.random(n_lm) >= no_obs_frac).astype(np.uint8)
    perm = rng.permutation(n_lm)
    kp_x_right = None
    if stereo:
        kp_x_right = np.full(n_kp, -1.0, np.float32)
        zk = np.full(n_kp, np.nan)
        zk[pick] = z
        ok = ~np.isnan(zk) & (rng.random(n_kp) < 0.8)
        kp_x_right[ok] = (kps["x"][ok] - camera["fxb"] / zk[ok] + 0.5 * rng.standard_normal(ok.sum())).astype(np.float32)
    turn = shift_px * 2 * np.pi / camera["cols"] if equirect else np.arctan(shift_px / fx)
    dR = _rodrigues(np.deg2rad(rot_deg) * rng.standard_normal(3) / np.sqrt(3)) @ _rot_y(turn)
    pose = np.eye(4)
    pose[:3, :3] = dR @ Rcw
    pose[:3, 3] = dR @ tcw + trans_m * rng.standard_normal(3) / np.sqrt(3)
    gt = np.eye(4)
    gt[:3, :3], gt[:3, 3] = Rcw, tcw
    axis = {"forward": np.array([0.0, 0.0, 1.0]), "backward": np.array([0.0, 0.0, -1.0]), "sideways": np.array([1.0, 0.0, 0.0])}[motion]
    step = 2.0 * true_baseline if true_baseline > 0 else 0.1
    center_last = -Rcw.T @ tcw - Rcw.T @ (step * axis)             # trans_lc = R_cw (c_curr - c_last) = step * axis
    last = np.eye(4)
    last[:3, :3], last[:3, 3] = Rcw, -Rcw @ center_last
    return dict(pose_cw=pose, last_pose_cw=last, gt_pose_cw=gt, kp_x_right=kp_x_right, true_baseline=float(true_baseline),
                table=dict(pos_w=pw[perm], desc=ldesc[perm], octave=octave[perm], angle=angle[perm], has_observation=has_obs[perm]))

def make_robust_frame(kps, desc, camera, seed=0, stereo=False, landmark_frac=0.6, clutter_frac=0.2, rotated_frac=0.05, erased_frac=0.05,
                      wrong_depth_frac=0.1, max_flips=20, baseline_m=0.5, rot_deg=2.0, trans_m=0.05, kf_keypoints=None):
    """The reference keyframe of frame_tracker::robust_match_based_track for one extracted frame (keypoints taken as undistorted), under a
    known relative pose.  A `landmark_frac` share of the frame's keypoints get a landmark at a random depth along their ray under the true
    pose; each is a keyframe keypoint (bearing of the landmark seen from the keyframe, descriptor = the frame keypoint's with a few flipped
    bits, angle within a few degrees of it).  Among them: `rotated_frac` turned 40-180 degrees (rejected by the orientation check),
    `erased_frac` whose landmark is will_be_erased (kf_valid 0) and `wrong_depth_frac` whose landmark sits at another depth along the
    keyframe's ray (the pair fits the epipolar geometry, the pose optimisation rejects it).  Clutter keypoints have random descriptors,
    bearings and positions.  The keyframe's keypoints come in a shuffled order.  last_pose_cw is the true pose perturbed by rot_deg /
    trans_m; the keyframe sits baseline_m away.  kf_keypoints caps the keyframe's size.  Perspective-family and equirectangular cameras."""
    rng = np.random.default_rng(seed)
    n_kp = len(kps)
    equirect = camera.get("model", "perspective") == "equirectangular"
    fx, fy, cx, cy = camera.get("fx", 1.0), camera.get("fy", 1.0), camera.get("cx", 0.0), camera.get("cy", 0.0)
    u, v = kps["x"].astype(np.float64), kps["y"].astype(np.float64)
    if equirect:                                                     # camera/equirectangular.cc:42-49
        lon, lat = (u / camera["cols"] - 0.5) * 2 * np.pi, -(v / camera["rows"] - 0.5) * np.pi
        rays = np.stack([np.cos(lat) * np.sin(lon), -np.sin(lat), np.cos(lat) * np.cos(lon)], 1)
    else:
        rays = np.stack([(u - cx) / fx, (v - cy) / fy, np.ones(n_kp)], 1)
    Rcw = _rot_y(0.3 * rng.standard_normal()) @ _rodrigues(0.05 * rng.standard_normal(3))
    tcw = rng.normal(0, 1.0, 3)
    dRk = _rodrigues(np.deg2rad(3.0) * rng.standard_normal(3) / np.sqrt(3))
    Rkw = dRk @ Rcw
    tkw = dRk @ tcw + baseline_m * np.array([1.0, 0.2 * rng.standard_normal(), 0.1 * rng.standard_normal()])
    pick = np.nonzero(rng.random(n_kp) < landmark_frac)[0]
    depth = rng.uniform(4, 30, len(pick))
    pc = rays[pick] * depth[:, None]                                 # perspective: z = depth; equirectangular: range = depth
    pw = (pc - tcw) @ Rcw
    pk = pw @ Rkw.T + tkw
    kb = pk / np.linalg.norm(pk, axis=1, keepdims=True)
    wrong = rng.random(len(pick)) < wrong_depth_frac
    scale = rng.uniform(1.3, 2.5, wrong.sum()) * rng.choice([1 / 1.8, 1.0], wrong.sum())
    pw[wrong] = ((pk[wrong] * scale[:, None]) - tkw) @ Rkw          # along the keyframe's ray, at another depth
    kdesc = np.empty((len(pick), 32), np.uint8)
    for j, k in enumerate(pick):
        row = desc[k].copy()
        for b in rng.choice(256, int(rng.integers(0, max_flips + 1)), replace=False):
            row[b >> 3] ^= np.uint8(1 << (b & 7))
        kdesc[j] = row
    kang = kps["angle"][pick].astype(np.float64) + rng.uniform(-6, 6, len(pick))
    turned = rng.random(len(pick)) < rotated_frac
    kang[turned] += rng.uniform(40, 180, turned.sum()) * rng.choice([-1, 1], turned.sum())
    n_cl = int(clutter_frac * len(pick))
    cb = rng.normal(0, 1, (n_cl, 3))
    cb[:, 2] = np.abs(cb[:, 2]) + 1.0
    cb /= np.linalg.norm(cb, axis=1, keepdims=True)
    cpw = ((cb * rng.uniform(4, 30, n_cl)[:, None]) - tkw) @ Rkw
    desc_all = np.concatenate([kdesc, rng.integers(0, 256, (n_cl, 32), dtype=np.uint8)])
    ang_all = np.mod(np.concatenate([kang, rng.uniform(0, 360, n_cl)]), 360.0).astype(np.float32)
    bear_all = np.concatenate([kb, cb])
    pos_all = np.concatenate([pw, cpw])
    valid = (rng.random(len(desc_all)) >= erased_frac).astype(np.uint8)
    perm = rng.permutation(len(desc_all))
    if kf_keypoints is not None:
        perm = perm[:int(kf_keypoints)]
    pos_all = pos_all[perm]
    pos_all[valid[perm] == 0] = 0.0                                  # not read for keypoints without a live landmark
    kp_x_right = None
    if stereo:
        kp_x_right = np.full(n_kp, -1.0, np.float32)
        zk = np.full(n_kp, np.nan)
        zk[pick] = pc[:, 2]
        ok = ~np.isnan(zk) & (rng.random(n_kp) < 0.8)
        kp_x_right[ok] = (kps["x"][ok] - camera["fxb"] / zk[ok] + 0.5 * rng.standard_normal(ok.sum())).astype(np.float32)
    gt = np.eye(4)
    gt[:3, :3], gt[:3, 3] = Rcw, tcw
    dR = _rodrigues(np.deg2rad(rot_deg) * rng.standard_normal(3) / np.sqrt(3))
    last = np.eye(4)
    last[:3, :3], last[:3, 3] = dR @ Rcw, dR @ tcw + trans_m * rng.standard_normal(3) / np.sqrt(3)
    return dict(last_pose_cw=last, gt_pose_cw=gt, kp_x_right=kp_x_right,
                keyframe=dict(desc=desc_all[perm], angle=ang_all[perm], bearings=bear_all[perm], valid=valid[perm], pos_w=pos_all))


def _hamming_rows(a, b, chunk=256):
    """Hamming distances (len(a), len(b)) between two sets of 32-byte descriptors."""
    out = np.empty((len(a), len(b)), np.int32)
    for s in range(0, len(a), chunk):
        out[s:s + chunk] = np.bitwise_count(a[s:s + chunk, None, :] ^ b[None, :, :]).sum(-1)
    return out


def make_bow_frame(kps, desc, camera, seed=0, stereo=False, n_nodes=64, split_frac=0.1, lookalike_frac=0.1, unnoded_frac=0.05, kf_unnoded_frac=0.02,
                   **robust_kw):
    """The reference keyframe of frame_tracker::bow_match_based_track: make_robust_frame(kps, desc, camera, seed, stereo, **robust_kw) plus
    the BoW node of every keypoint on both sides (kp_node, keyframe["node"]; -1 = no node lists the keypoint), drawn from a stream of
    its own.  A keyframe keypoint built from a frame keypoint (its descriptor within max_flips bits) shares that keypoint's node, except
    a `split_frac` share that lands in another node.  A `lookalike_frac` share of them gets a look-alike: the frame keypoint nearest to
    its source moves into the same node and the keyframe descriptor moves towards it until the best distance is <= 50 but fails the
    0.7 ratio test.  `unnoded_frac` of the frame's keypoints and `kf_unnoded_frac` of the keyframe's are in no node.  n_nodes = 1 puts
    every listed keypoint into one node (all pairs meet)."""
    fr = make_robust_frame(kps, desc, camera, seed=seed, stereo=stereo, **robust_kw)
    rng = np.random.default_rng([int(seed), 0xB0])
    desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
    kf = fr["keyframe"]
    kdesc = np.array(kf["desc"], np.uint8)
    n_kp, n_kf = len(desc), len(kdesc)
    d = _hamming_rows(kdesc, desc) if n_kp else np.zeros((n_kf, 0), np.int32)
    src = d.argmin(1) if n_kp else np.full(n_kf, -1)
    true = (d.min(1) <= robust_kw.get("max_flips", 20)) if n_kp else np.zeros(n_kf, bool)
    kp_node = rng.integers(0, n_nodes, n_kp).astype(np.int32)
    share = true & (rng.random(n_kf) >= split_frac)
    look = share & (rng.random(n_kf) < lookalike_frac)
    for j in np.nonzero(look)[0]:
        a = src[j]
        da = np.bitwise_count(desc ^ desc[a]).sum(-1)
        da[a] = 1 << 20
        b = int(da.argmin())
        D = int(da[b])
        k = int(np.floor(0.7 * D / 1.7)) + 1                     # 0.7 * (D - k) < k: the ratio test rejects; k <= 50 passes the threshold
        if k > 50 or k > D:
            continue
        bits = np.nonzero(np.unpackbits(desc[a] ^ desc[b], bitorder="little"))[0]
        x = np.unpackbits(desc[a], bitorder="little")
        x[rng.choice(bits, k, replace=False)] ^= 1
        kdesc[j] = np.packbits(x, bitorder="little")
        kp_node[b] = kp_node[a]
    knode = rng.integers(0, n_nodes, n_kf).astype(np.int32)
    knode[share] = kp_node[src[share]]
    split = true & ~share
    if n_nodes > 1:
        knode[split] = (kp_node[src[split]] + rng.integers(1, n_nodes, split.sum())) % n_nodes
    kp_node[rng.random(n_kp) < unnoded_frac] = -1
    knode[rng.random(n_kf) < kf_unnoded_frac] = -1
    return dict(fr, kp_node=kp_node, keyframe=dict(kf, desc=kdesc, node=knode))


def make_mapping_problem(seed, n_neighbours=10, n_keypoints=2000, model="perspective", stereo=False, num_levels=8, scale_factor=1.2):
    """A current keyframe and `n_neighbours` ordered covisibilities for the mapping module's landmark creation
    (mapping_module::create_new_landmarks, two_view_triangulator).  Returns (cur, neighbours): keyframe dicts in the shape of
    stella_vslam_b200.mapping (poses, camera, undistorted keypoints, octaves, bearings, descriptors, BoW nodes, no_landmark and, with
    `stereo`, x_right / depth).  model: "perspective" (640 x 480, f = 500) or "equirectangular" (1920 x 960; stereo is not defined there).
    Built in: points seen by the current keyframe and by several neighbours (so the row claims between ranks decide outcomes), far
    points with near-parallel rays, correspondences shifted along the epipolar line (points behind a camera, depth tests), perturbed
    x_right and pixel noise of varied strength (chi-square tests), inconsistent octaves (scale-ratio test) and keypoints that already
    carry a landmark."""
    rng = np.random.default_rng(seed)
    equirect = model == "equirectangular"
    assert not (equirect and stereo)
    sf = np.cumprod(np.concatenate([[np.float32(1.0)], np.full(num_levels - 1, np.float32(scale_factor))])).astype(np.float32)
    sigma_sq = (sf * sf).astype(np.float32)
    fx = fy = 500.0
    cx, cy, cols, rows = 320.0, 240.0, 1920.0, 960.0
    true_baseline = 0.1
    n_pts = int(1.2 * n_keypoints)
    depth = rng.uniform(2.0, 25.0, n_pts)
    far = rng.random(n_pts) < 0.05
    depth[far] = rng.uniform(200.0, 2000.0, far.sum())                    # near-parallel rays
    if equirect:
        d = rng.normal(0, 1, (n_pts, 3))
        d /= np.linalg.norm(d, axis=1, keepdims=True)
    else:
        d = np.stack([rng.uniform(-0.6, 0.6, n_pts), rng.uniform(-0.45, 0.45, n_pts), np.ones(n_pts)], 1)
        d /= np.linalg.norm(d, axis=1, keepdims=True)
    pts = d * depth[:, None]
    pdesc = rng.integers(0, 256, (n_pts, 32), dtype=np.uint8)
    pnode = rng.integers(0, 120, n_pts).astype(np.int32)
    octave_pt = rng.choice(num_levels, n_pts, p=np.array([.3, .22, .16, .12, .08, .06, .04, .02])).astype(np.int32)

    def pose(R, c):
        P, W = np.eye(4), np.eye(4)
        P[:3, :3], P[:3, 3] = R, -R @ c
        W[:3, :3], W[:3, 3] = R.T, c
        return P, W

    def flip(desc, n_bits):
        out = desc.copy()
        for k in range(len(out)):
            for b in rng.choice(256, n_bits[k], replace=False):
                out[k, b // 8] ^= np.uint8(1 << (b % 8))
        return out

    def view(R, c, n_kp, vis_frac, shifted_frac):
        P, W = pose(R, c)
        pc = pts @ R.T + P[:3, 3]
        if equirect:
            visible = np.ones(n_pts, bool)
        else:
            with np.errstate(divide="ignore", invalid="ignore"):
                u, v = fx * pc[:, 0] / pc[:, 2] + cx, fy * pc[:, 1] / pc[:, 2] + cy
            visible = (pc[:, 2] > 0.5) & (u > 0) & (u < 640) & (v > 0) & (v < 480)
        cand = np.flatnonzero(visible)
        n_obs = min(len(cand), int(vis_frac * n_kp))
        obs = np.sort(rng.choice(cand, n_obs, replace=False))
        n_cl = n_kp - n_obs
        pt_idx = np.concatenate([obs, np.full(n_cl, -1)])
        perm = rng.permutation(n_kp)
        pt_idx = pt_idx[perm]
        # camera-frame direction per keypoint: observed points (some shifted along the ray of the current keyframe), clutter at random
        X = np.where(pt_idx[:, None] >= 0, pts[np.maximum(pt_idx, 0)], 0.0)
        shifted = (pt_idx >= 0) & (rng.random(n_kp) < shifted_frac)
        s = rng.uniform(-1.5, 3.0, n_kp)
        X = np.where(shifted[:, None], X * s[:, None], X)                # the current keyframe sits at the origin
        Xc = X @ R.T + P[:3, 3]
        clutter = pt_idx < 0
        rnd = np.stack([rng.uniform(-0.6, 0.6, n_kp), rng.uniform(-0.45, 0.45, n_kp), np.ones(n_kp)], 1) * rng.uniform(2, 30, (n_kp, 1))
        if equirect:
            rnd = rng.normal(0, 1, (n_kp, 3)) * rng.uniform(2, 30, (n_kp, 1))
        Xc = np.where(clutter[:, None], rnd, Xc)
        bad = np.zeros(n_kp, bool) if equirect else (Xc[:, 2] <= 0.1)                              # shifted behind this camera: not observable, make it clutter
        Xc[bad] = rnd[bad]
        clutter |= bad
        noise_px = rng.choice([0.2, 0.7, 1.5, 2.5], n_kp, p=[.4, .3, .2, .1])
        oct_ = np.where(clutter, rng.integers(0, num_levels, n_kp), octave_pt[np.maximum(pt_idx, 0)]).astype(np.int32)
        wrong_oct = ~clutter & (rng.random(n_kp) < 0.04)
        oct_[wrong_oct] = np.where(oct_[wrong_oct] < 4, num_levels - 1, 0)
        if equirect:
            b = Xc / np.linalg.norm(Xc, axis=1, keepdims=True)
            lat, lon = -np.arcsin(b[:, 1]), np.arctan2(b[:, 0], b[:, 2])
            x = cols * (0.5 + lon / (2 * np.pi)) + rng.normal(0, 1, n_kp) * noise_px
            y = rows * (0.5 - lat / np.pi) + rng.normal(0, 1, n_kp) * noise_px
            x, y = x.astype(np.float32), y.astype(np.float32)
            lon2, lat2 = (x.astype(np.float64) / cols - 0.5) * 2 * np.pi, -(y.astype(np.float64) / rows - 0.5) * np.pi
            bearings = np.stack([np.cos(lat2) * np.sin(lon2), -np.sin(lat2), np.cos(lat2) * np.cos(lon2)], 1)
        else:
            x = (fx * Xc[:, 0] / Xc[:, 2] + cx + rng.normal(0, 1, n_kp) * noise_px).astype(np.float32)
            y = (fy * Xc[:, 1] / Xc[:, 2] + cy + rng.normal(0, 1, n_kp) * noise_px).astype(np.float32)
            bearings = np.stack([(x - cx) / fx, (y - cy) / fy, np.ones(n_kp)], 1)
            bearings /= np.linalg.norm(bearings, axis=1, keepdims=True)
        desc = np.where(clutter[:, None], rng.integers(0, 256, (n_kp, 32), dtype=np.uint8), pdesc[np.maximum(pt_idx, 0)])
        desc = flip(desc, rng.integers(0, 14, n_kp))
        node = np.where(clutter, rng.integers(0, 120, n_kp), pnode[np.maximum(pt_idx, 0)]).astype(np.int32)
        kf = dict(pose_cw=P, pose_wc=W, model=1 if equirect else 0, fx=fx, fy=fy, cx=cx, cy=cy, fx_inv=1.0 / fx, fy_inv=1.0 / fy,
                  focal_x_baseline=fx * true_baseline if stereo else 0.0, true_baseline=true_baseline if stereo else 0.0, cols=cols, rows=rows,
                  img_bounds=(0.0, 640.0, 0.0, 480.0),
                  scale_factor=np.float32(scale_factor), scale_factors=sf, level_sigma_sq=sigma_sq, x=x, y=y, octave=oct_,
                  bearings=np.ascontiguousarray(bearings), desc=np.ascontiguousarray(desc), node=node,
                  no_landmark=(rng.random(n_kp) >= 0.25).astype(np.uint8), x_right=None, depth=None, angle=np.zeros(n_kp, np.float32))
        if stereo:
            has = (rng.random(n_kp) < 0.5) & (Xc[:, 2] > 0.5) & (Xc[:, 2] < 60.0)
            z = Xc[:, 2].astype(np.float32)
            xr = (x - np.float32(fx * true_baseline) / z + rng.normal(0, 0.3, n_kp).astype(np.float32)).astype(np.float32)
            off = has & (rng.random(n_kp) < 0.08)
            xr[off] += rng.uniform(-6, 6, off.sum()).astype(np.float32)    # x_right off: 3-dof chi-square
            kf["x_right"] = np.where(has & (xr >= 0), xr, np.float32(-1)).astype(np.float32)
            kf["depth"] = np.where(kf["x_right"] >= 0, z, np.float32(-1)).astype(np.float32)
        return kf

    cur = view(np.eye(3), np.zeros(3), n_keypoints, 0.8, 0.0)
    neighbours = []
    for r in range(n_neighbours):
        c = rng.normal(0, 1, 3) * np.array([0.6, 0.2, 0.6])
        c *= rng.uniform(0.3, 1.2) / max(np.linalg.norm(c), 1e-9)
        R = _rodrigues(rng.normal(0, 0.06, 3))
        neighbours.append(view(R, c, n_keypoints, 0.7, 0.05))
    return cur, neighbours


def make_pnp_problem(seed=0, n=300, inlier_frac=0.5, model="perspective", case=None):
    """2D-3D matches of a lost frame for solve::pnp_solver, on make_pose_problem's geometry: a true pose, points at 2-60 m, inlier
    bearings rotated away from the true ray by less than half of their octave's threshold (scale_factors[octave] degrees), outliers with
    random bearings, octaves 0-7 with the float 1.2 recurrence.  model: "perspective" (bearings with z > 0, KITTI frustum) or "equirect"
    (all directions, negative z included, so compute_pcs' sign flip is exercised).  case: None, "coplanar" (world points on one plane:
    the pseudo-inverse of the barycentric coordinates drops a singular value <= 1e-6) or "min_inliers" (exactly 10 true inliers).
    Returns dict(bearings, points, octaves, scale_factors, gt_rot_cw, gt_trans_cw, gt_inlier); min sets are drawn by the caller."""
    rng = np.random.default_rng(seed)
    equirect = model == "equirect"
    sf = np.cumprod(np.concatenate([[np.float32(1.0)], np.full(7, np.float32(1.2))])).astype(np.float32)
    Rcw = _rot_y(0.3 * rng.standard_normal()) @ _rodrigues(0.05 * rng.standard_normal(3))
    tcw = rng.normal(0, 2.0, 3)
    depth = rng.uniform(2, 60, n)
    if equirect:
        d = rng.standard_normal((n, 3))
        pc = d / np.linalg.norm(d, axis=1, keepdims=True) * depth[:, None]
    else:
        u, v = rng.uniform(20, KITTI["cols"] - 20, n), rng.uniform(20, KITTI["rows"] - 20, n)
        pc = np.stack([(u - KITTI["cx"]) / KITTI["fx"] * depth, (v - KITTI["cy"]) / KITTI["fy"] * depth, depth], 1)
    if case == "coplanar" and n:
        # a plane in the world: the camera-frame points are pushed onto R (z_w = 0) expressed in the camera
        pw0 = (pc - tcw) @ Rcw
        pw0[:, 2] = 0.0
        pc = pw0 @ Rcw.T + tcw
        if not equirect:
            pc[:, 2] = np.abs(pc[:, 2]) + 2.0
            pw0 = (pc - tcw) @ Rcw
            pw0[:, 2] = 0.0
            pc = pw0 @ Rcw.T + tcw
    pw = (pc - tcw) @ Rcw
    if case == "coplanar":
        pw[:, 2] = 0.0
        pc = pw @ Rcw.T + tcw
    octaves = rng.integers(0, 8, n).astype(np.int32)
    n_in = 10 if case == "min_inliers" else int(round(inlier_frac * n))
    inl = np.zeros(n, bool)
    inl[rng.permutation(n)[:n_in]] = True
    ray = pc / np.linalg.norm(pc, axis=1, keepdims=True)
    thr = np.deg2rad(sf[octaves].astype(np.float64))
    # a perpendicular direction per ray, then a rotation by 5-45 % of the threshold: far from the decision boundary
    perp = np.cross(ray, rng.standard_normal((n, 3)))
    perp /= np.linalg.norm(perp, axis=1, keepdims=True)
    ang = rng.uniform(0.05, 0.45, n) * thr
    bear = np.cos(ang)[:, None] * ray + np.sin(ang)[:, None] * perp
    out = ~inl
    if out.any():
        if equirect:
            o = rng.standard_normal((out.sum(), 3))
        else:
            uo, vo = rng.uniform(20, KITTI["cols"] - 20, out.sum()), rng.uniform(20, KITTI["rows"] - 20, out.sum())
            o = np.stack([(uo - KITTI["cx"]) / KITTI["fx"], (vo - KITTI["cy"]) / KITTI["fy"], np.ones(out.sum())], 1)
        o /= np.linalg.norm(o, axis=1, keepdims=True)
        # keep the outliers clearly outside their threshold (at least 3 x the octave's threshold off the true ray): a random bearing
        # too close to the ray is replaced by the ray turned 4-6 thresholds away (z stays positive for the perspective frustum)
        far = np.sum(o * ray[out], 1) < np.cos(3 * thr[out])
        a = rng.uniform(4.0, 6.0, out.sum()) * thr[out]
        turned = np.cos(a)[:, None] * ray[out] + np.sin(a)[:, None] * perp[out]
        o[~far] = turned[~far]
        bear[out] = o
    return dict(bearings=bear, points=pw, octaves=octaves, scale_factors=sf, gt_rot_cw=Rcw, gt_trans_cw=tcw, gt_inlier=inl)


def make_essential_problem(seed=0, n=500, inlier_frac=0.6, model="perspective", case=None, noise=5e-4):
    """Matched bearings of two views for solve::essential_solver: a true R_21 / t_21 (unit translation), points at 2-30 m, inlier
    bearings of view 2 turned off their true ray by up to `noise` rad, outliers with view-2 bearings at least 3 deg away from their
    epipolar plane.  model: "perspective" (z > 0, KITTI frustum) or "equirect" (all directions, backward bearings included).
    case: None; "pure_rotation" (|t_21| = 1e-4 m); "planar" (all points on one plane); "duplicated" (a fifth of the matches are copies
    of others, so minimal sets with repeated bearings occur); "n5" (five noise-free inliers); "inliers8" / "inliers9" / "inliers10"
    (exactly 8, 9 or 10 noise-free inliers among 10, 11 or 14 matches, so RANSAC keeps exactly that many).
    Returns dict(bearings_1, bearings_2 (n x 3, in match order), E_21 (= [t_21]x R_21), R_21, t_21, gt_inlier)."""
    rng = np.random.default_rng(seed)
    equirect = model == "equirect"
    fixed = {"n5": (5, 5), "inliers8": (10, 8), "inliers9": (11, 9), "inliers10": (14, 10)}
    if case in fixed:
        n, n_in = fixed[case]
        noise = 0.0
    else:
        n_in = int(round(inlier_frac * n))
    R = _rodrigues(0.15 * rng.standard_normal(3))
    t = rng.standard_normal(3)
    t /= np.linalg.norm(t)
    if case == "pure_rotation":
        t *= 1e-4
    depth = rng.uniform(2, 30, n)
    if equirect:
        d = rng.standard_normal((n, 3))
        P = d / np.linalg.norm(d, axis=1, keepdims=True) * depth[:, None]
    else:
        u, v = rng.uniform(20, KITTI["cols"] - 20, n), rng.uniform(20, KITTI["rows"] - 20, n)
        P = np.stack([(u - KITTI["cx"]) / KITTI["fx"] * depth, (v - KITTI["cy"]) / KITTI["fy"] * depth, depth], 1)
    if case == "planar":  # the plane z = 8 + 0.2 x - 0.1 y (perspective) or x = 4 + 0.3 z (equirect)
        if equirect:
            P[:, 0] = 4.0 + 0.3 * P[:, 2]
        else:
            P[:, 2] = 8.0 + 0.2 * P[:, 0] - 0.1 * P[:, 1]
    unit = lambda a: a / np.linalg.norm(a, axis=-1, keepdims=True)
    b1 = unit(P)
    b2 = unit(P @ R.T + t)
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    E = tx @ R
    if noise > 0:
        perp = unit(np.cross(b2, rng.standard_normal((n, 3))))
        ang = rng.uniform(0, noise, n)
        b2 = np.cos(ang)[:, None] * b2 + np.sin(ang)[:, None] * perp
    inl = np.zeros(n, bool)
    inl[rng.permutation(n)[:n_in]] = True
    for j in np.flatnonzero(~inl):
        nrm = unit(E @ b1[j])
        while True:
            o = rng.standard_normal(3) if equirect else np.array([(rng.uniform(20, KITTI["cols"] - 20) - KITTI["cx"]) / KITTI["fx"],
                                                                   (rng.uniform(20, KITTI["rows"] - 20) - KITTI["cy"]) / KITTI["fy"], 1.0])
            o = unit(o)
            if abs(o @ nrm) > np.sin(np.deg2rad(3.0)):
                break
        b2[j] = o
    if case == "duplicated":
        k = n // 5
        src, dst = rng.choice(n, k, replace=False), rng.choice(n, k, replace=False)
        b1[dst], b2[dst], inl[dst] = b1[src], b2[src], inl[src]
    return dict(bearings_1=np.ascontiguousarray(b1), bearings_2=np.ascontiguousarray(b2), E_21=E, R_21=R, t_21=t, gt_inlier=inl)


EUROC_MONO = dict(fx=458.654, fy=457.296, cx=367.215, cy=248.375, cols=752, rows=480)  # example/euroc/EuRoC_mono.yaml


def make_twoview_problem(seed=0, n=500, inlier_frac=0.7, scene="general", case=None, noise=0.5, camera="euroc"):
    """Two monocular frames for homography_solver / fundamental_solver: undistorted pixel keypoints of both frames, with extra unmatched
    keypoints in each (normalisation runs over all of them), and matches in ascending order of the frame-1 index.  A true R_21 (a few
    degrees), t_21 (0.3 m), inlier keypoints of frame 2 moved by Gaussian pixel noise `noise`, outliers at least 6 px from their true
    epipolar line.  scene: "general" (depths 2-10 m) or "planar" (the plane n.X = 5 m in frame 1).  camera: "euroc" or "kitti".
    case: None; "pure_rotation" (t_21 = 0); "collinear" (noise-free, R_21 = I, t_21 along x; four fifths of the points on one 3D
    line parallel to the baseline, which images to one row of both frames, the same float y for every point, so normalisation keeps
    them exactly collinear and most minimal sets make H's coefficient matrix lose rank); "n7" / "n8" (7 or 8 matches); "inliers5" / "inliers9" / "inliers10"
    (exactly 5, 9 or 10 noise-free inliers among 10, 12 or 14 matches: RANSAC keeps exactly that many, so the recompute takes H's tall
    path at 10 rows and F's square or tall path); "duplicated" (a fifth of the matches copy the coordinates of others in both frames).
    Returns dict(keypts_1, keypts_2 ((n_k, 2) float32), matches_12 ((n, 2) int32), R_21, t_21, K, H_21 (planar or pure rotation, else
    None), F_21 (None under pure rotation), gt_inlier (match order), cols, rows)."""
    rng = np.random.default_rng(seed)
    cam = EUROC_MONO if camera == "euroc" else KITTI
    K = np.array([[cam["fx"], 0, cam["cx"]], [0, cam["fy"], cam["cy"]], [0, 0, 1.0]])
    Ki = np.linalg.inv(K)
    cols, rows = cam["cols"], cam["rows"]
    fixed = {"n7": (7, 7), "n8": (8, 8), "inliers5": (10, 5), "inliers9": (12, 9), "inliers10": (14, 10)}
    if case in fixed:
        n, n_in = fixed[case]
        if case.startswith("inliers"):
            noise = 0.0
    else:
        n_in = int(round(inlier_frac * n))
    if case == "collinear":
        noise = 0.0
    R = _rodrigues(0.05 * rng.standard_normal(3))
    t = rng.standard_normal(3)
    t *= 0.3 / np.linalg.norm(t)
    if case == "pure_rotation":
        t = np.zeros(3)
    nrm = np.array([0.1 * rng.standard_normal(), 0.1 * rng.standard_normal(), 1.0])
    if case == "collinear":
        R, t, nrm[0] = np.eye(3), np.array([0.3, 0.0, 0.0]), 0.0
    nrm /= np.linalg.norm(nrm)
    line_y = 0.3
    line_z = (5.0 - nrm[1] * line_y) / nrm[2] if scene == "planar" else 6.0
    P, p1, p2 = [], [], []
    while len(P) < n:
        if case == "collinear" and rng.uniform() < 0.8:
            X = np.array([rng.uniform(-2.0, 2.0), line_y, line_z])
        else:
            ray = Ki @ np.array([rng.uniform(10, cols - 10), rng.uniform(10, rows - 10), 1.0])
            X = ray * (5.0 / (nrm @ ray) if scene == "planar" else rng.uniform(2, 10))
        Y = R @ X + t
        if X[2] <= 0 or Y[2] <= 0:
            continue
        a, b = K @ (X / X[2]), K @ (Y / Y[2])
        if not (0 <= a[0] < cols and 0 <= a[1] < rows and 0 <= b[0] < cols and 0 <= b[1] < rows):
            continue
        P.append(X)
        p1.append(a[:2])
        p2.append(b[:2])
    p1, p2 = np.array(p1), np.array(p2)
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    F = None if case == "pure_rotation" else Ki.T @ tx @ R @ Ki
    H = K @ (R + np.outer(t, nrm) / 5.0) @ Ki if (scene == "planar" or case == "pure_rotation") else None
    if noise > 0:
        p2 = p2 + noise * rng.standard_normal(p2.shape)
    inl = np.zeros(n, bool)
    inl[rng.permutation(n)[:n_in]] = True
    for j in np.flatnonzero(~inl):
        while True:
            o = np.array([rng.uniform(0, cols), rng.uniform(0, rows)])
            if F is None:
                if np.linalg.norm(o - p2[j]) > 20.0:
                    break
                continue
            line = F @ np.array([p1[j, 0], p1[j, 1], 1.0])
            if abs(line @ np.array([o[0], o[1], 1.0])) / np.hypot(line[0], line[1]) > 6.0:
                break
        p2[j] = o
    if case == "duplicated":
        k = n // 5
        src, dst = rng.choice(n, k, replace=False), rng.choice(n, k, replace=False)
        p1[dst], p2[dst], inl[dst] = p1[src], p2[src], inl[src]
    n_extra = max(5, n // 3)
    kp1 = np.concatenate([p1, np.stack([rng.uniform(0, cols, n_extra), rng.uniform(0, rows, n_extra)], 1)])
    kp2 = np.concatenate([p2, np.stack([rng.uniform(0, cols, n_extra), rng.uniform(0, rows, n_extra)], 1)])
    perm1, perm2 = rng.permutation(len(kp1)), rng.permutation(len(kp2))
    kp1, kp2 = kp1[perm1], kp2[perm2]
    pos1, pos2 = np.argsort(perm1)[:n], np.argsort(perm2)[:n]  # where match j's keypoints landed
    order = np.argsort(pos1)
    matches = np.stack([pos1[order], pos2[order]], 1).astype(np.int32)
    return dict(keypts_1=np.ascontiguousarray(kp1, np.float32), keypts_2=np.ascontiguousarray(kp2, np.float32), matches_12=matches, R_21=R,
                t_21=t, K=K, H_21=H, F_21=F, gt_inlier=inl[order], cols=cols, rows=rows)


def make_pose_graph(n_keyframes=500, seed=0, fix_scale=False, laps=1.5, window=8, rot_noise=2e-3, trans_noise=0.01, scale_noise=2e-3,
                    lm_per_keyframe=4, min_num_shared_lms=100, return_description=False):
    """A loop-closure pose graph for optimize.graph_optimizer, built by optimize.build_essential_graph.

    The camera drives `laps` times around a circle of keyframes (laps > 1 revisits the ground of the first lap), facing along the
    track.  The keyframe poses are dead reckoning from noisy relative motions (rotation, translation and, unless fix_scale, scale drift
    as a monocular map drifts).  Covisibility weights (shared landmarks) come from the overlap of the true views: keyframes within about
    `window` steps, and the keyframes of other laps at the same place.  The spanning tree is the chain of keyframes (the root is keyframe
    0).  The last keyframe closes a loop with the first-lap keyframe at its place; its neighbours are pre-corrected through it as
    correct_loop does, and the loop connections join them to the loop keyframe's neighbours.  Landmarks: `lm_per_keyframe` per keyframe,
    in front of their reference keyframe; every third landmark of the current keyframe's neighbourhood is re-referenced to the loop
    keyframe (found_lm_to_ref_keyfrm_id).  Returns the graph dict (and the flat description with return_description)."""
    from stella_vslam_b200.optimize import build_essential_graph, sim3_from_rts, sim3_inverse, sim3_mul

    rng = np.random.default_rng(seed)
    n = int(n_keyframes)
    per_lap = max(8, int(round(n / laps)))
    radius = per_lap * 1.0 / (2 * np.pi)                      # 1 m between keyframes
    ang = 2 * np.pi * np.arange(n) / per_lap
    # true camera: at (r cos a, 0, r sin a), optical axis (z) along the track
    R_true, t_true = [], []
    for a in ang:
        Rwc = _rot_y(-a)                                       # camera z axis rotates with the heading
        c = np.array([radius * np.cos(a), 0.0, radius * np.sin(a)])
        R_true.append(Rwc.T)
        t_true.append(-Rwc.T @ c)
    R_true, t_true = np.array(R_true), np.array(t_true)
    # dead reckoning with drift
    R_est, t_est, sc = [R_true[0]], [t_true[0]], 1.0
    for i in range(1, n):
        R_rel = R_true[i] @ R_true[i - 1].T
        t_rel = t_true[i] - R_rel @ t_true[i - 1]
        if not fix_scale:
            sc *= 1.0 + scale_noise * rng.standard_normal()
        R_rel = _rodrigues(rot_noise * rng.standard_normal(3)) @ R_rel
        t_rel = sc * t_rel + trans_noise * rng.standard_normal(3)
        R_est.append(R_rel @ R_est[-1])
        t_est.append(R_rel @ t_est[-1] + t_rel)
    # covisibility weights from the overlap of the true views
    pos = np.stack([radius * np.cos(ang), np.zeros(n), radius * np.sin(ang)], 1)
    weights = []
    for i in range(n):
        d = np.linalg.norm(pos - pos[i], axis=1)
        dh = np.abs((ang - ang[i] + np.pi) % (2 * np.pi) - np.pi)
        w = (400 * np.clip(1 - d / (window * 1.25), 0, 1) * np.clip(np.cos(dh), 0, 1)).astype(int)
        w[i] = 0
        nz = np.nonzero(w > 0)[0]
        order = nz[np.argsort(-w[nz], kind="stable")]
        weights.append([(int(j), int(w[j])) for j in order])
    curr, loop = n - 1, int((n - 1) % per_lap)
    if loop >= curr - window:
        loop = 0
    kfs = []
    for i in range(n):
        kfs.append(dict(id=i, rot_cw=R_est[i], trans_cw=t_est[i], erased=False, parent=(i - 1 if i else None), children=([i + 1] if i + 1 < n else []),
                        loop_edges=[], covisibilities=weights[i]))
    # correct_loop: the current keyframe's Sim3 from the loop keyframe, its neighbours pre-corrected through it
    E = {i: sim3_from_rts(R_est[i], t_est[i], 1.0) for i in range(n)}
    R_cl = R_true[curr] @ R_true[loop].T
    t_cl = t_true[curr] - R_cl @ t_true[loop]
    corr_c = sim3_mul(sim3_from_rts(R_cl, t_cl, 1.0), E[loop])
    if not fix_scale:
        corr_c[7] = 1.0 / sc                                   # undo the scale the dead reckoning drifted by
    neigh = [curr] + [j for j, w in weights[curr] if w >= min_num_shared_lms and j > loop + window][:window]
    non_corrected = {j: E[j] for j in neigh}
    pre_corrected = {j: (corr_c if j == curr else sim3_mul(sim3_mul(E[j], sim3_inverse(E[curr])), corr_c)) for j in neigh}
    loop_side = [loop] + [j for j, w in weights[loop] if w >= min_num_shared_lms and j < loop + window][:window]
    loop_connections = []
    for j in neigh:
        conn = [k for k in loop_side if dict(weights[j]).get(k, 0) >= min_num_shared_lms or (j == curr and k == loop)]
        if conn:
            loop_connections.append((j, conn))
    # landmarks in front of their reference keyframe, in the drifted map
    landmarks, found, lid = [], {}, 0
    for i in range(n):
        for _ in range(lm_per_keyframe):
            pc = np.array([rng.uniform(-3, 3), rng.uniform(-2, 2), rng.uniform(2, 10)])
            pw = R_est[i].T @ (pc - t_est[i])
            landmarks.append((lid, pw, i))
            if i in pre_corrected and lid % 3 == 0:
                found[lid] = loop
            lid += 1
    desc = dict(keyframes=kfs, curr_id=curr, loop_id=loop, loop_connections=loop_connections, non_corrected_Sim3s=non_corrected,
                pre_corrected_Sim3s=pre_corrected, min_num_shared_lms=min_num_shared_lms, fix_scale=fix_scale, landmarks=landmarks,
                found_lm_to_ref_keyfrm_id=found)
    graph = build_essential_graph(**desc)
    return (graph, desc) if return_description else graph


def make_sim3_pair(seed=0, n_matches=300, models=("perspective", "perspective"), fix_scale=False, outlier_frac=0.2, pixel_sigma=1.0,
                   init_noise=(0.02, 0.05, 0.02)):
    """A loop candidate for optimize.transform_optimizer: keyframe 1 of the map and keyframe 2 of a drifted map see the same physical
    points, and the gathered pairs are already matched (gather_mutual_edges' output layout).

    The drifted map is the true one under a Sim3 (scale 1 under fix_scale): its landmarks (pos_w_2) and keyframe 2's pose are expressed
    in it, so the true Sim3_12 maps keyframe 2's camera frame, at the drifted scale, into keyframe 1's.  models: camera of keyframe 1 and
    2, "perspective" or "equirect".  Observations carry level-dependent noise (pixel_sigma * 1.2^octave); a fraction outlier_frac of
    the pairs has a gross error of 20-80 px on one of its two observations.  The initial Sim3 is the truth perturbed by init_noise =
    (rotation rad, translation m, log scale), as the loop detector's estimate would be.  Returns the problem dict plus gt_sim3_12 and
    gt_outlier."""
    from stella_vslam_b200.optimize import sim3_from_rts

    rng = np.random.default_rng(seed)
    n = int(n_matches)

    def camera(model):
        if model == "equirect":
            return dict(model=1, fx=0.0, fy=0.0, cx=0.0, cy=0.0, fxb=0.0, cols=3840.0, rows=1920.0)
        return dict(model=0, fx=KITTI["fx"], fy=KITTI["fy"], cx=KITTI["cx"], cy=KITTI["cy"], fxb=0.0, cols=float(KITTI["cols"]),
                    rows=float(KITTI["rows"]))

    cam1, cam2 = camera(models[0]), camera(models[1])
    # true poses (camera from world): keyframe 2 is a nearby view of keyframe 1's scene
    R1 = _rot_y(0.3 * rng.standard_normal()) @ _rodrigues(0.03 * rng.standard_normal(3))
    t1 = rng.normal(0, 1.0, 3)
    R21 = _rot_y(0.05 * rng.standard_normal()) @ _rodrigues(0.02 * rng.standard_normal(3))
    R2 = R21 @ R1
    t2 = R21 @ t1 + np.array([rng.uniform(-0.8, 0.8), 0.1 * rng.standard_normal(), 0.2 * rng.standard_normal()])

    def proj(cam, pc):
        if cam["model"] == 1:
            th, ph = np.arctan2(pc[:, 0], pc[:, 2]), -np.arcsin(pc[:, 1] / np.linalg.norm(pc, axis=1))
            return np.stack([cam["cols"] * (0.5 + th / (2 * np.pi)), cam["rows"] * (0.5 - ph / np.pi)], 1)
        return np.stack([cam["fx"] * pc[:, 0] / pc[:, 2] + cam["cx"], cam["fy"] * pc[:, 1] / pc[:, 2] + cam["cy"]], 1)

    def visible(cam, pc):
        if cam["model"] == 1:
            return np.linalg.norm(pc, axis=1) > 1.0
        uv = proj(cam, np.where(pc[:, 2:3] > 0.5, pc, 1.0))
        return (pc[:, 2] > 0.5) & (uv[:, 0] > 10) & (uv[:, 0] < cam["cols"] - 10) & (uv[:, 1] > 10) & (uv[:, 1] < cam["rows"] - 10)

    X = np.zeros((0, 3))
    while len(X) < n:                                        # points seen by both keyframes, 4-40 m from keyframe 1
        m = 4 * n + 64
        depth = rng.uniform(4, 40, m)
        if cam1["model"] == 1:
            d = rng.standard_normal((m, 3))
            pc1 = d / np.linalg.norm(d, axis=1, keepdims=True) * depth[:, None]
        else:
            u, v = rng.uniform(20, cam1["cols"] - 20, m), rng.uniform(20, cam1["rows"] - 20, m)
            pc1 = np.stack([(u - cam1["cx"]) / cam1["fx"] * depth, (v - cam1["cy"]) / cam1["fy"] * depth, depth], 1)
        Xw = (pc1 - t1) @ R1
        ok = visible(cam2, Xw @ R2.T + t2)
        X = np.concatenate([X, Xw[ok]])[:n]
    # the drifted map: P_B = s_d R_d X + t_d; keyframe 2's pose in it
    s_d = 1.0 if fix_scale else float(np.exp(0.2 * rng.standard_normal()))
    R_d = _rodrigues(0.1 * rng.standard_normal(3))
    t_d = rng.normal(0, 2.0, 3)
    pos_w_1 = X.copy()
    pos_w_2 = s_d * X @ R_d.T + t_d
    rot_2w = R2 @ R_d.T
    trans_2w = s_d * t2 - rot_2w @ t_d
    R12 = R1 @ R2.T
    gt = sim3_from_rts(R12, t1 - R12 @ t2, 1.0 / s_d)
    # observations with octave-dependent noise
    inv_sigma = (np.float32(1.0) / np.cumprod(np.concatenate([[np.float32(1.0)], np.full(7, np.float32(1.2))])).astype(np.float32) ** 2).astype(np.float32)
    lv1, lv2 = rng.integers(0, 8, n), rng.integers(0, 8, n)
    obs_1 = proj(cam1, X @ R1.T + t1) + (pixel_sigma / np.sqrt(inv_sigma[lv1].astype(np.float64)))[:, None] * rng.standard_normal((n, 2))
    obs_2 = proj(cam2, X @ R2.T + t2) + (pixel_sigma / np.sqrt(inv_sigma[lv2].astype(np.float64)))[:, None] * rng.standard_normal((n, 2))
    bad = rng.random(n) < outlier_frac
    which = rng.integers(0, 2, n)
    for o, side in ((obs_1, 0), (obs_2, 1)):
        sel = bad & (which == side)
        o[sel] += rng.choice([-1, 1], (sel.sum(), 2)) * rng.uniform(20, 80, (sel.sum(), 2))
    # initial estimate: the truth perturbed
    dR = _rodrigues(init_noise[0] * rng.standard_normal(3) / np.sqrt(3))
    s0 = 1.0 / s_d if fix_scale else float(np.exp(init_noise[2] * rng.standard_normal())) / s_d
    t0 = dR @ (t1 - R12 @ t2) + init_noise[1] * rng.standard_normal(3) / np.sqrt(3)
    init = sim3_from_rts(dR @ R12, t0, s0)
    return dict(n_matches=n, fix_scale=bool(fix_scale), sim3_12=init, rot_1w=R1, trans_1w=t1, rot_2w=rot_2w, trans_2w=trans_2w, cam_1=cam1,
                cam_2=cam2, obs_1=obs_1.astype(np.float32), inv_sigma_sq_1=inv_sigma[lv1], pos_w_2=pos_w_2, obs_2=obs_2.astype(np.float32),
                inv_sigma_sq_2=inv_sigma[lv2], pos_w_1=pos_w_1, gt_sim3_12=gt, gt_outlier=bad)


def make_rgbd_frames(w=640, h=480, seed=0, depthmap_factor=5000.0, n_planes=4, hole_frac=0.05, saturated_frac=0.01, float_specials_frac=0.03):
    """An RGB-D frame as a TUM RGB-D sensor gives it: the gray frame of make_frame and a depth map built from a few planes between 0.3 and
    10 m.  Returns (gray u8 (h, w), depth u16 (h, w) at `depthmap_factor` counts per metre, depth f32 (h, w) in metres).
    The u16 map has zero-depth holes and saturated (65535) pixels; the f32 variant is the u16 map over the factor, with NaN, negative
    values and +inf sprinkled in."""
    rng = np.random.default_rng(seed)
    gray = make_frame(w, h, seed=seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    depth = np.full((h, w), np.inf)
    for _ in range(n_planes):  # z = z0 + gx * (x - cx) + gy * (y - cy) over a random rectangle; the nearest plane wins
        z0 = rng.uniform(0.3, 10.0)
        gx, gy = rng.uniform(-4e-3, 4e-3, 2)
        x0, y0 = rng.integers(0, w // 2), rng.integers(0, h // 2)
        x1, y1 = rng.integers(x0 + w // 4, w + 1), rng.integers(y0 + h // 4, h + 1)
        z = np.clip(z0 + gx * (xx - w / 2) + gy * (yy - h / 2), 0.3, 10.0)
        inside = (xx >= x0) & (xx < x1) & (yy >= y0) & (yy < y1)
        depth = np.where(inside & (z < depth), z, depth)
    depth = np.where(np.isinf(depth), rng.uniform(0.3, 10.0), depth)  # background wall
    d16 = np.clip(np.rint(depth * depthmap_factor), 0, 65535).astype(np.uint16)
    holes = rng.random((h, w)) < hole_frac
    holes |= (xx >= rng.integers(0, w - 40)) & (xx < rng.integers(40, w)) & (yy < 12)  # a dropped band, as structured-light sensors lose
    d16[holes] = 0
    d16[rng.random((h, w)) < saturated_frac] = 65535
    d32 = (d16.astype(np.float32) * np.float32(1.0 / depthmap_factor)).astype(np.float32)
    special = rng.random((h, w)) < float_specials_frac
    kinds = rng.integers(0, 3, (h, w))
    d32[special & (kinds == 0)] = np.nan
    d32[special & (kinds == 1)] = -rng.uniform(0.1, 5.0, int((special & (kinds == 1)).sum())).astype(np.float32)
    d32[special & (kinds == 2)] = np.inf
    return gray, d16, d32


def make_cull_map(rng, n_covisibilities=30, n_keypoints=2000, observers=8, landmark_frac=0.8, redundant_frac=0.5, stereo_frac=0.3,
                  erased_frac=0.02, n_others=6, cur_id=1000, depth_thr=5.0):
    """A covisibility neighbourhood of a new keyframe as local_map_cleaner::remove_redundant_keyframes sees it, as an object graph:
    dict(cur_id, keyframes {id: keyframe}, landmarks [landmark], covisibilities [ids in rank order]).
      keyframe: id, is_root, octave (undist_keypts_ octaves), x_right / depth (None without stereo), depth_thr, landmarks (landmark
                index per keypoint, -1 for none), will_be_erased, cannot_be_erased;
      landmark: observations {keyframe id: keypoint index} in insertion order, num_observations (stereo observations count 2),
                will_be_erased.
    The covisibilities' ids are spread below cur_id with a few in the recent window and above it; the oldest is the spanning root with
    probability 1/2.  Besides them, cur_id and `n_others` keyframes observe landmarks (rank -1).  A landmark has about `observers`
    observers.  A share `redundant_frac` of the keyframes sees its keypoints at a raised floor octave, which makes them redundant
    against the other observers; with the observation counts falling as keyframes are erased, some ranks are removed and some later
    ones are kept only because of an earlier removal.  Stereo keyframes carry x_right (about 70 % matched, weight 2) and depths in
    [-1, 1.5 depth_thr) with some exactly at depth_thr."""
    pool = rng.choice(np.arange(max(cur_id - 4 * n_covisibilities - n_others, 0), min(cur_id + 4, 1 << 32)), n_covisibilities + n_others + 1, replace=False)
    pool = [int(k) for k in pool if k != cur_id][:n_covisibilities + n_others]
    covs = pool[:n_covisibilities]
    ids = covs + pool[n_covisibilities:] + [cur_id]
    root = min(covs) if covs and rng.random() < 0.5 else None
    keyframes = {}
    for kid in ids:
        floor = int(rng.integers(0, 7)) if rng.random() < redundant_frac else 0
        kf = dict(id=kid, is_root=kid == root, octave=rng.integers(floor, 8, n_keypoints).astype(np.int32), x_right=None, depth=None,
                  depth_thr=float(depth_thr), landmarks=np.full(n_keypoints, -1, np.int64), will_be_erased=False, cannot_be_erased=False)
        if rng.random() < stereo_frac:
            kf["x_right"] = np.where(rng.random(n_keypoints) < 0.7, rng.uniform(0.0, 640.0, n_keypoints), -1.0).astype(np.float32)
            d = rng.uniform(-1.0, 1.5 * depth_thr, n_keypoints)
            d[rng.random(n_keypoints) < 0.05] = depth_thr
            kf["depth"] = d.astype(np.float32)
        keyframes[kid] = kf
    free = {kid: list(rng.permutation(n_keypoints)) for kid in ids}
    landmarks = []
    for _ in range(int(len(ids) * n_keypoints * landmark_frac / observers)):
        k = int(min(len(ids), 1 + rng.poisson(observers - 1)))
        obs = {}
        for o in rng.choice(len(ids), k, replace=False):
            kid = ids[int(o)]
            if free[kid]:
                obs[kid] = int(free[kid].pop())
        if not obs:
            continue
        li = len(landmarks)
        num = 0
        for kid, idx in obs.items():
            keyframes[kid]["landmarks"][idx] = li
            xr = keyframes[kid]["x_right"]
            num += 2 if xr is not None and 0 <= xr[idx] else 1
        landmarks.append(dict(observations=obs, num_observations=num, will_be_erased=bool(rng.random() < erased_frac)))
    return dict(cur_id=cur_id, keyframes=keyframes, landmarks=landmarks, covisibilities=covs)


def gather_cull_problem(cull_map, covisibilities=None, redundant_obs_ratio_thr=0.9):
    """The flat tables of b200_remove_redundant_keyframes (mapping.pack_cull_problems' dict) for an object-graph map of make_cull_map,
    as the reference-side adapter gathers them: the covisibilities (default: the map's list) in rank order, and every live landmark
    their keypoints list once, with its observations by any keyframe (rank -1 outside the list)."""
    keyframes, landmarks = cull_map["keyframes"], cull_map["landmarks"]
    covs = cull_map["covisibilities"] if covisibilities is None else list(covisibilities)
    rank = {kid: r for r, kid in enumerate(covs)}
    rows = {}
    out_covs = []
    for kid in covs:
        kf = keyframes[kid]
        kl = np.full(len(kf["landmarks"]), -1, np.int32)
        for idx in np.flatnonzero(kf["landmarks"] >= 0):
            li = int(kf["landmarks"][idx])
            if not landmarks[li]["will_be_erased"]:
                kl[idx] = rows.setdefault(li, len(rows))
        out_covs.append(dict(id=kid, is_root=kf["is_root"], kp_landmark=kl, depth=kf["depth"], depth_thr=kf["depth_thr"]))
    off, o_rank, o_oct, o_w = [0], [], [], []
    for li in rows:
        for kid, idx in landmarks[li]["observations"].items():
            kf = keyframes[kid]
            o_rank.append(rank.get(kid, -1))
            o_oct.append(int(kf["octave"][idx]))
            o_w.append(2 if kf["x_right"] is not None and 0 <= kf["x_right"][idx] else 1)
        off.append(len(o_rank))
    return dict(cur_id=cull_map["cur_id"], redundant_obs_ratio_thr=redundant_obs_ratio_thr, covisibilities=out_covs,
                obs_offsets=np.array(off, np.int32), obs_rank=np.array(o_rank, np.int32), obs_octave=np.array(o_oct, np.int32),
                obs_weight=np.array(o_w, np.uint8))
