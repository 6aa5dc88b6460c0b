"""CPU restatement of initialize::perspective / initialize::bearing_vector (test infrastructure): loads tests/initialize_oracle.c (with
tests/motion_track_oracle.c's reproject_to_image), compiled on first use into a temporary directory (the tree is never written), and
composes it with the two-view and essential RANSAC oracles.

  reconstruct(problem, model, M, inlier)   reconstruct_with_H / _F / _E from a solver's matrix and inlier flags
  initialize(problem)                      the whole initialize(): RANSAC, the rel_cost_H choice, reconstruct
Problems are the dicts of stella_vslam_b200.initialize.initialize_batch; results carry the same keys.
"""
import ctypes as C
import math

import numpy as np

import cbuild
import essential_oracle as EO
import twoview_oracle as TO

_lib = None

MODEL_NONE, MODEL_H, MODEL_F, MODEL_E = 0, 1, 2, 3
NAMES = {MODEL_NONE: None, MODEL_H: "H", MODEL_F: "F", MODEL_E: "E"}
STAGE_NO_MODEL, STAGE_DECOMPOSE, STAGE_MIN_VALID, STAGE_AMBIGUOUS, STAGE_PARALLAX, STAGE_MIN_TRIANGULATED, STAGE_SUCCEEDED = range(7)
DEFAULTS = dict(num_ransac_iters=100, min_num_triangulated=50, min_num_valid_pts=50, parallax_deg_thr=1.0, reproj_err_thr=4.0)
_MODEL_CODES = {"perspective": 0, "equirectangular": 1, "fisheye": 2, "radial_division": 3}


def lib():
    global _lib
    if _lib is None:
        L = cbuild.load("initialize_oracle.c", "motion_track_oracle.c")
        vp, i32, u32 = C.c_void_p, C.c_int, C.c_uint32
        L.ino_choose_H.argtypes = [C.c_float, C.c_float, i32]
        L.ino_svd33.argtypes = [vp, vp, vp, vp]
        L.ino_decompose_H.argtypes = [vp, vp, vp, vp, vp, vp, C.POINTER(i32)]
        L.ino_decompose_E.argtypes = [vp, vp, vp]
        L.ino_essential_of_F.argtypes = [vp, vp, vp, vp]
        L.ino_essential_of_F.restype = None
        L.ino_midpoint.argtypes = [vp, vp, vp, vp, vp]
        L.ino_midpoint.restype = None
        L.ino_triangulate.argtypes = [vp, vp, i32, C.c_float, i32, vp, vp, vp, vp, i32, vp, vp, vp, vp, C.POINTER(i32), C.POINTER(C.c_float)]
        L.ino_select.argtypes = [i32, vp, vp, vp, u32, u32, C.c_double, C.POINTER(i32)]
        L.ino_reconstruct.argtypes = ([i32, vp, vp, vp, vp, u32, u32, C.c_double, C.c_float, i32, vp, vp, vp, vp, i32, vp, vp] +
                                      [C.POINTER(i32)] * 2 + [vp] * 7)
        _lib = L
    return _lib


def _d(a, shape):
    return np.ascontiguousarray(np.asarray(a, np.float64).reshape(shape))


def svd33(A):
    """(U, s, V, status) of JacobiSVD<Mat33_t>."""
    A = _d(A, 9)
    U, s, V = np.zeros(9), np.zeros(3), np.zeros(9)
    st = lib().ino_svd33(A.ctypes.data, U.ctypes.data, s.ctypes.data, V.ctypes.data)
    return U.reshape(3, 3), s, V.reshape(3, 3), st


def decompose_H(H, K1, K2):
    """homography_solver::decompose: (R (8, 3, 3), t (8, 3), normals (8, 3)) or None when the rank test rejects."""
    H, K1, K2 = _d(H, 9), _d(K1, 9), _d(K2, 9)
    R, t, n, st = np.zeros(72), np.zeros(24), np.zeros(24), C.c_int()
    ok = lib().ino_decompose_H(H.ctypes.data, K1.ctypes.data, K2.ctypes.data, R.ctypes.data, t.ctypes.data, n.ctypes.data, C.byref(st))
    return (R.reshape(8, 3, 3), t.reshape(8, 3), n.reshape(8, 3)) if ok else None


def decompose_E(E):
    """essential_solver::decompose: (R (4, 3, 3), t (4, 3))."""
    E = _d(E, 9)
    R, t = np.zeros(36), np.zeros(12)
    lib().ino_decompose_E(E.ctypes.data, R.ctypes.data, t.ctypes.data)
    return R.reshape(4, 3, 3), t.reshape(4, 3)


def essential_of_F(F, K1, K2):
    F, K1, K2 = _d(F, 9), _d(K1, 9), _d(K2, 9)
    E = np.zeros(9)
    lib().ino_essential_of_F(F.ctypes.data, K1.ctypes.data, K2.ctypes.data, E.ctypes.data)
    return E.reshape(3, 3)


def midpoint(b1, b2, R, t):
    b1, b2, R, t = _d(b1, 3), _d(b2, 3), _d(R, 9), _d(t, 3)
    p = np.zeros(3)
    lib().ino_midpoint(b1.ctypes.data, b2.ctypes.data, R.ctypes.data, t.ctypes.data, p.ctypes.data)
    return p


def choose_H(cost_H, cost_F, valid_H):
    return bool(lib().ino_choose_H(float(cost_H), float(cost_F), int(bool(valid_H))))


def select(nums_valid, num_triangulated, parallax_cos, min_num_valid_pts, min_num_triangulated, cos_thr):
    """find_most_plausible_pose's rules: (stage, best)."""
    nv, nt = np.ascontiguousarray(nums_valid, np.int32), np.ascontiguousarray(num_triangulated, np.int32)
    pc = np.ascontiguousarray(parallax_cos, np.float32)
    best = C.c_int()
    st = lib().ino_select(len(nv), nv.ctypes.data, nt.ctypes.data, pc.ctypes.data, int(min_num_valid_pts), int(min_num_triangulated),
                          float(cos_thr), C.byref(best))
    return st, best.value


def _cams(p):
    out = []
    for cam, b in ((p["cam_ref"], p.get("bounds_ref", (0, 0, 0, 0))), (p["cam_cur"], p.get("bounds_cur", (0, 0, 0, 0)))):
        out += [_MODEL_CODES[cam.get("model", "perspective")]] + [float(cam.get(k, 0.0)) for k in ("fx", "fy", "cx", "cy", "cols", "rows")]
        out += [float(np.float32(v)) for v in b]
    return np.ascontiguousarray(out, np.float64)


def K_of(cam):
    g = lambda k: float(cam.get(k, 0.0))  # noqa: E731
    return np.array([[g("fx"), 0.0, g("cx")], [0.0, g("fy"), g("cy")], [0.0, 0.0, 1.0]])


def matches_of(ref_matches_with_cur):
    """ref_cur_matches_ (ref order; negative entries are no match) as (n, 2) int32."""
    m = np.asarray(ref_matches_with_cur, np.int64).reshape(-1)
    idx = np.nonzero(m >= 0)[0]
    return np.ascontiguousarray(np.stack([idx, m[idx]], 1).astype(np.int32).reshape(-1, 2))


class _Frame:
    def __init__(self, p):
        self.ur = np.ascontiguousarray(np.asarray(p["undist_ref"], np.float32).reshape(-1, 2))
        self.br = _d(p["bearings_ref"], (-1, 3))
        self.uc = np.ascontiguousarray(np.asarray(p["undist_cur"], np.float32).reshape(-1, 2))
        self.bc = _d(p["bearings_cur"], (-1, 3))
        self.mt = matches_of(p["ref_matches_with_cur"])


def param(p, k):
    return p.get(k, DEFAULTS[k])


def cos_thr(p):
    return math.cos(float(np.float32(param(p, "parallax_deg_thr"))) / 180.0 * math.pi)


def triangulate(p, R, t, inlier, depth_is_positive):
    """base::triangulate for one hypothesis: (nums_valid, num_triangulated, parallax_cos, pts (n_ref, 3), flags (n_ref,))."""
    f = _Frame(p)
    Rt = np.ascontiguousarray(np.concatenate([np.asarray(R, np.float64).reshape(9), np.asarray(t, np.float64).reshape(3)]))
    inl = np.ascontiguousarray(np.asarray(inlier, np.uint8).reshape(-1))
    n_ref = len(f.ur)
    pts, fl = np.zeros((max(n_ref, 1), 3)), np.zeros(max(n_ref, 1), np.uint8)
    ntri, pc = C.c_int(), C.c_float()
    cams = _cams(p)
    nv = lib().ino_triangulate(cams.ctypes.data, Rt.ctypes.data, int(bool(depth_is_positive)), float(param(p, "reproj_err_thr")), n_ref,
                               f.ur.ctypes.data, f.br.ctypes.data, f.uc.ctypes.data, f.bc.ctypes.data, len(f.mt), f.mt.ctypes.data,
                               inl.ctypes.data, pts.ctypes.data, fl.ctypes.data, C.byref(ntri), C.byref(pc))
    return nv, ntri.value, np.float32(pc.value), pts[:n_ref], fl[:n_ref].astype(bool)


def reconstruct(p, model, M, inlier):
    """reconstruct_with_{H,F,E}: dict(status, stage, n_hypotheses, nums_valid, num_triangulated, parallax_cos, rot_ref_to_cur,
    trans_ref_to_cur (None when find_most_plausible_pose did not run), triangulated_pts, triangulated_flags (None unless succeeded))."""
    f = _Frame(p)
    code = {"H": MODEL_H, "F": MODEL_F, "E": MODEL_E}[model]
    M = _d(M, 9)
    inl = np.ascontiguousarray(np.asarray(inlier, np.uint8).reshape(-1))
    K1, K2 = _d(K_of(p["cam_ref"]), 9), _d(K_of(p["cam_cur"]), 9)
    cams = _cams(p)
    n_ref = len(f.ur)
    stage, nh = C.c_int(), C.c_int()
    nv, nt, pc = np.zeros(8, np.int32), np.zeros(8, np.int32), np.zeros(8, np.float32)
    R, t, pts, fl = np.zeros(9), np.zeros(3), np.zeros((max(n_ref, 1), 3)), np.zeros(max(n_ref, 1), np.uint8)
    st = lib().ino_reconstruct(code, M.ctypes.data, cams.ctypes.data, K1.ctypes.data, K2.ctypes.data, int(param(p, "min_num_triangulated")),
                               int(param(p, "min_num_valid_pts")), cos_thr(p), float(param(p, "reproj_err_thr")), n_ref, f.ur.ctypes.data,
                               f.br.ctypes.data, f.uc.ctypes.data, f.bc.ctypes.data, len(f.mt), f.mt.ctypes.data, inl.ctypes.data,
                               C.byref(stage), C.byref(nh), nv.ctypes.data, nt.ctypes.data, pc.ctypes.data, R.ctypes.data, t.ctypes.data,
                               pts.ctypes.data, fl.ctypes.data)
    k = nh.value
    ok = stage.value == STAGE_SUCCEEDED
    return dict(status=st, stage=stage.value, n_hypotheses=k, nums_valid=nv[:k], num_triangulated=nt[:k], parallax_cos=pc[:k],
                rot_ref_to_cur=R.reshape(3, 3) if k else None, trans_ref_to_cur=t if k else None,
                triangulated_pts=pts[:n_ref] if ok else None, triangulated_flags=fl[:n_ref].astype(bool) if ok else None)


def ransac(p):
    """The RANSAC stage of initialize(): the solvers' results, keyed "H" / "F" (perspective) or "E" (equirectangular); None for a solver
    that returned before drawing."""
    f = _Frame(p)
    iters = int(param(p, "num_ransac_iters"))
    if _MODEL_CODES[p["cam_ref"].get("model", "perspective")] == 1:
        ms = p.get("min_sets_E")
        return {"E": EO.essential_ransac(f.br[f.mt[:, 0]], f.bc[f.mt[:, 1]], np.zeros((0, 5)) if ms is None else np.asarray(ms)[:iters],
                                         recompute=False)}
    out = {}
    for k in ("H", "F"):
        ms = p.get("min_sets_" + k)
        size = 4 if k == "H" else 8
        out[k] = TO.twoview_ransac(k, f.ur, f.uc, f.mt, np.zeros((0, size)) if ms is None else ms, sigma=1.0, recompute=False)
    return out


def choose(r):
    """The model initialize() reconstructs with and its solver result, or (None, None)."""
    if "E" in r:
        return ("E", r["E"]) if r["E"]["valid"] else (None, None)
    if choose_H(r["H"]["best_cost"], r["F"]["best_cost"], r["H"]["valid"]):
        return "H", r["H"]
    if r["F"]["valid"]:
        return "F", r["F"]
    return None, None


def initialize(p):
    """initialize(): a result dict with the keys of initialize_batch."""
    r = ransac(p)
    n = len(matches_of(p["ref_matches_with_cur"]))
    out = dict(status=0, succeeded=False, model=None, stage=STAGE_NO_MODEL, n_matches=n, n_hypotheses=0, nums_valid=np.zeros(0, np.int32),
               num_triangulated=np.zeros(0, np.int32), parallax_cos=np.zeros(0, np.float32), rot_ref_to_cur=None, trans_ref_to_cur=None,
               triangulated_pts=None, triangulated_flags=None, inlier_flags=None)
    for k in ("H", "F", "E"):
        s = r.get(k)
        out["cost_" + k] = np.float32(s["best_cost"]) if s else np.float32(0.0)
        out["valid_" + k] = bool(s["valid"]) if s else False
        out["num_inliers_" + k] = s["num_inliers"] if s else 0
        out["status"] |= s["status"] if s else 0
    model, s = choose(r)
    if model is None:
        return out
    out["model"] = model
    out["inlier_flags"] = np.asarray(s["inlier_flags"], bool)
    rec = reconstruct(p, model, s["M_21"] if model != "E" else s["E_21"], s["inlier_flags"])
    out["status"] |= rec.pop("status")
    out.update(rec)
    out["succeeded"] = out["stage"] == STAGE_SUCCEEDED
    return out


# ---- synthetic problems ------------------------------------------------------------------------------------------------------------

def _bearings(pts, cam):
    """camera::perspective::convert_point_to_bearing of undistorted pixels (also fisheye / radial division)."""
    p = np.asarray(pts, np.float64).reshape(-1, 2)
    x, y = (p[:, 0] - cam["cx"]) / cam["fx"], (p[:, 1] - cam["cy"]) / cam["fy"]
    l2 = np.sqrt(x * x + y * y + 1.0)
    return np.stack([x / l2, y / l2, 1.0 / l2], 1)


def perspective_problem(seed=0, n=500, inlier_frac=0.7, scene="general", camera="euroc", model="perspective", noise=0.5, case=None,
                        draw_seed=None, **params):
    """A perspective-path problem from workloads.synth.make_twoview_problem: every keypoint of both frames, ref_matches_with_cur from the
    matches, bearings by the pinhole formula, the camera's image bounds.  model: "perspective", "fisheye" or "radial_division" (same
    intrinsics, finite coefficients).  Minimal sets drawn with b200_draw_min_sets from default engines (use_fixed_seed), or from
    engines seeded by draw_seed."""
    from workloads import synth
    pr = synth.make_twoview_problem(seed=seed, n=n, inlier_frac=inlier_frac, scene=scene, camera=camera, noise=noise, case=case)
    src = synth.EUROC_MONO if camera == "euroc" else synth.KITTI
    cam = dict(model=model, fx=src["fx"], fy=src["fy"], cx=src["cx"], cy=src["cy"])
    if model == "fisheye":
        cam.update(k1=0.01, k2=-0.002, k3=0.0, k4=0.0)
    elif model == "radial_division":
        cam.update(distortion=-1e-7)
    b = (0.0, float(pr["cols"]), 0.0, float(pr["rows"]))
    k1, k2, mt = pr["keypts_1"], pr["keypts_2"], pr["matches_12"]
    rm = np.full(len(k1), -1, np.int32)
    rm[mt[:, 0]] = mt[:, 1]
    p = dict(cam_ref=cam, cam_cur=cam, bounds_ref=b, bounds_cur=b, undist_ref=k1, bearings_ref=_bearings(k1, cam), undist_cur=k2,
             bearings_cur=_bearings(k2, cam), ref_matches_with_cur=rm, truth=dict(R=pr["R_21"], t=pr["t_21"], K=pr["K"], H=pr.get("H_21")))
    p.update(params)
    return with_min_sets(p, draw_seed)


def equirect_problem(seed=0, n=600, inlier_frac=0.7, cols=1920, rows=960, draw_seed=None, **params):
    """A bearing-vector problem: points 2-10 m around the first camera, a second pose 0.3 m away, bearings and equirectangular pixels of
    both views, outliers' current bearings replaced by random directions; extra unmatched keypoints in the ref frame."""
    rng = np.random.default_rng(seed)
    ang = 0.05 * rng.standard_normal(3)
    th = np.linalg.norm(ang)
    k = ang / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    R = np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx
    t = rng.standard_normal(3)
    t *= 0.3 / np.linalg.norm(t)
    d = rng.standard_normal((n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    X = d * rng.uniform(2.0, 10.0, (n, 1))
    Y = X @ R.T + t
    b1 = X / np.linalg.norm(X, axis=1, keepdims=True)
    b2 = Y / np.linalg.norm(Y, axis=1, keepdims=True)
    out = rng.uniform(size=n) > inlier_frac
    r = rng.standard_normal((int(out.sum()), 3))
    b2[out] = r / np.linalg.norm(r, axis=1, keepdims=True)

    def pix(b):
        lat, lon = -np.arcsin(b[:, 1]), np.arctan2(b[:, 0], b[:, 2])
        return np.stack([cols * (0.5 + lon / (2 * np.pi)), rows * (0.5 - lat / np.pi)], 1).astype(np.float32)

    extra = rng.standard_normal((n // 5, 3))
    extra /= np.linalg.norm(extra, axis=1, keepdims=True)
    b1 = np.concatenate([b1, extra])
    perm = rng.permutation(n)  # current keypoints in another order
    b2c = np.empty_like(b2)
    b2c[perm] = b2
    rm = np.full(len(b1), -1, np.int32)
    rm[:n] = perm
    cam = dict(model="equirectangular", cols=float(cols), rows=float(rows))
    p = dict(cam_ref=cam, cam_cur=cam, undist_ref=pix(b1), bearings_ref=b1, undist_cur=pix(b2c), bearings_cur=b2c, ref_matches_with_cur=rm,
             truth=dict(R=R, t=t))
    p.update(params)
    return with_min_sets(p, draw_seed)


def with_min_sets(p, draw_seed=None):
    """Adds the minimal sets initialize() would draw: each solver's engine default-constructed (use_fixed_seed), or seeded by
    draw_seed (the H, F / E engines by [draw_seed, 0], [draw_seed, 1])."""
    from stella_vslam_b200 import solve
    n = len(matches_of(p["ref_matches_with_cur"]))
    iters = int(param(p, "num_ransac_iters"))

    def eng(i):
        return solve.mt19937(None if draw_seed is None else [draw_seed, i])

    p = dict(p)
    if _MODEL_CODES[p["cam_ref"].get("model", "perspective")] == 1:
        p["min_sets_E"] = solve.draw_min_sets(n, iters, eng(0), set_size=5) if n >= 5 else None
    else:
        p["min_sets_H"] = solve.draw_min_sets(n, iters, eng(0), set_size=4) if n >= 8 else None
        p["min_sets_F"] = solve.draw_min_sets(n, iters, eng(1), set_size=8) if n >= 8 else None
    return p


def plane_problem(seed=0, n=800, inlier_frac=0.3, tilt=0.8, t_norm=0.5, fx=250.0, noise=0.0, draw_seed=None, **params):
    """A wide-angle (fx = fy = fx on 752 x 480) view of the plane n.X = 4 m, its normal tilted by `tilt` (standard deviation of the
    x and y components before normalising), and a second view rotated by a few hundredths of a radian and moved by t_norm metres
    mostly sideways (0: a pure rotation).  A fraction 1 - inlier_frac of the current keypoints is replaced by uniform pixels.  The
    sideways motion over a wide field of view puts part of the points behind a camera under the second Faugeras solution, so H
    reconstructions can succeed; t_norm = 0 makes K^-1 H K a rotation, whose equal singular values fail the rank test."""
    rng = np.random.default_rng(seed)
    cols, rows = 752, 480
    K = np.array([[fx, 0.0, 376.0], [0.0, fx, 240.0], [0.0, 0.0, 1.0]])
    Ki = np.linalg.inv(K)
    ang = 0.03 * rng.standard_normal(3)
    th = np.linalg.norm(ang)
    k = ang / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    R = np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx
    t = np.array([1.0, 0.2 * rng.standard_normal(), 0.2 * rng.standard_normal()])
    t *= t_norm / np.linalg.norm(t)
    nrm = np.array([tilt * rng.standard_normal(), tilt * rng.standard_normal(), 1.0])
    nrm /= np.linalg.norm(nrm)
    p1, p2 = [], []
    while len(p1) < n:
        u = np.array([rng.uniform(0, cols), rng.uniform(0, rows), 1.0])
        r = Ki @ u
        d = 4.0 / (nrm @ r)
        if d <= 0:
            continue
        Y = R @ (r * d) + t
        if Y[2] <= 0.1:
            continue
        q = K @ Y
        q = q[:2] / q[2]
        if not (0 < q[0] < cols and 0 < q[1] < rows):
            continue
        p1.append(u[:2])
        p2.append(q + noise * rng.standard_normal(2))
    p1, p2 = np.array(p1, np.float32), np.array(p2, np.float32)
    out = rng.uniform(size=n) > inlier_frac
    p2[out] = np.stack([rng.uniform(0, cols, out.sum()), rng.uniform(0, rows, out.sum())], 1).astype(np.float32)
    cam = dict(model="perspective", fx=fx, fy=fx, cx=376.0, cy=240.0)
    b = (0.0, float(cols), 0.0, float(rows))
    p = dict(cam_ref=cam, cam_cur=cam, bounds_ref=b, bounds_cur=b, undist_ref=p1, bearings_ref=_bearings(p1, cam), undist_cur=p2,
             bearings_cur=_bearings(p2, cam), ref_matches_with_cur=np.arange(n, dtype=np.int32), truth=dict(R=R, t=t, K=K))
    p.update(params)
    return with_min_sets(p, draw_seed)
