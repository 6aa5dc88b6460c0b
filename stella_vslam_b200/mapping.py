"""Host-side mirror of the mapping module's landmark creation: module::two_view_triangulator
(src/stella_vslam/module/two_view_triangulator.{h,cc}) and the numeric chain of mapping_module::create_new_landmarks
(match_for_triangulation per covisibility, then triangulation; src/stella_vslam/mapping_module.cc), the depth-seeded landmarks, and
the keyframe culling of module::local_map_cleaner::remove_redundant_keyframes on gathered tables.

Keyframes are dicts in the shape of workloads.synth.make_keyframe_pair, extended with the triangulator's fields:
    pose_cw, pose_wc (4x4), model (0 perspective family / 1 equirectangular), fx, fy, cx, cy, fx_inv, fy_inv, focal_x_baseline,
    true_baseline, cols, rows, img_bounds (perspective family), scale_factor, scale_factors, level_sigma_sq, x, y (undistorted keypoints), octave,
    x_right / depth (None = monocular), bearings (n x 3), desc (n x 32), no_landmark (u8), node (BoW node ids, optional).
"""
import ctypes as C

import numpy as np

from ._lib import check, lib
from .match import _matcher


class TriKeyframe(C.Structure):
    """b200_tri_keyframe_t (include/b200vslam.h)."""
    _fields_ = [("pose_cw", C.c_double * 16), ("pose_wc", C.c_double * 16), ("model", C.c_int32),
                ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double), ("fx_inv", C.c_double), ("fy_inv", C.c_double),
                ("focal_x_baseline", C.c_double), ("true_baseline", C.c_double), ("cols", C.c_double), ("rows", C.c_double),
                ("scale_factor", C.c_float), ("num_levels", C.c_int32), ("scale_factors", C.c_void_p), ("level_sigma_sq", C.c_void_p),
                ("n_keypoints", C.c_int32), ("x", C.c_void_p), ("y", C.c_void_p), ("octave", C.c_void_p), ("x_right", C.c_void_p),
                ("depth", C.c_void_p), ("bearings", C.c_void_p)]


class TriangulateProblem(C.Structure):
    """b200_triangulate_problem_t."""
    _fields_ = [("keyfrm_1", C.POINTER(TriKeyframe)), ("keyfrm_2", C.POINTER(TriKeyframe)), ("rays_parallax_deg_thr", C.c_float),
                ("n_matches", C.c_int32), ("matches", C.c_void_p), ("pos_w", C.c_void_p), ("ok", C.c_void_p), ("n_ok", C.c_int32)]


class NewLandmarksNeighbour(C.Structure):
    """b200_new_landmarks_neighbour_t."""
    _fields_ = [("keyfrm", C.POINTER(TriKeyframe)), ("desc", C.c_void_p), ("valid", C.c_void_p), ("node", C.c_void_p),
                ("E_12", C.c_double * 9), ("epiplane_in_keyfrm_2", C.c_double * 3), ("valid_epiplane", C.c_int32),
                ("match_out", C.c_void_p), ("n_matches", C.c_int32), ("n_created", C.c_int32)]


class NewLandmarksProblem(C.Structure):
    """b200_new_landmarks_problem_t."""
    _fields_ = [("keyfrm", C.POINTER(TriKeyframe)), ("desc", C.c_void_p), ("valid", C.c_void_p), ("node", C.c_void_p),
                ("n_neighbours", C.c_int32), ("neighbours", C.POINTER(NewLandmarksNeighbour)), ("created_rank", C.c_void_p),
                ("created_idx", C.c_void_p), ("created_pos_w", C.c_void_p), ("n_created", C.c_int32)]


RESIDUAL_RAD_THR = 0.2 * np.pi / 180.0  # match_for_triangulation's default residual


def _arr(keep, a, dt):
    if a is None:
        return None
    a = np.ascontiguousarray(a, dt)
    keep.append(a)
    return a.ctypes.data


def pack_keyframe(kf, keep, StructT=TriKeyframe):
    """dict -> TriKeyframe (arrays appended to `keep` stay alive with it)."""
    S = StructT()
    pose_cw = np.asarray(kf["pose_cw"], np.float64).reshape(16)
    pose_wc = np.asarray(kf["pose_wc"] if kf.get("pose_wc") is not None else np.linalg.inv(pose_cw.reshape(4, 4)), np.float64).reshape(16)
    for k in range(16):
        S.pose_cw[k], S.pose_wc[k] = float(pose_cw[k]), float(pose_wc[k])
    S.model = int(kf.get("model", 0))
    for f in ("fx", "fy", "cx", "cy", "focal_x_baseline", "true_baseline", "cols", "rows"):
        setattr(S, f, float(kf.get(f, 0.0)))
    S.fx_inv = float(kf.get("fx_inv", 1.0 / S.fx if S.fx else 0.0))
    S.fy_inv = float(kf.get("fy_inv", 1.0 / S.fy if S.fy else 0.0))
    sf = np.asarray(kf["scale_factors"], np.float32)
    S.scale_factor = float(kf.get("scale_factor", sf[1] if len(sf) > 1 else 1.0))
    S.num_levels = len(sf)
    S.scale_factors = _arr(keep, sf, np.float32)
    S.level_sigma_sq = _arr(keep, kf["level_sigma_sq"], np.float32)
    S.n_keypoints = len(kf["x"])
    S.x, S.y = _arr(keep, kf["x"], np.float32), _arr(keep, kf["y"], np.float32)
    S.octave = _arr(keep, kf["octave"], np.int32)
    S.x_right, S.depth = _arr(keep, kf.get("x_right"), np.float32), _arr(keep, kf.get("depth"), np.float32)
    S.bearings = _arr(keep, kf["bearings"], np.float64)
    keep.append(S)
    return S


def triangulate_pairs_batch(problems, device=0):
    """b200_triangulate_pairs.  problems: [(keyfrm_1, keyfrm_2, matches (n, 2), rays_parallax_deg_thr)].  Returns [(pos_w, ok)]."""
    if not problems:
        return []
    keep, views, arr = [], {}, (TriangulateProblem * len(problems))()
    outs = []
    for p, (k1, k2, matches, deg) in enumerate(problems):
        for kf in (k1, k2):
            if id(kf) not in views:
                views[id(kf)] = pack_keyframe(kf, keep)
        m = np.ascontiguousarray(np.asarray(matches, np.int32).reshape(-1, 2))
        pos, ok = np.zeros((len(m), 3)), np.zeros(len(m), np.uint8)
        keep += [m, pos, ok]
        outs.append((pos, ok))
        P = arr[p]
        P.keyfrm_1, P.keyfrm_2 = C.pointer(views[id(k1)]), C.pointer(views[id(k2)])
        P.rays_parallax_deg_thr = float(deg)
        P.n_matches, P.matches, P.pos_w, P.ok = len(m), m.ctypes.data, pos.ctypes.data, ok.ctypes.data
    _setup()
    check(lib().b200_triangulate_pairs(_matcher(device), len(problems), arr))
    return [(pos, ok.astype(bool)) for pos, ok in outs]


class two_view_triangulator:
    """module::two_view_triangulator(keyfrm_1, keyfrm_2, rays_parallax_deg_thr)."""

    def __init__(self, keyfrm_1, keyfrm_2, rays_parallax_deg_thr=1.0, device=0):
        self.keyfrm_1, self.keyfrm_2, self.rays_parallax_deg_thr, self.device = keyfrm_1, keyfrm_2, rays_parallax_deg_thr, device

    def triangulate(self, matches):
        """Every (idx_1, idx_2) of `matches`.  Returns (pos_w (n, 3), ok (n,) bool)."""
        return triangulate_pairs_batch([(self.keyfrm_1, self.keyfrm_2, matches, self.rays_parallax_deg_thr)], self.device)[0]


def epipolar_geometry(cur, ngh):
    """E_ngh_to_cur = essential_solver::create_E_21(ngh, cur) (mapping_module.cc) and the centre of `cur` as a bearing in `ngh`
    (robust.cc:22-27 with camera::*::reproject_to_bearing: a perspective-family camera reports it valid only in front of the camera
    AND inside ngh["img_bounds"] = (min_x, max_x, min_y, max_y), perspective.cc:150-169; equirectangular always)."""
    Pc, Pn = np.asarray(cur["pose_cw"], np.float64).reshape(4, 4), np.asarray(ngh["pose_cw"], np.float64).reshape(4, 4)
    rot_1w, trans_1w, rot_2w, trans_2w = Pn[:3, :3], Pn[:3, 3], Pc[:3, :3], Pc[:3, 3]
    rot_21 = rot_2w @ rot_1w.T
    t = -rot_21 @ trans_1w + trans_2w
    E = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]]) @ rot_21
    c_cur = -Pc[:3, :3].T @ Pc[:3, 3]
    e = Pn[:3, :3] @ c_cur + Pn[:3, 3]
    if int(ngh.get("model", 0)) == 1:
        valid = True
    elif e[2] <= 0.0:
        valid = False
    else:
        min_x, max_x, min_y, max_y = ngh["img_bounds"]
        z_inv = 1.0 / e[2]
        x, y = ngh["fx"] * e[0] * z_inv + ngh["cx"], ngh["fy"] * e[1] * z_inv + ngh["cy"]
        valid = min_x < x < max_x and min_y < y < max_y
    return E, e / np.linalg.norm(e), bool(valid)


def create_new_landmarks_batch(items, lowe_ratio=0.95, residual_rad_thr=RESIDUAL_RAD_THR, rays_parallax_deg_thr=1.0, bow=False,
                               max_candidates=0, return_matches=False, device=0):
    """b200_create_new_landmarks over several current keyframes.  items: [(cur_keyfrm, [neighbour keyframes in covisibility order])].
    Returns per item a dict: rank, idx (n, 2), pos_w (n, 3) of the created landmarks in creation order, n_matches / n_created per
    neighbour, and match_out per neighbour when return_matches."""
    keep, probs = [], (NewLandmarksProblem * max(len(items), 1))()
    results = []
    for k, (cur, nghs) in enumerate(items):
        P = probs[k]
        cs = pack_keyframe(cur, keep)
        n1 = cs.n_keypoints
        P.keyfrm = C.pointer(cs)
        P.desc = _arr(keep, cur["desc"], np.uint8)
        P.valid = _arr(keep, cur.get("no_landmark"), np.uint8)
        P.node = _arr(keep, cur["node"], np.int32) if bow else None
        nb = (NewLandmarksNeighbour * max(len(nghs), 1))()
        keep.append(nb)
        outs = dict(match_out=[])
        for r, ngh in enumerate(nghs):
            N = nb[r]
            N.keyfrm = C.pointer(pack_keyframe(ngh, keep))
            N.desc = _arr(keep, ngh["desc"], np.uint8)
            N.valid = _arr(keep, ngh.get("no_landmark"), np.uint8)
            N.node = _arr(keep, ngh["node"], np.int32) if bow else None
            E, epi, valid = epipolar_geometry(cur, ngh)
            for e in range(9):
                N.E_12[e] = float(E.reshape(9)[e])
            for e in range(3):
                N.epiplane_in_keyfrm_2[e] = float(epi[e])
            N.valid_epiplane = int(valid)
            if return_matches:
                mo = np.full(max(n1, 1), -2, np.int32)
                keep.append(mo)
                outs["match_out"].append(mo)
                N.match_out = mo.ctypes.data
        P.n_neighbours, P.neighbours = len(nghs), nb
        rank, idx, pos = np.zeros(max(n1, 1), np.int32), np.zeros((max(n1, 1), 2), np.int32), np.zeros((max(n1, 1), 3))
        keep += [rank, idx, pos]
        P.created_rank, P.created_idx, P.created_pos_w = rank.ctypes.data, idx.ctypes.data, pos.ctypes.data
        results.append((rank, idx, pos, nb, outs, n1, len(nghs)))
    _setup()
    check(lib().b200_create_new_landmarks(_matcher(device), len(items), probs, float(lowe_ratio), float(residual_rad_thr),
                                          float(rays_parallax_deg_thr), int(max_candidates)))
    out = []
    for k, (rank, idx, pos, nb, outs, n1, n_nb) in enumerate(results):
        n = probs[k].n_created
        d = dict(rank=rank[:n].copy(), idx=idx[:n].copy(), pos_w=pos[:n].copy(),
                 n_matches=np.array([nb[r].n_matches for r in range(n_nb)], np.int64),
                 n_created=np.array([nb[r].n_created for r in range(n_nb)], np.int64))
        if return_matches:
            d["match_out"] = [mo[:n1].copy() for mo in outs["match_out"]]
        out.append(d)
    return out


def create_new_landmarks(cur_keyfrm, neighbours, lowe_ratio=0.95, residual_deg_thr=0.2, bow=False, **kw):
    """mapping_module::create_new_landmarks after the baseline test, for one current keyframe and its ordered neighbours."""
    return create_new_landmarks_batch([(cur_keyfrm, neighbours)], lowe_ratio, residual_deg_thr * np.pi / 180.0, bow=bow, **kw)[0]


class DepthLandmarksProblem(C.Structure):
    """b200_depth_landmarks_problem_t."""
    _fields_ = [("mode", C.c_int32), ("model", C.c_int32), ("pose_wc", C.c_double * 16), ("fx_inv", C.c_double), ("fy_inv", C.c_double),
                ("cx", C.c_double), ("cy", C.c_double), ("depth_thr", C.c_double), ("n_keypoints", C.c_int32), ("x", C.c_void_p),
                ("y", C.c_void_p), ("octave", C.c_void_p), ("depth", C.c_void_p), ("has_landmark", C.c_void_p), ("num_levels", C.c_int32),
                ("scale_factors", C.c_void_p), ("inv_scale_factor_last", C.c_float), ("created_idx", C.c_void_p), ("pos_w", C.c_void_p),
                ("mean_normal", C.c_void_p), ("min_valid_dist", C.c_void_p), ("max_valid_dist", C.c_void_p), ("n_created", C.c_int32),
                ("status", C.c_int32)]


DEPTH_LANDMARKS_KEYFRAME, DEPTH_LANDMARKS_INITIAL = 0, 1
DEPTH_LANDMARKS_MAX_SORT = 8192  # B200_DEPTH_LM_MAX_SORT: keypoints with a valid depth one mode-0 problem may have


def depth_landmarks(problems, device=0, raise_on_error=True):
    """b200_depth_landmarks: the landmarks a stereo / RGB-D keyframe makes straight from its depths, for many frames in one call.
    Each problem is a dict: mode (0 = keyframe_inserter::create_new_keyframe, 1 = initializer::create_map_for_stereo), model (camera
    model code, default 0), pose_wc (4x4), fx_inv, fy_inv, cx, cy, depth_thr (mode 0), x, y, octave, depth (per undistorted keypoint),
    has_landmark (mode 0, optional), scale_factors, inv_scale_factor_last.  Returns per problem dict(idx, pos_w, mean_normal,
    min_valid_dist, max_valid_dist, status) with the landmarks in creation order.  raise_on_error=False returns the per-problem status
    (0, or the B200 error code of a rejected problem) instead of raising."""
    keep, arr = [], (DepthLandmarksProblem * max(len(problems), 1))()
    outs = []
    for k, pr in enumerate(problems):
        P = arr[k]
        n = len(pr["x"])
        P.mode, P.model = int(pr["mode"]), int(pr.get("model", 0))
        pose = np.asarray(pr["pose_wc"], np.float64).reshape(16)
        for e in range(16):
            P.pose_wc[e] = float(pose[e])
        P.fx_inv, P.fy_inv, P.cx, P.cy = (float(pr[f]) for f in ("fx_inv", "fy_inv", "cx", "cy"))
        P.depth_thr = float(pr.get("depth_thr", 0.0))
        P.n_keypoints = n
        P.x, P.y = _arr(keep, pr["x"], np.float32), _arr(keep, pr["y"], np.float32)
        P.octave, P.depth = _arr(keep, pr["octave"], np.int32), _arr(keep, pr["depth"], np.float32)
        P.has_landmark = _arr(keep, pr.get("has_landmark"), np.uint8)
        sf = np.asarray(pr["scale_factors"], np.float32)
        P.num_levels, P.scale_factors = len(sf), _arr(keep, sf, np.float32)
        P.inv_scale_factor_last = float(pr["inv_scale_factor_last"])
        m = max(n, 1)
        o = dict(idx=np.zeros(m, np.int32), pos_w=np.zeros((m, 3)), mean_normal=np.zeros((m, 3)), min_valid_dist=np.zeros(m, np.float32),
                 max_valid_dist=np.zeros(m, np.float32))
        keep.append(o)
        P.created_idx, P.pos_w, P.mean_normal = o["idx"].ctypes.data, o["pos_w"].ctypes.data, o["mean_normal"].ctypes.data
        P.min_valid_dist, P.max_valid_dist = o["min_valid_dist"].ctypes.data, o["max_valid_dist"].ctypes.data
        outs.append(o)
    _setup()
    rc = lib().b200_depth_landmarks(_matcher(device), len(problems), arr)
    if raise_on_error:
        check(rc)
    return [dict({f: v[:arr[k].n_created].copy() for f, v in o.items()}, status=int(arr[k].status)) for k, o in enumerate(outs)]


class CullKeyframe(C.Structure):
    """b200_cull_keyframe_t."""
    _fields_ = [("id", C.c_uint32), ("is_root", C.c_int32), ("n_keypoints", C.c_int32), ("kp_landmark", C.c_void_p), ("depth", C.c_void_p),
                ("depth_thr", C.c_double), ("n_valid", C.c_int32), ("n_redundant", C.c_int32), ("skipped", C.c_int32), ("removed", C.c_int32)]


class CullProblem(C.Structure):
    """b200_cull_problem_t."""
    _fields_ = [("cur_id", C.c_uint32), ("redundant_obs_ratio_thr", C.c_double), ("n_covisibilities", C.c_int32),
                ("covisibilities", C.POINTER(CullKeyframe)), ("n_landmarks", C.c_int32), ("obs_offsets", C.c_void_p), ("obs_rank", C.c_void_p),
                ("obs_octave", C.c_void_p), ("obs_weight", C.c_void_p), ("n_removed", C.c_int32), ("status", C.c_int32)]


CULL_SKIPPED_ROOT, CULL_SKIPPED_RECENT = 1, 2


def pack_cull_problems(problems):
    """Flat culling tables -> (CullProblem array, keep-alive list).  Each problem is a dict: cur_id, redundant_obs_ratio_thr,
    covisibilities (rank order; each a dict of id, is_root, kp_landmark, depth (None when the keyframe has no depths), depth_thr),
    obs_offsets, obs_rank, obs_octave, obs_weight (the landmark table in CSR form, b200_cull_problem_t)."""
    keep, arr = [], (CullProblem * max(len(problems), 1))()
    for k, pr in enumerate(problems):
        P = arr[k]
        P.cur_id = int(pr["cur_id"])
        P.redundant_obs_ratio_thr = float(pr["redundant_obs_ratio_thr"])
        covs = pr["covisibilities"]
        kfs = (CullKeyframe * max(len(covs), 1))()
        keep.append(kfs)
        for r, cv in enumerate(covs):
            K = kfs[r]
            K.id, K.is_root = int(cv["id"]), int(bool(cv.get("is_root", False)))
            K.n_keypoints = len(cv["kp_landmark"])
            K.kp_landmark = _arr(keep, cv["kp_landmark"], np.int32)
            K.depth = _arr(keep, cv.get("depth"), np.float32)
            K.depth_thr = float(cv.get("depth_thr", 0.0))
        P.n_covisibilities, P.covisibilities = len(covs), kfs
        off = np.asarray(pr["obs_offsets"], np.int32)
        P.n_landmarks = len(off) - 1
        P.obs_offsets = _arr(keep, off, np.int32)
        P.obs_rank, P.obs_octave = _arr(keep, pr["obs_rank"], np.int32), _arr(keep, pr["obs_octave"], np.int32)
        P.obs_weight = _arr(keep, pr["obs_weight"], np.uint8)
    return arr, keep


def cull_results(arr, problems):
    """Per problem dict(n_removed, status, skipped, n_valid, n_redundant, removed) (per-rank int arrays) read from a CullProblem array."""
    out = []
    for k, pr in enumerate(problems):
        P, n = arr[k], len(pr["covisibilities"])
        d = dict(n_removed=int(P.n_removed), status=int(P.status))
        for f in ("skipped", "n_valid", "n_redundant", "removed"):
            d[f] = np.array([getattr(P.covisibilities[r], f) for r in range(n)], np.int64)
        out.append(d)
    return out


def remove_redundant_keyframes(problems, device=0):
    """b200_remove_redundant_keyframes: local_map_cleaner::remove_redundant_keyframes' decisions for many maps in one launch, on flat
    tables as pack_cull_problems takes them (workloads.synth.gather_cull_problem builds them from an object-graph map).  The caller
    makes the reference's early return (redundant_obs_ratio_thr < 0 or no covisibility to search).  Returns cull_results."""
    arr, _keep = pack_cull_problems(problems)
    _setup()
    check(lib().b200_remove_redundant_keyframes(_matcher(device), len(problems), arr))
    return cull_results(arr, problems)


_argtypes_set = False


def _setup():
    global _argtypes_set
    if _argtypes_set:
        return
    L = lib()
    L.b200_triangulate_pairs.argtypes = [C.c_void_p, C.c_int, C.POINTER(TriangulateProblem)]
    L.b200_create_new_landmarks.argtypes = [C.c_void_p, C.c_int, C.POINTER(NewLandmarksProblem), C.c_float, C.c_float, C.c_float, C.c_int]
    L.b200_depth_landmarks.argtypes = [C.c_void_p, C.c_int, C.POINTER(DepthLandmarksProblem)]
    L.b200_remove_redundant_keyframes.argtypes = [C.c_void_p, C.c_int, C.POINTER(CullProblem)]
    _argtypes_set = True
