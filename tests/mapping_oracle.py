"""CPU restatement of the mapping module's landmark creation (test infrastructure): loads tests/mapping_oracle.c, compiled on first use
into a temporary directory (the tree is never written), and composes the chain of create_new_landmarks from oracle.pyoracle's
match_for_triangulation restatement and the triangulation, with the row claims between neighbour ranks."""
import ctypes as C

import numpy as np

import cbuild


class TriKeyframe(C.Structure):
    """orc_tri_keyframe_t (tests/mapping_oracle.c)."""
    _fields_ = [("pose_cw", C.c_double * 16), ("pose_wc", C.c_double * 16), ("model", C.c_int32),
                ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double), ("fx_inv", C.c_double), ("fy_inv", C.c_double),
                ("focal_x_baseline", C.c_double), ("true_baseline", C.c_double), ("cols", C.c_double), ("rows", C.c_double),
                ("scale_factor", C.c_float), ("num_levels", C.c_int32), ("scale_factors", C.c_void_p), ("level_sigma_sq", C.c_void_p),
                ("n_keypoints", C.c_int32), ("x", C.c_void_p), ("y", C.c_void_p), ("octave", C.c_void_p), ("x_right", C.c_void_p),
                ("depth", C.c_void_p), ("bearings", C.c_void_p)]


def pack_keyframe(kf, keep):
    S = TriKeyframe()

    def arr(a, dt):
        if a is None:
            return None
        a = np.ascontiguousarray(a, dt)
        keep.append(a)
        return a.ctypes.data

    S.pose_cw[:] = [float(v) for v in np.asarray(kf["pose_cw"], np.float64).reshape(16)]
    S.pose_wc[:] = [float(v) for v in np.asarray(kf["pose_wc"], np.float64).reshape(16)]
    S.model = int(kf["model"])
    for f in ("fx", "fy", "cx", "cy", "fx_inv", "fy_inv", "focal_x_baseline", "true_baseline", "cols", "rows"):
        setattr(S, f, float(kf[f]))
    S.scale_factor = float(kf["scale_factor"])
    S.num_levels = len(kf["scale_factors"])
    S.scale_factors, S.level_sigma_sq = arr(kf["scale_factors"], np.float32), arr(kf["level_sigma_sq"], np.float32)
    S.n_keypoints = len(kf["x"])
    S.x, S.y, S.octave = arr(kf["x"], np.float32), arr(kf["y"], np.float32), arr(kf["octave"], np.int32)
    S.x_right, S.depth, S.bearings = arr(kf.get("x_right"), np.float32), arr(kf.get("depth"), np.float32), arr(kf["bearings"], np.float64)
    keep.append(S)
    return S


def epipolar_geometry(cur, ngh):
    """E with bearing_cur . E bearing_ngh = 0, from the relative pose ngh -> cur (x_cur = R x_ngh + t, E = [t]x R), and the camera
    centre of `cur` seen from `ngh` as a unit bearing; valid as camera::*::reproject_to_bearing reports it (perspective family: in
    front of the camera and strictly inside the image bounds)."""
    Tc, Tn_wc = np.asarray(cur["pose_cw"], np.float64), np.asarray(ngh["pose_wc"], np.float64)
    T = Tc @ Tn_wc                                    # ngh camera -> cur camera
    R, t = T[:3, :3], T[:3, 3]
    E = np.array([[0.0, -t[2], t[1]], [t[2], 0.0, -t[0]], [-t[1], t[0], 0.0]]) @ R
    c = np.asarray(cur["pose_wc"], np.float64)[:3, 3]
    Pn = np.asarray(ngh["pose_cw"], np.float64)
    e = Pn[:3, :3] @ c + Pn[:3, 3]
    if int(ngh["model"]) == 1:
        valid = True
    else:
        b = ngh["img_bounds"]
        valid = e[2] > 0 and b[0] < ngh["fx"] * e[0] / e[2] + ngh["cx"] < b[1] and b[2] < ngh["fy"] * e[1] / e[2] + ngh["cy"] < b[3]
    return E, e / np.linalg.norm(e), bool(valid)


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = cbuild.load("mapping_oracle.c")
        P = C.POINTER(TriKeyframe)
        L.orc_triangulate_pairs.argtypes = [P, P, C.c_float, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_jacobi_svd4_null.argtypes = [C.c_void_p, C.c_void_p]
        L.orc_triangulator_constants.argtypes = [P, P, C.c_float, C.POINTER(C.c_float), C.POINTER(C.c_float)]
        _lib = L
    return _lib


def jacobi_svd4_null(A):
    """Null vector of a 4x4 by the Jacobi sweeps.  Returns (v, sweeps)."""
    A = np.ascontiguousarray(A, np.float64).reshape(16)
    v = np.zeros(4)
    n = lib().orc_jacobi_svd4_null(A.ctypes.data, v.ctypes.data)
    return v, n


def constants(k1, k2, deg=1.0):
    keep = []
    a, b = pack_keyframe(k1, keep), pack_keyframe(k2, keep)
    c, r = C.c_float(), C.c_float()
    lib().orc_triangulator_constants(C.byref(a), C.byref(b), deg, C.byref(c), C.byref(r))
    return np.float32(c.value), np.float32(r.value)


def triangulate_pairs(k1, k2, matches, rays_parallax_deg_thr=1.0):
    """two_view_triangulator(k1, k2, deg).triangulate over `matches` (n, 2).  Returns (pos_w (n, 3), ok (n,) bool); raises ValueError on
    the inputs the device entry point rejects with B200_ERR_INVALID."""
    keep = []
    a, b = pack_keyframe(k1, keep), pack_keyframe(k2, keep)
    m = np.ascontiguousarray(np.asarray(matches, np.int32).reshape(-1, 2))
    pos, ok = np.zeros((max(len(m), 1), 3)), np.zeros(max(len(m), 1), np.uint8)
    rc = lib().orc_triangulate_pairs(C.byref(a), C.byref(b), rays_parallax_deg_thr, len(m), m.ctypes.data, pos.ctypes.data, ok.ctypes.data)
    if rc == -1:
        raise ValueError("index / octave out of range or stereo keypoint on an equirectangular camera")
    if rc == -2:
        raise RuntimeError("Jacobi SVD did not converge")
    return pos[:len(m)], ok[:len(m)].astype(bool)


def triangulation_problem(cur, ngh, residual_rad_thr, bow, valid1):
    """The match_for_triangulation problem dict (oracle.pyoracle / b200_match_pairs layout) of (cur, ngh)."""
    E, epi, valid = epipolar_geometry(cur, ngh)
    sf = np.asarray(cur["scale_factors"], np.float32)

    def stereo(kf):
        return None if kf.get("x_right") is None else (np.asarray(kf["x_right"], np.float32) >= 0).astype(np.uint8)

    pr = dict(desc1=cur["desc"], valid1=valid1, bearing1=cur["bearings"], scale1=sf[np.asarray(cur["octave"], np.int64)], stereo1=stereo(cur),
              desc2=ngh["desc"], valid2=ngh.get("no_landmark"), bearing2=ngh["bearings"], stereo2=stereo(ngh), E_12=E,
              epiplane_in_keyfrm_2=epi, valid_epiplane=valid, residual_rad_thr=residual_rad_thr)
    if bow:
        pr.update(node1=cur["node"], node2=ngh["node"])
    return pr


def create_new_landmarks(cur, neighbours, lowe_ratio=0.95, residual_rad_thr=0.2 * np.pi / 180.0, rays_parallax_deg_thr=1.0, bow=False):
    """mapping_module::create_new_landmarks after the baseline test: per neighbour in order, match_for_triangulation on the rows that
    still carry no landmark, triangulate every match, and attach each created landmark to its row."""
    from oracle import pyoracle as O
    n1 = len(cur["x"])
    free = np.ones(n1, np.uint8) if cur.get("no_landmark") is None else np.asarray(cur["no_landmark"], np.uint8).copy()
    out = dict(rank=[], idx=[], pos_w=[], n_matches=[], n_created=[], match_out=[])
    for r, ngh in enumerate(neighbours):
        pr = triangulation_problem(cur, ngh, residual_rad_thr, bow, free.copy())
        if n1 == 0 or len(ngh["x"]) == 0:
            mo, n = np.full(n1, -1, np.int32), 0
        else:
            mo, n = O.match_pairs(pr, 1, lowe_ratio, False)
        out["match_out"].append(mo)
        out["n_matches"].append(n)
        idx_1 = np.flatnonzero(mo >= 0)
        pairs = np.stack([idx_1, mo[idx_1]], 1).astype(np.int32)
        pos, ok = triangulate_pairs(cur, ngh, pairs, rays_parallax_deg_thr) if len(pairs) else (np.zeros((0, 3)), np.zeros(0, bool))
        for k in np.flatnonzero(ok):
            out["rank"].append(r)
            out["idx"].append(pairs[k])
            out["pos_w"].append(pos[k])
            free[pairs[k][0]] = 0
        out["n_created"].append(int(ok.sum()))
    return dict(rank=np.array(out["rank"], np.int32), idx=np.array(out["idx"], np.int32).reshape(-1, 2),
                pos_w=np.array(out["pos_w"]).reshape(-1, 3), n_matches=np.array(out["n_matches"], np.int64),
                n_created=np.array(out["n_created"], np.int64), match_out=out["match_out"])
