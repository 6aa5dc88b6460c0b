"""ctypes loader for the CPU oracle (oracle/liboracle.so).  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this module.
The product package (stella_vslam_b200) never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle.so")


def build(force=False):
    """Compile the oracle with the committed Makefile (gcc only)."""
    if force or not os.path.exists(_LIB_PATH) or any(
            os.path.getmtime(os.path.join(_HERE, f)) > os.path.getmtime(_LIB_PATH)
            for f in os.listdir(_HERE) if f.endswith((".c", ".h"))):
        subprocess.check_call(["make", "-C", _HERE, "-s"] + (["-B"] if force else []))
    return _LIB_PATH


def build_ref():
    """Type-check the reference-side adapters against the reference's headers (`make ref`: records under oracle/_ref/, refreshed when
    an adapter, stub or the ABI header changes; a no-op where no stella_vslam checkout is available)."""
    subprocess.check_call(["make", "-C", _HERE, "-s", "-j8", "ref"])
    return os.path.join(_HERE, "_ref")


class Keypoint(C.Structure):
    _fields_ = [("x", C.c_float), ("y", C.c_float), ("size", C.c_float), ("angle", C.c_float),
                ("response", C.c_float), ("octave", C.c_int32)]


KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                     ("octave", "<i4")])


class OrbConfig(C.Structure):
    _fields_ = [("scale_factor", C.c_float), ("num_levels", C.c_int32), ("ini_fast_thr", C.c_int32),
                ("min_fast_thr", C.c_int32), ("min_area", C.c_uint32)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        u8p, f32p, i32p = C.POINTER(C.c_uint8), C.POINTER(C.c_float), C.POINTER(C.c_int32)
        L.orc_scale_factors.argtypes = [C.c_float, C.c_int, f32p, f32p, f32p, f32p]
        L.orc_level_size.argtypes = [C.c_int, C.c_int, C.c_float, i32p, i32p]
        L.orc_resize_linear_u8.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.orc_fast9_16_nms.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.orc_fast9_16_nms.restype = C.c_int
        L.orc_gaussian7_s2_u8.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int]
        L.orc_fast_atan2.argtypes = [C.c_float, C.c_float]
        L.orc_fast_atan2.restype = C.c_float
        L.orc_ic_angle.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.orc_ic_angle.restype = C.c_float
        L.orc_util_cos.argtypes = [C.c_float]
        L.orc_util_cos.restype = C.c_float
        L.orc_util_sin.argtypes = [C.c_float]
        L.orc_util_sin.restype = C.c_float
        L.orc_rbrief.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_float, C.c_float, C.c_void_p]
        L.orc_rect_mask.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
        L.orc_orb_extract.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.POINTER(OrbConfig),
                                      C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_orb_extract.restype = C.c_int
        L.orc_hamming_32.argtypes = [C.c_void_p, C.c_void_p]
        L.orc_hamming_32.restype = C.c_uint
        L.orc_hamming_64.argtypes = [C.c_void_p, C.c_void_p]
        L.orc_hamming_64.restype = C.c_uint
        L.orc_angle_diff.argtypes = [C.c_float, C.c_float]
        L.orc_angle_diff.restype = C.c_float
        L.orc_brute_force_match.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                            C.c_float, C.c_int, C.c_void_p]
        L.orc_brute_force_match.restype = C.c_int
        L.orc_frontend_batch.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(OrbConfig), C.c_int, C.c_float, C.c_int,
                                         C.c_int, C.c_void_p, C.c_void_p]
        L.orc_frontend_batch.restype = C.c_int
        if hasattr(L, "orc_lba_solve"):
            L.orc_lba_solve.restype = C.c_int
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def scale_factors(scale_factor=1.2, n=8):
    out = [np.zeros(n, np.float32) for _ in range(4)]
    lib().orc_scale_factors(scale_factor, n, *[o.ctypes.data_as(C.POINTER(C.c_float)) for o in out])
    return out  # sf, inv_sf, sigma_sq, inv_sigma_sq


def level_sizes(w, h, scale_factor=1.2, n=8):
    sf = scale_factors(scale_factor, n)[0]
    sizes = [(w, h)]
    for l in range(1, n):
        lw, lh = C.c_int32(), C.c_int32()
        lib().orc_level_size(w, h, float(sf[l]), C.byref(lw), C.byref(lh))
        sizes.append((lw.value, lh.value))
    return sizes


def resize_linear(src, dw, dh):
    src = np.ascontiguousarray(src, np.uint8)
    dst = np.empty((dh, dw), np.uint8)
    lib().orc_resize_linear_u8(_p(src), src.shape[1], src.shape[0], src.strides[0], _p(dst), dw, dh, dw)
    return dst


def fast9_16_nms(img, thr):
    """cv::FAST(img, thr, nonmax=True) on a (possibly non-contiguous) 2-D u8 view."""
    assert img.dtype == np.uint8 and img.strides[1] == 1
    h, w = img.shape
    cap = w * h
    xs, ys, sc = np.empty(cap, np.int16), np.empty(cap, np.int16), np.empty(cap, np.uint8)
    n = lib().orc_fast9_16_nms(img.ctypes.data, img.strides[0], w, h, thr, _p(xs), _p(ys), _p(sc), cap)
    return xs[:n].copy(), ys[:n].copy(), sc[:n].copy()


def gaussian7(src):
    src = np.ascontiguousarray(src, np.uint8)
    dst = np.empty_like(src)
    lib().orc_gaussian7_s2_u8(_p(src), src.shape[1], src.shape[0], src.strides[0], _p(dst), dst.strides[0])
    return dst


def fast_atan2(y, x):
    return lib().orc_fast_atan2(float(y), float(x))


def ic_angle(img, x, y):
    img = np.ascontiguousarray(img, np.uint8)
    return lib().orc_ic_angle(_p(img), img.strides[0], int(x), int(y))


def rbrief(blurred, x, y, angle_deg):
    blurred = np.ascontiguousarray(blurred, np.uint8)
    d = np.zeros(32, np.uint8)
    lib().orc_rbrief(_p(blurred), blurred.strides[0], float(x), float(y), float(angle_deg), _p(d))
    return d


def rect_mask(cols, rows, rects):
    r = np.ascontiguousarray(np.asarray(rects, np.float32).reshape(-1, 4))
    m = np.empty((rows, cols), np.uint8)
    lib().orc_rect_mask(cols, rows, _p(r), r.shape[0], _p(m), cols)
    return m


def orb_extract(img, mask=None, scale_factor=1.2, num_levels=8, ini_fast_thr=20, min_fast_thr=7, min_area=800,
                want_pyramid=False, cap=None):
    """feature::orb_extractor::extract.  Returns dict(kps=structured array, desc=(N,32) u8, level_counts, raw_counts[, pyramid])."""
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape
    cfg = OrbConfig(scale_factor, num_levels, ini_fast_thr, min_fast_thr, min_area)
    if cap is None:
        cap = max(1024, (w * h) // 64)
    kps = np.zeros(cap, KP_DTYPE)
    desc = np.zeros((cap, 32), np.uint8)
    lc, rc = np.zeros(num_levels, np.int32), np.zeros(num_levels, np.int32)
    pyr, pyr_ptrs = None, None
    if want_pyramid:
        pyr = [np.empty((lh, lw), np.uint8) for (lw, lh) in level_sizes(w, h, scale_factor, num_levels)]
        pyr_ptrs = (C.c_void_p * num_levels)(*[p.ctypes.data for p in pyr])
    if mask is not None:
        mask = np.ascontiguousarray(mask, np.uint8)
    n = lib().orc_orb_extract(_p(img), w, h, img.strides[0], _p(mask), mask.strides[0] if mask is not None else 0,
                              C.byref(cfg), _p(kps), _p(desc), cap, _p(lc), _p(rc), pyr_ptrs)
    if n < 0:
        raise RuntimeError("oracle keypoint capacity too small")
    out = dict(kps=kps[:n].copy(), desc=desc[:n].copy(), level_counts=lc, raw_counts=rc)
    if want_pyramid:
        out["pyramid"] = pyr
    return out


def hamming_32(a, b):
    a, b = np.ascontiguousarray(a, np.uint8), np.ascontiguousarray(b, np.uint8)
    return lib().orc_hamming_32(_p(a), _p(b))


def hamming_64(a, b):
    a, b = np.ascontiguousarray(a, np.uint8), np.ascontiguousarray(b, np.uint8)
    return lib().orc_hamming_64(_p(a), _p(b))


def brute_force_match(desc1, angle1, desc2, angle2, valid2=None, lowe_ratio=0.8, check_orientation=True):
    desc1, desc2 = np.ascontiguousarray(desc1, np.uint8), np.ascontiguousarray(desc2, np.uint8)
    angle1, angle2 = np.ascontiguousarray(angle1, np.float32), np.ascontiguousarray(angle2, np.float32)
    n1, n2 = desc1.shape[0], desc2.shape[0]
    if valid2 is not None:
        valid2 = np.ascontiguousarray(valid2, np.uint8)
    pairs = np.zeros((max(n1, 1), 2), np.int32)
    n = lib().orc_brute_force_match(_p(desc1), _p(angle1), n1, _p(desc2), _p(angle2), _p(valid2), n2, lowe_ratio,
                                    int(check_orientation), _p(pairs))
    return pairs[:n].copy()


def frontend_batch(frames, n, min_area=800, lowe_ratio=0.8, check_orientation=True, threads=1, cap=4096):
    """Timed CPU baseline: extract n frames (cycling through `frames`) on `threads` pthreads, match each to its predecessor."""
    frames = np.ascontiguousarray(frames, np.uint8)
    nu, h, w = frames.shape
    cfg = OrbConfig(1.2, 8, 20, 7, min_area)
    counts, matches = np.zeros(n, np.int32), np.zeros(n, np.int32)
    lib().orc_frontend_batch(_p(frames), nu, n, w, h, C.byref(cfg), cap, lowe_ratio, int(check_orientation), threads, _p(counts), _p(matches))
    if (counts < 0).any():
        raise RuntimeError("oracle keypoint capacity too small")
    return counts, matches


# ---- grid-guided projection matchers --------------------------------------------------------------------------------------
class GuidedProblem(C.Structure):
    """orc_guided_t (oracle.h)."""
    _fields_ = [("n_train", C.c_int32), ("t_x", C.c_void_p), ("t_y", C.c_void_p), ("t_octave", C.c_void_p), ("t_angle", C.c_void_p),
                ("t_x_right", C.c_void_p), ("t_desc", C.c_void_p), ("t_occupied", C.c_void_p),
                ("min_x", C.c_float), ("max_x", C.c_float), ("min_y", C.c_float), ("max_y", C.c_float),
                ("grid_cols", C.c_int32), ("grid_rows", C.c_int32), ("n_queries", C.c_int32),
                ("q_desc", C.c_void_p), ("q_x", C.c_void_p), ("q_y", C.c_void_p), ("q_margin", C.c_void_p), ("q_min_level", C.c_void_p),
                ("q_max_level", C.c_void_p), ("q_x_right", C.c_void_p), ("q_angle", C.c_void_p), ("q_valid", C.c_void_p),
                ("q_has_observation", C.c_void_p), ("q_reproj", C.c_void_p), ("inv_level_sigma_sq", C.c_void_p),
                ("do_reprojection_matching", C.c_int32)]


_GUIDED_FIELDS = (("t_x", "f4"), ("t_y", "f4"), ("t_octave", "u1"), ("t_angle", "f4"), ("t_x_right", "f4"), ("t_desc", "u1"),
                  ("t_occupied", "u1"), ("q_desc", "u1"), ("q_x", "f4"), ("q_y", "f4"), ("q_margin", "f4"), ("q_min_level", "i1"),
                  ("q_max_level", "i1"), ("q_x_right", "f4"), ("q_angle", "f4"), ("q_valid", "u1"), ("q_has_observation", "u1"), ("q_reproj", "f8"),
                  ("inv_level_sigma_sq", "f4"))


def match_guided(prob, mode, thr=100, lowe_ratio=0.8, check_orientation=True):
    """orc_match_guided on a problem dict (keys: _GUIDED_FIELDS, bounds, grid).  Returns (match_out, occupied_after, n)."""
    S, keep = GuidedProblem(), {}
    for name, dt in _GUIDED_FIELDS:
        v = prob.get(name)
        if v is None and name == "t_occupied":
            v = np.zeros(len(prob["t_x"]), np.uint8)
        if v is None:
            setattr(S, name, None)
            continue
        a = np.ascontiguousarray(v, np.dtype(dt))
        if name == "t_occupied":
            a = a.copy()
        keep[name] = a
        setattr(S, name, a.ctypes.data)
    S.n_train, S.n_queries = len(keep["t_x"]), len(keep["q_x"])
    S.min_x, S.max_x, S.min_y, S.max_y = [float(v) for v in prob["bounds"]]
    S.grid_cols, S.grid_rows = prob.get("grid", (64, 48))
    S.do_reprojection_matching = int(bool(prob.get("do_reprojection_matching", False)))
    out = np.full(max(S.n_queries, 1), -2, np.int32)
    L = lib()
    L.orc_match_guided.argtypes = [C.POINTER(GuidedProblem), C.c_int, C.c_uint, C.c_float, C.c_int, C.c_void_p]
    n = L.orc_match_guided(C.byref(S), mode, thr, lowe_ratio, int(check_orientation), out.ctypes.data)
    return out[:S.n_queries].copy(), keep["t_occupied"], n


def cross_check(idx2_in_1, idx1_in_2):
    a, b = np.ascontiguousarray(idx2_in_1, np.int32), np.ascontiguousarray(idx1_in_2, np.int32)
    out = np.full(max(len(a), 1), -2, np.int32)
    n = lib().orc_cross_check(_p(a), len(a), _p(b), len(b), _p(out))
    return out[:len(a)].copy(), n


# ---- all-pairs matchers with greedy state (bow_tree / match_for_triangulation) ------------------------------------------
class PairsProblem(C.Structure):
    """orc_pairs_t (oracle.h)."""
    _fields_ = [("n1", C.c_int32), ("desc1", C.c_void_p), ("angle1", C.c_void_p), ("valid1", C.c_void_p), ("node1", C.c_void_p),
                ("bearing1", C.c_void_p), ("scale1", C.c_void_p), ("stereo1", C.c_void_p),
                ("n2", C.c_int32), ("desc2", C.c_void_p), ("angle2", C.c_void_p), ("valid2", C.c_void_p), ("node2", C.c_void_p),
                ("bearing2", C.c_void_p), ("stereo2", C.c_void_p),
                ("E_12", C.c_double * 9), ("epiplane_in_2", C.c_double * 3), ("valid_epiplane", C.c_int32), ("residual_rad_thr", C.c_float)]


_PAIRS_FIELDS = (("desc1", "u1"), ("angle1", "f4"), ("valid1", "u1"), ("node1", "i4"), ("bearing1", "f8"), ("scale1", "f4"), ("stereo1", "u1"),
                 ("desc2", "u1"), ("angle2", "f4"), ("valid2", "u1"), ("node2", "i4"), ("bearing2", "f8"), ("stereo2", "u1"))


def match_pairs(prob, variant, lowe_ratio=0.6, check_orientation=True):
    """orc_match_pairs on a problem dict.  Returns (match_out per row, n)."""
    S, keep = PairsProblem(), {}
    for name, dt in _PAIRS_FIELDS:
        v = prob.get(name)
        if v is None:
            setattr(S, name, None)
            continue
        keep[name] = np.ascontiguousarray(v, np.dtype(dt))
        setattr(S, name, keep[name].ctypes.data)
    S.n1, S.n2 = len(keep["desc1"].reshape(-1, 32)), len(keep["desc2"].reshape(-1, 32))
    E = np.asarray(prob.get("E_12", np.zeros((3, 3))), np.float64).reshape(9)
    epi = np.asarray(prob.get("epiplane_in_keyfrm_2", np.zeros(3)), np.float64).reshape(3)
    for k in range(9):
        S.E_12[k] = float(E[k])
    for k in range(3):
        S.epiplane_in_2[k] = float(epi[k])
    S.valid_epiplane = int(bool(prob.get("valid_epiplane", False)))
    S.residual_rad_thr = float(prob.get("residual_rad_thr", 0.0))
    out = np.full(max(S.n1, 1), -2, np.int32)
    L = lib()
    L.orc_match_pairs.argtypes = [C.POINTER(PairsProblem), C.c_int, C.c_float, C.c_int, C.c_void_p]
    n = L.orc_match_pairs(C.byref(S), variant, lowe_ratio, int(check_orientation), out.ctypes.data)
    return out[:S.n1].copy(), n


# ---- match::stereo ------------------------------------------------------------------------------------------------------------
def stereo_compute(pyr_left, pyr_right, kps_left, desc_left, kps_right, desc_right, focal_x_baseline, true_baseline, scale_factor=1.2):
    """stereo::compute (stereo.cc:20-114).  pyr_*: lists of tight u8 level images; kps_*: KP_DTYPE arrays.  Returns (x_right, depths)."""
    n_levels = len(pyr_left)
    pl = [np.ascontiguousarray(a, np.uint8) for a in pyr_left]
    prr = [np.ascontiguousarray(a, np.uint8) for a in pyr_right]
    widths = np.array([a.shape[1] for a in pl], np.int32)
    heights = np.array([a.shape[0] for a in pl], np.int32)
    lp = (C.c_void_p * n_levels)(*[a.ctypes.data for a in pl])
    rp = (C.c_void_p * n_levels)(*[a.ctypes.data for a in prr])
    sf, inv = scale_factors(scale_factor, n_levels)[:2]
    kl, kr = np.ascontiguousarray(kps_left, KP_DTYPE), np.ascontiguousarray(kps_right, KP_DTYPE)
    dl, dr = np.ascontiguousarray(desc_left, np.uint8), np.ascontiguousarray(desc_right, np.uint8)
    xr, dep = np.zeros(max(len(kl), 1), np.float32), np.zeros(max(len(kl), 1), np.float32)
    L = lib()
    L.orc_stereo_compute.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                     C.c_int, C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_void_p, C.c_void_p]
    sf, inv = np.ascontiguousarray(sf, np.float32), np.ascontiguousarray(inv, np.float32)
    n = L.orc_stereo_compute(lp, rp, _p(widths), _p(heights), _p(kl), _p(dl), len(kl), _p(kr), _p(dr), len(kr), _p(sf), _p(inv),
                             focal_x_baseline, true_baseline, _p(xr), _p(dep))
    return xr[:len(kl)].copy(), dep[:len(kl)].copy(), n


# ---- local BA ---------------------------------------------------------------------------------------------------------
class Camera(C.Structure):
    _fields_ = [("model", C.c_int32), ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
                ("fxb", C.c_double), ("cols", C.c_double), ("rows", C.c_double)]


class LbaProblem(C.Structure):
    _fields_ = [("n_poses", C.c_int32), ("n_points", C.c_int32), ("n_edges", C.c_int32), ("n_cams", C.c_int32),
                ("pose_cw", C.c_void_p), ("pose_fixed", C.c_void_p), ("points", C.c_void_p), ("point_fixed", C.c_void_p),
                ("e_pose", C.c_void_p), ("e_point", C.c_void_p), ("e_cam", C.c_void_p), ("e_obs", C.c_void_p),
                ("e_inv_sigma_sq", C.c_void_p), ("e_delta", C.c_void_p), ("e_robust", C.c_void_p), ("e_can_be_outlier", C.c_void_p),
                ("cams", C.c_void_p)]


class LbaStats(C.Structure):
    _fields_ = [("iterations", C.c_int32 * 2), ("n_outliers", C.c_int32), ("chi2", C.c_double * 2), ("lambda_init", C.c_double),
                ("lambda_final", C.c_double * 2)]


def pack_lba_problem(prob, ProblemT=LbaProblem, CameraT=Camera):
    """dict from synth.make_ba_problem -> (ctypes struct, keep-alive list)."""
    keep = []

    def arr(x, dt):
        if x is None:
            return None
        a = np.ascontiguousarray(x, dt)
        keep.append(a)
        return a.ctypes.data

    cams = (CameraT * len(prob["cams"]))(*[CameraT(c["model"], c["fx"], c["fy"], c["cx"], c["cy"], c["fxb"], c["cols"], c["rows"])
                                            for c in prob["cams"]])
    keep.append(cams)
    K, L, E = len(prob["pose_cw"]), len(prob["points"]), len(prob["e_pose"])
    P = ProblemT(K, L, E, len(prob["cams"]), arr(prob["pose_cw"], np.float64), arr(prob["pose_fixed"], np.uint8),
                 arr(prob["points"], np.float64), arr(prob.get("point_fixed"), np.uint8), arr(prob["e_pose"], np.int32),
                 arr(prob["e_point"], np.int32), arr(prob["e_cam"], np.uint8), arr(prob["e_obs"], np.float32),
                 arr(prob["e_inv_sigma_sq"], np.float32), arr(prob["e_delta"], np.float32), arr(prob.get("e_robust"), np.uint8),
                 arr(prob.get("e_can_be_outlier"), np.uint8), C.cast(cams, C.c_void_p))
    return P, keep


def lba_solve(prob, iters1=5, iters2=10, force_stop=None):
    """local_bundle_adjuster_g2o::optimize steps 5-8 on the CPU oracle.  force_stop: optional 1-element uint8 array."""
    L_ = lib()
    L_.orc_lba_solve.argtypes = [C.POINTER(LbaProblem), C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(LbaStats)]
    P, keep = pack_lba_problem(prob)
    K, L, E = P.n_poses, P.n_points, P.n_edges
    pose_out, pts_out, outl = np.zeros((K, 4, 4)), np.zeros((L, 3)), np.zeros(E, np.uint8)
    st = LbaStats()
    rc = L_.orc_lba_solve(C.byref(P), iters1, iters2, _p(force_stop), _p(pose_out), _p(pts_out), _p(outl), C.byref(st))
    return dict(rc=rc, pose_cw=pose_out, points=pts_out, outliers=outl, iterations=list(st.iterations), n_outliers=st.n_outliers,
                chi2=list(st.chi2), lambda_init=st.lambda_init, lambda_final=list(st.lambda_final))


def global_ba_solve(prob, num_iter=10, gain_threshold=1e-3, force_stop=None):
    """global_bundle_adjuster::optimize / optimize_for_initialization on the CPU oracle (one LM round, no outlier pass)."""
    L_ = lib()
    L_.orc_global_ba_solve.argtypes = [C.POINTER(LbaProblem), C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(LbaStats)]
    P, keep = pack_lba_problem(prob)
    pose_out, pts_out = np.zeros((P.n_poses, 4, 4)), np.zeros((P.n_points, 3))
    st = LbaStats()
    rc = L_.orc_global_ba_solve(C.byref(P), int(num_iter), float(gain_threshold), _p(force_stop), _p(pose_out), _p(pts_out), C.byref(st))
    return dict(rc=rc, pose_cw=pose_out, points=pts_out, iterations=st.iterations[0], chi2=st.chi2[0], lambda_init=st.lambda_init,
                lambda_final=st.lambda_final[0])


def lba_linearize(prob, pose_cw=None, points=None, level=None, robust=None):
    """orc_lba_linearize: per edge the residual (E,3), robust weight (E,), landmark Jacobian (E,3,3) and pose Jacobian (E,3,6) that
    the oracle's build_system uses at the state (pose_cw, points) -- default: the problem's -- with the edges of level != 0 left out
    (all zero).  robust: per-edge Huber switch (default: the problem's e_robust).  Test infrastructure only."""
    L_ = lib()
    L_.orc_lba_linearize.argtypes = [C.POINTER(LbaProblem)] + [C.c_void_p] * 8
    L_.orc_lba_linearize.restype = C.c_int
    P, keep = pack_lba_problem(prob)
    E = P.n_edges
    args = [None if a is None else np.ascontiguousarray(a, dt) for a, dt in
            ((pose_cw, np.float64), (points, np.float64), (level, np.uint8), (robust, np.uint8))]
    err, w, Ji, Jj = np.zeros((E, 3)), np.zeros(E), np.zeros((E, 3, 3)), np.zeros((E, 3, 6))
    n = L_.orc_lba_linearize(C.byref(P), *[_p(a) for a in args], _p(err), _p(w), _p(Ji), _p(Jj))
    return dict(n_active=n, err=err, weight=w, Ji=Ji, Jj=Jj)


def pose_optimize(prob, num_trials_robust=2, num_trials=2, num_each_iter=10):
    """orc_pose_optimize on a flattened frame (synth.make_pose_problem).  Returns (num_valid_obs, pose (4,4), outlier_flags bool)."""
    P, keep = pack_lba_problem(prob)
    pose = np.zeros((4, 4))
    flags = np.zeros(max(P.n_edges, 1), np.uint8)
    L = lib()
    L.orc_pose_optimize.argtypes = [C.POINTER(LbaProblem), C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    L.orc_pose_optimize.restype = C.c_uint
    n = L.orc_pose_optimize(C.byref(P), num_trials_robust, num_trials, num_each_iter, pose.ctypes.data, flags.ctypes.data)
    return int(n), pose, flags[:P.n_edges].astype(bool)


def undistort_keypoints(camera, kps):
    """camera::perspective::undistort_keypoints + convert_keypoints_to_bearings (camera_oracle.c).  Returns (undist_kps, bearings)."""
    kps = np.ascontiguousarray(kps, KP_DTYPE)
    n = len(kps)
    out = kps.copy()
    xy = np.ascontiguousarray(np.stack([kps["x"], kps["y"]], 1), np.float32)
    L = lib()
    equi = camera.get("model", "perspective") == "equirectangular"
    g = lambda k: float(camera.get(k, 0.0))
    if not equi:
        L.orc_undistort_points.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_void_p, C.c_int, C.c_double, C.c_void_p]
        L.orc_undistort_points.restype = None
        dist = np.array([g("k1"), g("k2"), g("p1"), g("p2"), g("k3")], np.float64)
        und = np.zeros_like(xy)
        if n:
            L.orc_undistort_points(xy.ctypes.data, n, g("fx"), g("fy"), g("cx"), g("cy"), dist.ctypes.data, 20, 1e-6, und.ctypes.data)
        out["x"], out["y"] = und[:, 0], und[:, 1]
        out["response"] = 0          # undist_keypts.resize(): default KeyPoint, only pt / angle / size / octave are set (perspective.cc:266-272)
        xy = und
    b = np.zeros((n, 3))
    L.orc_points_to_bearings.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, C.c_void_p]
    L.orc_points_to_bearings.restype = None
    if n:
        xy = np.ascontiguousarray(xy, np.float32)
        L.orc_points_to_bearings(xy.ctypes.data, n, 1 if equi else 0, g("fx"), g("fy"), g("cx"), g("cy"), g("cols"), g("rows"), b.ctypes.data)
    return out, b


def landmark_descriptor(descs):
    """orc_landmark_descriptor: index of the representative descriptor (data/landmark.cc:199-256)."""
    d = np.ascontiguousarray(descs, np.uint8).reshape(-1, 32)
    return lib().orc_landmark_descriptor(_p(d), len(d))


def can_observe(camera, pose_cw, landmarks, ray_cos_thr=0.5, img_bounds=None, num_levels=8, log_scale_factor=None):
    """orc_can_observe (data::frame::can_observe).  Same arguments and result layout as feature.orb_extractor.can_observe."""
    pos = np.ascontiguousarray(landmarks["pos_w"], np.float64).reshape(-1, 3)
    nml = np.ascontiguousarray(landmarks["mean_normal"], np.float64).reshape(-1, 3)
    lo = np.ascontiguousarray(landmarks["min_valid_dist"], np.float32)
    hi = np.ascontiguousarray(landmarks["max_valid_dist"], np.float32)
    n = len(pos)
    g = lambda k: float(camera.get(k, 0.0))
    bounds = np.ascontiguousarray(img_bounds if img_bounds is not None else (0.0, g("cols"), 0.0, g("rows")), np.float32)
    T = np.ascontiguousarray(pose_cw, np.float64).reshape(4, 4)
    Rt = np.concatenate([T[:3, :3].reshape(9), T[:3, 3]])
    twc = np.array([-((T[0, r] * T[0, 3] + T[1, r] * T[1, 3]) + T[2, r] * T[2, 3]) for r in range(3)])
    if log_scale_factor is None:
        log_scale_factor = np.log(np.float32(1.2)).astype(np.float32) if hasattr(np.log(np.float32(1.2)), "astype") else np.float32(np.log(np.float32(1.2)))
    ok, rp = np.zeros(max(n, 1), np.uint8), np.zeros((max(n, 1), 2))
    xr, lv = np.zeros(max(n, 1), np.float32), np.zeros(max(n, 1), np.uint32)
    L = lib()
    L.orc_can_observe.argtypes = [C.c_int] + [C.c_double] * 7 + [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_float, C.c_uint, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_can_observe.restype = None
    L.orc_can_observe(1 if camera.get("model", "perspective") == "equirectangular" else 0, g("fx"), g("fy"), g("cx"), g("cy"), g("fxb"), g("cols"),
                      g("rows"), _p(bounds), _p(Rt), _p(twc), n, _p(pos), _p(nml), _p(lo), _p(hi), float(ray_cos_thr), int(num_levels),
                      float(log_scale_factor), _p(ok), _p(rp), _p(xr), _p(lv))
    return dict(observable=ok[:n].astype(bool), reproj=rp[:n], x_right=xr[:n], pred_scale_level=lv[:n])


def landmark_geometry(pos_w, cam_center_lists, ref_center, ref_scale_factor, inv_scale_factor_last):
    """orc_landmark_geometry (data/landmark.cc:256-311).  Same arguments / results as match.landmark_geometry."""
    n = len(cam_center_lists)
    cnt = np.array([len(c) for c in cam_center_lists], np.int32)
    offsets = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32)
    flat = np.ascontiguousarray(np.concatenate([np.asarray(c, np.float64).reshape(-1, 3) for c in cam_center_lists]) if n and cnt.sum() else np.zeros((1, 3)))
    pos, ref = np.ascontiguousarray(pos_w, np.float64).reshape(-1, 3), np.ascontiguousarray(ref_center, np.float64).reshape(-1, 3)
    sf = np.ascontiguousarray(ref_scale_factor, np.float32)
    mn, mx, mi = np.zeros((max(n, 1), 3)), np.zeros(max(n, 1), np.float32), np.zeros(max(n, 1), np.float32)
    L = lib()
    L.orc_landmark_geometry.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_landmark_geometry.restype = None
    L.orc_landmark_geometry(n, _p(pos), _p(offsets), _p(flat), _p(ref), _p(sf), float(inv_scale_factor_last), _p(mn), _p(mx), _p(mi))
    return mn[:n], mx[:n], mi[:n]


def convert_to_grayscale(img, in_color_order="BGR"):
    """orc_convert_to_grayscale: (h, w, 3|4) uint8 -> (h, w) uint8."""
    img = np.ascontiguousarray(img, np.uint8)
    h, w, c = img.shape
    out = np.empty((h, w), np.uint8)
    L = lib()
    L.orc_convert_to_grayscale.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int]
    L.orc_convert_to_grayscale.restype = None
    L.orc_convert_to_grayscale(_p(img), w, h, img.strides[0], c, 1 if in_color_order == "RGB" else 0, _p(out), out.strides[0])
    return out


def track_local_map(camera, kps, desc, frame, scale_factors, inv_level_sigma_sq, log_scale_factor, margin=5.0, lowe_ratio=0.8, thr=100,
                    ray_cos_thr=0.5, img_bounds=None, grid=(64, 48), monocular=True, num_trials_robust=2, num_trials=2, num_each_iter=10):
    """The per-frame steady state of tracking_module::track_local_map, stage by stage with the oracle's functions:
    undistort_keypoints (perspective.cc:245-275) -> search_local_landmarks (tracking_module.cc:533-606: can_observe over the local
    landmarks, projection::match_frame_and_landmarks projection.cc:13-93) -> pose_optimizer::optimize (pose_optimizer_g2o.cc:38-175).
    kps / desc: the frame's (distorted) keypoints and descriptors; frame: dict(pose_cw, landmarks, [kp_x_right], [kp_landmark]) as
    stella_vslam_b200.tracking.local_map_tracker.pack takes it.  Returns the same dict as local_map_tracker.track."""
    kps = np.ascontiguousarray(kps, KP_DTYPE)
    n_kp = len(kps)
    lm = frame["landmarks"]
    n_lm = len(np.asarray(lm["pos_w"]).reshape(-1, 3))
    sf = np.asarray(scale_factors, np.float32)
    num_levels = len(sf)
    und, _ = undistort_keypoints(camera, kps)
    g = lambda k: float(camera.get(k, 0.0))
    bounds = img_bounds if img_bounds is not None else (0.0, g("cols"), 0.0, g("rows"))
    co = can_observe(camera, frame["pose_cw"], lm, ray_cos_thr, bounds, num_levels, log_scale_factor)
    skip = np.zeros(n_lm, bool) if lm.get("skip") is None else np.asarray(lm["skip"]).astype(bool)
    has_obs = np.ones(n_lm, bool) if lm.get("has_observation") is None else np.asarray(lm["has_observation"]).astype(bool)
    observable = co["observable"] & ~skip
    kp_lm = np.full(n_kp, -1, np.int32) if frame.get("kp_landmark") is None else np.asarray(frame["kp_landmark"], np.int32).copy()
    occupied = np.array([(l >= 0 and has_obs[l]) for l in kp_lm], np.uint8)          # `lm && lm->has_observation()` (projection.cc:50-53)
    lvl = co["pred_scale_level"].astype(np.int64)
    pr = dict(t_x=und["x"], t_y=und["y"], t_octave=und["octave"].astype(np.uint8), t_desc=np.ascontiguousarray(desc, np.uint8),
              t_x_right=frame.get("kp_x_right"), t_occupied=occupied, bounds=bounds, grid=grid,
              q_desc=np.ascontiguousarray(lm["desc"], np.uint8), q_x=co["reproj"][:, 0].astype(np.float32), q_y=co["reproj"][:, 1].astype(np.float32),
              q_margin=np.float32(margin) * sf[lvl], q_min_level=np.maximum(0, lvl - 1), q_max_level=np.minimum(num_levels - 1, lvl + 1),
              q_x_right=co["x_right"], q_valid=observable.astype(np.uint8), q_has_observation=has_obs.astype(np.uint8))
    match_out, _, n_matches = match_guided(pr, 0, thr=thr, lowe_ratio=lowe_ratio, check_orientation=False)
    for q in range(n_lm):                                   # frm.add_landmark(local_lm, best_idx) in iteration order (projection.cc:87)
        if match_out[q] >= 0:
            kp_lm[match_out[q]] = q
    idx = np.nonzero(kp_lm >= 0)[0]                         # one edge per keypoint with a landmark, keypoint order (pose_optimizer_g2o.cc:88-111)
    xr = np.full(n_kp, -1.0, np.float32) if frame.get("kp_x_right") is None else np.asarray(frame["kp_x_right"], np.float32)
    isig = np.asarray(inv_level_sigma_sq, np.float32)
    chi = np.float32(np.sqrt(np.float32(5.99146))) if monocular else np.float32(np.sqrt(np.float32(7.81473)))
    pos = np.asarray(lm["pos_w"], np.float64).reshape(-1, 3)
    cam = dict(model=1 if camera.get("model", "perspective") == "equirectangular" else 0, fx=g("fx"), fy=g("fy"), cx=g("cx"), cy=g("cy"),
               fxb=g("fxb"), cols=g("cols"), rows=g("rows"))
    ne = len(idx)
    pp = dict(pose_cw=np.asarray(frame["pose_cw"], np.float64).reshape(1, 4, 4), pose_fixed=np.zeros(1, np.uint8), points=pos[kp_lm[idx]].reshape(-1, 3),
              point_fixed=np.ones(ne, np.uint8), e_pose=np.zeros(ne, np.int32), e_point=np.arange(ne, dtype=np.int32), e_cam=np.zeros(ne, np.uint8),
              e_obs=np.stack([und["x"][idx], und["y"][idx], xr[idx]], 1).astype(np.float32), e_inv_sigma_sq=isig[und["octave"][idx].astype(np.int64)],
              e_delta=np.full(ne, chi, np.float32), e_robust=None, e_can_be_outlier=None, cams=[cam])
    outlier = np.zeros(n_kp, bool)
    if ne >= 5:
        n_valid, pose, flags = pose_optimize(pp, num_trials_robust, num_trials, num_each_iter)
        outlier[idx] = flags
    else:
        n_valid, pose = 0, np.asarray(frame["pose_cw"], np.float64).reshape(4, 4).copy()
    return dict(observable=observable, kp_landmark=kp_lm, kp_outlier=outlier, pose_cw=pose, n_matches=int(n_matches), n_valid=int(n_valid),
                n_keypoints=n_kp)
