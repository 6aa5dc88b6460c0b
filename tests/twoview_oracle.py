"""CPU restatement of solve::homography_solver / fundamental_solver (test infrastructure): loads tests/twoview_oracle.c, compiled on
first use into a temporary directory (the tree is never written)."""
import ctypes as C

import numpy as np

import cbuild

_lib = None

MODEL_H, MODEL_F = 0, 1
STATUS_SVD = 2


def lib():
    global _lib
    if _lib is None:
        L = cbuild.load("twoview_oracle.c")
        vp, i32 = C.c_void_p, C.c_int
        L.orc_normalize.argtypes = [i32, vp, vp, vp, vp, vp]
        L.orc_normalize.restype = None
        L.orc_estimate.argtypes = [i32, i32, vp, vp, vp, C.POINTER(i32)]
        L.orc_svd_n9.argtypes = [i32, vp, vp, vp, C.POINTER(i32)]
        L.orc_inverse33.argtypes = [vp, vp]
        L.orc_inverse33.restype = None
        L.orc_check_inliers.argtypes = [i32, vp, vp, i32, vp, vp, C.c_float, vp, C.POINTER(C.c_float)]
        L.orc_check_inliers.restype = C.c_uint
        L.orc_error.argtypes = [i32, vp, vp, vp]
        L.orc_error.restype = C.c_double
        L.orc_twoview_ransac.argtypes = ([i32, i32, vp, i32, vp, i32, vp, C.c_float, i32, i32, vp] + [C.POINTER(i32)] * 3 +
                                         [C.POINTER(C.c_float), vp, vp])
        _lib = L
    return _lib


def _f(a, shape=(-1, 2)):
    return np.ascontiguousarray(np.asarray(a, np.float32).reshape(shape))


def _d(a, shape=None):
    a = np.ascontiguousarray(a, np.float64)
    return a if shape is None else a.reshape(shape)


def _model(m):
    return {"H": MODEL_H, "F": MODEL_F, MODEL_H: MODEL_H, MODEL_F: MODEL_F}[m]


def normalize(pts):
    """solve::normalize: (normalised points (n, 2) float32, mean float32[2], l1 float32[2], transform (3, 3))."""
    pts = _f(pts)
    out, mean, l1, T = np.zeros_like(pts), np.zeros(2, np.float32), np.zeros(2, np.float32), np.zeros(9)
    lib().orc_normalize(len(pts), pts.ctypes.data, out.ctypes.data, mean.ctypes.data, l1.ctypes.data, T.ctypes.data)
    return out, mean, l1, T.reshape(3, 3)


def estimate(model, p1, p2):
    """compute_H_21 / compute_F_21 on normalised points: (3 x 3 or None when H is degenerate, status)."""
    p1, p2 = _f(p1), _f(p2)
    M, st = np.zeros(9), C.c_int()
    ok = lib().orc_estimate(_model(model), len(p1), p1.ctypes.data, p2.ctypes.data, M.ctypes.data, C.byref(st))
    return (M.reshape(3, 3) if ok else None), st.value


def svd_n9(A):
    """JacobiSVD of the m x 9 A: (V's last column, singular values, rank, status)."""
    A = _d(A, (-1, 9))
    v, sv, rank = np.zeros(9), np.zeros(9), C.c_int()
    st = lib().orc_svd_n9(len(A), A.ctypes.data, v.ctypes.data, sv.ctypes.data, C.byref(rank))
    return v, sv[:min(len(A), 9)], rank.value, st


def inverse33(M):
    M, R = _d(M, 9), np.zeros(9)
    lib().orc_inverse33(M.ctypes.data, R.ctypes.data)
    return R.reshape(3, 3)


def error(model, M, k1, k2):
    """One match's error: H's symmetric transfer error, F's Sampson distance."""
    M, k1, k2 = _d(M, 9), _f(k1, 2), _f(k2, 2)
    return lib().orc_error(_model(model), M.ctypes.data, k1.ctypes.data, k2.ctypes.data)


def check_inliers(model, kp1, kp2, matches, M, sigma=1.0):
    """(num_inliers, flags, cost as float32)."""
    kp1, kp2, M = _f(kp1), _f(kp2), _d(M, 9)
    mt = np.ascontiguousarray(np.asarray(matches, np.int32).reshape(-1, 2))
    fl, cost = np.zeros(max(len(mt), 1), np.uint8), C.c_float()
    num = lib().orc_check_inliers(_model(model), kp1.ctypes.data, kp2.ctypes.data, len(mt), mt.ctypes.data, M.ctypes.data, float(sigma),
                                  fl.ctypes.data, C.byref(cost))
    return num, fl[:len(mt)].astype(bool), np.float32(cost.value)


def twoview_ransac(model, keypts_1, keypts_2, matches_12, min_sets, sigma=1.0, recompute=True):
    """find_via_ransac on the given minimal sets.  Returns dict(status, valid, best_iter, num_inliers, best_cost (float32), M_21 (None
    unless valid), inlier_flags (None on the early return))."""
    m = _model(model)
    kp1, kp2 = _f(keypts_1), _f(keypts_2)
    mt = np.ascontiguousarray(np.asarray(matches_12, np.int32).reshape(-1, 2))
    n = len(mt)
    ms = np.ascontiguousarray(np.asarray(min_sets, np.int32).reshape(-1, 4 if m == MODEL_H else 8))
    M, fl = np.zeros(9), np.zeros(max(n, 1), np.uint8)
    valid, it, ninl, cost = C.c_int(), C.c_int(), C.c_int(), C.c_float()
    st = lib().orc_twoview_ransac(m, len(kp1), kp1.ctypes.data, len(kp2), kp2.ctypes.data, n, mt.ctypes.data, float(sigma), len(ms),
                                  int(bool(recompute)), ms.ctypes.data, C.byref(valid), C.byref(it), C.byref(ninl), C.byref(cost),
                                  M.ctypes.data, fl.ctypes.data)
    return dict(status=st, valid=bool(valid.value), best_iter=it.value, num_inliers=ninl.value, best_cost=np.float32(cost.value),
                M_21=M.reshape(3, 3) if valid.value else None, inlier_flags=None if n < 8 else fl[:n].astype(bool))
