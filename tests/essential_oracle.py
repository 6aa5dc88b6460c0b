"""CPU restatement of solve::essential_solver (test infrastructure): loads tests/essential_oracle.c, compiled on first use into a temporary
directory (the tree is never written)."""
import ctypes as C

import numpy as np

import cbuild

_lib = None

STATUS_SCHUR, STATUS_SVD, STATUS_WIDE_KER = 1, 2, 4


def lib():
    global _lib
    if _lib is None:
        L = cbuild.load("essential_oracle.c")
        vp, i32 = C.c_void_p, C.c_int
        L.orc_nullspace5.argtypes = [vp, vp, vp, C.POINTER(i32)]
        L.orc_lu_kernel.argtypes = [i32, vp, vp]
        L.orc_lu_solve10.argtypes = [vp, vp, vp]
        L.orc_constraint_matrix.argtypes = [vp, vp]
        L.orc_constraint_matrix.restype = None
        L.orc_eigen10.argtypes = [vp, vp, vp, vp]
        L.orc_minimal.argtypes = [vp, vp, vp, C.POINTER(i32)]
        L.orc_nonminimal.argtypes = [i32, vp, vp, vp]
        L.orc_check_inliers.argtypes = [i32, vp, vp, vp, vp, C.POINTER(C.c_float)]
        L.orc_check_inliers.restype = C.c_uint
        L.orc_cos_angle_thr.restype = C.c_float
        L.orc_essential_ransac.argtypes = [i32, vp, vp, i32, i32, vp] + [C.POINTER(i32)] * 4 + [C.POINTER(C.c_float), vp, vp]
        _lib = L
    return _lib


def _d(a, shape=None):
    a = np.ascontiguousarray(a, np.float64)
    return a if shape is None else a.reshape(shape)


def nullspace5(b1, b2):
    """(basis 9 x 4 or None when dimensionOfKernel() < 4, wide): the five-point nullspace."""
    b1, b2 = _d(b1, (5, 3)), _d(b2, (5, 3))
    basis, wide = np.zeros((9, 4)), C.c_int()
    ok = lib().orc_nullspace5(b1.ctypes.data, b2.ctypes.data, basis.ctypes.data, C.byref(wide))
    return (basis if ok else None), bool(wide.value)


def lu_kernel(A):
    A = _d(A)
    n = A.shape[0]
    K = np.zeros((n, n))
    k = lib().orc_lu_kernel(n, A.ctypes.data, K.ctypes.data)
    return K[:, :k]


def lu_solve10(A, B):
    """FullPivLU(A).solve(B): (X, rank)."""
    A, B = _d(A, (10, 10)), _d(B, (10, 10))
    X = np.zeros((10, 10))
    r = lib().orc_lu_solve10(A.ctypes.data, B.ctypes.data, X.ctypes.data)
    return X, r


def constraint_matrix(basis):
    basis = _d(basis, (9, 4))
    M = np.zeros((10, 20))
    lib().orc_constraint_matrix(basis.ctypes.data, M.ctypes.data)
    return M


def eigen10(A):
    """EigenSolver: (eigenvalues (complex, 10), V with the real eigenvectors in the columns of the real eigenvalues).  Raises on failure."""
    A = _d(A, (10, 10))
    re, im, V = np.zeros(10), np.zeros(10), np.zeros((10, 10))
    if lib().orc_eigen10(A.ctypes.data, re.ctypes.data, im.ctypes.data, V.ctypes.data) < 0:
        raise RuntimeError("RealSchur did not converge")
    return re + 1j * im, V


def minimal(b1, b2):
    """compute_E_21_minimal on five pairs: (candidates (k, 3, 3), status bits)."""
    b1, b2 = _d(b1, (5, 3)), _d(b2, (5, 3))
    E, fl = np.zeros((10, 9)), C.c_int()
    k = lib().orc_minimal(b1.ctypes.data, b2.ctypes.data, E.ctypes.data, C.byref(fl))
    return E[:k].reshape(-1, 3, 3), fl.value


def nonminimal(b1, b2):
    b1, b2 = _d(b1, (-1, 3)), _d(b2, (-1, 3))
    E = np.zeros(9)
    st = lib().orc_nonminimal(len(b1), b1.ctypes.data, b2.ctypes.data, E.ctypes.data)
    return E.reshape(3, 3), st


def check_inliers(b1, b2, E):
    """(num_inliers, flags, cost as float32)."""
    b1, b2, E = _d(b1, (-1, 3)), _d(b2, (-1, 3)), _d(E, 9)
    fl, cost = np.zeros(max(len(b1), 1), np.uint8), C.c_float()
    num = lib().orc_check_inliers(len(b1), b1.ctypes.data, b2.ctypes.data, E.ctypes.data, fl.ctypes.data, C.byref(cost))
    return num, fl[:len(b1)].astype(bool), np.float32(cost.value)


def cos_angle_thr():
    return np.float32(lib().orc_cos_angle_thr())


def essential_ransac(b1, b2, min_sets, recompute=True):
    """find_via_ransac on the given minimal sets (max_num_iter x 5).  Returns dict(status, valid, best_iter, best_candidate, num_inliers,
    best_cost (float32), E_21 (None unless valid), inlier_flags (None on the early return))."""
    b1, b2 = _d(b1, (-1, 3)), _d(b2, (-1, 3))
    n = len(b1)
    ms = np.ascontiguousarray(np.asarray(min_sets, np.int32).reshape(-1, 5))
    E, fl = np.zeros(9), np.zeros(max(n, 1), np.uint8)
    valid, it, cand, ninl, cost = C.c_int(), C.c_int(), C.c_int(), C.c_int(), C.c_float()
    st = lib().orc_essential_ransac(n, b1.ctypes.data, b2.ctypes.data, len(ms), int(bool(recompute)), ms.ctypes.data, C.byref(valid),
                                    C.byref(it), C.byref(cand), C.byref(ninl), C.byref(cost), E.ctypes.data, fl.ctypes.data)
    return dict(status=st, valid=bool(valid.value), best_iter=it.value, best_candidate=cand.value, num_inliers=ninl.value,
                best_cost=np.float32(cost.value), E_21=E.reshape(3, 3) if valid.value else None,
                inlier_flags=None if n < 5 else fl[:n].astype(bool))
