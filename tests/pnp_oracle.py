"""CPU restatement of solve::pnp_solver (test infrastructure): loads tests/pnp_oracle.c, compiled on first use into a temporary
directory (the tree is never written)."""
import ctypes as C

import numpy as np

import cbuild

_lib = None


def lib():
    global _lib
    if _lib is None:
        L = cbuild.load("pnp_oracle.c")
        vp, i32, u32 = C.c_void_p, C.c_int, C.c_uint
        L.orc_svd_square.argtypes = [i32, vp, vp, vp, vp, vp]
        L.orc_svd_solve_6xk.argtypes = [i32, vp, vp, vp, vp]
        L.orc_householder_qr_solve_6x4.argtypes = [vp, vp, vp]
        L.orc_householder_qr_solve_6x4.restype = None
        L.orc_max_cos_error.argtypes = [C.c_float]
        L.orc_max_cos_error.restype = C.c_float
        L.orc_epnp_compute_pose.argtypes = [i32, vp, vp, u32, vp, vp, C.POINTER(i32), C.POINTER(C.c_double)]
        L.orc_pnp_ransac.argtypes = [i32, vp, vp, vp, u32, u32, u32, i32, vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32),
                                     C.POINTER(C.c_double), vp, vp, vp]
        _lib = L
    return _lib


def _d(a, shape=None):
    a = np.ascontiguousarray(a, np.float64)
    return a if shape is None else a.reshape(shape)


def svd_square(A, want_v=True):
    """JacobiSVD of a square matrix: (U, V or None, singular values, number of nonzero singular values).  Raises on no convergence."""
    A = _d(A)
    n = A.shape[0]
    W, U, V, sv = np.zeros((n, n)), np.zeros((n, n)), np.zeros((n, n)), np.zeros(n)
    nz = lib().orc_svd_square(n, A.ctypes.data, W.ctypes.data, U.ctypes.data, V.ctypes.data if want_v else None, sv.ctypes.data)
    if nz < 0:
        raise RuntimeError("Jacobi SVD did not converge")
    return U, (V if want_v else None), sv, nz


def svd_solve_6xk(A, rhs):
    """JacobiSVD<MatX_t>(A (6 x k), ComputeFullU | ComputeFullV).solve(rhs): (x, rank, singular values)."""
    A = _d(A)
    k = A.shape[1]
    assert A.shape[0] == 6 and k in (3, 4, 5)
    rhs = _d(rhs, 6)
    x, sv = np.zeros(k), np.zeros(k)
    r = lib().orc_svd_solve_6xk(k, A.ctypes.data, rhs.ctypes.data, x.ctypes.data, sv.ctypes.data)
    if r < 0:
        raise RuntimeError("Jacobi SVD did not converge")
    return x, r, sv


def householder_qr_solve(A, b):
    A, b = _d(A, (6, 4)), _d(b, 6)
    x = np.zeros(4)
    lib().orc_householder_qr_solve_6x4(A.ctypes.data, b.ctypes.data, x.ctypes.data)
    return x


def max_cos_errors(scale_factors, octaves):
    sf = np.asarray(scale_factors, np.float32)
    return np.array([lib().orc_max_cos_error(float(sf[o])) for o in np.asarray(octaves, np.int64)], np.float32)


def compute_pose(bearings, points, num_iter=5, rot_cw=None, trans_cw=None):
    """pnp_solver::compute_pose: (rot_cw, trans_cw, reproj_error, wrote).  rot_cw / trans_cw are kept as given when no candidate wrote."""
    b, p = _d(bearings, (-1, 3)), _d(points, (-1, 3))
    R = np.zeros((3, 3)) if rot_cw is None else _d(rot_cw, (3, 3)).copy()
    t = np.zeros(3) if trans_cw is None else _d(trans_cw, 3).copy()
    wrote, err = C.c_int(), C.c_double()
    st = lib().orc_epnp_compute_pose(len(b), b.ctypes.data, p.ctypes.data, int(num_iter), R.ctypes.data, t.ctypes.data, C.byref(wrote),
                                      C.byref(err))
    if st < 0:
        raise RuntimeError("Jacobi SVD did not converge")
    return R, t, err.value, bool(wrote.value)


def pnp_ransac(prob, min_sets):
    """find_via_ransac on the given minimal sets.  prob: dict(bearings, points, octaves, scale_factors, min_num_inliers=10,
    gauss_newton_num_iter=10, recompute=True).  Returns dict(status, valid, best_iter, num_inliers, min_cost, rot_cw, trans_cw, inlier_flags)."""
    b, p = _d(prob["bearings"], (-1, 3)), _d(prob["points"], (-1, 3))
    n = len(b)
    mc = max_cos_errors(prob["scale_factors"], prob["octaves"]) if n else np.zeros(0, np.float32)
    mc = np.ascontiguousarray(mc)
    ms = np.ascontiguousarray(np.asarray(min_sets, np.int32).reshape(-1, 4))
    R, t, flags = np.zeros((3, 3)), np.zeros(3), np.zeros(max(n, 1), np.uint8)
    valid, best, ninl, cost = C.c_int(), C.c_int(), C.c_int(), C.c_double()
    st = lib().orc_pnp_ransac(n, b.ctypes.data, p.ctypes.data, mc.ctypes.data, int(prob.get("min_num_inliers", 10)),
                              int(prob.get("gauss_newton_num_iter", 10)), len(ms), int(bool(prob.get("recompute", True))), ms.ctypes.data,
                              C.byref(valid), C.byref(best), C.byref(ninl), C.byref(cost), R.ctypes.data, t.ctypes.data, flags.ctypes.data)
    return dict(status=0 if st == 0 else -1, valid=bool(valid.value), best_iter=best.value, num_inliers=ninl.value, min_cost=cost.value,
                rot_cw=R, trans_cw=t, inlier_flags=flags[:n].astype(bool))
