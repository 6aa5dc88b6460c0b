"""CPU restatement of optimize::graph_optimizer (test infrastructure): loads tests/pgo_oracle.c, compiled on first use into a temporary
directory (the tree is never written).  Sim3s are 8-vectors (q x y z w, t, s), as b200_sim3_t."""
import ctypes as C

import numpy as np

import cbuild

_lib = None


def lib():
    global _lib
    if _lib is None:
        L = cbuild.load("pgo_oracle.c")
        vp, i32 = C.c_void_p, C.c_int
        for name in ("orc_sim3_exp", "orc_sim3_log", "orc_sim3_inverse"):
            getattr(L, name).argtypes = [vp, vp]
        for name in ("orc_sim3_mul", "orc_sim3_map"):
            getattr(L, name).argtypes = [vp, vp, vp]
        L.orc_sim3_from_rts.argtypes = [vp, vp, C.c_double, vp]
        L.orc_edge_error.argtypes = [vp, vp, vp, vp]
        L.orc_edge_jacobian.argtypes = [vp, vp, vp, i32, i32, vp]
        L.orc_rcm.argtypes = [i32, vp, i32, vp, vp, vp, vp, C.POINTER(C.c_int64)]
        L.orc_graph_optimize.argtypes = [i32, i32, i32, vp, vp, vp, vp, vp, i32, vp, vp, i32, C.c_double, vp, vp, vp, vp]
        L.orc_graph_linearize.argtypes = [i32, i32, vp, vp, vp, vp, vp, C.c_double, i32, vp, vp]
        for name in ("orc_sim3_exp", "orc_sim3_log", "orc_sim3_inverse", "orc_sim3_mul", "orc_sim3_map", "orc_sim3_from_rts", "orc_edge_error",
                     "orc_edge_jacobian", "orc_graph_linearize"):
            getattr(L, name).restype = None
        _lib = L
    return _lib


def _d(a, n=None):
    a = np.ascontiguousarray(a, np.float64)
    return a if n is None else a.reshape(n)


def exp(u):
    out = np.zeros(8)
    lib().orc_sim3_exp(_d(u, 7).ctypes.data, out.ctypes.data)
    return out


def log(g):
    out = np.zeros(7)
    lib().orc_sim3_log(_d(g, 8).ctypes.data, out.ctypes.data)
    return out


def mul(a, b):
    out = np.zeros(8)
    lib().orc_sim3_mul(_d(a, 8).ctypes.data, _d(b, 8).ctypes.data, out.ctypes.data)
    return out


def inverse(a):
    out = np.zeros(8)
    lib().orc_sim3_inverse(_d(a, 8).ctypes.data, out.ctypes.data)
    return out


def map(a, p):  # noqa: A001 - g2o::Sim3::map
    out = np.zeros(3)
    lib().orc_sim3_map(_d(a, 8).ctypes.data, _d(p, 3).ctypes.data, out.ctypes.data)
    return out


def from_rts(R, t, s=1.0):
    out = np.zeros(8)
    lib().orc_sim3_from_rts(_d(R, 9).ctypes.data, _d(t, 3).ctypes.data, float(s), out.ctypes.data)
    return out


def edge_error(meas, v1, v2):
    out = np.zeros(7)
    lib().orc_edge_error(_d(meas, 8).ctypes.data, _d(v1, 8).ctypes.data, _d(v2, 8).ctypes.data, out.ctypes.data)
    return out


def edge_jacobian(meas, v1, v2, side, fix_scale=False):
    """d error / d update of vertex `side` (7x7, rows = error components), g2o's central difference at delta 1e-9."""
    out = np.zeros((7, 7))
    lib().orc_edge_jacobian(_d(meas, 8).ctypes.data, _d(v1, 8).ctypes.data, _d(v2, 8).ctypes.data, int(side), int(bool(fix_scale)),
                            out.ctypes.data)
    return out


def graph_linearize(graph, delta=1e-9, order=2):
    """Every edge's error (m,7) and both vertex Jacobians (m,2,7,7) by a central difference of `order` 2 (g2o's, bit-identical to
    edge_jacobian at delta 1e-9) or 4 at step `delta`; the Jacobian of a fixed vertex is zero."""
    est = _d(graph["estimate"], (-1, 8))
    fixed = np.ascontiguousarray(graph["fixed"], np.uint8)
    e1, e2 = np.ascontiguousarray(graph["e_v1"], np.int32), np.ascontiguousarray(graph["e_v2"], np.int32)
    meas = _d(graph["e_meas"], (-1, 8))
    err, J = np.zeros((len(e1), 7)), np.zeros((len(e1), 2, 7, 7))
    lib().orc_graph_linearize(len(e1), int(bool(graph.get("fix_scale", False))), est.ctypes.data, fixed.ctypes.data, e1.ctypes.data,
                              e2.ctypes.data, meas.ctypes.data, float(delta), int(order), err.ctypes.data, J.ctypes.data)
    return err, J


def rcm(graph):
    """(order of the free vertices, envelope doubles of the 32x32-tile envelope)."""
    nv = len(graph["estimate"])
    fixed = np.ascontiguousarray(graph["fixed"], np.uint8)
    e1, e2 = np.ascontiguousarray(graph["e_v1"], np.int32), np.ascontiguousarray(graph["e_v2"], np.int32)
    order, pos = np.zeros(nv + 1, np.int32), np.zeros(nv, np.int32)
    env = C.c_int64()
    nf = lib().orc_rcm(nv, fixed.ctypes.data, len(e1), e1.ctypes.data, e2.ctypes.data, order.ctypes.data, pos.ctypes.data, C.byref(env))
    return order[:nf].copy(), env.value


def graph_optimize(graph, max_iter=50, gain_threshold=1e-3):
    """graph: dict(estimate (n,8), fixed (n,), e_v1, e_v2, e_meas (m,8), fix_scale, points (k,3), point_ref (k,)).
    Returns dict(estimate, pose_cw, points, iterations, trials, chi2_init, chi2_final, lambda_init, lambda_final, envelope_doubles,
    chi2_history: the chi2 after every iteration)."""
    est = _d(graph["estimate"], (-1, 8))
    nv = len(est)
    fixed = np.ascontiguousarray(graph["fixed"], np.uint8)
    e1, e2 = np.ascontiguousarray(graph["e_v1"], np.int32), np.ascontiguousarray(graph["e_v2"], np.int32)
    meas = _d(graph["e_meas"], (-1, 8))
    pts = _d(graph.get("points", np.zeros((0, 3))), (-1, 3))
    pref = np.ascontiguousarray(graph.get("point_ref", np.zeros(0)), np.int32)
    est_out, pose, pts_out, st = np.zeros((nv, 8)), np.zeros((nv, 4, 4)), np.zeros((len(pts), 3)), np.zeros(8 + max(int(max_iter), 0))
    lib().orc_graph_optimize(nv, len(e1), int(bool(graph.get("fix_scale", False))), est.ctypes.data, fixed.ctypes.data, e1.ctypes.data,
                             e2.ctypes.data, meas.ctypes.data, len(pts), pts.ctypes.data, pref.ctypes.data, int(max_iter), float(gain_threshold),
                             est_out.ctypes.data, pose.ctypes.data, pts_out.ctypes.data, st.ctypes.data)
    return dict(estimate=est_out, pose_cw=pose, points=pts_out, iterations=int(st[0]), trials=int(st[1]), chi2_init=st[2], chi2_final=st[3],
                lambda_init=st[4], lambda_final=st[5], envelope_doubles=int(st[6]), chi2_history=st[8:8 + int(st[0])].copy())
