"""CPU restatement of optimize::transform_optimizer (test infrastructure): loads tests/transform_oracle.c (which includes
tests/pgo_oracle.c for the g2o::Sim3 algebra), compiled on first use into a temporary directory (the tree is never written).  Sim3s are
8-vectors (q x y z w, t, s), as b200_sim3_t; a camera is a dict(model, fx, fy, cx, cy, cols, rows) as b200_camera_t."""
import ctypes as C

import numpy as np

import cbuild

_lib = None


def lib():
    global _lib
    if _lib is None:
        L = cbuild.load("transform_oracle.c")
        vp, i32 = C.c_void_p, C.c_int
        L.orc_transform_edge.argtypes = [vp, i32, vp, vp, vp, C.c_float, vp]
        L.orc_transform_edge.restype = C.c_double
        L.orc_transform_jacobian.argtypes = [vp, i32, vp, vp, vp, C.c_float, i32, vp]
        L.orc_transform_jacobian.restype = None
        L.orc_transform_optimize.argtypes = [i32, i32] + [vp] * 13 + [C.c_float, i32, vp, vp, vp]
        L.orc_transform_optimize.restype = C.c_uint
        _lib = L
    return _lib


def _d(a, n=None):
    a = np.ascontiguousarray(a, np.float64)
    return a if n is None else a.reshape(n)


def _cam(c):
    return _d([c["model"], c.get("fx", 0.0), c.get("fy", 0.0), c.get("cx", 0.0), c.get("cy", 0.0), c.get("cols", 0.0), c.get("rows", 0.0)], 7)


def transform_edge(sim3_12, side, pc, cam, obs, inv_sigma_sq):
    """computeError of edge_12 (side 0: Sim3_12.map) or edge_21 (side 1: Sim3_12.inverse().map) at the camera-frame point pc.
    Returns (error (2,), chi2)."""
    e = np.zeros(2)
    o = np.ascontiguousarray(obs, np.float32).reshape(2)
    chi = lib().orc_transform_edge(_d(sim3_12, 8).ctypes.data, int(side), _d(pc, 3).ctypes.data, _cam(cam).ctypes.data, o.ctypes.data,
                                   float(inv_sigma_sq), e.ctypes.data)
    return e, chi


def transform_jacobian(sim3_12, side, pc, cam, obs, inv_sigma_sq, fix_scale=False):
    """d error / d update (2x7), g2o's central difference at delta 1e-9 through transform_vertex::oplusImpl."""
    J = np.zeros((2, 7))
    o = np.ascontiguousarray(obs, np.float32).reshape(2)
    lib().orc_transform_jacobian(_d(sim3_12, 8).ctypes.data, int(side), _d(pc, 3).ctypes.data, _cam(cam).ctypes.data, o.ctypes.data,
                                 float(inv_sigma_sq), int(bool(fix_scale)), J.ctypes.data)
    return J


def transform_optimize(pr, chi_sq=10.0, num_iter=10):
    """pr: dict as workloads.synth.make_sim3_pair returns (sim3_12, rot_1w, trans_1w, rot_2w, trans_2w, cam_1, cam_2, obs_1,
    inv_sigma_sq_1, pos_w_2, obs_2, inv_sigma_sq_2, pos_w_1, fix_scale).  Returns dict(sim3_12, keep, num_inliers, n_outliers_round1,
    iterations, trials, chi2, lambda_init, failed_at: per round the iteration whose LM step failed, -1 for none)."""
    n = len(pr["obs_1"])
    f32 = lambda k, shape: np.ascontiguousarray(pr[k], np.float32).reshape(shape)
    arrs = [_d(pr["sim3_12"], 8), _d(pr["rot_1w"], 9), _d(pr["trans_1w"], 3), _d(pr["rot_2w"], 9), _d(pr["trans_2w"], 3), _cam(pr["cam_1"]),
            _cam(pr["cam_2"]), f32("obs_1", (n, 2)), f32("inv_sigma_sq_1", n), _d(pr["pos_w_2"], (n, 3)), f32("obs_2", (n, 2)),
            f32("inv_sigma_sq_2", n), _d(pr["pos_w_1"], (n, 3))]
    out, keep, st = np.zeros(8), np.zeros(max(n, 1), np.uint8), np.zeros(11)
    good = lib().orc_transform_optimize(n, int(bool(pr.get("fix_scale", False))), *[a.ctypes.data for a in arrs], float(chi_sq), int(num_iter),
                                        out.ctypes.data, keep.ctypes.data, st.ctypes.data)
    return dict(sim3_12=out, keep=keep[:n].copy(), num_inliers=int(good), n_outliers_round1=int(st[0]), iterations=[int(st[1]), int(st[6])],
                trials=[int(st[2]), int(st[7])], chi2=[st[3], st[8]], lambda_init=[st[4], st[9]], failed_at=[int(st[5]), int(st[10])])
