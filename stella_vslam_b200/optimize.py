"""Host-side mirror of optimize::local_bundle_adjuster (src/stella_vslam/optimize/local_bundle_adjuster.h:15-24,
local_bundle_adjuster_g2o.{h,cc}, local_bundle_adjuster_factory.h:15-33).

The reference's optimize(map_db, curr_keyfrm, force_stop_flag) first flattens the covisibility window into vertices and
edges (steps 1-4) and writes the result back under the map mutex (step 8); both stay on the host.  This module takes the
flattened problem (the layout of b200_lba_problem_t) and runs steps 5-7 on the GPU.
"""
import ctypes as C
import math

import numpy as np

from ._lib import ERR_ABORTED, check, lib, ptr


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


def _bind():
    L = lib()
    vp = C.c_void_p
    L.b200_lba_create.argtypes = [C.c_int, C.POINTER(vp)]
    L.b200_lba_destroy.argtypes = [vp]
    L.b200_lba_solve.argtypes = [vp, C.POINTER(LbaProblem), C.c_int, C.c_int, vp, vp, vp, vp, C.POINTER(LbaStats)]
    L.b200_lba_solve_batch.argtypes = [vp, C.c_int, C.POINTER(LbaProblem), C.c_int, C.c_int, vp, vp, vp, vp, C.POINTER(LbaStats), vp]
    L.b200_lba_last_profile.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(C.c_int)]
    L.b200_pose_optimize.argtypes = [vp, C.c_int, C.POINTER(LbaProblem), C.c_int, C.c_int, C.c_int, vp, vp, vp]
    L.b200_global_ba_solve.argtypes = [vp, C.POINTER(LbaProblem), C.c_int, C.c_double, vp, vp, vp, C.POINTER(LbaStats)]
    L.b200_graph_optimize.argtypes = [vp, C.POINTER(PoseGraph), C.c_int, C.c_double, C.POINTER(PgoStats)]
    L.b200_pgo_envelope.argtypes = [C.POINTER(PoseGraph), C.POINTER(C.c_int32), vp, C.POINTER(C.c_int64)]
    L.b200_transform_optimize.argtypes = [vp, C.c_int, C.POINTER(TransformProblem), C.c_float, C.c_int]
    return L


def pack_problem(prob):
    """dict (see synth.make_ba_problem) -> (LbaProblem, keep-alive list)."""
    keep = []

    def arr(x, dt):
        if x is None:
            return None
        a = np.ascontiguousarray(x, dt)
        keep.append(a)
        return a.ctypes.data

    cams = (Camera * len(prob["cams"]))(*[Camera(c["model"], c["fx"], c["fy"], c["cx"], c["cy"], c["fxb"], c["cols"], c["rows"])
                                          for c in prob["cams"]])
    keep.append(cams)
    P = LbaProblem(len(prob["pose_cw"]), len(prob["points"]), len(prob["e_pose"]), len(prob["cams"]), arr(prob["pose_cw"], np.float64),
                   arr(prob["pose_fixed"], np.uint8), arr(prob["points"], np.float64), arr(prob.get("point_fixed"), np.uint8),
                   arr(prob["e_pose"], np.int32), arr(prob["e_point"], np.int32), arr(prob["e_cam"], np.uint8),
                   arr(prob["e_obs"], np.float32), arr(prob["e_inv_sigma_sq"], np.float32), arr(prob["e_delta"], np.float32),
                   arr(prob.get("e_robust"), np.uint8), arr(prob.get("e_can_be_outlier"), np.uint8), C.cast(cams, C.c_void_p))
    return P, keep


class local_bundle_adjuster:
    """optimize::local_bundle_adjuster with the "b200" backend (factory key Mapping.backend, local_bundle_adjuster_factory.h:17-32)."""

    def __init__(self, num_first_iter=5, num_second_iter=10, device=0):
        self.num_first_iter_ = int(num_first_iter)    # local_bundle_adjuster_g2o.h:25-27
        self.num_second_iter_ = int(num_second_iter)
        self._L = _bind()
        self._h = C.c_void_p()
        check(self._L.b200_lba_create(device, C.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None):
            self._L.b200_lba_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def prepare(self, problem):
        """Pack a problem once (ctypes struct + output buffers) for repeated, low-overhead optimize_prepared() calls."""
        P, keep = pack_problem(problem)
        K, L, E = P.n_poses, P.n_points, P.n_edges
        return dict(P=P, keep=keep, pose=np.zeros((K, 4, 4)), pts=np.zeros((L, 3)), outl=np.zeros(E, np.uint8), st=LbaStats())

    def optimize_prepared(self, prep, force_stop_flag=None):
        rc = self._L.b200_lba_solve(self._h, C.byref(prep["P"]), self.num_first_iter_, self.num_second_iter_, ptr(force_stop_flag),
                                    ptr(prep["pose"]), ptr(prep["pts"]), ptr(prep["outl"]), C.byref(prep["st"]))
        if rc == ERR_ABORTED:
            return None
        check(rc)
        launches = C.c_int()
        self._L.b200_lba_last_profile(self._h, None, C.byref(launches))
        return launches.value

    def prepare_batch(self, problems):
        """Pack several windows once (ctypes structs, pointer tables, output buffers) for repeated optimize_prepared_batch() calls."""
        packed = [pack_problem(pr) for pr in problems]
        n = len(packed)
        arr = (LbaProblem * n)(*[pk[0] for pk in packed])
        pose = [np.zeros((pk[0].n_poses, 4, 4)) for pk in packed]
        pts = [np.zeros((pk[0].n_points, 3)) for pk in packed]
        outl = [np.zeros(max(pk[0].n_edges, 1), np.uint8) for pk in packed]
        tab = lambda arrs: (C.c_void_p * n)(*[a.ctypes.data for a in arrs])
        return dict(n=n, arr=arr, keep=packed, pose=pose, pts=pts, outl=outl, pose_tab=tab(pose), pts_tab=tab(pts), outl_tab=tab(outl),
                    st=(LbaStats * n)(), status=np.zeros(n, np.int32))

    def optimize_prepared_batch(self, prep, force_stop_flags=None):
        """b200_lba_solve_batch on a prepared batch.  force_stop_flags: optional list of 1-element uint8 arrays / None per window.
        Returns the number of kernel launches the whole batch took; per-window status in prep["status"]."""
        flags = None
        if force_stop_flags is not None:
            flags = (C.c_void_p * prep["n"])(*[(f.ctypes.data if f is not None else None) for f in force_stop_flags])
        rc = self._L.b200_lba_solve_batch(self._h, prep["n"], prep["arr"], self.num_first_iter_, self.num_second_iter_, flags, prep["pose_tab"],
                                          prep["pts_tab"], prep["outl_tab"], prep["st"], ptr(prep["status"]))
        check(rc)
        launches = C.c_int()
        self._L.b200_lba_last_profile(self._h, None, C.byref(launches))
        return launches.value

    def optimize_batch(self, problems, force_stop_flags=None):
        """Several independent windows in one launch sequence (b200_lba_solve_batch).  Returns one result per window: a dict like
        optimize(), or None for a window whose flag was already set (local_bundle_adjuster_g2o.cc:308-310)."""
        if not problems:
            return []
        prep = self.prepare_batch(problems)
        launches = self.optimize_prepared_batch(prep, force_stop_flags)
        ms = C.c_float()
        self._L.b200_lba_last_profile(self._h, C.byref(ms), None)
        out = []
        for w in range(prep["n"]):
            if prep["status"][w] == ERR_ABORTED:
                out.append(None)
                continue
            st = prep["st"][w]
            E = prep["arr"][w].n_edges
            out.append(dict(pose_cw=prep["pose"][w], points=prep["pts"][w], outliers=prep["outl"][w][:E], iterations=list(st.iterations),
                            n_outliers=st.n_outliers, chi2=list(st.chi2), lambda_init=st.lambda_init, lambda_final=list(st.lambda_final),
                            gpu_ms=ms.value, launches=launches))
        return out

    def optimize(self, problem, force_stop_flag=None):
        """problem: flattened window (dict).  force_stop_flag: optional 1-element uint8 array (read AND written, like the
        reference's bool*).  Returns None if the flag was already set (local_bundle_adjuster_g2o.cc:308-310), else a dict."""
        P, keep = pack_problem(problem)
        K, L, E = P.n_poses, P.n_points, P.n_edges
        pose_out, pts_out, outl = np.zeros((K, 4, 4)), np.zeros((L, 3)), np.zeros(E, np.uint8)
        st = LbaStats()
        rc = self._L.b200_lba_solve(self._h, C.byref(P), self.num_first_iter_, self.num_second_iter_, ptr(force_stop_flag), ptr(pose_out),
                                    ptr(pts_out), ptr(outl), C.byref(st))
        if rc == ERR_ABORTED:
            return None
        check(rc)
        ms, launches = C.c_float(), C.c_int()
        self._L.b200_lba_last_profile(self._h, C.byref(ms), C.byref(launches))
        return dict(pose_cw=pose_out, points=pts_out, outliers=outl, iterations=list(st.iterations), n_outliers=st.n_outliers,
                    chi2=list(st.chi2), lambda_init=st.lambda_init, lambda_final=list(st.lambda_final), gpu_ms=ms.value,
                    launches=launches.value)


class global_bundle_adjuster:
    """optimize::global_bundle_adjuster (optimize/global_bundle_adjuster.h:18-62): one LM round over the whole map; Huber is the
    problem's e_robust array (use_huber_kernel_)."""

    def __init__(self, num_iter=10, use_huber_kernel=True, verbose=False, device=0):
        self.num_iter_, self.use_huber_kernel_, self.verbose_ = int(num_iter), bool(use_huber_kernel), bool(verbose)
        self._L = _bind()
        self._h = C.c_void_p()
        check(self._L.b200_lba_create(device, C.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None):
            self._L.b200_lba_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def optimize(self, problem, force_stop_flag=None, gain_threshold=1e-3):
        """global_bundle_adjuster::optimize (:258-420; gain threshold 1e-3) / optimize_for_initialization (:201-256; the caller's
        gain_threshold).  Returns None when the caller's flag aborted the solve (the reference returns false), else a dict."""
        pr = dict(problem)
        if not self.use_huber_kernel_:
            pr["e_robust"] = np.zeros(len(pr["e_pose"]), np.uint8)
        P, keep = pack_problem(pr)
        pose_out, pts_out = np.zeros((P.n_poses, 4, 4)), np.zeros((P.n_points, 3))
        st = LbaStats()
        rc = self._L.b200_global_ba_solve(self._h, C.byref(P), self.num_iter_, float(gain_threshold), ptr(force_stop_flag), ptr(pose_out),
                                          ptr(pts_out), C.byref(st))
        if rc == ERR_ABORTED:
            return None
        check(rc)
        ms, launches = C.c_float(), C.c_int()
        self._L.b200_lba_last_profile(self._h, C.byref(ms), C.byref(launches))
        return dict(pose_cw=pose_out, points=pts_out, iterations=st.iterations[0], chi2=st.chi2[0], lambda_init=st.lambda_init,
                    lambda_final=st.lambda_final[0], gpu_ms=ms.value, launches=launches.value)


class pose_optimizer:
    """optimize::pose_optimizer (optimize/pose_optimizer.h:24-40, pose_optimizer_g2o.{h,cc}; factory defaults
    pose_optimizer_factory.h:18-47): motion-only BA of frames, one CUDA launch for a whole batch."""

    def __init__(self, num_trials_robust=2, num_trials=2, num_each_iter=10, device=0):
        self.num_trials_robust_, self.num_trials_, self.num_each_iter_ = int(num_trials_robust), int(num_trials), int(num_each_iter)
        self._L = _bind()
        self._h = C.c_void_p()
        check(self._L.b200_lba_create(device, C.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None):
            self._L.b200_lba_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def optimize_batch(self, problems):
        """problems: flattened frames (synth.make_pose_problem layout: one pose, fixed landmarks, one edge per observation).
        Returns [(num_valid_obs, optimized_pose (4,4), outlier_flags (n,) bool)] like pose_optimizer::optimize (:38-44)."""
        if not problems:
            return []
        packed = [pack_problem(pr) for pr in problems]
        arr = (LbaProblem * len(problems))(*[pk[0] for pk in packed])
        n_edges = [pk[0].n_edges for pk in packed]
        pose = np.zeros((len(problems), 4, 4))
        flags = np.zeros(max(sum(n_edges), 1), np.uint8)
        valid = np.zeros(len(problems), np.uint32)
        check(self._L.b200_pose_optimize(self._h, len(problems), arr, self.num_trials_robust_, self.num_trials_, self.num_each_iter_,
                                         ptr(pose), ptr(flags), ptr(valid)))
        out, off = [], 0
        for i, ne in enumerate(n_edges):
            out.append((int(valid[i]), pose[i].copy(), flags[off:off + ne].astype(bool)))
            off += ne
        return out

    def optimize(self, problem):
        return self.optimize_batch([problem])[0]


def create(yaml_node=None, device=0):
    """local_bundle_adjuster_factory::create (local_bundle_adjuster_factory.h:17-32): Mapping.backend must be "b200" here;
    "g2o"/"gtsam" are the reference's CPU backends and are not part of this library."""
    node = yaml_node or {}
    backend = node.get("backend", "b200")
    if backend != "b200":
        raise RuntimeError(f"Invalid backend: {backend}")
    return local_bundle_adjuster(node.get("num_first_iter", 5), node.get("num_second_iter", 10), device)


# ---------------------------------------------------------------------------------------------------------------------------------
# optimize::graph_optimizer (optimize/graph_optimizer.{h,cc}): the Sim3 pose-graph optimisation of a loop closure
# ---------------------------------------------------------------------------------------------------------------------------------
class Sim3(C.Structure):
    """b200_sim3_t: g2o::Sim3 as rotation().coeffs() (x y z w), translation(), scale()."""
    _fields_ = [("q", C.c_double * 4), ("t", C.c_double * 3), ("s", C.c_double)]


class PoseGraph(C.Structure):
    """b200_pose_graph_t (include/b200vslam.h)."""
    _fields_ = [("n_vertices", C.c_int32), ("n_edges", C.c_int32), ("fix_scale", C.c_int32), ("estimate", C.c_void_p), ("fixed", C.c_void_p),
                ("e_v1", C.c_void_p), ("e_v2", C.c_void_p), ("e_meas", C.c_void_p), ("n_points", C.c_int32), ("points", C.c_void_p),
                ("point_ref", C.c_void_p), ("estimate_out", C.c_void_p), ("pose_cw_out", C.c_void_p), ("points_out", C.c_void_p)]


class PgoStats(C.Structure):
    """b200_pgo_stats_t (include/b200vslam.h)."""
    _fields_ = [("iterations", C.c_int32), ("trials", C.c_int32), ("chi2_init", C.c_double), ("chi2_final", C.c_double),
                ("lambda_init", C.c_double), ("lambda_final", C.c_double), ("envelope_doubles", C.c_int64), ("factor_flops", C.c_int64),
                ("launches", C.c_int32), ("lin_ms", C.c_float), ("factor_ms", C.c_float), ("solve_ms", C.c_float), ("total_ms", C.c_float)]


PGO_MAX_ENVELOPE_DOUBLES = 1 << 28   # B200_PGO_MAX_ENVELOPE_DOUBLES


# g2o::Sim3 on the host, as 8-vectors (q x y z w, t, s), in the evaluation order of csrc/sim3.cuh: what build_essential_graph needs
def _quat_rotate(q, v):
    uv = [q[1] * v[2] - q[2] * v[1], q[2] * v[0] - q[0] * v[2], q[0] * v[1] - q[1] * v[0]]
    uv = [u + u for u in uv]
    c = [q[1] * uv[2] - q[2] * uv[1], q[2] * uv[0] - q[0] * uv[2], q[0] * uv[1] - q[1] * uv[0]]
    return [v[i] + q[3] * uv[i] + c[i] for i in range(3)]


def _quat_normalize(q):
    if q[3] < 0:
        q = [-x for x in q]
    n = math.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
    return [x / n for x in q]


def sim3_from_rts(R, t, s=1.0):
    """g2o::Sim3(const Matrix3& R, const Vector3& t, double s): Quaternion(R), normalised."""
    R = [float(x) for x in np.asarray(R, np.float64).reshape(9)]
    tr = R[0] + R[4] + R[8]
    if tr > 0:
        tr = math.sqrt(tr + 1.0)
        w = 0.5 * tr
        tr = 0.5 / tr
        q = [(R[7] - R[5]) * tr, (R[2] - R[6]) * tr, (R[3] - R[1]) * tr, w]
    else:
        i = 0
        if R[4] > R[0]:
            i = 1
        if R[8] > R[i * 3 + i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        tr = math.sqrt(R[i * 3 + i] - R[j * 3 + j] - R[k * 3 + k] + 1.0)
        q = [0.0] * 4
        q[i] = 0.5 * tr
        tr = 0.5 / tr
        q[3] = (R[k * 3 + j] - R[j * 3 + k]) * tr
        q[j] = (R[j * 3 + i] + R[i * 3 + j]) * tr
        q[k] = (R[k * 3 + i] + R[i * 3 + k]) * tr
    t = [float(x) for x in np.asarray(t, np.float64).reshape(3)]
    return np.array(_quat_normalize(q) + t + [float(s)])


def sim3_mul(a, b):
    """g2o::Sim3::operator*."""
    a, b = [float(x) for x in a], [float(x) for x in b]
    q = [a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1],
         a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2],
         a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0],
         a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2]]
    rt = _quat_rotate(a[:4], b[4:7])
    return np.array(q + [a[7] * rt[i] + a[4 + i] for i in range(3)] + [a[7] * b[7]])


def sim3_inverse(a):
    """g2o::Sim3::inverse() (its constructor normalises the rotation)."""
    a = [float(x) for x in a]
    qc = [-a[0], -a[1], -a[2], a[3]]
    f = -1. / a[7]
    t = _quat_rotate(qc, [f * a[4], f * a[5], f * a[6]])
    return np.array(_quat_normalize(qc) + t + [1. / a[7]])


def build_essential_graph(keyframes, curr_id, loop_id, loop_connections, non_corrected_Sim3s=None, pre_corrected_Sim3s=None,
                          min_num_shared_lms=100, fix_scale=False, landmarks=None, found_lm_to_ref_keyfrm_id=None):
    """graph_optimizer::optimize steps 1-3 (graph_optimizer.cc:43-250) from a flat description of the map.

    keyframes: curr_keyfrm->graph_node_->get_keyframes_from_root() in order, each a dict with
        id, rot_cw (3x3), trans_cw (3), erased (will_be_erased), parent (spanning parent id or None for the root), children (spanning
        children ids), loop_edges (ids), covisibilities ([(id, num_shared_lms)] in the order of ordered_covisibilities_: descending).
    loop_connections: [(id1, [id2, ...])] in the order of the caller's std::map.
    non_corrected_Sim3s / pre_corrected_Sim3s: {id: Sim3 8-vector}.
    landmarks: optional [(lm_id, pos_w (3), ref_keyfrm_id)] of the non-erased landmarks in all_lms order; found_lm_to_ref_keyfrm_id:
        {lm_id: keyframe id}.
    Returns the graph dict of graph_optimizer.optimize (plus vertex_ids, the keyframe id of every vertex)."""
    non_corrected_Sim3s = non_corrected_Sim3s or {}
    pre_corrected_Sim3s = pre_corrected_Sim3s or {}
    found = found_lm_to_ref_keyfrm_id or {}
    kf_by_id = {k["id"]: k for k in keyframes}
    Sim3s_cw, vidx, est, fixed, vertex_ids = {}, {}, [], [], []
    for k in keyframes:                                              # 2. vertices (:70-106)
        if k.get("erased", False):
            continue
        kid = k["id"]
        if kid in pre_corrected_Sim3s:
            s = np.asarray(pre_corrected_Sim3s[kid], np.float64)
        else:
            s = sim3_from_rts(k["rot_cw"], k["trans_cw"], 1.0)
        Sim3s_cw[kid] = s
        vidx[kid] = len(est)
        est.append(s)
        fixed.append(kid == loop_id or kid == curr_id or k.get("parent") is None)
        vertex_ids.append(kid)
    e_v1, e_v2, meas = [], [], []
    inserted = set()

    def insert_edge(id1, id2, S21):
        e_v1.append(vidx[id1])
        e_v2.append(vidx[id2])
        meas.append(S21)
        inserted.add((min(id1, id2), max(id1, id2)))

    def shared(k, other):
        return dict(k.get("covisibilities", ())).get(other, 0)

    for id1, connected in loop_connections:                          # loop edges over the threshold (:130-160)
        S_w1 = sim3_inverse(Sim3s_cw[id1])
        for id2 in connected:
            if not (id1 == curr_id and id2 == loop_id) and shared(kf_by_id[id1], id2) < min_num_shared_lms:
                continue
            insert_edge(id1, id2, sim3_mul(Sim3s_cw[id2], S_w1))

    def sim3_2w(id2):
        return np.asarray(non_corrected_Sim3s[id2], np.float64) if id2 in non_corrected_Sim3s else Sim3s_cw[id2]

    for k in keyframes:                                              # non-loop edges (:162-250)
        if k.get("erased", False):                                   # no vertex: the reference's Sim3s_cw.at(id1) would throw
            continue
        id1 = k["id"]
        S_w1 = sim3_inverse(np.asarray(non_corrected_Sim3s[id1], np.float64) if id1 in non_corrected_Sim3s else Sim3s_cw[id1])
        parent = k.get("parent")
        if parent is not None:
            if id1 <= parent:                                        # :166-172 skips the rest of this keyframe, not only the edge
                continue
            insert_edge(id1, parent, sim3_mul(sim3_2w(parent), S_w1))
        loop_edges = set(k.get("loop_edges", ()))
        for id2 in k.get("loop_edges", ()):
            if id1 > id2:
                insert_edge(id1, id2, sim3_mul(sim3_2w(id2), S_w1))
        children = set(k.get("children", ()))
        for id2, w in k.get("covisibilities", ()):
            if w < min_num_shared_lms or parent is None:
                continue
            if id2 == parent or id2 in children or id2 in loop_edges:
                continue
            if kf_by_id[id2].get("erased", False):
                continue
            if id1 <= id2 or (min(id1, id2), max(id1, id2)) in inserted:
                continue
            insert_edge(id1, id2, sim3_mul(sim3_2w(id2), S_w1))
    graph = dict(estimate=np.array(est).reshape(-1, 8), fixed=np.array(fixed, np.uint8), e_v1=np.array(e_v1, np.int32),
                 e_v2=np.array(e_v2, np.int32), e_meas=np.array(meas).reshape(-1, 8), fix_scale=bool(fix_scale), vertex_ids=vertex_ids,
                 points=np.zeros((0, 3)), point_ref=np.zeros(0, np.int32))
    if landmarks:                                                    # 5. landmark references (:283-300)
        graph["points"] = np.array([lm[1] for lm in landmarks], np.float64).reshape(-1, 3)
        graph["point_ref"] = np.array([vidx[found.get(lm[0], lm[2])] for lm in landmarks], np.int32)
    return graph


def pack_pose_graph(graph):
    """graph dict -> (PoseGraph with output buffers, keep-alive dict holding estimate_out / pose_cw_out / points_out)."""
    keep = {}

    def arr(name, x, dt, shape=None):
        a = np.ascontiguousarray(x, dt)
        if shape is not None:
            a = a.reshape(shape)
        keep[name] = a
        return a.ctypes.data

    nv, ne = len(graph["estimate"]), len(graph["e_v1"])
    pts = np.asarray(graph.get("points", np.zeros((0, 3))), np.float64).reshape(-1, 3)
    G = PoseGraph()
    G.n_vertices, G.n_edges, G.fix_scale = nv, ne, int(bool(graph.get("fix_scale", False)))
    G.estimate = arr("estimate", graph["estimate"], np.float64, (-1, 8))
    G.fixed = arr("fixed", graph["fixed"], np.uint8)
    G.e_v1 = arr("e_v1", graph["e_v1"], np.int32)
    G.e_v2 = arr("e_v2", graph["e_v2"], np.int32)
    G.e_meas = arr("e_meas", np.asarray(graph["e_meas"], np.float64).reshape(-1, 8), np.float64)
    G.n_points = len(pts)
    G.points = arr("points", pts, np.float64)
    G.point_ref = arr("point_ref", graph.get("point_ref", np.zeros(0)), np.int32)
    keep["estimate_out"], keep["pose_cw_out"], keep["points_out"] = np.zeros((nv, 8)), np.zeros((nv, 4, 4)), np.zeros((len(pts), 3))
    G.estimate_out, G.pose_cw_out = keep["estimate_out"].ctypes.data, keep["pose_cw_out"].ctypes.data
    G.points_out = keep["points_out"].ctypes.data if len(pts) else None
    return G, keep


def pgo_envelope(graph):
    """b200_pgo_envelope (host only): (reverse Cuthill-McKee order of the free vertices, envelope doubles)."""
    L = _bind()
    G, keep = pack_pose_graph(graph)
    nf, env = C.c_int32(), C.c_int64()
    order = np.zeros(max(len(graph["estimate"]), 1), np.int32)
    check(L.b200_pgo_envelope(C.byref(G), C.byref(nf), ptr(order), C.byref(env)))
    return order[:nf.value].copy(), env.value


class graph_optimizer:
    """optimize::graph_optimizer (optimize/graph_optimizer.h:20-45): the loop closure's Sim3 essential-graph optimisation on the GPU.
    build_essential_graph() restates how the reference builds the vertices and edges; optimize() runs steps 4-5."""

    def __init__(self, min_num_shared_lms=100, fix_scale=False, device=0, max_iter=50, gain_threshold=1e-3):
        self.min_num_shared_lms_, self.fix_scale_ = int(min_num_shared_lms), bool(fix_scale)   # GraphOptimizer.min_num_shared_lms
        self.max_iter_, self.gain_threshold_ = int(max_iter), float(gain_threshold)
        self._L = _bind()
        self._h = C.c_void_p()
        check(self._L.b200_lba_create(device, C.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None):
            self._L.b200_lba_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def build_essential_graph(self, keyframes, curr_id, loop_id, loop_connections, non_corrected_Sim3s=None, pre_corrected_Sim3s=None,
                              landmarks=None, found_lm_to_ref_keyfrm_id=None):
        return build_essential_graph(keyframes, curr_id, loop_id, loop_connections, non_corrected_Sim3s, pre_corrected_Sim3s,
                                     self.min_num_shared_lms_, self.fix_scale_, landmarks, found_lm_to_ref_keyfrm_id)

    def optimize(self, graph):
        """graph: dict(estimate (n,8), fixed (n,), e_v1, e_v2, e_meas (m,8), fix_scale, points (k,3), point_ref (k,)).
        Returns dict(estimate, pose_cw (n,4,4), points (k,3), iterations, trials, chi2_init, chi2_final, lambda_init, lambda_final,
        envelope_doubles, factor_flops, launches, lin_ms, factor_ms, solve_ms, total_ms)."""
        G, keep = pack_pose_graph(graph)
        st = PgoStats()
        check(self._L.b200_graph_optimize(self._h, C.byref(G), self.max_iter_, self.gain_threshold_, C.byref(st)))
        out = dict(estimate=keep["estimate_out"], pose_cw=keep["pose_cw_out"], points=keep["points_out"])
        out.update({name: getattr(st, name) for name, _ in PgoStats._fields_})
        return out


# ---------------------------------------------------------------------------------------------------------------------------------
# optimize::transform_optimizer (optimize/transform_optimizer.{h,cc}): the Sim3 refinement of a loop candidate
# ---------------------------------------------------------------------------------------------------------------------------------
class TransformProblem(C.Structure):
    """b200_transform_problem_t (include/b200vslam.h)."""
    _fields_ = [("n_matches", C.c_int32), ("fix_scale", C.c_int32), ("sim3_12", Sim3), ("rot_1w", C.c_double * 9), ("trans_1w", C.c_double * 3),
                ("rot_2w", C.c_double * 9), ("trans_2w", C.c_double * 3), ("cam_1", Camera), ("cam_2", Camera), ("obs_1", C.c_void_p),
                ("inv_sigma_sq_1", C.c_void_p), ("pos_w_2", C.c_void_p), ("obs_2", C.c_void_p), ("inv_sigma_sq_2", C.c_void_p),
                ("pos_w_1", C.c_void_p), ("sim3_12_out", Sim3), ("keep", C.c_void_p), ("num_inliers", C.c_uint32),
                ("n_outliers_round1", C.c_int32), ("iterations", C.c_int32 * 2), ("trials", C.c_int32 * 2), ("chi2", C.c_double * 2),
                ("lambda_init", C.c_double * 2)]


def _camera(c):
    return Camera(int(c["model"]), *[float(c.get(k, 0.0)) for k in ("fx", "fy", "cx", "cy", "fxb", "cols", "rows")])


def gather_mutual_edges(keyfrm_1, keyfrm_2, matched_lms_in_keyfrm_2):
    """transform_optimizer::optimize step 3 (transform_optimizer.cc:58-94): the pairs that get a forward and a backward edge.

    keyfrm_1 / keyfrm_2: dict(id, rot_cw (3x3), trans_cw (3), camera (b200_camera_t fields), undist_keypts (n, 2), octaves (n,),
        inv_level_sigma_sq (per octave), landmarks (keyframe 1: get_landmarks(), a list of landmarks or None per keypoint)).
    A landmark: dict(pos_w (3), will_be_erased (bool), observations {keyframe id: keypoint index}).
    matched_lms_in_keyfrm_2: a landmark or None per keypoint of keyframe 1.
    Returns (problem dict in the layout of transform_optimizer.optimize without sim3_12, idx1 of every pair in ascending order)."""
    lms_1 = keyfrm_1["landmarks"]
    idx1s, idx2s, lm1s, lm2s = [], [], [], []
    for idx1, lm_2 in enumerate(matched_lms_in_keyfrm_2):
        if lm_2 is None:
            continue
        lm_1 = lms_1[idx1]
        if lm_1 is None:
            continue
        if lm_1.get("will_be_erased", False) or lm_2.get("will_be_erased", False):
            continue
        idx2 = lm_2.get("observations", {}).get(keyfrm_2["id"], -1)   # get_index_in_keyframe
        if idx2 < 0:
            continue
        idx1s.append(idx1)
        idx2s.append(idx2)
        lm1s.append(lm_1)
        lm2s.append(lm_2)

    def obs(kf, idx):
        kp = np.asarray(kf["undist_keypts"], np.float32).reshape(-1, 2)
        sig = np.asarray(kf["inv_level_sigma_sq"], np.float32)
        octv = np.asarray(kf["octaves"], np.int64)
        idx = np.asarray(idx, np.int64)
        return kp[idx].reshape(-1, 2), sig[octv[idx]]

    obs_1, w1 = obs(keyfrm_1, idx1s)
    obs_2, w2 = obs(keyfrm_2, idx2s)
    prob = dict(n_matches=len(idx1s), rot_1w=np.asarray(keyfrm_1["rot_cw"], np.float64), trans_1w=np.asarray(keyfrm_1["trans_cw"], np.float64),
                rot_2w=np.asarray(keyfrm_2["rot_cw"], np.float64), trans_2w=np.asarray(keyfrm_2["trans_cw"], np.float64),
                cam_1=keyfrm_1["camera"], cam_2=keyfrm_2["camera"], obs_1=obs_1, inv_sigma_sq_1=w1,
                pos_w_2=np.array([lm["pos_w"] for lm in lm2s], np.float64).reshape(-1, 3), obs_2=obs_2, inv_sigma_sq_2=w2,
                pos_w_1=np.array([lm["pos_w"] for lm in lm1s], np.float64).reshape(-1, 3))
    return prob, np.array(idx1s, np.int64)


def pack_transform_problem(problem, fix_scale):
    """problem dict -> (TransformProblem, keep-alive dict holding the keep output)."""
    keep = {}

    def arr(name, x, dt, shape):
        a = np.ascontiguousarray(np.asarray(x, dt).reshape(shape))
        keep[name] = a
        return a.ctypes.data

    n = len(problem["obs_1"])
    P = TransformProblem()
    P.n_matches, P.fix_scale = n, int(bool(fix_scale))
    s = np.asarray(problem["sim3_12"], np.float64).reshape(8)
    P.sim3_12 = Sim3((C.c_double * 4)(*s[:4]), (C.c_double * 3)(*s[4:7]), float(s[7]))
    P.rot_1w = (C.c_double * 9)(*np.asarray(problem["rot_1w"], np.float64).reshape(9))
    P.trans_1w = (C.c_double * 3)(*np.asarray(problem["trans_1w"], np.float64).reshape(3))
    P.rot_2w = (C.c_double * 9)(*np.asarray(problem["rot_2w"], np.float64).reshape(9))
    P.trans_2w = (C.c_double * 3)(*np.asarray(problem["trans_2w"], np.float64).reshape(3))
    P.cam_1, P.cam_2 = _camera(problem["cam_1"]), _camera(problem["cam_2"])
    P.obs_1 = arr("obs_1", problem["obs_1"], np.float32, (n, 2))
    P.inv_sigma_sq_1 = arr("inv_sigma_sq_1", problem["inv_sigma_sq_1"], np.float32, n)
    P.pos_w_2 = arr("pos_w_2", problem["pos_w_2"], np.float64, (n, 3))
    P.obs_2 = arr("obs_2", problem["obs_2"], np.float32, (n, 2))
    P.inv_sigma_sq_2 = arr("inv_sigma_sq_2", problem["inv_sigma_sq_2"], np.float32, n)
    P.pos_w_1 = arr("pos_w_1", problem["pos_w_1"], np.float64, (n, 3))
    keep["keep"] = np.zeros(max(n, 1), np.uint8)
    P.keep = keep["keep"].ctypes.data
    return P, keep


def _transform_result(P, keep):
    o = P.sim3_12_out
    return dict(sim3_12=np.array(list(o.q) + list(o.t) + [o.s]), keep=keep["keep"][:P.n_matches].copy(), num_inliers=int(P.num_inliers),
                n_outliers_round1=int(P.n_outliers_round1), iterations=list(P.iterations), trials=list(P.trials), chi2=list(P.chi2),
                lambda_init=list(P.lambda_init))


class transform_optimizer:
    """optimize::transform_optimizer (optimize/transform_optimizer.h:17-48): the Sim3 refinement of loop candidates on the GPU, one
    launch for a whole batch.  gather_mutual_edges() restates how the reference picks the pairs; optimize() runs the rest of
    transform_optimizer::optimize on them."""

    def __init__(self, fix_scale, num_iter=10, device=0):
        self.fix_scale_, self.num_iter_ = bool(fix_scale), int(num_iter)
        self._L = _bind()
        self._h = C.c_void_p()
        check(self._L.b200_lba_create(device, C.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None):
            self._L.b200_lba_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def optimize_batch(self, problems, chi_sq=10.0):
        """problems: dicts (workloads.synth.make_sim3_pair layout; sim3_12 is the initial Sim3_12 as an 8-vector q x y z w, t, s).
        Returns per problem dict(sim3_12: the refined Sim3_12, or the input when the second round did not run; keep (n,) uint8: 1 where
        the entry stays in matched_lms_in_keyfrm_2; num_inliers: the return value; n_outliers_round1, iterations, trials, chi2,
        lambda_init)."""
        if not problems:
            return []
        packed = [pack_transform_problem(pr, self.fix_scale_) for pr in problems]
        arr = (TransformProblem * len(packed))(*[pk[0] for pk in packed])
        check(self._L.b200_transform_optimize(self._h, len(packed), arr, float(chi_sq), self.num_iter_))
        return [_transform_result(arr[i], pk[1]) for i, pk in enumerate(packed)]

    def optimize(self, problem, chi_sq=10.0):
        return self.optimize_batch([problem], chi_sq)[0]
