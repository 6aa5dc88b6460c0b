"""Host-side mirrors of initialize::perspective and initialize::bearing_vector (src/stella_vslam/initialize/{base,perspective,
bearing_vector}.{h,cc}): monocular map initialisation on the device (b200_initialize on a b200_lba_t handle).  One call runs, for every
frame pair, the RANSAC of the H and F solvers (perspective, fisheye and radial-division cameras) or of the E solver (equirectangular),
the rel_cost_H choice, the decomposition of the chosen model, the triangulation of every pose hypothesis and
find_most_plausible_pose.  The minimal sets are drawn on the host from each solver's own engine (solve.draw_min_sets).

A frame is a dict: camera (a camera dict as _lib.camera_intrinsics takes it), img_bounds ((min_x, max_x, min_y, max_y); unused by
equirectangular cameras), undist_keypts ((n, 2) pixels) and bearings ((n, 3)).
"""
import ctypes as C

import numpy as np

from . import solve
from ._lib import CAMERA_MODELS, CameraIntrinsics, camera_intrinsics, check

MODEL_NONE, MODEL_H, MODEL_F, MODEL_E = 0, 1, 2, 3
MODEL_NAMES = {MODEL_NONE: None, MODEL_H: "H", MODEL_F: "F", MODEL_E: "E"}
STAGE_NO_MODEL, STAGE_DECOMPOSE, STAGE_MIN_VALID, STAGE_AMBIGUOUS, STAGE_PARALLAX, STAGE_MIN_TRIANGULATED, STAGE_SUCCEEDED = range(7)

# module/initializer.cc's defaults
DEFAULTS = dict(num_ransac_iters=100, min_num_triangulated=50, min_num_valid_pts=50, parallax_deg_thr=1.0, reproj_err_thr=4.0)


class InitProblem(C.Structure):
    """b200_init_problem_t (include/b200vslam.h)."""
    _fields_ = [("cam_ref", CameraIntrinsics), ("cam_cur", CameraIntrinsics), ("img_bounds_ref", C.c_float * 4), ("img_bounds_cur", C.c_float * 4),
                ("n_ref", C.c_int32), ("n_cur", C.c_int32), ("undist_ref", C.c_void_p), ("bearings_ref", C.c_void_p), ("undist_cur", C.c_void_p),
                ("bearings_cur", C.c_void_p), ("ref_matches_with_cur", C.c_void_p), ("num_ransac_iters", C.c_uint32),
                ("min_num_triangulated", C.c_uint32), ("min_num_valid_pts", C.c_uint32), ("parallax_deg_thr", C.c_float),
                ("reproj_err_thr", C.c_float), ("min_sets_H", C.c_void_p), ("min_sets_F", C.c_void_p), ("min_sets_E", C.c_void_p),
                ("status", C.c_int32), ("succeeded", C.c_int32), ("model", C.c_int32), ("stage", C.c_int32), ("n_matches", C.c_int32),
                ("cost_H", C.c_float), ("cost_F", C.c_float), ("cost_E", C.c_float), ("valid_H", C.c_int32), ("valid_F", C.c_int32),
                ("valid_E", C.c_int32), ("num_inliers_H", C.c_int32), ("num_inliers_F", C.c_int32), ("num_inliers_E", C.c_int32),
                ("n_hypotheses", C.c_int32), ("nums_valid", C.c_int32 * 8), ("num_triangulated", C.c_int32 * 8), ("parallax_cos", C.c_float * 8),
                ("rot_ref_to_cur", C.c_double * 9), ("trans_ref_to_cur", C.c_double * 3), ("triangulated_pts", C.c_void_p),
                ("triangulated_flags", C.c_void_p), ("inlier_flags", C.c_void_p)]


def _L():
    L = solve._L()
    if not getattr(L, "_init_bound", False):
        L.b200_initialize.argtypes = [C.c_void_p, C.c_int, C.POINTER(InitProblem)]
        L._init_bound = True
    return L


def _arr(a, dtype, cols):
    return np.ascontiguousarray(np.asarray(a, dtype).reshape(-1, cols))


def _pack(prob, keep):
    S = InitProblem()
    S.cam_ref, S.cam_cur = camera_intrinsics(prob["cam_ref"]), camera_intrinsics(prob["cam_cur"])
    S.img_bounds_ref[:] = [float(v) for v in prob.get("bounds_ref", (0.0, 0.0, 0.0, 0.0))]
    S.img_bounds_cur[:] = [float(v) for v in prob.get("bounds_cur", (0.0, 0.0, 0.0, 0.0))]
    ur, br = _arr(prob["undist_ref"], np.float32, 2), _arr(prob["bearings_ref"], np.float64, 3)
    uc, bc = _arr(prob["undist_cur"], np.float32, 2), _arr(prob["bearings_cur"], np.float64, 3)
    if len(ur) != len(br) or len(uc) != len(bc):
        raise ValueError("each frame needs one bearing per undistorted keypoint")
    m = np.ascontiguousarray(np.asarray(prob["ref_matches_with_cur"], np.int32).reshape(-1))
    if len(m) != len(ur):
        raise ValueError("ref_matches_with_cur needs one entry per ref keypoint")
    n_ref = len(ur)
    pts, tri, inl = np.zeros((max(n_ref, 1), 3)), np.zeros(max(n_ref, 1), np.uint8), np.zeros(max(n_ref, 1), np.uint8)
    sets = {}
    for k, size in (("H", 4), ("F", 8), ("E", 5)):
        v = prob.get("min_sets_" + k)
        sets[k] = None if v is None else _arr(v, np.int32, size)
    keep += [ur, br, uc, bc, m, pts, tri, inl] + [v for v in sets.values() if v is not None]
    S.n_ref, S.n_cur = n_ref, len(uc)
    S.undist_ref, S.bearings_ref, S.undist_cur, S.bearings_cur = ur.ctypes.data, br.ctypes.data, uc.ctypes.data, bc.ctypes.data
    S.ref_matches_with_cur = m.ctypes.data
    for k in DEFAULTS:
        setattr(S, k, prob.get(k, DEFAULTS[k]))
    S.min_sets_H, S.min_sets_F, S.min_sets_E = [None if sets[k] is None else sets[k].ctypes.data for k in ("H", "F", "E")]
    S.triangulated_pts, S.triangulated_flags, S.inlier_flags = pts.ctypes.data, tri.ctypes.data, inl.ctypes.data
    return S, (pts, tri, inl)


def _result(S, bufs):
    pts, tri, inl = bufs
    nh = S.n_hypotheses
    return dict(status=S.status, succeeded=bool(S.succeeded), model=MODEL_NAMES[S.model], stage=S.stage, n_matches=S.n_matches,
                cost_H=np.float32(S.cost_H), cost_F=np.float32(S.cost_F), cost_E=np.float32(S.cost_E), valid_H=bool(S.valid_H),
                valid_F=bool(S.valid_F), valid_E=bool(S.valid_E), num_inliers_H=S.num_inliers_H, num_inliers_F=S.num_inliers_F,
                num_inliers_E=S.num_inliers_E, n_hypotheses=nh, nums_valid=np.array(S.nums_valid[:nh], np.int32),
                num_triangulated=np.array(S.num_triangulated[:nh], np.int32), parallax_cos=np.array(S.parallax_cos[:nh], np.float32),
                rot_ref_to_cur=np.array(S.rot_ref_to_cur).reshape(3, 3) if nh else None,
                trans_ref_to_cur=np.array(S.trans_ref_to_cur) if nh else None,
                triangulated_pts=pts[:S.n_ref].copy() if S.succeeded else None,
                triangulated_flags=tri[:S.n_ref].astype(bool) if S.succeeded else None,
                inlier_flags=inl[:S.n_matches].astype(bool) if S.model != MODEL_NONE else None)


def initialize_batch(problems, device=0):
    """b200_initialize over dicts(cam_ref, cam_cur (camera dicts), bounds_ref, bounds_cur, undist_ref, bearings_ref, undist_cur,
    bearings_cur, ref_matches_with_cur, min_sets_H and min_sets_F (perspective cameras) or min_sets_E (equirectangular), and the
    parameters of DEFAULTS).  Returns per problem dict(status, succeeded, model ("H", "F", "E" or None), stage (STAGE_*), n_matches,
    cost_* / valid_* / num_inliers_* of the solvers, n_hypotheses, nums_valid / num_triangulated / parallax_cos per hypothesis,
    rot_ref_to_cur / trans_ref_to_cur (None when find_most_plausible_pose did not run; zeros when it rejected), triangulated_pts /
    triangulated_flags per ref keypoint (None unless succeeded), inlier_flags (the chosen solver's, None when no model was chosen))."""
    keep, bufs = [], []
    arr = (InitProblem * max(len(problems), 1))()
    for i, pr in enumerate(problems):
        arr[i], b = _pack(pr, keep)
        bufs.append(b)
    check(_L().b200_initialize(solve._handle(device), len(problems), arr))
    return [_result(S, b) for S, b in zip(arr[:len(problems)], bufs)]


def draw_min_sets(n_matches, num_ransac_iters, bearing, use_fixed_seed=False):
    """The minimal sets one initialize() call draws: each solver is constructed per attempt with its own engine (util::create_random_engine)
    and draws only when its RANSAC runs (8 matches for H and F, 5 for E).  Returns a dict of min_sets_H / min_sets_F or min_sets_E."""
    if bearing:
        return {"min_sets_E": solve.draw_min_sets(n_matches, num_ransac_iters, solve._random_engine(use_fixed_seed), set_size=5)
                if n_matches >= 5 else None}
    if n_matches < 8:
        return {"min_sets_H": None, "min_sets_F": None}
    return {"min_sets_H": solve.draw_min_sets(n_matches, num_ransac_iters, solve._random_engine(use_fixed_seed), set_size=4),
            "min_sets_F": solve.draw_min_sets(n_matches, num_ransac_iters, solve._random_engine(use_fixed_seed), set_size=8)}


class base:
    """initialize::base: the reference frame, the parameters, and the members find_most_plausible_pose leaves behind.  A Jacobi SVD
    or RealSchur that hits its bound does not raise, as the reference returns normally: status() is then B200_ERR_INVALID."""

    _bearing = False

    def __init__(self, ref_frm, num_ransac_iters=100, min_num_triangulated=50, min_num_valid_pts=50, parallax_deg_thr=1.0, reproj_err_thr=4.0,
                 use_fixed_seed=False, device=0):
        is_equirect = CAMERA_MODELS[ref_frm["camera"].get("model", "perspective")] == 1
        if is_equirect != self._bearing:
            raise ValueError(f"{type(self).__name__} does not take a {ref_frm['camera'].get('model', 'perspective')} camera")
        self.ref_frm_ = ref_frm
        self.params_ = dict(num_ransac_iters=int(num_ransac_iters), min_num_triangulated=int(min_num_triangulated),
                            min_num_valid_pts=int(min_num_valid_pts), parallax_deg_thr=float(parallax_deg_thr), reproj_err_thr=float(reproj_err_thr))
        self.use_fixed_seed_ = use_fixed_seed
        self.device = device
        self.rot_ref_to_cur_ = np.eye(3)  # base.h: Mat33_t::Identity()
        self.trans_ref_to_cur_ = np.zeros(3)
        self.triangulated_pts_ = np.zeros((0, 3))
        self.is_triangulated_ = []
        self.last_result_ = None
        self.status_ = 0

    def initialize(self, cur_frm, ref_matches_with_cur):
        """initialize(cur_frm, ref_matches_with_cur): True when a map could be initialised."""
        m = np.asarray(ref_matches_with_cur, np.int32).reshape(-1)
        r, f = self.ref_frm_, cur_frm
        prob = dict(cam_ref=r["camera"], cam_cur=f["camera"], bounds_ref=r.get("img_bounds", (0.0, 0.0, 0.0, 0.0)),
                    bounds_cur=f.get("img_bounds", (0.0, 0.0, 0.0, 0.0)), undist_ref=r["undist_keypts"], bearings_ref=r["bearings"],
                    undist_cur=f["undist_keypts"], bearings_cur=f["bearings"], ref_matches_with_cur=m, **self.params_,
                    **draw_min_sets(int((m >= 0).sum()), self.params_["num_ransac_iters"], self._bearing, self.use_fixed_seed_))
        res = initialize_batch([prob], self.device)[0]
        self.status_ = res["status"]
        self.last_result_ = res
        if res["rot_ref_to_cur"] is not None:
            self.rot_ref_to_cur_, self.trans_ref_to_cur_ = res["rot_ref_to_cur"], res["trans_ref_to_cur"]
        if res["succeeded"]:
            self.triangulated_pts_, self.is_triangulated_ = res["triangulated_pts"], [bool(v) for v in res["triangulated_flags"]]
        return res["succeeded"]

    def status(self):
        """B200_OK, or B200_ERR_INVALID when a Jacobi sweep or RealSchur of the last initialize() hit its bound."""
        return self.status_

    def get_rotation_ref_to_cur(self):
        return self.rot_ref_to_cur_.copy()

    def get_translation_ref_to_cur(self):
        return self.trans_ref_to_cur_.copy()

    def get_triangulated_pts(self):
        return self.triangulated_pts_.copy()

    def get_triangulated_flags(self):
        return list(self.is_triangulated_)


class perspective(base):
    """initialize::perspective: H and F RANSAC, reconstruction with the model rel_cost_H picks (perspective, fisheye and radial-division
    cameras)."""


class bearing_vector(base):
    """initialize::bearing_vector: E RANSAC and its reconstruction (equirectangular cameras)."""
    _bearing = True
