"""Host-side mirrors of solve::pnp_solver (src/stella_vslam/solve/pnp_solver.{h,cc}): EPnP inside RANSAC on the device
(b200_pnp_ransac / b200_epnp_compute_pose on a b200_lba_t handle), with the minimal sets drawn on the host exactly as
util::create_random_array draws them from the solver's std::mt19937 (b200_draw_min_sets).

Arrays: bearings and points are (n, 3) float64, octaves (n,) int, scale_factors the ORB pyramid's float32 scale factors.

And of solve::essential_solver (src/stella_vslam/solve/essential_solver.{h,cc}): the five-point minimal solver inside RANSAC on the
device (b200_essential_ransac), the minimal sets drawn on the host by util::create_random_array(5, ...) (b200_draw_min_sets).

And of solve::homography_solver and solve::fundamental_solver (homography_solver.{h,cc}, fundamental_solver.{h,cc}), monocular
initialisation's two RANSAC solvers, H and F problems together in one call (b200_twoview_ransac), the minimal sets of 4 and 8 drawn
by b200_draw_min_sets.
"""
import ctypes as C

import numpy as np

from ._lib import check, lib


class PnpProblem(C.Structure):
    """b200_pnp_problem_t (include/b200vslam.h)."""
    _fields_ = [("n_matches", C.c_int32), ("bearings", C.c_void_p), ("points", C.c_void_p), ("octaves", C.c_void_p),
                ("num_levels", C.c_int32), ("scale_factors", C.c_void_p), ("min_num_inliers", C.c_uint32),
                ("gauss_newton_num_iter", C.c_uint32), ("max_num_iter", C.c_uint32), ("recompute", C.c_int32), ("min_sets", C.c_void_p),
                ("status", C.c_int32), ("valid", C.c_int32), ("best_iter", C.c_int32), ("num_inliers", C.c_int32),
                ("min_cost", C.c_double), ("rot_cw", C.c_double * 9), ("trans_cw", C.c_double * 3), ("inlier_flags", C.c_void_p)]


class EpnpProblem(C.Structure):
    """b200_epnp_problem_t (include/b200vslam.h)."""
    _fields_ = [("n", C.c_int32), ("bearings", C.c_void_p), ("points", C.c_void_p), ("num_iter", C.c_uint32),
                ("rot_cw", C.c_double * 9), ("trans_cw", C.c_double * 3), ("reproj_error", C.c_double), ("wrote", C.c_int32),
                ("status", C.c_int32)]


class EssentialProblem(C.Structure):
    """b200_essential_problem_t (include/b200vslam.h)."""
    _fields_ = [("n_matches", C.c_int32), ("bearings_1", C.c_void_p), ("bearings_2", C.c_void_p), ("min_set_size", C.c_uint32),
                ("max_num_iter", C.c_uint32), ("recompute", C.c_int32), ("min_sets", C.c_void_p),
                ("status", C.c_int32), ("valid", C.c_int32), ("best_iter", C.c_int32), ("best_candidate", C.c_int32),
                ("num_inliers", C.c_int32), ("best_cost", C.c_float), ("E_21", C.c_double * 9), ("inlier_flags", C.c_void_p)]


class Mt19937(C.Structure):
    """b200_mt19937_t: std::mt19937's state."""
    _fields_ = [("state", C.c_uint32 * 624), ("index", C.c_uint32)]


def _L():
    L = lib()
    if not getattr(L, "_pnp_bound", False):
        vp = C.c_void_p
        L.b200_lba_create.argtypes = [C.c_int, C.POINTER(vp)]
        L.b200_pnp_ransac.argtypes = [vp, C.c_int, C.POINTER(PnpProblem)]
        L.b200_epnp_compute_pose.argtypes = [vp, C.c_int, C.POINTER(EpnpProblem)]
        L.b200_mt19937_seed.argtypes = [C.POINTER(Mt19937), C.POINTER(C.c_uint32), C.c_int]
        L.b200_mt19937_next.argtypes = [C.POINTER(Mt19937)]
        L.b200_mt19937_next.restype = C.c_uint32
        L.b200_draw_min_sets.argtypes = [C.POINTER(Mt19937), C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_int32)]
        L.b200_draw_min_sets_batch.argtypes = [vp, C.c_int, C.POINTER(Mt19937), C.c_uint32, C.POINTER(C.c_uint32), C.c_uint32, C.POINTER(C.c_int32)]
        L.b200_essential_ransac.argtypes = [vp, C.c_int, C.POINTER(EssentialProblem)]
        L.b200_twoview_ransac.argtypes = [vp, C.c_int, C.POINTER(TwoviewProblem)]
        L._pnp_bound = True
    return L


_HANDLES = {}


def _handle(device=0):
    """One b200_lba_t per device for the PnP entry points (the handle of optimize.pose_optimizer serves as well)."""
    if device not in _HANDLES:
        h = C.c_void_p()
        check(_L().b200_lba_create(device, C.byref(h)))
        _HANDLES[device] = h
    return _HANDLES[device]


def mt19937(seed_seq=None):
    """A std::mt19937: default-constructed (seed 5489) when seed_seq is None or empty, else seeded by std::seed_seq over the words."""
    e = Mt19937()
    words = np.ascontiguousarray(np.asarray([] if seed_seq is None else seed_seq, np.uint32))
    check(_L().b200_mt19937_seed(C.byref(e), words.ctypes.data_as(C.POINTER(C.c_uint32)) if len(words) else None, len(words)))
    return e


def _random_engine(use_fixed_seed):
    """util::create_random_engine: a default-constructed engine, or one seeded by std::seed_seq over ten std::random_device words."""
    return mt19937(None if use_fixed_seed else np.frombuffer(np.random.bytes(40), np.uint32))


def draw_min_sets(n_matches, max_num_iter, engine=None, set_size=4):
    """max_num_iter calls of util::create_random_array(set_size, 0, n_matches - 1, engine), (max_num_iter, set_size) int32.  engine: an
    Mt19937 (advanced in place) or None for a default-constructed one.  set_size 4 is PnP's minimal set, 5 the essential solver's."""
    e = mt19937() if engine is None else engine
    k = int(set_size)
    out = np.zeros((max(int(max_num_iter), 1), max(k, 1)), np.int32)
    check(_L().b200_draw_min_sets(C.byref(e), k, int(n_matches), int(max_num_iter), out.ctypes.data_as(C.POINTER(C.c_int32))))
    return out[:int(max_num_iter)]


def draw_min_sets_batch(n_matches, max_num_iter, engines=None, set_size=5, device=0):
    """The device sampler (b200_draw_min_sets_batch): engine p (engines None: default-constructed ones) draws max_num_iter minimal sets
    from n_matches[p] matches, (len(n_matches), max_num_iter, set_size) int32.  The engines are not advanced."""
    nm = np.ascontiguousarray(np.asarray(n_matches, np.uint32).reshape(-1))
    n = len(nm)
    k, it = int(set_size), int(max_num_iter)
    arr = None
    if engines is not None:
        arr = (Mt19937 * max(n, 1))()
        for i, e in enumerate(engines):
            arr[i] = e
    out = np.zeros((max(n, 1), max(it, 1), max(k, 1)), np.int32)
    check(_L().b200_draw_min_sets_batch(_handle(device), n, arr, k, nm.ctypes.data_as(C.POINTER(C.c_uint32)), it,
                                        out.ctypes.data_as(C.POINTER(C.c_int32))))
    return out[:n, :it, :k]


def _run_batch(entry, StructT, pack, problems, device):
    """Packs each problem dict into a StructT with pack(problem, keep) -> (struct, inlier flag buffer), then calls the entry point named
    entry on the batch.  Returns the filled structs and the flag buffers, one per problem."""
    keep, flags = [], []
    arr = (StructT * max(len(problems), 1))()
    for i, pr in enumerate(problems):
        arr[i], fl = pack(pr, keep)
        flags.append(fl)
    check(getattr(_L(), entry)(_handle(device), len(problems), arr))
    return arr[:len(problems)], flags


class _ransac_solver:
    """What the RANSAC solvers share: the engine is the solver's member, so find_via_ransac continues its state across calls; the
    validity, status and inlier flags of the last call."""

    def __init__(self, use_fixed_seed, device):
        self.device = device
        self.random_engine_ = _random_engine(use_fixed_seed)
        self.solution_is_valid_ = False
        self.is_inlier_match_ = []
        self.status_ = 0

    def _find_via_ransac(self, early_return, max_num_iter, set_size, batch, problem):
        """Returns before any draw when early_return (None), else draws the minimal sets from the engine, solves the one problem with
        batch and returns its result dict."""
        if early_return:
            self.solution_is_valid_ = False
            return None
        ms = draw_min_sets(self.num_matches_, max_num_iter, self.random_engine_, set_size=set_size)
        r = batch([dict(problem, min_sets=ms)], self.device)[0]
        self.status_ = r["status"]
        self.solution_is_valid_ = r["valid"]
        self.is_inlier_match_ = [bool(v) for v in r["inlier_flags"]]
        return r

    def solution_is_valid(self):
        return self.solution_is_valid_


def _pack(prob, keep):
    S = PnpProblem()
    b = np.ascontiguousarray(np.asarray(prob["bearings"], np.float64).reshape(-1, 3))
    p = np.ascontiguousarray(np.asarray(prob["points"], np.float64).reshape(-1, 3))
    o = np.ascontiguousarray(np.asarray(prob["octaves"], np.int32).reshape(-1))
    sf = np.ascontiguousarray(np.asarray(prob["scale_factors"], np.float32).reshape(-1))
    ms = np.ascontiguousarray(np.asarray(prob.get("min_sets", np.zeros((0, 4))), np.int32).reshape(-1, 4))
    fl = np.zeros(max(len(b), 1), np.uint8)
    keep += [b, p, o, sf, ms, fl]
    S.n_matches = len(b)
    S.bearings, S.points, S.octaves = b.ctypes.data, p.ctypes.data, o.ctypes.data
    S.num_levels, S.scale_factors = len(sf), sf.ctypes.data
    S.min_num_inliers = int(prob.get("min_num_inliers", 10))
    S.gauss_newton_num_iter = int(prob.get("gauss_newton_num_iter", 10))
    S.max_num_iter = len(ms)
    S.recompute = int(bool(prob.get("recompute", True)))
    S.min_sets = ms.ctypes.data
    S.inlier_flags = fl.ctypes.data
    return S, fl


def pnp_ransac_batch(problems, device=0):
    """b200_pnp_ransac over dicts(bearings, points, octaves, scale_factors, min_sets (max_num_iter x 4), min_num_inliers=10,
    gauss_newton_num_iter=10, recompute=True).  Returns per problem dict(status, valid, best_iter, num_inliers, min_cost, rot_cw, trans_cw,
    inlier_flags (None on the early return)); rot_cw / trans_cw are None unless valid."""
    arr, flags = _run_batch("b200_pnp_ransac", PnpProblem, _pack, problems, device)
    out = []
    for S, fl in zip(arr, flags):
        n = S.n_matches
        early = n < 4 or n < S.min_num_inliers
        out.append(dict(status=S.status, valid=bool(S.valid), best_iter=S.best_iter, num_inliers=S.num_inliers, min_cost=S.min_cost,
                        rot_cw=np.array(S.rot_cw).reshape(3, 3) if S.valid else None, trans_cw=np.array(S.trans_cw) if S.valid else None,
                        inlier_flags=None if early else fl[:n].astype(bool)))
    return out


def compute_pose_batch(problems, device=0):
    """b200_epnp_compute_pose over dicts(bearings, points, num_iter=5, rot_cw=None, trans_cw=None).  Returns per problem
    dict(rot_cw, trans_cw, reproj_error, wrote, status); rot_cw / trans_cw are the given ones (zeros if None) when nothing was written."""
    keep = []
    arr = (EpnpProblem * max(len(problems), 1))()
    for i, pr in enumerate(problems):
        b = np.ascontiguousarray(np.asarray(pr["bearings"], np.float64).reshape(-1, 3))
        p = np.ascontiguousarray(np.asarray(pr["points"], np.float64).reshape(-1, 3))
        keep += [b, p]
        S = arr[i]
        S.n, S.bearings, S.points, S.num_iter = len(b), b.ctypes.data, p.ctypes.data, int(pr.get("num_iter", 5))
        S.rot_cw[:] = [float(v) for v in np.asarray(pr["rot_cw"] if pr.get("rot_cw") is not None else np.zeros(9), np.float64).reshape(9)]
        S.trans_cw[:] = [float(v) for v in np.asarray(pr["trans_cw"] if pr.get("trans_cw") is not None else np.zeros(3), np.float64).reshape(3)]
    check(_L().b200_epnp_compute_pose(_handle(device), len(problems), arr))
    return [dict(rot_cw=np.array(arr[i].rot_cw).reshape(3, 3), trans_cw=np.array(arr[i].trans_cw), reproj_error=arr[i].reproj_error,
                 wrote=bool(arr[i].wrote), status=arr[i].status) for i in range(len(problems))]


class pnp_solver(_ransac_solver):
    """solve::pnp_solver.  The engine is the solver's member: find_via_ransac continues its state across calls."""

    def __init__(self, valid_bearings, octaves, valid_points, scale_factors, min_num_inliers=10, use_fixed_seed=False,
                 gauss_newton_num_iter=10, device=0):
        self.bearings_ = np.ascontiguousarray(np.asarray(valid_bearings, np.float64).reshape(-1, 3))
        self.points_ = np.ascontiguousarray(np.asarray(valid_points, np.float64).reshape(-1, 3))
        self.octaves_ = np.asarray(octaves, np.int32).reshape(-1)
        self.scale_factors_ = np.asarray(scale_factors, np.float32).reshape(-1)
        n = len(self.bearings_)
        if len(self.points_) != n or len(self.octaves_) != n:
            raise ValueError("bearings, octaves and points must have one entry per match")
        if n and (self.octaves_.min() < 0 or self.octaves_.max() >= len(self.scale_factors_)):
            raise IndexError("octave outside the scale factors")  # std::vector::at throws in the reference
        super().__init__(use_fixed_seed, device)
        self.num_matches_ = n
        self.min_num_inliers_ = int(min_num_inliers)
        self.gauss_newton_num_iter_ = int(gauss_newton_num_iter)
        self.best_rot_cw_ = np.zeros((3, 3))
        self.best_trans_cw_ = np.zeros(3)

    def find_via_ransac(self, max_num_iter, recompute=True):
        n = self.num_matches_
        r = self._find_via_ransac(n < 4 or n < self.min_num_inliers_, max_num_iter, 4, pnp_ransac_batch,
                                  dict(bearings=self.bearings_, points=self.points_, octaves=self.octaves_, scale_factors=self.scale_factors_,
                                       min_num_inliers=self.min_num_inliers_, gauss_newton_num_iter=self.gauss_newton_num_iter_,
                                       recompute=recompute))
        if r is not None and r["valid"]:
            self.best_rot_cw_, self.best_trans_cw_ = r["rot_cw"], r["trans_cw"]

    def get_best_rotation(self):
        return self.best_rot_cw_.copy()

    def get_best_translation(self):
        return self.best_trans_cw_.copy()

    def get_best_cam_pose(self):
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = self.best_rot_cw_, self.best_trans_cw_
        return T

    def get_inlier_flags(self):
        return list(self.is_inlier_match_)

    @staticmethod
    def compute_pose(bearing_vectors, pos_ws, rot_cw=None, trans_cw=None, num_iter=5, device=0):
        """Returns (reproj_error, rot_cw, trans_cw); the given rot_cw / trans_cw come back unchanged when no candidate was written."""
        r = compute_pose_batch([dict(bearings=bearing_vectors, points=pos_ws, num_iter=num_iter, rot_cw=rot_cw, trans_cw=trans_cw)], device)[0]
        check(r["status"])
        return r["reproj_error"], r["rot_cw"], r["trans_cw"]


def _pack_essential(prob, keep):
    S = EssentialProblem()
    b1 = np.ascontiguousarray(np.asarray(prob["bearings_1"], np.float64).reshape(-1, 3))
    b2 = np.ascontiguousarray(np.asarray(prob["bearings_2"], np.float64).reshape(-1, 3))
    if len(b1) != len(b2):
        raise ValueError("bearings_1 and bearings_2 must have one row per match")
    k = int(prob.get("min_set_size", 5))
    ms = np.ascontiguousarray(np.asarray(prob.get("min_sets", np.zeros((0, k))), np.int32).reshape(-1, max(k, 1)))
    fl = np.zeros(max(len(b1), 1), np.uint8)
    keep += [b1, b2, ms, fl]
    S.n_matches = len(b1)
    S.bearings_1, S.bearings_2 = b1.ctypes.data, b2.ctypes.data
    S.min_set_size = k
    S.max_num_iter = len(ms)
    S.recompute = int(bool(prob.get("recompute", True)))
    S.min_sets = ms.ctypes.data
    S.inlier_flags = fl.ctypes.data
    return S, fl


def essential_ransac_batch(problems, device=0):
    """b200_essential_ransac over dicts(bearings_1, bearings_2 (n x 3, gathered through matches_12), min_sets (max_num_iter x 5),
    recompute=True, min_set_size=5).  Returns per problem dict(status, valid, best_iter, best_candidate, num_inliers, best_cost (float32),
    E_21 (None unless valid), inlier_flags (None on the early return))."""
    arr, flags = _run_batch("b200_essential_ransac", EssentialProblem, _pack_essential, problems, device)
    return [dict(status=S.status, valid=bool(S.valid), best_iter=S.best_iter, best_candidate=S.best_candidate, num_inliers=S.num_inliers,
                 best_cost=np.float32(S.best_cost), E_21=np.array(S.E_21).reshape(3, 3) if S.valid else None,
                 inlier_flags=None if S.n_matches < S.min_set_size else fl[:S.n_matches].astype(bool)) for S, fl in zip(arr, flags)]


class essential_solver(_ransac_solver):
    """solve::essential_solver.  matches_12: (first, second) index pairs into bearings_1 / bearings_2.  The engine is the solver's
    member: find_via_ransac continues its state across calls."""

    def __init__(self, bearings_1, bearings_2, matches_12, use_fixed_seed=False, device=0):
        b1 = np.asarray(bearings_1, np.float64).reshape(-1, 3)
        b2 = np.asarray(bearings_2, np.float64).reshape(-1, 3)
        m = np.asarray(matches_12, np.int64).reshape(-1, 2)
        if len(m) and (m.min() < 0 or m[:, 0].max() >= len(b1) or m[:, 1].max() >= len(b2)):
            raise IndexError("match index outside the bearings")  # std::vector::at throws in the reference
        super().__init__(use_fixed_seed, device)
        self.bearings_1_ = np.ascontiguousarray(b1[m[:, 0]])
        self.bearings_2_ = np.ascontiguousarray(b2[m[:, 1]])
        self.num_matches_ = len(m)
        self.best_cost_ = np.float32(0.0)
        self.best_E_21_ = np.zeros((3, 3))

    def find_via_ransac(self, max_num_iter, recompute=True, min_set_size=5):
        if int(min_set_size) != 5:
            raise ValueError("essential_solver: only the five-point minimal set (min_set_size = 5) is supported")
        r = self._find_via_ransac(self.num_matches_ < min_set_size, max_num_iter, 5, essential_ransac_batch,
                                  dict(bearings_1=self.bearings_1_, bearings_2=self.bearings_2_, recompute=recompute))
        if r is not None:
            self.best_cost_ = r["best_cost"]
            if r["valid"]:
                self.best_E_21_ = r["E_21"]

    def get_best_cost(self):
        return self.best_cost_

    def get_best_E_21(self):
        return self.best_E_21_.copy()

    def get_inlier_matches(self):
        return list(self.is_inlier_match_)


# ---- solve::homography_solver / solve::fundamental_solver (src/stella_vslam/solve/homography_solver.cc, fundamental_solver.cc) ----

MODEL_H, MODEL_F = 0, 1
_SET_SIZE = {MODEL_H: 4, MODEL_F: 8}


class TwoviewProblem(C.Structure):
    """b200_twoview_problem_t (include/b200vslam.h)."""
    _fields_ = [("model", C.c_int32), ("n_keypts_1", C.c_int32), ("keypts_1", C.c_void_p), ("n_keypts_2", C.c_int32),
                ("keypts_2", C.c_void_p), ("n_matches", C.c_int32), ("matches_12", C.c_void_p), ("sigma", C.c_float),
                ("max_num_iter", C.c_uint32), ("recompute", C.c_int32), ("min_sets", C.c_void_p),
                ("status", C.c_int32), ("valid", C.c_int32), ("best_iter", C.c_int32), ("num_inliers", C.c_int32),
                ("best_cost", C.c_float), ("M_21", C.c_double * 9), ("inlier_flags", C.c_void_p)]


def _model_id(model):
    m = {"H": MODEL_H, "F": MODEL_F, MODEL_H: MODEL_H, MODEL_F: MODEL_F}.get(model)
    if m is None:
        raise ValueError(f"two-view model must be 'H' or 'F', not {model!r}")
    return m


def _keypts(k):
    """(n, 2) float32 pixel coordinates: an array, or a sequence of objects with .pt / (x, y) pairs."""
    return np.ascontiguousarray(np.asarray(k, np.float32).reshape(-1, 2))


def _pack_twoview(prob, keep):
    S = TwoviewProblem()
    m = _model_id(prob["model"])
    k1, k2 = _keypts(prob["keypts_1"]), _keypts(prob["keypts_2"])
    mt = np.ascontiguousarray(np.asarray(prob["matches_12"], np.int32).reshape(-1, 2))
    k = _SET_SIZE[m]
    ms = np.ascontiguousarray(np.asarray(prob.get("min_sets", np.zeros((0, k))), np.int32).reshape(-1, k))
    fl = np.zeros(max(len(mt), 1), np.uint8)
    keep += [k1, k2, mt, ms, fl]
    S.model = m
    S.n_keypts_1, S.keypts_1 = len(k1), k1.ctypes.data
    S.n_keypts_2, S.keypts_2 = len(k2), k2.ctypes.data
    S.n_matches, S.matches_12 = len(mt), mt.ctypes.data
    S.sigma = float(prob.get("sigma", 1.0))
    S.max_num_iter = len(ms)
    S.recompute = int(bool(prob.get("recompute", True)))
    S.min_sets = ms.ctypes.data
    S.inlier_flags = fl.ctypes.data
    return S, fl


def twoview_ransac_batch(problems, device=0):
    """b200_twoview_ransac over dicts(model ("H" or "F"), keypts_1, keypts_2 (all undistorted keypoints of each frame, (n, 2) pixels),
    matches_12 ((n, 2) keypoint index pairs), min_sets (max_num_iter x 4 for H, x 8 for F), sigma=1.0, recompute=True).  H and F
    problems mix freely in one call.  Returns per problem dict(status, valid, best_iter, num_inliers, best_cost (float32), M_21 (None
    unless valid), inlier_flags (None on the early return, n < 8))."""
    arr, flags = _run_batch("b200_twoview_ransac", TwoviewProblem, _pack_twoview, problems, device)
    return [dict(status=S.status, valid=bool(S.valid), best_iter=S.best_iter, num_inliers=S.num_inliers, best_cost=np.float32(S.best_cost),
                 M_21=np.array(S.M_21).reshape(3, 3) if S.valid else None, inlier_flags=None if S.n_matches < 8 else fl[:S.n_matches].astype(bool))
            for S, fl in zip(arr, flags)]


class _twoview_solver(_ransac_solver):
    """The shared surface of homography_solver and fundamental_solver.  undist_keypts_*: every undistorted keypoint of each frame
    ((n, 2) pixels); matches_12: (first, second) index pairs.  The engine is the solver's member: find_via_ransac continues its state
    across calls, and use_fixed_seed gives each solver its own default-constructed engine, as util::create_random_engine does."""

    _model = None

    def __init__(self, undist_keypts_1, undist_keypts_2, matches_12, sigma, use_fixed_seed=False, device=0):
        super().__init__(use_fixed_seed, device)
        self.undist_keypts_1_ = _keypts(undist_keypts_1)
        self.undist_keypts_2_ = _keypts(undist_keypts_2)
        m = np.asarray(matches_12, np.int64).reshape(-1, 2)
        if len(m) and (m.min() < 0 or m[:, 0].max() >= len(self.undist_keypts_1_) or m[:, 1].max() >= len(self.undist_keypts_2_)):
            raise IndexError("match index outside the keypoints")  # std::vector::at throws in the reference
        self.matches_12_ = np.ascontiguousarray(m.astype(np.int32))
        self.num_matches_ = len(m)
        self.sigma_ = np.float32(sigma)
        self.best_cost_ = np.float32(0.0)
        self.best_M_21_ = np.zeros((3, 3))

    def find_via_ransac(self, max_num_iter, recompute=True):
        r = self._find_via_ransac(self.num_matches_ < 8, max_num_iter, _SET_SIZE[self._model], twoview_ransac_batch,
                                  dict(model=self._model, keypts_1=self.undist_keypts_1_, keypts_2=self.undist_keypts_2_,
                                       matches_12=self.matches_12_, sigma=self.sigma_, recompute=recompute))
        if r is not None:
            self.best_cost_ = r["best_cost"]
            if r["valid"]:
                self.best_M_21_ = r["M_21"]

    def get_best_cost(self):
        return self.best_cost_

    def get_inlier_matches(self):
        return list(self.is_inlier_match_)


class homography_solver(_twoview_solver):
    """solve::homography_solver: the four-point DLT inside RANSAC (min_sets of 4, early return below 8 matches)."""
    _model = MODEL_H

    def get_best_H_21(self):
        return self.best_M_21_.copy()


class fundamental_solver(_twoview_solver):
    """solve::fundamental_solver: the normalised eight-point algorithm inside RANSAC."""
    _model = MODEL_F

    def get_best_F_21(self):
        return self.best_M_21_.copy()
