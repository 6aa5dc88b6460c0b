"""Host-side mirrors of the device-resident tracking chains (include/b200vslam.h) for a batch of frames whose keypoints / descriptors are
the results of the last extract of an orb_extractor and never leave the GPU:
  local_map_tracker   b200_track_local_map: tracking_module::search_local_landmarks (tracking_module.cc:533-606) + pose_optimizer::optimize
  frame_tracker       b200_motion_based_track: module::frame_tracker::motion_based_track (module/frame_tracker.cc:20-59)
                      b200_robust_match_based_track: module::frame_tracker::robust_match_based_track (module/frame_tracker.cc:97-131)
                      b200_bow_match_based_track: module::frame_tracker::bow_match_based_track (module/frame_tracker.cc:61-95)"""
import ctypes as C

import numpy as np

from . import _lib, feature, match, optimize, solve
from ._lib import CameraIntrinsics, check, lib, ptr


class TrackParams(C.Structure):
    """b200_track_params_t"""
    _fields_ = [("cam", CameraIntrinsics), ("focal_x_baseline", C.c_double), ("monocular", C.c_int32), ("img_bounds", C.c_float * 4),
                ("grid_cols", C.c_int32), ("grid_rows", C.c_int32), ("num_levels", C.c_uint32), ("log_scale_factor", C.c_float),
                ("scale_factors", C.c_void_p), ("inv_level_sigma_sq", C.c_void_p), ("margin", C.c_float), ("lowe_ratio", C.c_float),
                ("hamming_thr", C.c_uint32), ("ray_cos_thr", C.c_float), ("num_trials_robust", C.c_int32), ("num_trials", C.c_int32),
                ("num_each_iter", C.c_int32), ("max_candidates", C.c_int32)]


class TrackFrame(C.Structure):
    """b200_track_frame_t"""
    _fields_ = [("frame", C.c_int32), ("pose_cw", C.c_void_p), ("n_keypoints_in", C.c_int32), ("kp_x_right", C.c_void_p),
                ("kp_landmark", C.c_void_p), ("n_landmarks", C.c_int32), ("lm_pos_w", C.c_void_p), ("lm_mean_normal", C.c_void_p),
                ("lm_min_valid_dist", C.c_void_p), ("lm_max_valid_dist", C.c_void_p), ("lm_desc", C.c_void_p), ("lm_skip", C.c_void_p),
                ("lm_has_observation", C.c_void_p), ("kp_cap", C.c_int32), ("lm_observable", C.c_void_p), ("kp_landmark_out", C.c_void_p),
                ("kp_outlier", C.c_void_p), ("pose_cw_out", C.c_double * 16), ("n_keypoints", C.c_int32), ("n_matches", C.c_int32),
                ("n_valid", C.c_uint32)]


class MotionTrackFrame(C.Structure):
    """b200_motion_track_frame_t"""
    _fields_ = [("frame", C.c_int32), ("pose_cw", C.c_void_p), ("last_pose_cw", C.c_void_p), ("n_keypoints_in", C.c_int32), ("kp_x_right", C.c_void_p),
                ("n_landmarks", C.c_int32), ("lm_pos_w", C.c_void_p), ("lm_desc", C.c_void_p), ("lm_octave", C.c_void_p), ("lm_angle", C.c_void_p),
                ("lm_has_observation", C.c_void_p), ("kp_cap", C.c_int32), ("kp_landmark_out", C.c_void_p), ("pose_cw_out", C.c_double * 16),
                ("n_keypoints", C.c_int32), ("n_matches_first", C.c_int32), ("n_matches", C.c_int32), ("retried", C.c_int32), ("n_valid", C.c_uint32),
                ("tracked", C.c_int32)]


class RobustTrackFrame(C.Structure):
    """b200_robust_track_frame_t"""
    _fields_ = [("frame", C.c_int32), ("last_pose_cw", C.c_void_p), ("n_keypoints_in", C.c_int32), ("kp_x_right", C.c_void_p), ("engine", C.c_void_p),
                ("n_kf_keypoints", C.c_int32), ("kf_desc", C.c_void_p), ("kf_angle", C.c_void_p), ("kf_bearings", C.c_void_p), ("kf_valid", C.c_void_p),
                ("kf_pos_w", C.c_void_p), ("kp_cap", C.c_int32), ("kp_landmark_out", C.c_void_p), ("pose_cw_out", C.c_double * 16),
                ("n_keypoints", C.c_int32), ("n_matches", C.c_int32), ("essential_valid", C.c_int32), ("status", C.c_int32), ("n_inliers", C.c_int32),
                ("applied", C.c_int32), ("n_valid", C.c_uint32), ("tracked", C.c_int32)]


class BowTrackFrame(C.Structure):
    """b200_bow_track_frame_t"""
    _fields_ = [("frame", C.c_int32), ("last_pose_cw", C.c_void_p), ("n_keypoints_in", C.c_int32), ("kp_node", C.c_void_p), ("kp_x_right", C.c_void_p),
                ("n_kf_keypoints", C.c_int32), ("kf_desc", C.c_void_p), ("kf_angle", C.c_void_p), ("kf_node", C.c_void_p), ("kf_valid", C.c_void_p),
                ("kf_pos_w", C.c_void_p), ("kp_cap", C.c_int32), ("kp_landmark_out", C.c_void_p), ("pose_cw_out", C.c_double * 16),
                ("n_keypoints", C.c_int32), ("n_matches", C.c_int32), ("applied", C.c_int32), ("n_valid", C.c_uint32), ("tracked", C.c_int32)]


def _bind():
    L = lib()
    if not getattr(L, "_track_bound", False):
        L.b200_track_local_map.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(TrackParams), C.c_int, C.POINTER(TrackFrame)]
        L.b200_track_stage_ms.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_float)]
        L.b200_motion_based_track.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(TrackParams), C.c_double, C.c_uint32, C.c_int,
                                              C.POINTER(MotionTrackFrame)]
        L.b200_motion_track_stage_ms.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_float)]
        L.b200_robust_match_based_track.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(TrackParams), C.c_uint32, C.c_int,
                                                    C.POINTER(RobustTrackFrame)]
        L.b200_robust_track_stage_ms.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_float)]
        L.b200_bow_match_based_track.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(TrackParams), C.c_uint32, C.c_int,
                                                 C.POINTER(BowTrackFrame)]
        L.b200_bow_track_stage_ms.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_float)]
        L._track_bound = True
    return L


def _track_params(extractor, camera, margin, lowe_ratio, hamming_thr, ray_cos_thr, num_trials_robust, num_trials, num_each_iter, grid, img_bounds,
                  max_candidates):
    """b200_track_params_t of an extractor and a camera dict, plus the arrays it points to (keep them alive with it)."""
    op = extractor.orb_params_
    sf = np.ascontiguousarray(op.scale_factors_, np.float32)
    isig = np.ascontiguousarray(op.inv_level_sigma_sq_, np.float32)
    p = TrackParams()
    p.cam = camera_intrinsics(camera)
    p.focal_x_baseline = float(camera.get("fxb", 0.0))
    p.monocular = 1 if camera.get("setup", "monocular") == "monocular" else 0
    if img_bounds is not None:
        b = img_bounds
    elif p.cam.model in (2, 3):  # fisheye / radial division: camera::*::compute_image_bounds
        b = feature.camera_image_bounds(camera, extractor)
    else:
        b = (0.0, camera.get("cols", 0.0), 0.0, camera.get("rows", 0.0))
    p.img_bounds = (C.c_float * 4)(*[float(v) for v in b])
    p.grid_cols, p.grid_rows = int(grid[0]), int(grid[1])
    p.num_levels = int(op.num_levels_)
    p.log_scale_factor = float(op.log_scale_factor_)
    p.scale_factors = sf.ctypes.data
    p.inv_level_sigma_sq = isig.ctypes.data
    p.margin, p.lowe_ratio, p.hamming_thr, p.ray_cos_thr = float(margin), float(lowe_ratio), int(hamming_thr), float(ray_cos_thr)
    p.num_trials_robust, p.num_trials, p.num_each_iter = int(num_trials_robust), int(num_trials), int(num_each_iter)
    p.max_candidates = int(max_candidates)
    return p, (sf, isig)


def _default_kp_cap(extractor):
    """The extractor's largest keypoint count at its last image size."""
    b, h, w = extractor._shape
    return lib().b200_orb_max_keypoints(extractor._h, w, h)


def _stage_ms(fn, names, device):
    """{name: ms} of the calling thread's matcher's last call of one chain, read with fn (b200_*_stage_ms)."""
    out = {}
    for i, nm in enumerate(names):
        v = C.c_float()
        check(fn(match._matcher(device), i, C.byref(v)))
        out[nm] = v.value
    return out


def camera_intrinsics(camera):
    """b200_camera_intrinsics_t of a camera dict (perspective, equirectangular, fisheye or radial_division; see _lib.camera_intrinsics)."""
    return _lib.camera_intrinsics(camera)


class local_map_tracker:
    """One instance owns the pose-optimiser handle of the chain; the matcher handle is the calling thread's (match._matcher)."""

    STAGES = ("undistort_observe", "grid", "candidates", "resolve", "edges", "pose_optimize", "chain")

    def __init__(self, extractor, camera, margin=5.0, lowe_ratio=0.8, hamming_thr=match.HAMMING_DIST_THR_HIGH, ray_cos_thr=0.5,
                 num_trials_robust=2, num_trials=2, num_each_iter=10, grid=(64, 48), img_bounds=None, max_candidates=0, device=0):
        self._L = _bind()
        self.extractor = extractor
        self.device = device
        self._opt = optimize.pose_optimizer(num_trials_robust, num_trials, num_each_iter, device)
        self._prm, self._keep = _track_params(extractor, camera, margin, lowe_ratio, hamming_thr, ray_cos_thr, num_trials_robust, num_trials,
                                              num_each_iter, grid, img_bounds, max_candidates)

    def pack(self, frames, kp_cap):
        """frames: dicts(frame, pose_cw (4,4), landmarks=dict(pos_w, mean_normal, min_valid_dist, max_valid_dist, desc[, skip, has_observation])
        [, kp_x_right, kp_landmark]).  Returns (ctypes array, keep-alive list, output arrays)."""
        arr = (TrackFrame * len(frames))()
        keep, outs = [], []
        for i, fr in enumerate(frames):
            lm = fr["landmarks"]
            pos = np.ascontiguousarray(lm["pos_w"], np.float64).reshape(-1, 3)
            n = len(pos)
            a = dict(pose=np.ascontiguousarray(fr["pose_cw"], np.float64).reshape(4, 4), pos=pos,
                     nml=np.ascontiguousarray(lm["mean_normal"], np.float64).reshape(-1, 3),
                     lo=np.ascontiguousarray(lm["min_valid_dist"], np.float32), hi=np.ascontiguousarray(lm["max_valid_dist"], np.float32),
                     desc=np.ascontiguousarray(lm["desc"], np.uint8).reshape(-1, 32),
                     skip=None if lm.get("skip") is None else np.ascontiguousarray(lm["skip"], np.uint8),
                     hobs=None if lm.get("has_observation") is None else np.ascontiguousarray(lm["has_observation"], np.uint8),
                     xr=None if fr.get("kp_x_right") is None else np.ascontiguousarray(fr["kp_x_right"], np.float32),
                     kl=None if fr.get("kp_landmark") is None else np.ascontiguousarray(fr["kp_landmark"], np.int32))
            o = dict(observable=np.zeros(max(n, 1), np.uint8), kp_landmark=np.full(max(kp_cap, 1), -1, np.int32),
                     kp_outlier=np.zeros(max(kp_cap, 1), np.uint8))
            T = arr[i]
            T.frame = int(fr.get("frame", i))
            T.pose_cw = a["pose"].ctypes.data
            T.n_keypoints_in = len(a["xr"]) if a["xr"] is not None else (len(a["kl"]) if a["kl"] is not None else 0)
            T.kp_x_right, T.kp_landmark = ptr(a["xr"]), ptr(a["kl"])
            T.n_landmarks = n
            T.lm_pos_w, T.lm_mean_normal, T.lm_min_valid_dist, T.lm_max_valid_dist = ptr(a["pos"]), ptr(a["nml"]), ptr(a["lo"]), ptr(a["hi"])
            T.lm_desc, T.lm_skip, T.lm_has_observation = ptr(a["desc"]), ptr(a["skip"]), ptr(a["hobs"])
            T.kp_cap = int(kp_cap)
            T.lm_observable, T.kp_landmark_out, T.kp_outlier = ptr(o["observable"]), ptr(o["kp_landmark"]), ptr(o["kp_outlier"])
            keep.append(a)
            outs.append(o)
        return arr, keep, outs

    def run_packed(self, packed):
        arr = packed[0]
        check(self._L.b200_track_local_map(self.extractor._h, match._matcher(self.device), self._opt._h, C.byref(self._prm), len(arr), arr))

    def track(self, frames, kp_cap=None):
        """Returns, per frame: dict(observable bool (n_lm,), kp_landmark int32 (n_kp,), kp_outlier bool (n_kp,), pose_cw (4,4), n_matches, n_valid)."""
        if kp_cap is None:
            kp_cap = _default_kp_cap(self.extractor)
        packed = self.pack(frames, kp_cap)
        self.run_packed(packed)
        res = []
        for T, o, a in zip(packed[0], packed[2], packed[1]):
            nk = T.n_keypoints
            res.append(dict(observable=o["observable"][:len(a["pos"])].astype(bool), kp_landmark=o["kp_landmark"][:nk].copy(),
                            kp_outlier=o["kp_outlier"][:nk].astype(bool), pose_cw=np.array(T.pose_cw_out[:]).reshape(4, 4),
                            n_matches=int(T.n_matches), n_valid=int(T.n_valid), n_keypoints=int(nk)))
        return res

    def stage_ms(self):
        return _stage_ms(self._L.b200_track_stage_ms, self.STAGES, self.device)


class frame_tracker:
    """module::frame_tracker for a batch of frames: motion_based_track (module/frame_tracker.cc:20-59) with match::projection(0.9, true)
    (b200_motion_based_track), bow_match_based_track (:61-95) with match::bow_tree(0.7, true) (b200_bow_match_based_track) and
    robust_match_based_track (:97-131) with match::robust(0.8, true) (b200_robust_match_based_track).
    margin = margin_last_frame_projection (20; 10 in the KITTI example).  true_baseline defaults to the camera's fxb / fx
    (camera::base::true_baseline_).  use_fixed_seed: the reference's member; the robust matcher's essential solver then draws from a
    default-constructed engine, otherwise from one seeded by ten random words.  One instance owns the pose-optimiser handle; the matcher
    handle is the calling thread's (match._matcher)."""

    STAGES = ("undistort_queries", "grid", "first_search", "second_search", "edges", "pose_optimize", "chain")
    ROBUST_STAGES = ("undistort_bearings", "brute_force", "sampler", "essential", "edges", "pose_optimize", "chain")
    BOW_STAGES = ("undistort_angles", "candidates", "resolve", "gate", "edges", "pose_optimize", "chain")

    def __init__(self, extractor, camera, margin=20.0, num_matches_thr=10, hamming_thr=match.HAMMING_DIST_THR_HIGH, num_trials_robust=2, num_trials=2,
                 num_each_iter=10, grid=(64, 48), img_bounds=None, max_candidates=0, true_baseline=None, device=0, use_fixed_seed=False):
        self._L = _bind()
        self.extractor = extractor
        self.device = device
        self.num_matches_thr = int(num_matches_thr)
        self.use_fixed_seed = bool(use_fixed_seed)
        fx = float(camera.get("fx", 0.0))
        self.true_baseline = float(true_baseline) if true_baseline is not None else (float(camera.get("fxb", 0.0)) / fx if fx else 0.0)
        self._opt = optimize.pose_optimizer(num_trials_robust, num_trials, num_each_iter, device)
        # lowe_ratio is robust(0.8, true)'s (the motion chain does not read it); ray_cos_thr and log_scale_factor are used by neither chain
        self._prm, self._keep = _track_params(extractor, camera, margin, 0.8, hamming_thr, 0.5, num_trials_robust, num_trials, num_each_iter, grid,
                                              img_bounds, max_candidates)
        # bow_tree(0.7, true); max_candidates bounds the gated candidates of one keyframe keypoint there (0 = 64)
        self._prm_bow, self._keep_bow = _track_params(extractor, camera, margin, 0.7, hamming_thr, 0.5, num_trials_robust, num_trials, num_each_iter,
                                                      grid, img_bounds, max_candidates)

    def pack(self, frames, kp_cap):
        """frames: dicts(frame, pose_cw (4,4), [last_pose_cw (4,4)], table=dict(pos_w, desc, octave, angle[, has_observation]) [, kp_x_right]).
        Returns (ctypes array, keep-alive list, output arrays)."""
        arr = (MotionTrackFrame * len(frames))()
        keep, outs = [], []
        for i, fr in enumerate(frames):
            tb = fr["table"]
            pos = np.ascontiguousarray(tb["pos_w"], np.float64).reshape(-1, 3)
            n = len(pos)
            opt = lambda v, dt: None if v is None else np.ascontiguousarray(v, dt)
            a = dict(pose=np.ascontiguousarray(fr["pose_cw"], np.float64).reshape(4, 4), last=opt(fr.get("last_pose_cw"), np.float64), pos=pos,
                     desc=np.ascontiguousarray(tb["desc"], np.uint8).reshape(-1, 32), oct=np.ascontiguousarray(tb["octave"], np.uint8),
                     ang=np.ascontiguousarray(tb["angle"], np.float32), hobs=opt(tb.get("has_observation"), np.uint8),
                     xr=opt(fr.get("kp_x_right"), np.float32))
            o = dict(kp_landmark=np.full(max(kp_cap, 1), -1, np.int32))
            T = arr[i]
            T.frame = int(fr.get("frame", i))
            T.pose_cw, T.last_pose_cw = a["pose"].ctypes.data, ptr(a["last"])
            T.n_keypoints_in = len(a["xr"]) if a["xr"] is not None else 0
            T.kp_x_right = ptr(a["xr"])
            T.n_landmarks = n
            T.lm_pos_w, T.lm_desc, T.lm_octave, T.lm_angle, T.lm_has_observation = ptr(a["pos"]), ptr(a["desc"]), ptr(a["oct"]), ptr(a["ang"]), ptr(a["hobs"])
            T.kp_cap = int(kp_cap)
            T.kp_landmark_out = ptr(o["kp_landmark"])
            keep.append(a)
            outs.append(o)
        return arr, keep, outs

    def run_packed(self, packed):
        arr = packed[0]
        check(self._L.b200_motion_based_track(self.extractor._h, match._matcher(self.device), self._opt._h, C.byref(self._prm), self.true_baseline,
                                              self.num_matches_thr, len(arr), arr))

    def motion_based_track(self, frames, kp_cap=None):
        """Returns, per frame: dict(kp_landmark int32 (n_kp,) after discard_outliers, pose_cw (4,4), n_keypoints, n_matches_first, n_matches,
        retried, n_valid, tracked)."""
        if kp_cap is None:
            kp_cap = _default_kp_cap(self.extractor)
        packed = self.pack(frames, kp_cap)
        self.run_packed(packed)
        res = []
        for T, o in zip(packed[0], packed[2]):
            nk = T.n_keypoints
            res.append(dict(kp_landmark=o["kp_landmark"][:nk].copy(), pose_cw=np.array(T.pose_cw_out[:]).reshape(4, 4), n_keypoints=int(nk),
                            n_matches_first=int(T.n_matches_first), n_matches=int(T.n_matches), retried=bool(T.retried), n_valid=int(T.n_valid),
                            tracked=bool(T.tracked)))
        return res

    def stage_ms(self):
        return _stage_ms(self._L.b200_motion_track_stage_ms, self.STAGES, self.device)

    def pack_robust(self, frames, kp_cap):
        """frames: dicts(frame, last_pose_cw (4,4), keyframe=dict(desc (n, 32), angle, bearings (n, 3), valid, pos_w (n, 3)) [, kp_x_right]
        [, engine (solve.mt19937)]).  A frame without an engine draws from a default-constructed one when use_fixed_seed, else from one
        seeded by ten random words (util::create_random_engine).  Returns (ctypes array, keep-alive list, output arrays)."""
        arr = (RobustTrackFrame * len(frames))()
        keep, outs = [], []
        for i, fr in enumerate(frames):
            kf = fr["keyframe"]
            desc = np.ascontiguousarray(kf["desc"], np.uint8).reshape(-1, 32)
            n = len(desc)
            opt = lambda v, dt: None if v is None else np.ascontiguousarray(v, dt)
            eng = fr.get("engine")
            if eng is None and not self.use_fixed_seed:
                eng = solve._random_engine(False)
            a = dict(last=np.ascontiguousarray(fr["last_pose_cw"], np.float64).reshape(4, 4), desc=desc,
                     ang=np.ascontiguousarray(kf["angle"], np.float32), bear=np.ascontiguousarray(kf["bearings"], np.float64).reshape(-1, 3),
                     valid=np.ascontiguousarray(kf["valid"], np.uint8), pos=np.ascontiguousarray(kf["pos_w"], np.float64).reshape(-1, 3),
                     xr=opt(fr.get("kp_x_right"), np.float32), eng=eng)
            o = dict(kp_landmark=np.full(max(kp_cap, 1), -1, np.int32))
            T = arr[i]
            T.frame = int(fr.get("frame", i))
            T.last_pose_cw = a["last"].ctypes.data
            T.n_keypoints_in = len(a["xr"]) if a["xr"] is not None else 0
            T.kp_x_right = ptr(a["xr"])
            T.engine = C.addressof(eng) if eng is not None else None
            T.n_kf_keypoints = n
            T.kf_desc, T.kf_angle, T.kf_bearings, T.kf_valid, T.kf_pos_w = ptr(a["desc"]), ptr(a["ang"]), ptr(a["bear"]), ptr(a["valid"]), ptr(a["pos"])
            T.kp_cap = int(kp_cap)
            T.kp_landmark_out = ptr(o["kp_landmark"])
            keep.append(a)
            outs.append(o)
        return arr, keep, outs

    def run_robust_packed(self, packed):
        arr = packed[0]
        check(self._L.b200_robust_match_based_track(self.extractor._h, match._matcher(self.device), self._opt._h, C.byref(self._prm),
                                                    self.num_matches_thr, len(arr), arr))

    def robust_match_based_track(self, frames, kp_cap=None):
        """Returns, per frame: dict(kp_landmark int32 (n_kp,) after discard_outliers and pose_cw (4,4) -- both None when not applied (the
        reference leaves the frame as it was) --, n_keypoints, n_matches, essential_valid, status, n_inliers, applied, n_valid, tracked)."""
        if kp_cap is None:
            kp_cap = _default_kp_cap(self.extractor)
        packed = self.pack_robust(frames, kp_cap)
        self.run_robust_packed(packed)
        res = []
        for T, o in zip(packed[0], packed[2]):
            nk = T.n_keypoints
            applied = bool(T.applied)
            res.append(dict(kp_landmark=o["kp_landmark"][:nk].copy() if applied else None,
                            pose_cw=np.array(T.pose_cw_out[:]).reshape(4, 4) if applied else None, n_keypoints=int(nk), n_matches=int(T.n_matches),
                            essential_valid=bool(T.essential_valid), status=int(T.status), n_inliers=int(T.n_inliers), applied=applied,
                            n_valid=int(T.n_valid), tracked=bool(T.tracked)))
        return res

    def robust_stage_ms(self):
        return _stage_ms(self._L.b200_robust_track_stage_ms, self.ROBUST_STAGES, self.device)

    def pack_bow(self, frames, kp_cap):
        """frames: dicts(frame, last_pose_cw (4,4), kp_node (n_kp,), keyframe=dict(desc (n, 32), angle, node, valid, pos_w (n, 3))
        [, kp_x_right]).  kp_node / keyframe node: the BoW node of each keypoint (the key of bow_feat_vec_ that lists it), -1 = none.
        Returns (ctypes array, keep-alive list, output arrays)."""
        arr = (BowTrackFrame * len(frames))()
        keep, outs = [], []
        for i, fr in enumerate(frames):
            kf = fr["keyframe"]
            desc = np.ascontiguousarray(kf["desc"], np.uint8).reshape(-1, 32)
            opt = lambda v, dt: None if v is None else np.ascontiguousarray(v, dt)
            a = dict(last=np.ascontiguousarray(fr["last_pose_cw"], np.float64).reshape(4, 4), node=np.ascontiguousarray(fr["kp_node"], np.int32),
                     desc=desc, ang=np.ascontiguousarray(kf["angle"], np.float32), knode=np.ascontiguousarray(kf["node"], np.int32),
                     valid=np.ascontiguousarray(kf["valid"], np.uint8), pos=np.ascontiguousarray(kf["pos_w"], np.float64).reshape(-1, 3),
                     xr=opt(fr.get("kp_x_right"), np.float32))
            o = dict(kp_landmark=np.full(max(kp_cap, 1), -1, np.int32))
            T = arr[i]
            T.frame = int(fr.get("frame", i))
            T.last_pose_cw = a["last"].ctypes.data
            T.n_keypoints_in = len(a["node"])
            T.kp_node, T.kp_x_right = ptr(a["node"]), ptr(a["xr"])
            T.n_kf_keypoints = len(desc)
            T.kf_desc, T.kf_angle, T.kf_node, T.kf_valid, T.kf_pos_w = ptr(a["desc"]), ptr(a["ang"]), ptr(a["knode"]), ptr(a["valid"]), ptr(a["pos"])
            T.kp_cap = int(kp_cap)
            T.kp_landmark_out = ptr(o["kp_landmark"])
            keep.append(a)
            outs.append(o)
        return arr, keep, outs

    def run_bow_packed(self, packed):
        arr = packed[0]
        check(self._L.b200_bow_match_based_track(self.extractor._h, match._matcher(self.device), self._opt._h, C.byref(self._prm_bow),
                                                 self.num_matches_thr, len(arr), arr))

    def bow_match_based_track(self, frames, kp_cap=None):
        """Returns, per frame: dict(kp_landmark int32 (n_kp,) after discard_outliers and pose_cw (4,4) -- both None when not applied (the
        reference leaves the frame as it was) --, n_keypoints, n_matches, applied, n_valid, tracked)."""
        if kp_cap is None:
            kp_cap = _default_kp_cap(self.extractor)
        packed = self.pack_bow(frames, kp_cap)
        self.run_bow_packed(packed)
        res = []
        for T, o in zip(packed[0], packed[2]):
            nk = T.n_keypoints
            applied = bool(T.applied)
            res.append(dict(kp_landmark=o["kp_landmark"][:nk].copy() if applied else None,
                            pose_cw=np.array(T.pose_cw_out[:]).reshape(4, 4) if applied else None, n_keypoints=int(nk), n_matches=int(T.n_matches),
                            applied=applied, n_valid=int(T.n_valid), tracked=bool(T.tracked)))
        return res

    def bow_stage_ms(self):
        return _stage_ms(self._L.b200_bow_track_stage_ms, self.BOW_STAGES, self.device)
