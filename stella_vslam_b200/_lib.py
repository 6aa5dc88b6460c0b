"""ctypes binding of libb200vslam.so (the C ABI declared in include/b200vslam.h).

There is no fallback: if the CUDA extension is missing or no sm_90 (Hopper) device is present, calls fail loudly.
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libb200vslam.so")

OK, ERR_INVALID, ERR_CUDA, ERR_CAPACITY, ERR_ABORTED = 0, -1, -2, -3, -4


class B200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"b200vslam error {code}: {msg}")
        self.code = code


class OrbParams(C.Structure):
    _fields_ = [("scale_factor", C.c_float), ("num_levels", C.c_int32), ("ini_fast_thr", C.c_int32),
                ("min_fast_thr", C.c_int32), ("min_area", C.c_uint32), ("n_mask_rects", C.c_int32),
                ("mask_rects", C.POINTER(C.c_float)), ("device", C.c_int32), ("max_batch", C.c_int32)]


KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                     ("octave", "<i4")])

_lib = None

# every symbol include/b200vslam.h declares (tests check that the .so exports all of them)
class CameraIntrinsics(C.Structure):
    """b200_camera_intrinsics_t (include/b200vslam.h)."""
    _fields_ = [("model", C.c_int32), ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
                ("k1", C.c_double), ("k2", C.c_double), ("p1", C.c_double), ("p2", C.c_double), ("k3", C.c_double),
                ("cols", C.c_double), ("rows", C.c_double), ("k4", C.c_double), ("distortion", C.c_double)]


# camera::base::model_type_t names -> the model codes of b200_camera_intrinsics_t
CAMERA_MODELS = {"perspective": 0, "equirectangular": 1, "fisheye": 2, "radial_division": 3}


def camera_intrinsics(camera):
    """b200_camera_intrinsics_t of a camera dict: model ("perspective" when absent, "equirectangular", "fisheye",
    "radial_division"), fx, fy, cx, cy, k1, k2, p1, p2, k3, k4, distortion, cols, rows; missing values are 0."""
    name = camera.get("model", "perspective")
    if name not in CAMERA_MODELS:
        raise ValueError(f"unknown camera model {name!r}; expected one of {sorted(CAMERA_MODELS)}")
    return CameraIntrinsics(CAMERA_MODELS[name], *[float(camera.get(k, 0.0)) for k in
                            ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2", "k3", "cols", "rows", "k4", "distortion")])


class RectifierParams(C.Structure):
    """b200_rectifier_params_t (include/b200vslam.h)."""
    _fields_ = [("model", C.c_int32), ("cols", C.c_int32), ("rows", C.c_int32), ("K_rect", C.c_double * 9), ("K", (C.c_double * 9) * 2),
                ("R", (C.c_double * 9) * 2), ("D", (C.c_double * 8) * 2), ("n_dist", C.c_int32 * 2), ("device", C.c_int32)]


class GuidedProblem(C.Structure):
    """b200_guided_problem_t (include/b200vslam.h)."""
    _fields_ = [("n_train", C.c_int32), ("t_x", C.c_void_p), ("t_y", C.c_void_p), ("t_octave", C.c_void_p), ("t_angle", C.c_void_p),
                ("t_x_right", C.c_void_p), ("t_desc", C.c_void_p), ("t_occupied", C.c_void_p),
                ("min_x", C.c_float), ("max_x", C.c_float), ("min_y", C.c_float), ("max_y", C.c_float),
                ("grid_cols", C.c_int32), ("grid_rows", C.c_int32), ("n_queries", C.c_int32),
                ("q_desc", C.c_void_p), ("q_x", C.c_void_p), ("q_y", C.c_void_p), ("q_margin", C.c_void_p), ("q_min_level", C.c_void_p),
                ("q_max_level", C.c_void_p), ("q_x_right", C.c_void_p), ("q_angle", C.c_void_p), ("q_valid", C.c_void_p),
                ("q_has_observation", C.c_void_p), ("q_reproj", C.c_void_p), ("inv_level_sigma_sq", C.c_void_p), ("n_levels", C.c_int32), ("do_reprojection_matching", C.c_int32),
                ("match_out", C.c_void_p), ("n_matches", C.c_int32)]


GUIDED_FIELDS = (("t_x", "f4"), ("t_y", "f4"), ("t_octave", "u1"), ("t_angle", "f4"), ("t_x_right", "f4"), ("t_desc", "u1"), ("t_occupied", "u1"),
                 ("q_desc", "u1"), ("q_x", "f4"), ("q_y", "f4"), ("q_margin", "f4"), ("q_min_level", "i1"), ("q_max_level", "i1"),
                 ("q_x_right", "f4"), ("q_angle", "f4"), ("q_valid", "u1"), ("q_has_observation", "u1"), ("q_reproj", "f8"),
                 ("inv_level_sigma_sq", "f4"))


def pack_guided_problem(prob, StructT=None):
    """dict -> (struct, keep-alive arrays).  Keys: GUIDED_FIELDS (missing / None -> NULL), bounds=(min_x,max_x,min_y,max_y),
    grid=(cols, rows).  The struct's match_out / t_occupied point into the returned arrays."""
    import numpy as np
    S = (StructT or GuidedProblem)()
    keep = {}
    for name, dt in GUIDED_FIELDS:
        v = prob.get(name)
        if v is None:
            setattr(S, name, None)
            continue
        a = np.ascontiguousarray(v, np.dtype(dt))
        if name == "t_occupied":
            a = a.copy()
        keep[name] = a
        setattr(S, name, a.ctypes.data)
    S.n_train = len(keep["t_x"]) if "t_x" in keep else 0
    S.n_queries = len(keep["q_x"]) if "q_x" in keep else 0
    S.min_x, S.max_x, S.min_y, S.max_y = [float(v) for v in prob["bounds"]]
    S.grid_cols, S.grid_rows = prob.get("grid", (64, 48))
    S.do_reprojection_matching = int(bool(prob.get("do_reprojection_matching", False)))
    if hasattr(S, "n_levels"):
        S.n_levels = len(keep["inv_level_sigma_sq"]) if "inv_level_sigma_sq" in keep else 0
    if hasattr(S, "match_out"):
        keep["match_out"] = np.full(max(S.n_queries, 1), -2, np.int32)
        S.match_out = keep["match_out"].ctypes.data
    return S, keep


class PairsProblem(C.Structure):
    """b200_pairs_problem_t (include/b200vslam.h)."""
    _fields_ = [("n1", C.c_int32), ("desc1", C.c_void_p), ("angle1", C.c_void_p), ("valid1", C.c_void_p), ("node1", C.c_void_p),
                ("bearing1", C.c_void_p), ("scale1", C.c_void_p), ("stereo1", C.c_void_p),
                ("n2", C.c_int32), ("desc2", C.c_void_p), ("angle2", C.c_void_p), ("valid2", C.c_void_p), ("node2", C.c_void_p),
                ("bearing2", C.c_void_p), ("stereo2", C.c_void_p),
                ("E_12", C.c_double * 9), ("epiplane_in_keyfrm_2", C.c_double * 3), ("valid_epiplane", C.c_int32),
                ("residual_rad_thr", C.c_float), ("match_out", C.c_void_p), ("n_matches", C.c_int32)]


PAIRS_FIELDS = (("desc1", "u1"), ("angle1", "f4"), ("valid1", "u1"), ("node1", "i4"), ("bearing1", "f8"), ("scale1", "f4"), ("stereo1", "u1"),
                ("desc2", "u1"), ("angle2", "f4"), ("valid2", "u1"), ("node2", "i4"), ("bearing2", "f8"), ("stereo2", "u1"))


def pack_pairs_problem(prob, StructT=None):
    """dict -> (struct, keep-alive arrays).  Keys: PAIRS_FIELDS (missing / None -> NULL), E_12 (3x3), epiplane_in_keyfrm_2 (3),
    valid_epiplane, residual_rad_thr."""
    import numpy as np
    S = (StructT or PairsProblem)()
    keep = {}
    for name, dt in PAIRS_FIELDS:
        v = prob.get(name)
        if v is None:
            setattr(S, name, None)
            continue
        a = np.ascontiguousarray(v, np.dtype(dt))
        keep[name] = a
        setattr(S, name, a.ctypes.data)
    S.n1 = len(keep["desc1"].reshape(-1, 32)) if "desc1" in keep else 0
    S.n2 = len(keep["desc2"].reshape(-1, 32)) if "desc2" in keep else 0
    E = np.asarray(prob.get("E_12", np.zeros((3, 3))), np.float64).reshape(9)
    epi = np.asarray(prob.get("epiplane_in_keyfrm_2", np.zeros(3)), np.float64).reshape(3)
    for k in range(9):
        S.E_12[k] = float(E[k])
    for k in range(3):
        S.epiplane_in_keyfrm_2[k] = float(epi[k])
    S.valid_epiplane = int(bool(prob.get("valid_epiplane", False)))
    S.residual_rad_thr = float(prob.get("residual_rad_thr", 0.0))
    if hasattr(S, "match_out"):
        keep["match_out"] = np.full(max(S.n1, 1), -2, np.int32)
        S.match_out = keep["match_out"].ctypes.data
    return S, keep


SYMBOLS = [
    "b200_last_error", "b200_device_count", "b200_version", "b200_host_alloc", "b200_host_free",
    "b200_orb_default_params", "b200_orb_create", "b200_orb_destroy", "b200_orb_max_keypoints", "b200_orb_extract",
    "b200_orb_extract_device", "b200_orb_set_stream", "b200_orb_bind_outputs", "b200_orb_reserve", "b200_orb_fetch", "b200_orb_device_results", "b200_orb_sync", "b200_orb_level_info",
    "b200_orb_pyramid_level_device", "b200_orb_pyramid_level_host", "b200_orb_pyramid_level_view", "b200_convert_to_grayscale", "b200_convert_to_grayscale_device", "b200_keypoints_undistort", "b200_frame_can_observe", "b200_orb_stage_ms", "b200_orb_enable_timing", "b200_orb_raw_corner_counts",
    "b200_matcher_create", "b200_matcher_destroy", "b200_hamming_matrix", "b200_match_bruteforce",
    "b200_match_bruteforce_device", "b200_match_guided", "b200_match_cross_check", "b200_match_pairs", "b200_stereo_compute", "b200_landmark_descriptors", "b200_landmark_geometry", "b200_matcher_set_stream", "b200_matcher_sync", "b200_matcher_set_async_resolve", "b200_matcher_join", "b200_matcher_enable_timing", "b200_matcher_stage_ms",
    "b200_lba_create", "b200_lba_destroy", "b200_lba_solve", "b200_lba_solve_batch", "b200_pose_optimize", "b200_lba_last_profile", "b200_lba_enable_profile", "b200_lba_kernel_ms",
    "b200_global_ba_solve", "b200_track_local_map", "b200_track_stage_ms", "b200_motion_based_track", "b200_motion_track_stage_ms", "b200_bow_match_based_track", "b200_bow_track_stage_ms", "b200_orb_export_keyframe_blobs", "b200_keyframe_blob_to_keypoints",
    "b200_triangulate_pairs", "b200_create_new_landmarks", "b200_rgbd_depths", "b200_depth_landmarks", "b200_remove_redundant_keyframes",
    "b200_rectifier_create", "b200_rectifier_destroy", "b200_rectifier_set_stream", "b200_rectifier_maps", "b200_stereo_rectify",
    "b200_stereo_rectify_device",
    "b200_pnp_ransac", "b200_epnp_compute_pose", "b200_mt19937_seed", "b200_mt19937_next", "b200_pnp_draw_min_sets",
    "b200_draw_min_sets", "b200_essential_ransac", "b200_twoview_ransac", "b200_initialize",
    "b200_graph_optimize", "b200_pgo_envelope", "b200_transform_optimize",
]


def lib():
    """Load the shared library (raises if it has not been built: run `python __graft_entry__.py` / build())."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise B200Error(ERR_CUDA, f"{LIB_PATH} is missing: the CUDA extension must be built (__graft_entry__.build()); "
                                  "there is no CPU fallback")
    L = C.CDLL(LIB_PATH)
    vp, sz, i32 = C.c_void_p, C.c_size_t, C.c_int
    L.b200_last_error.restype = C.c_char_p
    L.b200_version.restype = C.c_char_p
    L.b200_host_alloc.argtypes = [C.POINTER(vp), sz]
    L.b200_host_free.argtypes = [vp]
    L.b200_orb_default_params.argtypes = [C.POINTER(OrbParams)]
    L.b200_orb_default_params.restype = None
    L.b200_orb_create.argtypes = [C.POINTER(OrbParams), C.POINTER(vp)]
    L.b200_orb_destroy.argtypes = [vp]
    L.b200_orb_max_keypoints.argtypes = [vp, i32, i32]
    L.b200_orb_extract.argtypes = [vp, vp, i32, i32, sz, sz, i32, vp, sz, vp, vp, i32, vp]
    L.b200_orb_extract_device.argtypes = [vp, vp, i32, i32, sz, sz, i32, vp, sz]
    L.b200_orb_set_stream.argtypes = [vp, vp, i32]
    L.b200_orb_reserve.argtypes = [vp, i32, i32, i32]
    L.b200_orb_bind_outputs.argtypes = [vp, vp, vp, vp, i32]
    L.b200_orb_fetch.argtypes = [vp, vp, vp, i32, vp]
    L.b200_orb_device_results.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(i32)]
    L.b200_orb_sync.argtypes = [vp]
    L.b200_orb_level_info.argtypes = [vp, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(sz), C.POINTER(C.c_float)]
    L.b200_orb_pyramid_level_device.argtypes = [vp, i32, i32, C.POINTER(vp)]
    L.b200_orb_pyramid_level_host.argtypes = [vp, i32, i32, vp, sz]
    L.b200_orb_stage_ms.argtypes = [vp, i32, C.POINTER(C.c_float)]
    L.b200_orb_enable_timing.argtypes = [vp, i32]
    L.b200_matcher_create.argtypes = [i32, C.POINTER(vp)]
    L.b200_matcher_destroy.argtypes = [vp]
    L.b200_matcher_sync.argtypes = [vp]
    L.b200_hamming_matrix.argtypes = [vp, vp, i32, vp, i32, vp]
    L.b200_match_bruteforce.argtypes = [vp, i32, vp, vp, sz, vp, vp, vp, vp, sz, vp, vp, vp, C.c_float, i32, vp, i32, vp]
    L.b200_match_bruteforce_device.argtypes = [vp, i32, vp, vp, sz, vp, vp, vp, vp, sz, vp, vp, vp, i32, i32, C.c_float, i32,
                                               vp, i32, vp]
    L.b200_match_guided.argtypes = [vp, i32, C.POINTER(GuidedProblem), i32, C.c_uint, C.c_float, i32, i32]
    L.b200_match_cross_check.argtypes = [vp, i32, vp, i32, vp, C.POINTER(i32)]
    L.b200_match_pairs.argtypes = [vp, i32, C.POINTER(PairsProblem), i32, C.c_float, i32, i32]
    L.b200_stereo_compute.argtypes = [vp, vp, i32, vp, i32, vp, vp, i32, vp, vp, i32, C.c_float, C.c_float, vp, vp, C.POINTER(i32)]
    L.b200_orb_pyramid_level_view.argtypes = [vp, i32, i32, C.POINTER(vp), C.POINTER(sz), C.POINTER(i32), C.POINTER(i32)]
    L.b200_keypoints_undistort.argtypes = [vp, C.POINTER(CameraIntrinsics), vp, i32, vp, vp]
    L.b200_landmark_descriptors.argtypes = [vp, i32, vp, vp, vp, vp]
    L.b200_frame_can_observe.argtypes = [vp, C.POINTER(CameraIntrinsics), C.c_double, vp, vp, i32, vp, vp, vp, vp, C.c_float, C.c_uint, C.c_float,
                                         vp, vp, vp, vp]
    L.b200_landmark_geometry.argtypes = [vp, i32, vp, vp, vp, vp, vp, C.c_float, vp, vp, vp]
    L.b200_rgbd_depths.argtypes = [vp, i32, C.POINTER(CameraIntrinsics), C.c_double, C.c_double, i32, vp, i32, i32, sz, sz, i32, vp, vp, vp, vp, vp]
    L.b200_convert_to_grayscale.argtypes = [vp, vp, i32, i32, sz, i32, i32, vp, sz]
    L.b200_convert_to_grayscale_device.argtypes = [vp, vp, i32, i32, sz, sz, i32, i32, vp, sz, sz, i32]
    L.b200_matcher_set_stream.argtypes = [vp, vp, i32]
    L.b200_rectifier_create.argtypes = [C.POINTER(RectifierParams), C.POINTER(vp)]
    L.b200_rectifier_destroy.argtypes = [vp]
    L.b200_rectifier_set_stream.argtypes = [vp, vp, i32]
    L.b200_rectifier_maps.argtypes = [vp, i32, vp, vp]
    L.b200_stereo_rectify.argtypes = [vp, i32, vp, sz, vp, sz, vp, sz, vp, sz]
    L.b200_stereo_rectify_device.argtypes = [vp, i32, vp, vp, sz, sz, vp, vp, sz, sz, i32]
    _lib = L
    return L


def check(rc, allow=()):
    if rc != OK and rc not in allow:
        raise B200Error(rc, lib().b200_last_error().decode(errors="replace"))
    return rc


def ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(C.c_void_p)
    if isinstance(a, int):
        return C.c_void_p(a)
    if hasattr(a, "data_ptr"):  # torch tensor
        return C.c_void_p(a.data_ptr())
    raise TypeError(type(a))


class _PinnedOwner:
    def __init__(self, address):
        self.address = address

    def __del__(self):
        try:
            lib().b200_host_free(C.c_void_p(self.address))
        except Exception:
            pass


_PINNED = {}


def pinned_empty(shape, dtype):
    """numpy array backed by cudaHostAlloc'd memory (freed by pinned_free or at interpreter exit)."""
    dtype = np.dtype(dtype)
    n = int(np.prod(shape)) * dtype.itemsize
    p = C.c_void_p()
    check(lib().b200_host_alloc(C.byref(p), max(n, 1)))
    buf = (C.c_uint8 * max(n, 1)).from_address(p.value)
    arr = np.frombuffer(buf, dtype=np.uint8, count=n).view(dtype).reshape(shape)
    _PINNED[arr.ctypes.data] = _PinnedOwner(p.value)
    return arr


def pinned_free(arr):
    _PINNED.pop(arr.ctypes.data, None)
