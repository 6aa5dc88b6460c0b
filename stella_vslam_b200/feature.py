"""Host-side mirror of the reference's feature:: surface (src/stella_vslam/feature/orb_params.h, orb_extractor.h).

Same names, argument meaning and error behaviour as the C++ classes, on top of the C ABI (include/b200vslam.h):
  feature::orb_params      orb_params.cc:12-71
  feature::orb_extractor   orb_extractor.h:51-71, orb_extractor.cc:16-136
cv::Mat inputs become 2-D uint8 numpy arrays; std::vector<cv::KeyPoint> becomes a structured array with the
cv::KeyPoint fields the reference fills (class_id is always -1 and is not stored).
"""
import ctypes as C
import math

import numpy as np

from . import _lib
from ._lib import KP_DTYPE, OrbParams, check, lib, ptr


class descriptor_type:  # feature/orb_extractor.h:17-44
    ORB = 0
    HASH_SIFT = 1


class orb_params:
    """feature::orb_params: pyramid scale tables built with the reference's float recurrences (orb_params.cc:37-71)."""

    def __init__(self, name="default ORB feature extraction setting", scale_factor=1.2, num_levels=8, ini_fast_thr=20,
                 min_fast_thr=7):
        self.name_ = name
        self.scale_factor_ = np.float32(scale_factor)
        self.log_scale_factor_ = np.float32(np.log(np.float32(scale_factor)))
        self.num_levels_ = int(num_levels)
        self.ini_fast_thr_ = int(ini_fast_thr)
        self.min_fast_thr_ = int(min_fast_thr)
        sf, inv, sig, isig = [np.float32(1.0)], [np.float32(1.0)], [np.float32(1.0)], [np.float32(1.0)]
        s = np.float32(1.0)
        for _ in range(1, self.num_levels_):
            s = self.scale_factor_ * s
            sf.append(s)
            inv.append((np.float32(1.0) / self.scale_factor_) * inv[-1])
            sig.append(s * s)
            isig.append(np.float32(1.0) / (s * s))
        self.scale_factors_ = np.array(sf, np.float32)
        self.inv_scale_factors_ = np.array(inv, np.float32)
        self.level_sigma_sq_ = np.array(sig, np.float32)
        self.inv_level_sigma_sq_ = np.array(isig, np.float32)

    @classmethod
    def from_yaml(cls, node):
        """orb_params(const YAML::Node&) (orb_params.cc:22-27): `node` is the dict of the `Feature:` block."""
        return cls(node.get("name", "default ORB feature extraction setting"), node.get("scale_factor", 1.2),
                   node.get("num_levels", 8), node.get("ini_fast_threshold", 20), node.get("min_fast_threshold", 7))

    def to_json(self):
        return {"name": self.name_, "scale_factor": float(self.scale_factor_), "num_levels": self.num_levels_,
                "ini_fast_threshold": self.ini_fast_thr_, "min_fast_threshold": self.min_fast_thr_}


class orb_extractor:
    """feature::orb_extractor on the GPU.  `extract` handles one frame like the reference; `extract_batch` takes a
    stack of same-sized frames (the GPU-native entry: one launch sequence for the whole batch)."""

    def __init__(self, orb_params_, min_area, desc_type=descriptor_type.ORB, mask_rects=(), device=0, max_batch=1):
        if desc_type == descriptor_type.HASH_SIFT:
            # orb_extractor.cc:117-122 without USE_CUDA_EFFICIENT_DESCRIPTORS
            raise RuntimeError("cuda_efficient_features is not available")
        if desc_type != descriptor_type.ORB:
            raise RuntimeError("Invalid descriptor_type")  # orb_extractor.cc:125
        self.orb_params_ = orb_params_
        self.mask_rects_ = [list(map(float, r)) for r in mask_rects]
        self.image_pyramid_ = []
        self._rects = np.ascontiguousarray(np.array(self.mask_rects_, np.float32).reshape(-1, 4))
        p = OrbParams()
        lib().b200_orb_default_params(C.byref(p))
        p.scale_factor = float(orb_params_.scale_factor_)
        p.num_levels = orb_params_.num_levels_
        p.ini_fast_thr = orb_params_.ini_fast_thr_
        p.min_fast_thr = orb_params_.min_fast_thr_
        p.min_area = int(min_area)
        p.n_mask_rects = self._rects.shape[0]
        p.mask_rects = self._rects.ctypes.data_as(C.POINTER(C.c_float)) if self._rects.size else None
        p.device = device
        p.max_batch = max_batch
        self._h = C.c_void_p()
        check(lib().b200_orb_create(C.byref(p), C.byref(self._h)))
        self._shape = None

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            lib().b200_orb_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- reference signature: extract(in_image, in_image_mask, keypts, out_descriptors) ------------------------------
    def extract(self, in_image, in_image_mask=None):
        """Returns (keypts, descriptors).  Empty image -> ([], None-like empty) as orb_extractor.cc:30-32,72-74."""
        img = np.asarray(in_image)
        if img.size == 0:
            return np.zeros(0, KP_DTYPE), np.zeros((0, 32), np.uint8)
        k, d = self.extract_batch(img[None], in_image_mask)
        return k[0], d[0]

    def extract_batch(self, images, in_image_mask=None, cap=None):
        images = np.asarray(images)
        assert images.dtype == np.uint8 and images.ndim == 3, "image.type() == CV_8UC1"  # orb_extractor.cc:36
        images = np.ascontiguousarray(images)
        b, h, w = images.shape
        if b == 0 or h == 0 or w == 0:
            return [], []
        mask = None
        if in_image_mask is not None and np.asarray(in_image_mask).size:
            mask = np.ascontiguousarray(in_image_mask, np.uint8)
            assert mask.shape == (h, w), "image mask must have the image's size"
        if cap is None:
            cap = check_pos(lib().b200_orb_max_keypoints(self._h, w, h))
        kps = np.zeros((b, max(cap, 1)), KP_DTYPE)
        desc = np.zeros((b, max(cap, 1), 32), np.uint8)
        counts = np.zeros(b, np.int32)
        check(lib().b200_orb_extract(self._h, ptr(images), w, h, images.strides[1], images.strides[0], b, ptr(mask),
                                     mask.strides[0] if mask is not None else 0, ptr(kps), ptr(desc), cap, ptr(counts)))
        self._shape = (b, h, w)
        self._last_images = images
        return [kps[f, :counts[f]].copy() for f in range(b)], [desc[f, :counts[f]].copy() for f in range(b)]

    def image_pyramid(self, frame=0):
        """orb_extractor::image_pyramid_ (orb_extractor.h:71) of the last extract, copied back to the host."""
        if self._shape is None:
            return []
        out = [self._last_images[frame]]
        for l in range(1, self.orb_params_.num_levels_):
            w, h = C.c_int(), C.c_int()
            check(lib().b200_orb_level_info(self._h, l, C.byref(w), C.byref(h), None, None))
            lv = np.empty((h.value, w.value), np.uint8)
            check(lib().b200_orb_pyramid_level_host(self._h, frame, l, ptr(lv), lv.strides[0]))
            out.append(lv)
        self.image_pyramid_ = out
        return out

    def undistort_keypoints(self, camera, dist_keypts, want_bearings=True):
        """camera::*::undistort_keypoints + camera::base::convert_keypoints_to_bearings (camera/perspective.cc:245-275, 117-122;
        equirectangular.cc:42-49; fisheye.cc:281-309, 156-161; radial_division.cc:83-105; called right after extract,
        system.cc:386-395).  camera: dict(model="perspective"|"equirectangular"|"fisheye"|"radial_division", fx, fy, cx, cy,
        k1, k2, p1, p2, k3 (perspective), k1, k2, k3, k4 (fisheye), distortion (radial division), cols, rows).
        Returns (undist_keypts, bearings (n, 3) float64 | None)."""
        kps = np.ascontiguousarray(dist_keypts, KP_DTYPE)
        n = len(kps)
        cam = _lib.camera_intrinsics(camera)
        out = np.zeros(n, KP_DTYPE)
        bearings = np.zeros((n, 3)) if want_bearings else None
        if n:
            check(lib().b200_keypoints_undistort(self._h, C.byref(cam), ptr(kps), n, ptr(out), ptr(bearings)))
        return out, bearings

    def rgbd_depths(self, camera, depth_maps, depthmap_factor, focal_x_baseline, n_frames=None, cap=None):
        """system::create_RGBD_frame after the extraction (system.cc:467-530) for the first n_frames frames of the last extract (all of
        them by default): undistorted keypoints and bearings as undistort_keypoints gives them, the depth sampled at each distorted
        keypoint after util::convert_to_true_depth(depthmap_factor), and x_right = undist_x - focal_x_baseline / depth (-1 / -1 where
        the depth is not positive).  depth_maps: (h, w) or (n, h, w) uint16 (CV_16UC1) or float32 (CV_32FC1) numpy array of the
        extracted frames' size.  Returns one dict(undist_keypts, bearings, depths, x_right) per frame."""
        maps = np.asarray(depth_maps)
        if maps.ndim == 2:
            maps = maps[None]
        types = {np.dtype(np.uint16): 2, np.dtype(np.float32): 5}  # B200_DEPTH_16UC1 / B200_DEPTH_32FC1
        if maps.ndim != 3 or maps.dtype not in types:
            raise ValueError(f"depth maps must be (h, w) or (n, h, w) uint16 or float32 arrays, got {maps.dtype} {maps.shape}")
        maps = np.ascontiguousarray(maps)
        n = maps.shape[0] if n_frames is None else int(n_frames)
        if n > maps.shape[0]:
            raise ValueError(f"{n} frames requested, {maps.shape[0]} depth maps given")
        if cap is None:
            cap = check_pos(lib().b200_orb_max_keypoints(self._h, maps.shape[2], maps.shape[1]))
        und = np.zeros((max(n, 1), max(cap, 1)), KP_DTYPE)
        bearings = np.zeros((max(n, 1), max(cap, 1), 3))
        depths, x_right = np.zeros((max(n, 1), max(cap, 1)), np.float32), np.zeros((max(n, 1), max(cap, 1)), np.float32)
        counts = np.zeros(max(n, 1), np.int32)
        cam = _lib.camera_intrinsics(camera)
        check(lib().b200_rgbd_depths(self._h, n, C.byref(cam), float(focal_x_baseline), float(depthmap_factor), types[maps.dtype], ptr(maps),
                                     maps.shape[2], maps.shape[1], maps.strides[1], maps.strides[0], cap, ptr(und), ptr(bearings), ptr(depths),
                                     ptr(x_right), ptr(counts)))
        return [dict(undist_keypts=und[f, :counts[f]].copy(), bearings=bearings[f, :counts[f]].copy(), depths=depths[f, :counts[f]].copy(),
                     x_right=x_right[f, :counts[f]].copy()) for f in range(n)]

    def can_observe(self, camera, pose_cw, landmarks, ray_cos_thr=0.5, img_bounds=None):
        """data::frame::can_observe (data/frame.cc:59-84) for the local landmarks (tracking_module.cc:559-594).
        landmarks: dict(pos_w (n,3), mean_normal (n,3), min_valid_dist (n,), max_valid_dist (n,)).
        Returns dict(observable bool (n,), reproj (n,2), x_right (n,), pred_scale_level (n,)) -- the inputs of
        match.projection.match_frame_and_landmarks.  Without img_bounds, fisheye and radial-division cameras use
        camera_image_bounds(camera, self), the other models (0, cols, 0, rows)."""
        pos = np.ascontiguousarray(landmarks["pos_w"], np.float64).reshape(-1, 3)
        nml = np.ascontiguousarray(landmarks["mean_normal"], np.float64).reshape(-1, 3)
        lo = np.ascontiguousarray(landmarks["min_valid_dist"], np.float32)
        hi = np.ascontiguousarray(landmarks["max_valid_dist"], np.float32)
        n = len(pos)
        cam = _lib.camera_intrinsics(camera)
        if img_bounds is None:
            img_bounds = camera_image_bounds(camera, self) if cam.model in (2, 3) else (0.0, camera.get("cols", 0.0), 0.0, camera.get("rows", 0.0))
        bounds = np.ascontiguousarray(img_bounds, np.float32)
        pose = np.ascontiguousarray(pose_cw, np.float64).reshape(4, 4)
        ok, rp = np.zeros(max(n, 1), np.uint8), np.zeros((max(n, 1), 2))
        xr, lv = np.zeros(max(n, 1), np.float32), np.zeros(max(n, 1), np.uint32)
        check(lib().b200_frame_can_observe(self._h, C.byref(cam), float(camera.get("fxb", 0.0)), ptr(bounds), ptr(pose), n, ptr(pos), ptr(nml), ptr(lo),
                                           ptr(hi), float(ray_cos_thr), int(self.orb_params_.num_levels_), float(self.orb_params_.log_scale_factor_),
                                           ptr(ok), ptr(rp), ptr(xr), ptr(lv)))
        return dict(observable=ok[:n].astype(bool), reproj=rp[:n], x_right=xr[:n], pred_scale_level=lv[:n])

    def convert_to_grayscale(self, img, in_color_order="BGR"):
        """util::convert_to_grayscale (util/image_converter.cc:8-39): (h, w, 3|4) uint8 -> (h, w) uint8; a 1-channel image or
        in_color_order == "Gray" is returned unchanged."""
        img = np.asarray(img)
        if img.ndim == 2 or in_color_order == "Gray":
            return img
        img = np.ascontiguousarray(img, np.uint8)
        h, w, c = img.shape
        out = np.empty((h, w), np.uint8)
        check(lib().b200_convert_to_grayscale(self._h, ptr(img), w, h, img.strides[0], c, 1 if in_color_order == "RGB" else 0, ptr(out), out.strides[0]))
        return out

    def enable_timing(self, on=True):
        check(lib().b200_orb_enable_timing(self._h, int(on)))

    def stage_ms(self):
        out = []
        for s in range(6):
            v = C.c_float()
            check(lib().b200_orb_stage_ms(self._h, s, C.byref(v)))
            out.append(v.value)
        return out


class stereo_rectifier:
    """util::stereo_rectifier (util/stereo_rectifier.cc:12-66) on the GPU: both eyes' undistort-and-rectify maps are built once when
    the object is made, and `rectify` is cv::remap(INTER_LINEAR) of a pair, bit-exact to OpenCV.  Frames are 8-bit with 1, 3 or 4
    channels: (h, w) or (h, w, c) numpy arrays for `rectify`, torch CUDA tensors for `rectify_device`."""

    MODELS = {"perspective": 0, "fisheye": 1}

    def __init__(self, model, cols, rows, K_rect, K_left, D_left, R_left, K_right, D_right, R_right, device=0):
        if model not in self.MODELS:  # stereo_rectifier.cc:52-54 (equirectangular)
            raise RuntimeError("Invalid model type for stereo rectification: " + str(model))
        p = _lib.RectifierParams()
        p.model, p.cols, p.rows, p.device = self.MODELS[model], int(cols), int(rows), int(device)
        p.K_rect[:] = [float(v) for v in np.asarray(K_rect, np.float64).reshape(9)]
        for eye, (K, D, R) in enumerate(((K_left, D_left, R_left), (K_right, D_right, R_right))):
            D = np.asarray(D, np.float64).reshape(-1)
            if len(D) > 8:
                raise RuntimeError(f"{len(D)} distortion coefficients: the thin-prism and tilt models are not supported")
            p.K[eye][:] = [float(v) for v in np.asarray(K, np.float64).reshape(9)]
            p.R[eye][:] = [float(v) for v in np.asarray(R, np.float64).reshape(9)]
            p.D[eye][:len(D)] = [float(v) for v in D]
            p.n_dist[eye] = len(D)
        self.model_type_, self.cols_, self.rows_ = model, int(cols), int(rows)
        self._h = C.c_void_p()
        check(lib().b200_rectifier_create(C.byref(p), C.byref(self._h)))

    @staticmethod
    def load_model_type(rectifier_node):
        """stereo_rectifier::load_model_type (stereo_rectifier.cc:75-89): `model` defaults to "perspective"."""
        m = rectifier_node.get("model", "perspective")
        if m not in ("perspective", "fisheye", "equirectangular"):
            raise RuntimeError("Invalid camera model: " + str(m))
        return m

    @staticmethod
    def parse_vector_as_mat(shape, vec):
        """stereo_rectifier::parse_vector_as_mat: the first rows x cols entries of a YAML list as a float64 matrix (row-major)."""
        cols, rows = shape
        v = np.asarray(vec, np.float64).reshape(-1)
        if v.size < rows * cols:
            raise RuntimeError(f"expected {rows * cols} values, got {v.size}")
        return v[:rows * cols].reshape(rows, cols).copy()

    @classmethod
    def from_yaml(cls, camera_node, rectifier_node, device=0):
        """stereo_rectifier(camera, yaml_node) (stereo_rectifier.cc:16-56).  camera_node: the `Camera:` block as a dict (the camera
        the rectified frames feed), rectifier_node: the `StereoRectifier:` block."""
        return cls(**cls.parse_yaml(camera_node, rectifier_node), device=device)

    @classmethod
    def parse_yaml(cls, camera_node, rectifier_node):
        """The constructor's checks and parsing, in the reference's order, as keyword arguments of stereo_rectifier(...).  K_rect is
        the rectified camera's cv_cam_matrix_, which the reference stores as CV_32F: fx, fy, cx, cy are rounded to float."""
        model = cls.load_model_type(rectifier_node)
        if camera_node.get("setup") != "stereo":
            raise RuntimeError("When stereo rectification is used, 'setup' must be set to 'stereo'")
        if camera_node.get("model") != "perspective":
            raise RuntimeError("When stereo rectification is used, 'model' must be set to 'perspective'")
        f32 = [float(np.float32(camera_node[k])) for k in ("fx", "fy", "cx", "cy")]
        K_rect = np.array([[f32[0], 0.0, f32[2]], [0.0, f32[1], f32[3]], [0.0, 0.0, 1.0]])
        mat = cls.parse_vector_as_mat
        args = dict(K_left=mat((3, 3), rectifier_node["K_left"]), K_right=mat((3, 3), rectifier_node["K_right"]),
                    R_left=mat((3, 3), rectifier_node["R_left"]), R_right=mat((3, 3), rectifier_node["R_right"]),
                    D_left=np.asarray(rectifier_node["D_left"], np.float64).reshape(-1), D_right=np.asarray(rectifier_node["D_right"], np.float64).reshape(-1))
        if model == "equirectangular":  # the camera's model string, as camera::base::get_model_type_string gives it
            raise RuntimeError("Invalid model type for stereo rectification: " + camera_node["model"])
        return dict(model=model, cols=int(camera_node["cols"]), rows=int(camera_node["rows"]), K_rect=K_rect, **args)

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            lib().b200_rectifier_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def maps(self, eye):
        """(map_x, map_y) float32 (rows, cols) of eye 0 (left) or 1 (right): the reference's undist_map_{x,y}_{l,r}_."""
        mx, my = np.empty((self.rows_, self.cols_), np.float32), np.empty((self.rows_, self.cols_), np.float32)
        check(lib().b200_rectifier_maps(self._h, int(eye), ptr(mx), ptr(my)))
        return mx, my

    def _channels(self, img):
        if img.dtype != np.uint8 or img.shape[:2] != (self.rows_, self.cols_) or img.ndim not in (2, 3) or (img.ndim == 3 and img.shape[2] not in (1, 3, 4)):
            raise ValueError(f"expected uint8 ({self.rows_}, {self.cols_}[, 1|3|4]) frames, got {img.dtype} {img.shape}")
        return 1 if img.ndim == 2 else img.shape[2]

    def rectify(self, in_img_l, in_img_r):
        """stereo_rectifier::rectify: (out_img_l, out_img_r) with the inputs' shape and type."""
        l, r = np.ascontiguousarray(in_img_l), np.ascontiguousarray(in_img_r)
        c = self._channels(l)
        if self._channels(r) != c:
            raise ValueError("both eyes must have the same number of channels")
        ol, orr = np.empty_like(l), np.empty_like(r)
        check(lib().b200_stereo_rectify(self._h, c, ptr(l), l.strides[0], ptr(r), r.strides[0], ptr(ol), ol.strides[0], ptr(orr), orr.strides[0]))
        return ol, orr

    def set_stream(self, stream=None):
        """Run rectify_device on a torch / CUDA stream (an object with .cuda_stream, or a raw handle); None restores the own stream."""
        if stream is None:
            check(lib().b200_rectifier_set_stream(self._h, None, 1))
        else:
            check(lib().b200_rectifier_set_stream(self._h, C.c_void_p(getattr(stream, "cuda_stream", stream)), 0))

    def rectify_device(self, left, right, out_left, out_right):
        """b200_stereo_rectify_device on torch uint8 CUDA tensors of shape (B, rows, cols[, c]).  Each tensor's strides give the row
        pitch and the frame stride (dims 0 and 1), so views such as out[0::2] / out[1::2] of one (2B, rows, cols) tensor interleave
        the eyes.  Enqueued on the rectifier's stream (see set_stream) without synchronising."""
        if left.dim() not in (3, 4) or tuple(left.shape[1:3]) != (self.rows_, self.cols_) or left.shape != right.shape \
                or out_left.shape != left.shape or out_right.shape != left.shape:
            raise ValueError("left, right and outputs must be (B, rows, cols[, c]) tensors of the rectifier's size")
        c = 1 if left.dim() == 3 else int(left.shape[3])
        for a, b in ((left, right), (out_left, out_right)):
            for t in (a, b):
                if t.stride()[:2] != a.stride()[:2] or t.stride(2) != c or (t.dim() == 4 and t.stride(3) != 1):
                    raise ValueError("rows must be dense (channels interleaved) and both eyes must share pitch and frame stride")
        b = int(left.shape[0])
        check(lib().b200_stereo_rectify_device(self._h, c, ptr(left), ptr(right), left.stride(1), left.stride(0), ptr(out_left), ptr(out_right),
                                               out_left.stride(1), out_left.stride(0), b))


def camera_image_bounds(camera, extractor):
    """camera::*::compute_image_bounds (perspective.cc:70-95, equirectangular.cc:32-36, fisheye.cc:68-135, radial_division.cc:61-81):
    (min_x, max_x, min_y, max_y) as the floats of camera::image_bounds.  The corner / edge-midpoint keypoints are undistorted by
    extractor.undistort_keypoints (the device's undistortion); float and double steps are those of the reference."""
    cam = _lib.camera_intrinsics(camera)
    f32 = lambda v: float(np.float32(v))
    g = lambda k: float(camera.get(k, 0.0))
    cols, rows = f32(int(g("cols"))), f32(int(g("rows")))  # cols_ / rows_ are unsigned int
    no_dist = {0: all(g(k) == 0 for k in ("k1", "k2", "p1", "p2", "k3")), 1: True,
               2: all(g(k) == 0 for k in ("k1", "k2", "k3", "k4")), 3: g("distortion") == 0.0}[cam.model]
    if no_dist:
        return (0.0, cols, 0.0, rows)

    def undistort(pts):  # cv::KeyPoint(x, y, 1.0): float coordinates
        kps = np.zeros(len(pts), KP_DTYPE)
        kps["x"], kps["y"], kps["size"] = [p[0] for p in pts], [p[1] for p in pts], 1.0
        und, _ = extractor.undistort_keypoints(camera, kps, want_bearings=False)
        return [(float(k["x"]), float(k["y"])) for k in und]

    fx, fy, cx, cy = g("fx"), g("fy"), g("cx"), g("cy")
    if cam.model == 2:
        pwx, pwy = (0.0 - cx) / fx, (0.0 - cy) / fy
        if math.sqrt(pwx * pwx + pwy * pwy) > math.pi / 2:  # super-wide FOV: the four corners are out of view (fisheye.cc:83-115)
            u = undistort([(f32(cx), 0.0), (cols, f32(cy)), (0.0, f32(cy)), (f32(cx), rows)])
            deg_thr = 5.0  # constexpr float 5.0; deg_thr * M_PI / 180.0 is double
            dist_thr_x, dist_thr_y = f32(fx / math.tan(deg_thr * math.pi / 180.0)), f32(fy / math.tan(deg_thr * math.pi / 180.0))
            min_x_thr, max_x_thr = f32(-dist_thr_x + cx), f32(dist_thr_x + cx)
            min_y_thr, max_y_thr = f32(-dist_thr_y + cy), f32(dist_thr_y + cy)
            umin_x, umax_x, umin_y, umax_y = u[2][0], u[1][0], u[0][1], u[3][1]
            return (min_x_thr if (umin_x < min_x_thr or umin_x > cx) else umin_x, max_x_thr if (umax_x > max_x_thr or umax_x < cx) else umax_x,
                    min_y_thr if (umin_y < min_y_thr or umin_y > cy) else umin_y, max_y_thr if (umax_y > max_y_thr or umax_y < cy) else umax_y)
    u = undistort([(0.0, 0.0), (cols, 0.0), (0.0, rows), (cols, rows)])
    return (min(u[0][0], u[2][0]), max(u[1][0], u[3][0]), min(u[0][1], u[1][1]), max(u[2][1], u[3][1]))


def check_pos(v):
    if v < 0:
        check(v)
    return v
