"""Keyframe serialisation formats of the reference (SURVEY 8f N4), host-side mirror:
  data::convert_keypoints_to_json / convert_json_to_keypoints       src/stella_vslam/data/common.cc:32-55
  data::convert_descriptors_to_json / convert_json_to_descriptors   src/stella_vslam/data/common.cc:57-81
  data::keyframe::to_db / from_stmt blobs                           src/stella_vslam/data/keyframe.cc:298-347, 191-235
The bytes come from the GPU in the blob layout (b200_orb_export_keyframe_blobs); the JSON forms are views of the same bytes."""
import ctypes as C

import numpy as np

from ._lib import KP_DTYPE, CameraIntrinsics, camera_intrinsics, check, lib, ptr

# cv::KeyPoint as stored in the `undist_keypts` blob: 28 bytes
CV_KEYPOINT_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"), ("octave", "<i4"), ("class_id", "<i4")])
assert CV_KEYPOINT_DTYPE.itemsize == 28


def export_keyframe_blobs(extractor, frame=0, camera=None):
    """(undist_keypts blob, descriptor blob) of frame `frame` of the extractor's last batch, as bytes-compatible numpy arrays:
    keypoints (n,) CV_KEYPOINT_DTYPE -- `.tobytes()` is what keyframe::to_db binds (:324-330) -- and descriptors (n, 32) uint8 (:343-347)."""
    L = lib()
    L.b200_orb_export_keyframe_blobs.argtypes = [C.c_void_p, C.c_int, C.POINTER(CameraIntrinsics), C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int32)]
    b, h, w = extractor._shape
    cap = L.b200_orb_max_keypoints(extractor._h, w, h)
    kp = np.zeros(max(cap, 1), CV_KEYPOINT_DTYPE)
    desc = np.zeros((max(cap, 1), 32), np.uint8)
    n = C.c_int32()
    cam = None
    if camera is not None:
        cam = camera_intrinsics(camera)
    check(L.b200_orb_export_keyframe_blobs(extractor._h, int(frame), C.byref(cam) if cam is not None else None, ptr(kp), ptr(desc), cap, C.byref(n)))
    return kp[:n.value].copy(), desc[:n.value].copy()


def keypoints_from_blob(blob):
    """keyframe::from_stmt (:198-201): raw cv::KeyPoint bytes (or a CV_KEYPOINT_DTYPE array) -> the library's keypoint records."""
    src = np.frombuffer(blob, CV_KEYPOINT_DTYPE) if isinstance(blob, (bytes, bytearray, memoryview)) else np.ascontiguousarray(blob, CV_KEYPOINT_DTYPE)
    out = np.zeros(len(src), KP_DTYPE)
    L = lib()
    L.b200_keyframe_blob_to_keypoints.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    check(L.b200_keyframe_blob_to_keypoints(ptr(np.ascontiguousarray(src)), len(src), ptr(out)))
    return out


def convert_descriptors_to_json(descriptors):
    """common.cc:57-69: one list of eight uint32 per descriptor row (`desc.ptr<uint32_t>()`, host byte order = little endian)."""
    d = np.ascontiguousarray(descriptors, np.uint8).reshape(-1, 32)
    return d.view("<u4").reshape(-1, 8).tolist()


def convert_json_to_descriptors(json_descriptors):
    """common.cc:71-81."""
    a = np.asarray(json_descriptors, dtype=np.uint64).reshape(-1, 8)
    assert (a <= 0xFFFFFFFF).all(), "descriptor words are uint32"
    return a.astype("<u4").view(np.uint8).reshape(-1, 32)


def convert_keypoints_to_json(keypts):
    """common.cc:32-41: pt, ang, oct (size / response / class_id are not stored)."""
    return [{"pt": [float(k["x"]), float(k["y"])], "ang": float(k["angle"]), "oct": int(np.uint32(k["octave"]))} for k in keypts]


def convert_json_to_keypoints(json_keypts):
    """common.cc:43-55: cv::KeyPoint(x, y, size = 0, angle, response = 0, octave, class_id = -1)."""
    out = np.zeros(len(json_keypts), CV_KEYPOINT_DTYPE)
    for i, j in enumerate(json_keypts):
        out[i] = (np.float32(j["pt"][0]), np.float32(j["pt"][1]), 0.0, np.float32(j["ang"]), 0.0, int(j["oct"]), -1)
    return out
