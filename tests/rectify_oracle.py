"""CPU restatement of util::stereo_rectifier (test infrastructure): loads tests/rectify_oracle.c, compiled on first use into a temporary
directory (the tree is never written).  Maps as cv::initUndistortRectifyMap / cv::fisheye::initUndistortRectifyMap build them (CV_32F),
their fixed-point form and cv::remap INTER_LINEAR / BORDER_CONSTANT 0."""
import ctypes as C

import numpy as np

import cbuild

_lib = None


def lib():
    global _lib
    if _lib is None:
        L = cbuild.load("rectify_oracle.c")
        vp, sz, i32 = C.c_void_p, C.c_size_t, C.c_int
        L.orc_rect_map.argtypes = [i32, i32, i32, vp, vp, i32, vp, vp, vp, vp]
        L.orc_rect_fixed.argtypes = [sz, vp, vp, vp, vp]
        L.orc_rect_fixed.restype = None
        L.orc_rect_weights.argtypes = [vp]
        L.orc_remap.argtypes = [i32, i32, i32, vp, sz, i32, i32, vp, vp, vp, sz]
        L.orc_remap.restype = None
        _lib = L
    return _lib


def _d(a, n):
    return np.ascontiguousarray(np.asarray(a, np.float64).reshape(n))


def rect_map(model, cols, rows, K, D, R, K_rect):
    """(map_x, map_y) float32 (rows, cols).  model: "perspective" | "fisheye".  Raises ValueError where the library returns
    B200_ERR_INVALID (coefficient count, singular K_rect R)."""
    D = np.asarray(D, np.float64).reshape(-1)
    K, R, Kr, Dc = _d(K, 9), _d(R, 9), _d(K_rect, 9), np.ascontiguousarray(np.concatenate([D, np.zeros(8)])[:8])
    mx, my = np.empty((rows, cols), np.float32), np.empty((rows, cols), np.float32)
    rc = lib().orc_rect_map({"perspective": 0, "fisheye": 1}[model], cols, rows, K.ctypes.data, Dc.ctypes.data, len(D), R.ctypes.data,
                            Kr.ctypes.data, mx.ctypes.data, my.ctypes.data)
    if rc:
        raise ValueError("unsupported distortion model or singular K_rect * R")
    return mx, my


def fixed_point(map_x, map_y):
    """(sxy int16 (rows, cols, 2), frac uint16 (rows, cols))."""
    mx, my = np.ascontiguousarray(map_x, np.float32), np.ascontiguousarray(map_y, np.float32)
    sxy, frac = np.empty(mx.shape + (2,), np.int16), np.empty(mx.shape, np.uint16)
    lib().orc_rect_fixed(mx.size, mx.ctypes.data, my.ctypes.data, sxy.ctypes.data, frac.ctypes.data)
    return sxy, frac


def weights():
    """(1024, 4) int32 bilinear weight table and the number of entries whose weights do not sum to 32768."""
    t = np.empty((1024, 4), np.int32)
    bad = lib().orc_rect_weights(t.ctypes.data)
    return t, bad


def remap(src, map_x, map_y):
    """cv::remap(src, dst, map_x, map_y, INTER_LINEAR) of a (h, w) or (h, w, c) uint8 image; dst has the maps' size."""
    src = np.ascontiguousarray(src, np.uint8)
    c = 1 if src.ndim == 2 else src.shape[2]
    sxy, frac = fixed_point(map_x, map_y)
    rows, cols = frac.shape
    dst = np.empty((rows, cols) + (() if src.ndim == 2 else (c,)), np.uint8)
    lib().orc_remap(cols, rows, c, src.ctypes.data, src.strides[0], src.shape[1], src.shape[0], sxy.ctypes.data, frac.ctypes.data,
                    dst.ctypes.data, dst.strides[0])
    return dst


def rectify_pair(calib, left, right):
    """stereo_rectifier::rectify with the maps of `calib` (workloads.synth calibration dict)."""
    out = []
    for eye, img in enumerate((left, right)):
        mx, my = rect_map(calib["model"], calib["cols"], calib["rows"], calib["K"][eye], calib["D"][eye], calib["R"][eye], calib["K_rect"])
        out.append(remap(img, mx, my))
    return tuple(out)
