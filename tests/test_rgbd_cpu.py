"""CPU checks of the RGB-D frame step and the depth-seeded landmarks: the depth conversion arithmetic pinned against cv2, the CPU
restatement (tests/rgbd_oracle.c) against plain numpy / Python transcriptions of the reference, and the ctypes mirrors' layout."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import rgbd_oracle as RO  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SF = np.cumprod(np.concatenate([[np.float32(1.0)], np.full(7, np.float32(1.2))])).astype(np.float32)
INV_LAST = np.float32(np.float32(1.0) / SF[-1])


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32 if np.asarray(a).dtype == np.float32 else np.uint64)


def _alpha_for(scale, max_value):
    """An alpha for which cv::normalize(NORM_INF)'s scale alpha / max_value is exactly `scale`, so that it calls convertTo(CV_32F, scale)."""
    a = scale * max_value
    for _ in range(1000):
        q = a / max_value
        if q == scale:
            return a
        a = math.nextafter(a, math.inf if q < scale else -math.inf)
    raise AssertionError("no alpha reproduces the scale")


# ---- util::convert_to_true_depth = convertTo(CV_32F, 1.0 / depthmap_factor), pinned against cv2 ----------------------------------------
@pytest.mark.parametrize("factor", [5000.0, 1000.0, 5208.0, 0.7])
def test_cv2_u16_conversion_is_float_product(factor):
    cv2 = pytest.importorskip("cv2")
    src = np.arange(65536, dtype=np.uint16).reshape(256, 256)  # every uint16 value; the maximum is 65535
    scale = 1.0 / factor
    got = cv2.normalize(src, None, _alpha_for(scale, 65535.0), 0, cv2.NORM_INF, cv2.CV_32F)
    want = src.astype(np.float32) * np.float32(scale)
    assert np.array_equal(_bits(got), _bits(want))
    # the double product rounded once is a different function, so the probe does discriminate
    if factor in (5000.0, 1000.0):
        assert (_bits((src.astype(np.float64) * scale).astype(np.float32)) != _bits(want)).sum() > 100
    # and the oracle samples exactly these values
    kps = np.zeros(65536, RO.CM.O.KP_DTYPE)
    kps["x"], kps["y"] = np.tile(np.arange(256), 256).astype(np.float32), np.repeat(np.arange(256), 256).astype(np.float32)
    d, _ = RO.depths(kps, kps["x"], src, factor, 40.0)
    pos = want.reshape(-1) > 0
    assert np.array_equal(_bits(d[pos]), _bits(want.reshape(-1)[pos])) and np.all(d[~pos] == -1)


@pytest.mark.parametrize("factor", [1.0, 5000.0, 1000.0])
def test_cv2_f32_conversion(factor):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(int(factor))
    M = 4096.0  # a power-of-two maximum makes alpha / M exactly 1 / factor
    v = rng.uniform(-M, M, 4096).astype(np.float32)
    v[:8] = [M, 0.0, -0.0, np.nan, -1.0, 1e-30, -1e-30, np.float32(1e-42)]
    src = v.reshape(64, 64)
    scale = 1.0 / factor
    got = cv2.normalize(src, None, _alpha_for(scale, M), 0, cv2.NORM_INF, cv2.CV_32F)  # NORM_INF skips the NaN
    want = src.copy() if factor == 1.0 else src * np.float32(scale)  # factor 1: convertTo copies the data
    fin = ~np.isnan(want)
    nz = fin & (want != 0)
    # bit for bit, except that the scaled conversion adds its zero shift, which turns -0 into +0 (either is an invalid depth)
    assert np.array_equal(_bits(got[nz]), _bits(want[nz])) and np.all(got[fin & ~nz] == 0) and np.all(np.isnan(got[~fin]))
    if factor == 1.0:
        assert np.array_equal(_bits(got[fin]), _bits(want[fin]))
    # +inf cannot go through normalize (it is the norm); IEEE gives inf * scale = inf, and the oracle keeps it as a valid depth
    kps = np.zeros(6, RO.CM.O.KP_DTYPE)
    kps["x"] = np.arange(6, dtype=np.float32)
    dm = np.array([[np.inf, np.nan, -2.5, 0.0, -0.0, 2.5]], np.float32)
    d, xr = RO.depths(kps, kps["x"] + np.float32(0.25), dm, factor, 40.0)
    assert d[0] == np.inf and xr[0] == np.float32(0.25)
    assert np.all(d[1:5] == -1) and np.all(xr[1:5] == -1)
    assert d[5] == (np.float32(2.5) if factor == 1.0 else np.float32(2.5) * np.float32(scale))


# ---- the oracle's per-keypoint depth and x_right against numpy ------------------------------------------------------------------------------
def _numpy_depths(kps, ux, dm, factor, fxb):
    xi, yi = kps["x"].astype(np.int64), kps["y"].astype(np.int64)  # truncation toward zero: the coordinates are non-negative
    raw = dm[yi, xi]
    scale = np.float32(1.0 / factor)
    d = raw.astype(np.float32) * scale if (dm.dtype == np.uint16 or factor != 1.0) else raw.astype(np.float32)
    ok = d > 0
    depths = np.where(ok, d, np.float32(-1)).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        xr = (ux.astype(np.float64) - fxb / d.astype(np.float64)).astype(np.float32)
    return depths, np.where(ok, xr, np.float32(-1)).astype(np.float32)


@pytest.mark.parametrize("kind", ["u16", "f32"])
def test_oracle_depths_vs_numpy(kind):
    from workloads import synth
    _, d16, d32 = synth.make_rgbd_frames(seed=4)
    dm = d16 if kind == "u16" else d32
    rng = np.random.default_rng(1)
    n = 5000
    kps = np.zeros(n, RO.CM.O.KP_DTYPE)
    octave = rng.integers(0, 8, n)
    # level-`octave` pixel coordinates scaled to level 0: non-integer, so truncation and rounding differ
    kps["x"] = (rng.uniform(0, 639 / SF[octave]) * SF[octave]).astype(np.float32)
    kps["y"] = (rng.uniform(0, 479 / SF[octave]) * SF[octave]).astype(np.float32)
    kps["x"][:4], kps["y"][:4] = [0.0, 639.99, 10.5, 10.999], [0.0, 479.99, 10.5, 10.999]
    kps["octave"] = octave
    assert np.any(np.floor(kps["x"]) != np.rint(kps["x"]))
    ux = kps["x"] + rng.normal(0, 3, n).astype(np.float32)
    for factor in ((5000.0, 1000.0) if kind == "u16" else (1.0, 5000.0)):
        got = RO.depths(kps, ux, dm, factor, RO.TUM_FXB)
        want = _numpy_depths(kps, ux, dm, factor, RO.TUM_FXB)
        assert np.array_equal(_bits(got[0]), _bits(want[0])) and np.array_equal(_bits(got[1]), _bits(want[1]))
        assert (got[0] > 0).sum() > n // 2 and (got[0] == -1).sum() > 20


# ---- the landmark walk ----------------------------------------------------------------------------------------------------------------------
def _walk_mode0(depth, has_lm, depth_thr):
    """keyframe_inserter.cc:160-212, transcribed."""
    pairs = sorted((np.float32(d), idx) for idx, d in enumerate(depth) if 0 < d)
    out = []
    for count, (d, idx) in enumerate(pairs):
        if 100 < count and depth_thr < float(d):
            break
        if has_lm is not None and has_lm[idx]:
            continue
        out.append(idx)
    return out


def _walk_mode1(depth):
    """initializer.cc:363-387, transcribed."""
    return [idx for idx, z in enumerate(depth) if not (z <= 0) and 0 < z]


def _problem(mode, depth, has_lm=None, depth_thr=3.0, seed=0):
    rng = np.random.default_rng(seed)
    n = len(depth)
    a = rng.normal(0, 0.3, 3)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    R = np.eye(3) + math.sin(0.4) * K + (1 - math.cos(0.4)) * K @ K
    R, _ = np.linalg.qr(R)
    pose = np.eye(4)
    pose[:3, :3], pose[:3, 3] = R, rng.normal(0, 2, 3)
    return dict(mode=mode, pose_wc=pose, fx_inv=1.0 / 517.306408, fy_inv=1.0 / 516.469215, cx=318.643040, cy=255.313989, depth_thr=depth_thr,
                x=rng.uniform(0, 640, n).astype(np.float32), y=rng.uniform(0, 480, n).astype(np.float32), octave=rng.integers(0, 8, n).astype(np.int32),
                depth=np.asarray(depth, np.float32), has_landmark=has_lm, scale_factors=SF, inv_scale_factor_last=INV_LAST)


def walk_cases():
    rng = np.random.default_rng(7)
    cases = {}
    d = rng.choice(np.float32([0.5, 1.0, 1.0, 2.0, 2.0, 2.0, 4.0]), 400)  # many ties in depth
    cases["ties"] = (d, rng.random(400) < 0.2)
    d = np.concatenate([rng.uniform(0.3, 2.9, 150), rng.uniform(3.1, 9.0, 150)]).astype(np.float32)  # > 100 below and above depth_thr
    rng.shuffle(d)
    cases["many_below_and_above"] = (d, rng.random(300) < 0.3)
    d = np.concatenate([rng.uniform(0.3, 2.9, 40), rng.uniform(3.1, 9.0, 200)]).astype(np.float32)  # < 100 below: the walk stops at 101
    cases["few_below"] = (d, None)
    order = np.argsort(d, kind="stable")
    hl = np.zeros(240, bool)
    hl[order[[0, 5, 99, 100, 101, 150]]] = True  # skipped keypoints before and after position 100
    cases["skips_around_100"] = (d, hl)
    cases["no_valid_depth"] = (np.array([-1, 0, np.nan, -0.5] * 30, np.float32), None)
    d = rng.uniform(0.3, 9.0, 500).astype(np.float32)
    d[rng.random(500) < 0.3] = -1
    d[rng.random(500) < 0.05] = np.inf
    cases["invalid_and_inf"] = (d, rng.random(500) < 0.1)
    return cases


@pytest.mark.parametrize("name", sorted(walk_cases()))
def test_mode0_walk(name):
    depth, hl = walk_cases()[name]
    pr = _problem(0, depth, None if hl is None else hl.astype(np.uint8))
    got = RO.depth_landmarks(pr)
    want = _walk_mode0(pr["depth"], hl, pr["depth_thr"])
    assert got["idx"].tolist() == want
    if name == "no_valid_depth":
        assert len(want) == 0
    if name == "many_below_and_above":
        assert 101 < len(want) + (hl[want].sum() if len(want) else 0) < 300


@pytest.mark.parametrize("name", sorted(walk_cases()))
def test_mode1_walk(name):
    depth, hl = walk_cases()[name]
    pr = _problem(1, depth, None if hl is None else hl.astype(np.uint8))  # has_landmark is not read in mode 1
    assert RO.depth_landmarks(pr)["idx"].tolist() == _walk_mode1(pr["depth"])


def test_unprojection_and_geometry_vs_numpy():
    rng = np.random.default_rng(3)
    pr = _problem(1, rng.uniform(0.3, 10.0, 300).astype(np.float32), seed=3)
    got = RO.depth_landmarks(pr)
    P = pr["pose_wc"]
    for k, idx in enumerate(got["idx"]):
        z = float(pr["depth"][idx])
        ux = float(np.float32((float(pr["x"][idx]) - pr["cx"]) * z * pr["fx_inv"]))
        uy = float(np.float32((float(pr["y"][idx]) - pr["cy"]) * z * pr["fy_inv"]))
        pw = [((P[r, 0] * ux + P[r, 1] * uy) + P[r, 2] * z) + P[r, 3] for r in range(3)]
        assert got["pos_w"][k].tolist() == pw
        v = [pw[r] - P[r, 3] for r in range(3)]
        nrm = math.sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2])
        m = [0.0 + v[r] / nrm for r in range(3)]
        mn = math.sqrt((m[0] * m[0] + m[1] * m[1]) + m[2] * m[2])
        assert got["mean_normal"][k].tolist() == [m[r] / mn for r in range(3)]
        mx = np.float32(nrm * float(SF[pr["octave"][idx]]))
        assert got["max_valid_dist"][k] == mx and got["min_valid_dist"][k] == np.float32(mx * INV_LAST)
        # and the point lies on the keypoint's ray at the given depth
        pc = P[:3, :3].T @ (np.array(pw) - P[:3, 3])
        assert abs(pc[2] - z) < 1e-9 * max(1.0, z)


# ---- ctypes mirrors --------------------------------------------------------------------------------------------------------------------------
def test_ctypes_layout(tmp_path):
    from stella_vslam_b200 import mapping
    mirrors = {"b200_depth_landmarks_problem_t": mapping.DepthLandmarksProblem}
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "b200vslam.h"', "int main(void) {"]
    for cname, T in mirrors.items():
        lines.append(f'  printf("{cname} __sizeof__ %zu\\n", sizeof({cname}));')
        for fname, _ in T._fields_:
            lines.append(f'  printf("{cname} {fname} %zu\\n", offsetof({cname}, {fname}));')
    lines.append('  printf("consts %d %d %d %d %d\\n", B200_DEPTH_16UC1, B200_DEPTH_32FC1, B200_DEPTH_LM_KEYFRAME, B200_DEPTH_LM_INITIAL, '
                 'B200_DEPTH_LM_MAX_SORT);')
    lines += ["  return 0;", "}"]
    src, exe = tmp_path / "probe.c", tmp_path / "probe.exe"
    src.write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    want = {}
    for ln in subprocess.check_output([str(exe)], text=True).splitlines():
        parts = ln.split()
        if parts[0] == "consts":
            assert [int(v) for v in parts[1:]] == [2, 5, mapping.DEPTH_LANDMARKS_KEYFRAME, mapping.DEPTH_LANDMARKS_INITIAL,
                                                   mapping.DEPTH_LANDMARKS_MAX_SORT]
            continue
        want[(parts[0], parts[1])] = int(parts[2])
    for cname, T in mirrors.items():
        assert C.sizeof(T) == want[(cname, "__sizeof__")]
        for fname, _ in T._fields_:
            assert getattr(T, fname).offset == want[(cname, fname)], (cname, fname)
