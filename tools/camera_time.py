"""Time the fisheye front end on one GPU:
  undistort    b200_keypoints_undistort + bearings for 64 x 2 000 keypoints of a TUM-VI fisheye camera (one call, one launch): the
               end-to-end host-call wall time (upload, kernel, download) and the kernel time from torch.profiler;
  chain        stage 0 of b200_track_local_map (undistort + can_observe + query build) for a 64-frame batch of 512 x 512 frames with the
               TUM-VI fisheye calibration, against the same batch with EuRoC's perspective intrinsics (CUDA events of the chain);
  cv2          single-thread cv2.fisheye.undistortPoints on the same 128 000 points, called as camera::fisheye calls it (float K and D).
Medians of the repetitions.  Prints the card and its power limit (read-only nvidia-smi query, in the same run).

    python tools/camera_time.py [--reps 20] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402

from stella_vslam_b200 import _lib, feature, tracking  # noqa: E402
from workloads import synth  # noqa: E402

TUM_VI = dict(model="fisheye", fx=190.97847715128717, fy=190.9733070521226, cx=254.93170605935475, cy=256.8974428996504, k1=0.0034823894022493434,
              k2=0.0007150348452162257, k3=-0.0020532361418706202, k4=0.00020293673591811182, cols=512.0, rows=512.0)
EUROC = dict(model="perspective", fx=458.654, fy=457.296, cx=367.215, cy=248.375, k1=-0.28340811, k2=0.07395907, p1=0.00019359, p2=1.76187114e-05,
             k3=0.0, cols=512.0, rows=512.0)


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True)
        return q.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def median_ms(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return round(float(np.median(ts)) * 1e3, 4)


def kernel_ms(fn, name):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            fn()
    ev = [e for e in prof.events() if name in e.name]
    return round(sum(e.device_time for e in ev) / max(len(ev), 1) / 1e3, 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card=card())
    ex = feature.orb_extractor(feature.orb_params(), 800, max_batch=64)
    rng = np.random.default_rng(0)
    kps = np.zeros(64 * 2000, _lib.KP_DTYPE)
    kps["x"], kps["y"] = rng.uniform(0, 512, len(kps)), rng.uniform(0, 512, len(kps))
    kps["size"], kps["octave"] = 31.0, rng.integers(0, 8, len(kps))
    run = lambda: ex.undistort_keypoints(TUM_VI, kps)
    res["undistort_128k_host_call_ms"] = median_ms(run, a.reps)
    res["undistort_128k_kernel_ms"] = kernel_ms(run, "undistort_bearings_kernel")
    try:
        import cv2
        cv2.setNumThreads(1)
        K = np.array([[TUM_VI["fx"], 0, TUM_VI["cx"]], [0, TUM_VI["fy"], TUM_VI["cy"]], [0, 0, 1]], np.float32)
        D = np.array([TUM_VI[k] for k in ("k1", "k2", "k3", "k4")], np.float32)
        pts = np.stack([kps["x"], kps["y"]], 1).reshape(-1, 1, 2).astype(np.float32)
        res["cv2_fisheye_undistort_128k_1thread_ms"] = median_ms(lambda: cv2.fisheye.undistortPoints(pts, K, D, R=None, P=K), max(3, a.reps // 4))
    except ImportError:
        res["cv2_fisheye_undistort_128k_1thread_ms"] = None
    imgs = np.stack([synth.make_frame(512, 512, seed=600 + i) for i in range(64)])
    fk, fd = ex.extract_batch(imgs)
    res["chain_keypoints"] = int(sum(len(k) for k in fk))
    for label, cam in (("tum_vi_fisheye", TUM_VI), ("euroc_perspective", EUROC)):
        c = dict(cam, fxb=0.0, setup="monocular")
        und = [ex.undistort_keypoints(c, k, want_bearings=False)[0] for k in fk]
        frames = [dict(synth.make_tracking_frame(und[i], fd[i], c, ex.orb_params_.scale_factors_, seed=700 + i), frame=i) for i in range(64)]
        tr = tracking.local_map_tracker(ex, c, grid=(16, 16))
        packed = tr.pack(frames, _lib.lib().b200_orb_max_keypoints(ex._h, 512, 512))
        tr.run_packed(packed)
        st = []
        for _ in range(a.reps):
            tr.run_packed(packed)
            st.append((tr.stage_ms()["undistort_observe"], tr.stage_ms()["chain"]))
        res[f"chain64_{label}_stage0_ms"] = round(float(np.median([s[0] for s in st])), 4)
        res[f"chain64_{label}_whole_ms"] = round(float(np.median([s[1] for s in st])), 4)
    print(json.dumps(res), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
