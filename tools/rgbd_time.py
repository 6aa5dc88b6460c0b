"""Time the RGB-D front end and the depth-seeded landmarks on one GPU:
  rgbd_depths     b200_rgbd_depths for 64 TUM-sized (640 x 480) RGB-D frames with the TUM RGB-D calibration: the end-to-end host-call wall
                  time (depth-map upload, kernel, download) and the kernel time from torch.profiler;
  depth_landmarks b200_depth_landmarks for 64 keyframes of about 2 000 keypoints, mode 0 (keyframe_inserter) and mode 1
                  (create_map_for_stereo): host-call and kernel time;
  cpu             the single-thread CPU restatement (tests/rgbd_oracle.c, with the camera oracles' undistortion) on the same inputs.
Medians of the repetitions.  Prints the card and its power limit (read-only nvidia-smi query, in the same run).

    python tools/rgbd_time.py [--reps 20] [--out FILE.json]
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

import rgbd_oracle as RO  # noqa: E402
from stella_vslam_b200 import feature, mapping  # noqa: E402
from workloads import synth  # noqa: E402


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
    frames = [synth.make_rgbd_frames(640, 480, seed=900 + i) for i in range(64)]
    gray, d16 = np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames])
    ex = feature.orb_extractor(feature.orb_params(), 800, max_batch=64)
    kps, _ = ex.extract_batch(gray)
    res["rgbd_keypoints"] = int(sum(len(k) for k in kps))
    cam = RO.TUM_RGBD
    run = lambda: ex.rgbd_depths(cam, d16, 5000.0, RO.TUM_FXB)
    res["rgbd_depths_64_host_call_ms"] = median_ms(run, a.reps)
    res["rgbd_depths_64_kernel_ms"] = kernel_ms(run, "rgbd_depths_kernel")
    res["rgbd_cpu_64_1thread_ms"] = median_ms(lambda: [RO.rgbd_frame(cam, kps[f], d16[f], 5000.0, RO.TUM_FXB) for f in range(64)], max(3, a.reps // 4))
    rgbd = run()
    prm = ex.orb_params_
    for mode in (0, 1):
        probs = []
        for f, fr in enumerate(rgbd):
            pose = np.eye(4)
            pose[:3, 3] = [0.05 * f, 0.0, 0.0]
            probs.append(dict(mode=mode, pose_wc=pose, fx_inv=1.0 / cam["fx"], fy_inv=1.0 / cam["fy"], cx=cam["cx"], cy=cam["cy"], depth_thr=RO.TUM_DEPTH_THR,
                              x=fr["undist_keypts"]["x"], y=fr["undist_keypts"]["y"], octave=fr["undist_keypts"]["octave"], depth=fr["depths"],
                              has_landmark=None, scale_factors=prm.scale_factors_, inv_scale_factor_last=prm.inv_scale_factors_[-1]))
        go = lambda: mapping.depth_landmarks(probs)
        res[f"depth_landmarks_mode{mode}_created"] = int(sum(len(r["idx"]) for r in go()))
        res[f"depth_landmarks_mode{mode}_64_host_call_ms"] = median_ms(go, a.reps)
        res[f"depth_landmarks_mode{mode}_64_kernel_ms"] = kernel_ms(go, "depth_landmarks_kernel")
        res[f"depth_landmarks_mode{mode}_cpu_64_1thread_ms"] = median_ms(lambda: [RO.depth_landmarks(p) for p in probs], max(3, a.reps // 4))
    print(json.dumps(res), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
