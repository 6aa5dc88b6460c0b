"""Time robust-match tracking (frame_tracker::robust_match_based_track) on one GPU, for KITTI-like stereo (1241 x 376) and EuRoC-like monocular
(752 x 480, with distortion) frames of about 2 000 keypoints, with 1 and 64 frames per call:
  chain           b200_robust_match_based_track: host-call wall time (keyframe upload, the device chain, download, one synchronise) and the
                  device time per stage (b200_robust_track_stage_ms, CUDA events);
  stage_by_stage  the host path it replaces, frame by frame: b200_match_bruteforce, b200_draw_min_sets, b200_essential_ransac and
                  b200_pose_optimize, composed in Python (tests/robust_track_oracle.py with the device stages plugged in; the frames'
                  undistorted keypoints and bearings are already on the host, as in the reference's data::frame);
  cpu             the single-thread CPU restatement (tests/robust_track_oracle.py with the oracle's matcher, RANSAC and pose optimiser).
Each frame's reference keyframe is a synth.make_robust_frame.  Medians of the repetitions, after a warm-up call of every shape.  Prints the
card and its power limit (read-only nvidia-smi query, in the same run).

    python tools/robust_track_time.py [--reps 20] [--cpu-reps 2] [--out FILE.json]
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

import camera_models_oracle as CM  # noqa: E402
import robust_track_oracle as RT  # noqa: E402
from stella_vslam_b200 import feature, match, optimize, solve, tracking  # noqa: E402
from workloads import synth  # noqa: E402

CONFIGS = {
    "kitti_stereo": (dict(model="perspective", fx=718.856, fy=718.856, cx=607.1928, cy=185.2157, fxb=386.1448, cols=1241.0, rows=376.0, setup="stereo"),
                     1241, 376, 150),
    "euroc_mono": (dict(model="perspective", fx=458.654, fy=457.296, cx=367.215, cy=248.375, k1=-0.28340811, k2=0.07395907, p1=0.00019359,
                        p2=1.76187114e-05, k3=0.0, fxb=0.0, cols=752.0, rows=480.0, setup="monocular"), 752, 480, 100),
}


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


def run(name, n_frames, reps, cpu_reps):
    cam, w, h, min_area = CONFIGS[name]
    stereo = cam["setup"] != "monocular"
    n_img = min(n_frames, 8)
    ex = feature.orb_extractor(feature.orb_params(), min_area, max_batch=n_frames)
    imgs = np.stack([synth.make_frame(w, h, seed=100 + i % n_img) for i in range(n_frames)])
    kps, descs = ex.extract_batch(imgs)
    ub = [CM.undistort_keypoints(cam, k) for k in kps]
    frames = [dict(synth.make_robust_frame(ub[i][0], descs[i], cam, seed=200 + i, stereo=stereo), frame=i) for i in range(n_frames)]
    tr = tracking.frame_tracker(ex, cam, use_fixed_seed=True)
    res = dict(frames=n_frames, keypoints_mean=round(float(np.mean([len(k) for k in kps])), 1),
               kf_keypoints_mean=round(float(np.mean([len(f["keyframe"]["desc"]) for f in frames])), 1))
    got = tr.robust_match_based_track(frames)
    res["matches_mean"] = round(float(np.mean([g["n_matches"] for g in got])), 1)
    res["tracked"] = int(sum(g["tracked"] for g in got))
    res["chain_host_ms"] = median_ms(lambda: tr.robust_match_based_track(frames), reps)
    stage = {k: [] for k in tracking.frame_tracker.ROBUST_STAGES}
    for _ in range(reps):
        tr.robust_match_based_track(frames)
        for k, v in tr.robust_stage_ms().items():
            stage[k].append(v)
    res["chain_stage_ms"] = {k: round(float(np.median(v)), 4) for k, v in stage.items()}
    res["sampler_share"] = round(res["chain_stage_ms"]["sampler"] / res["chain_stage_ms"]["chain"], 4)
    po = optimize.pose_optimizer()
    rb = match.robust(0.8, True)
    isig = ex.orb_params_.inv_level_sigma_sq_

    def path(i, device):
        kw = {}
        if device:
            kw = dict(match_fn=lambda d1, a1, d2, a2, v2, lowe, ori: rb.brute_force_match(d1, a1, d2, a2, v2),
                      ransac_fn=lambda b1, b2, ms, rc: solve.essential_ransac_batch([dict(bearings_1=b1, bearings_2=b2, min_sets=ms, recompute=rc)])[0],
                      pose_fn=lambda pp, a, b, c: po.optimize(pp))
        return RT.robust_match_based_track(cam, kps[i], descs[i], frames[i], isig, monocular=not stereo, undistort_fn=lambda c, k: ub[i], **kw)

    res["stage_by_stage_host_ms"] = median_ms(lambda: [path(i, True) for i in range(n_frames)], reps)
    res["cpu_ms"] = median_ms(lambda: [path(i, False) for i in range(n_frames)], cpu_reps)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--cpu-reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card=card())
    print(json.dumps(dict(card=res["card"])), flush=True)
    for name in CONFIGS:
        for n in (1, 64):
            res[f"{name}_x{n}"] = run(name, n, a.reps, a.cpu_reps)
            print(json.dumps({f"{name}_x{n}": res[f"{name}_x{n}"]}), flush=True)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
