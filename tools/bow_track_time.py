"""Time BoW-match tracking (frame_tracker::bow_match_based_track) on one GPU, for KITTI-like stereo (1241 x 376) and EuRoC-like monocular
(752 x 480, with distortion) frames of about 2 000 keypoints, with 1 and 64 frames per call:
  chain           b200_bow_match_based_track: host-call wall time (keyframe upload, the device chain, download, one synchronise) and the
                  device time per stage (b200_bow_track_stage_ms, CUDA events); candidate_share = the candidate pass over the chain;
  stage_by_stage  the device path composed in Python, frame by frame: b200_keypoints_undistort, b200_match_pairs (variant B200_PAIRS_BOW)
                  and b200_pose_optimize (tests/bow_track_oracle.py with the device stages plugged in);
  cpu             the single-thread CPU restatement (tests/bow_track_oracle.py with the oracle's undistortion, matcher and pose optimiser).
Each frame's reference keyframe and BoW nodes are a synth.make_bow_frame (64 nodes).  Medians of the repetitions, after a warm-up call of
every shape.  Prints the card and its power limit (read-only nvidia-smi query, in the same run).

    python tools/bow_track_time.py [--reps 20] [--cpu-reps 2] [--out FILE.json]
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
import bow_track_oracle as BT  # noqa: E402
from stella_vslam_b200 import feature, match, optimize, tracking  # noqa: E402
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
    und = [CM.undistort_keypoints(cam, k)[0] for k in kps]
    frames = [dict(synth.make_bow_frame(und[i], descs[i], cam, seed=200 + i, stereo=stereo), frame=i) for i in range(n_frames)]
    tr = tracking.frame_tracker(ex, cam)
    res = dict(frames=n_frames, keypoints_mean=round(float(np.mean([len(k) for k in kps])), 1),
               kf_keypoints_mean=round(float(np.mean([len(f["keyframe"]["desc"]) for f in frames])), 1))
    got = tr.bow_match_based_track(frames)
    res["matches_mean"] = round(float(np.mean([g["n_matches"] for g in got])), 1)
    res["tracked"] = int(sum(g["tracked"] for g in got))
    res["chain_host_ms"] = median_ms(lambda: tr.bow_match_based_track(frames), reps)
    stage = {k: [] for k in tracking.frame_tracker.BOW_STAGES}
    for _ in range(reps):
        tr.bow_match_based_track(frames)
        for k, v in tr.bow_stage_ms().items():
            stage[k].append(v)
    res["chain_stage_ms"] = {k: round(float(np.median(v)), 4) for k, v in stage.items()}
    res["candidate_share"] = round(res["chain_stage_ms"]["candidates"] / res["chain_stage_ms"]["chain"], 4)
    po = optimize.pose_optimizer()
    isig = ex.orb_params_.inv_level_sigma_sq_

    def path(i, device):
        kw = {}
        if device:
            kw = dict(undistort_fn=lambda c, k: ex.undistort_keypoints(c, k),
                      match_fn=lambda p: match.match_pairs_batch([p], match.PAIRS_BOW, 0.7, True)[0],
                      pose_fn=lambda pp, a, b, c: po.optimize(pp))
        return BT.bow_match_based_track(cam, kps[i], descs[i], frames[i], isig, monocular=not stereo, **kw)

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
