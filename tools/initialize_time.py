"""Time monocular initialisation (b200_initialize) for 1 and 64 frame pairs with 100 RANSAC iterations -- EuRoC-sized perspective pairs
(800 matches) and equirectangular pairs (600 matches) -- against the stage-by-stage path (b200_twoview_ransac for H and F, or
b200_essential_ransac for E, then the reconstruction on the host) and the single-thread CPU restatement.  "host" is the wall time of one
call, which ends in a synchronise; "kernels" is the sum of the call's kernel times from torch.profiler (the upload and download are
not included).  Prints the card name and power limit of the same run.  Needs an sm_90 GPU.

    python tools/initialize_time.py [--reps 20]
"""
import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import initialize_oracle as O  # noqa: E402
from stella_vslam_b200 import initialize as I, solve  # noqa: E402


def stage_by_stage(probs):
    if probs[0]["cam_ref"].get("model") == "equirectangular":
        out = []
        for p in probs:
            mt = O.matches_of(p["ref_matches_with_cur"])
            s = solve.essential_ransac_batch([dict(bearings_1=p["bearings_ref"][mt[:, 0]], bearings_2=p["bearings_cur"][mt[:, 1]],
                                                   min_sets=p["min_sets_E"], recompute=False)])[0]
            out.append(O.reconstruct(p, "E", s["E_21"], s["inlier_flags"]) if s["valid"] else None)
        return out
    out = []
    sols = solve.twoview_ransac_batch([dict(model=k, keypts_1=p["undist_ref"], keypts_2=p["undist_cur"],
                                            matches_12=O.matches_of(p["ref_matches_with_cur"]), min_sets=p["min_sets_" + k], recompute=False)
                                       for p in probs for k in ("H", "F")])
    for i, p in enumerate(probs):
        h, f = sols[2 * i], sols[2 * i + 1]
        s, model = (h, "H") if O.choose_H(h["best_cost"], f["best_cost"], h["valid"]) else (f, "F")
        out.append(O.reconstruct(p, model, s["M_21"], s["inlier_flags"]) if s["valid"] else None)
    return out


def timed(fn, reps):
    fn()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t) / reps * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("initialize_time: no CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"card: {card}")
    sets = {"perspective": [O.perspective_problem(seed=500 + i, n=800) for i in range(64)],
            "equirectangular": [O.equirect_problem(seed=i) for i in range(64)]}
    for (kind, base), n in [(kv, n) for kv in sets.items() for n in (1, 64)]:
        probs = base[:n]
        host_ms = timed(lambda: I.initialize_batch(probs), a.reps)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            I.initialize_batch(probs)
            torch.cuda.synchronize()
        dev_ms = sum(e.device_time_total for e in prof.key_averages() if e.device_time_total > 0 and "Memcpy" not in e.key) / 1e3
        stage_ms = timed(lambda: stage_by_stage(probs), max(1, a.reps // 4))
        cpu_ms = timed(lambda: [O.initialize(p) for p in probs], max(1, a.reps // 10))
        print(f"{kind:15s} pairs={n:3d}  b200_initialize host {host_ms:8.2f} ms (kernels {dev_ms:7.3f} ms)  stage-by-stage {stage_ms:8.2f} ms  "
              f"CPU oracle {cpu_ms:8.2f} ms")


if __name__ == "__main__":
    main()
