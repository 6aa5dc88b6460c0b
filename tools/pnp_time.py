"""Time relocalisation's PnP (solve::pnp_solver::find_via_ransac(30, false)) on one GPU against the single-thread CPU restatement
(tests/pnp_oracle.c, the stand-in for the reference's serial loop over candidates):
  one problem   n = 300 matches, 30 hypotheses, one b200_pnp_ransac call;
  a batch       64 lost frames x 16 candidate keyframes = 1024 problems, n uniform in [50, 1000], one call.
The GPU figures are END-TO-END HOST-CALL times of the Python entry point (ctypes packing, upload, kernels, download, the synchronisation
inside the call): wall time per call, median of the repetitions.  The minimal sets are drawn beforehand, as the library's sampler does
before each call.  Prints the card and its power limit (read-only nvidia-smi query).

    python tools/pnp_time.py [--reps 20] [--out FILE.json]
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

import pnp_oracle as O  # noqa: E402
from stella_vslam_b200 import solve  # noqa: E402
from workloads import synth  # noqa: E402


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True)
        return q.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def problems(ns, seed0):
    out = []
    for i, n in enumerate(ns):
        pr = synth.make_pnp_problem(seed0 + i, int(n), 0.3 + 0.4 * ((i * 7) % 10) / 10, "equirect" if i % 4 == 3 else "perspective")
        out.append(dict(bearings=pr["bearings"], points=pr["points"], octaves=pr["octaves"], scale_factors=pr["scale_factors"], recompute=False,
                        min_sets=solve.draw_min_sets(int(n), 30, solve.mt19937((seed0 + i,)))))
    return out


def time_gpu(probs, reps):
    solve.pnp_ransac_batch(probs)  # warm-up: module load, arena growth
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        solve.pnp_ransac_batch(probs)
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3


def time_cpu(probs, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        for p in probs:
            O.pnp_ransac(p, p["min_sets"])
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    one = problems([300], 1)
    rng = np.random.default_rng(0)
    batch = problems(rng.integers(50, 1001, 1024), 100)
    res = dict(card=card(), one_problem_gpu_ms=time_gpu(one, a.reps), one_problem_cpu_ms=time_cpu(one, a.reps),
               batch_1024_gpu_ms=time_gpu(batch, max(3, a.reps // 4)), batch_1024_cpu_ms=time_cpu(batch, 2))
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
