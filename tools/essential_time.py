"""Time robust matching's essential-matrix RANSAC (solve::essential_solver::find_via_ransac(1000, true), five-point) on one GPU against
the single-thread CPU restatement (tests/essential_oracle.c, the stand-in for the reference's serial loop):
  one problem   n = 500 matches, 1 000 iterations, one b200_essential_ransac call (the tracker's fallback: one frame x one keyframe);
  a batch       256 problems, n uniform in [50, 1500], 1 000 iterations each, one call (a relocalisation round), with the kernel
                time of each of the three launches from torch.profiler in a separate pass.
The GPU host-call figures are END-TO-END wall times of the Python entry point (ctypes packing, upload, kernels, download, the
synchronisation inside the call), median of the repetitions.  The minimal sets are drawn beforehand, as the library's sampler does
before each call.  Prints the card and its power limit (read-only nvidia-smi query, in the same run).

    python tools/essential_time.py [--reps 10] [--out FILE.json] [--no-oracle]
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

from stella_vslam_b200 import solve  # noqa: E402
from workloads import synth  # noqa: E402


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True)
        return q.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def problems(ns, seed0, iters=1000):
    out = []
    for i, n in enumerate(ns):
        p = synth.make_essential_problem(seed0 + i, int(n), 0.3 + 0.5 * ((i * 7) % 10) / 10, "equirect" if i % 4 == 3 else "perspective")
        out.append(dict(bearings_1=p["bearings_1"], bearings_2=p["bearings_2"], recompute=True,
                        min_sets=solve.draw_min_sets(int(n), iters, solve.mt19937((seed0 + i,)), set_size=5)))
    return out


def time_gpu(probs, reps):
    solve.essential_ransac_batch(probs)  # warm-up: module load, arena growth
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        solve.essential_ransac_batch(probs)
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3


def kernel_ms(probs):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            solve.essential_ransac_batch(probs)
    out = {}
    for k in ("essential_hypothesis_kernel", "essential_score_kernel", "essential_select_kernel"):
        ev = [e for e in prof.events() if k in e.name]
        out[k] = round(sum(e.device_time for e in ev) / max(len(ev), 1) / 1e3, 3)
    return out


def time_cpu(probs):
    import essential_oracle as O
    t0 = time.perf_counter()
    for p in probs:
        O.essential_ransac(p["bearings_1"], p["bearings_2"], p["min_sets"], True)
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    one = problems([500], 1)
    rng = np.random.default_rng(0)
    batch = problems(rng.integers(50, 1501, 256), 100)
    res = dict(card=card(), one_problem_gpu_ms=round(time_gpu(one, a.reps), 3), one_problem_kernel_ms=kernel_ms(one),
               batch_256_gpu_ms=round(time_gpu(batch, max(3, a.reps // 2)), 3), batch_256_kernel_ms=kernel_ms(batch),
               batch_matches=int(sum(len(p["bearings_1"]) for p in batch)))
    if not a.no_oracle:
        res["one_problem_cpu_ms"] = round(time_cpu(one), 1)
        res["batch_256_cpu_ms"] = round(time_cpu(batch), 1)
    print(json.dumps(res), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
