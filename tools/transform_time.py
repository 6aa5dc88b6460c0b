"""Time loop detection's Sim3 refinement on the GPU (b200_transform_optimize) against the CPU oracle's single-thread time, on the
loop candidates of workloads/synth.make_sim3_pair.  g2o itself is not part of this project and is not timed here.

    python tools/transform_time.py [--reps 200] [--batch 1024] [--no-oracle]

Reports, with the card's name and power limit read in the same run:
- one problem of 300 perspective pairs: host-call time of one b200_transform_optimize call (upload, launch, download, synchronise),
  which is what the reference-side adapter pays per candidate;
- a batch of `--batch` problems of 20-1000 pairs (mixed camera models): host-call time of the whole call and the device time of its
  kernel (torch.profiler, CUDA activity, in a separate pass);
- the single-thread CPU oracle (tests/transform_oracle.c) on the same inputs."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def _host_ms(fn, reps):
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        ts.append(1e3 * (time.perf_counter() - t))
    return float(np.median(ts)), float(np.min(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    from stella_vslam_b200 import optimize
    from workloads import synth
    gpu = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True).strip()
    print(json.dumps(dict(gpu=gpu)), flush=True)
    opt = optimize.transform_optimizer(False)

    one = synth.make_sim3_pair(1, 300)
    packed = [optimize.pack_transform_problem(one, False)]
    arr1 = (optimize.TransformProblem * 1)(packed[0][0])
    call1 = lambda: opt._L.b200_transform_optimize(opt._h, 1, arr1, 10.0, 10)
    for _ in range(20):
        call1()
    med, mn = _host_ms(call1, a.reps)
    row = dict(case="one problem, 300 pairs", host_call_ms_median=round(med, 4), host_call_ms_min=round(mn, 4),
               iterations=list(arr1[0].iterations), trials=list(arr1[0].trials))
    if not a.no_oracle:
        import transform_oracle as O
        O.transform_optimize(one)
        row["oracle_ms_median"] = round(_host_ms(lambda: O.transform_optimize(one), 20)[0], 4)
    print(json.dumps(row), flush=True)

    rng = np.random.default_rng(7)
    models = [("perspective", "perspective"), ("equirect", "equirect"), ("perspective", "equirect"), ("equirect", "perspective")]
    probs = [synth.make_sim3_pair(int(rng.integers(1 << 30)), int(rng.integers(20, 1001)), models=models[k % 4],
                                  outlier_frac=float(rng.uniform(0.1, 0.3))) for k in range(a.batch)]
    packed = [optimize.pack_transform_problem(pr, False) for pr in probs]
    arr = (optimize.TransformProblem * len(packed))(*[pk[0] for pk in packed])
    callb = lambda: opt._L.b200_transform_optimize(opt._h, len(packed), arr, 10.0, 10)
    for _ in range(3):
        callb()
    med, mn = _host_ms(callb, 10)
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            callb()
    kern = [e for e in prof.events() if "transform_optimize_kernel" in e.name]
    dev_ms = sum(e.device_time for e in kern) / max(len(kern), 1) / 1e3
    row = dict(case=f"batch of {a.batch} problems, 20-1000 pairs", pairs=int(sum(len(p["obs_1"]) for p in probs)), host_call_ms_median=round(med, 3),
               host_call_ms_min=round(mn, 3), kernel_ms=round(dev_ms, 3), kernel_launches_profiled=len(kern), torch=torch.__version__)
    if not a.no_oracle:
        import transform_oracle as O
        t = time.perf_counter()
        for pr in probs:
            O.transform_optimize(pr)
        row["oracle_ms"] = round(1e3 * (time.perf_counter() - t), 1)
    print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
