"""Time keyframe culling (b200_remove_redundant_keyframes) on one GPU, for 1 and 64 maps of 30 covisibilities x about 2 000 keypoints
with about 8 observers per landmark (workloads.synth.make_cull_map):
  host_call  wall time of the C-ABI call on packed tables (staging, upload, launch, download, synchronise);
  device     CUDA events on the call's stream around the same call (the stream idles while the host checks and stages, so this
             includes that work as well as the upload, the kernel and the download);
  kernel     cull_keyframes_kernel alone, from torch.profiler;
  cpu        the single-thread C restatement (tests/cull_oracle.c) on the same tables.
Medians of the repetitions.  Prints the card and its power limit (read-only nvidia-smi query, in the same run).

    python tools/cull_time.py [--reps 20] [--out FILE.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402

import cull_oracle as CO  # noqa: E402
from stella_vslam_b200 import _lib, mapping  # noqa: E402
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    res = dict(card=card())
    rng = np.random.default_rng(2024)
    probs = [synth.gather_cull_problem(synth.make_cull_map(rng, n_covisibilities=30, n_keypoints=2000, observers=8)) for _ in range(64)]
    res["keypoints_per_map"] = int(np.mean([sum(len(c["kp_landmark"]) for c in p["covisibilities"]) for p in probs]))
    res["landmarks_per_map"] = int(np.mean([len(p["obs_offsets"]) - 1 for p in probs]))
    res["observations_per_map"] = int(np.mean([len(p["obs_rank"]) for p in probs]))
    L = _lib.lib()
    mapping._setup()
    h = C.c_void_p()
    _lib.check(L.b200_matcher_create(0, C.byref(h)))
    stream = torch.cuda.Stream()
    _lib.check(L.b200_matcher_set_stream(h, C.c_void_p(stream.cuda_stream), 0))
    for n in (1, 64):
        arr, keep = mapping.pack_cull_problems(probs[:n])
        call = lambda: _lib.check(L.b200_remove_redundant_keyframes(h, n, arr))  # noqa: E731
        call()
        res[f"removed_{n}"] = int(sum(arr[k].n_removed for k in range(n)))
        res[f"host_call_{n}_ms"] = median_ms(call, a.reps)
        dev = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            call()
            e1.record(stream)
            e1.synchronize()
            dev.append(e0.elapsed_time(e1))
        res[f"device_{n}_ms"] = round(float(np.median(dev)), 4)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                call()
        ev = [e for e in prof.events() if "cull_keyframes_kernel" in e.name]
        res[f"kernel_{n}_ms"] = round(sum(e.device_time for e in ev) / max(len(ev), 1) / 1e3, 4)
        want = CO.remove_redundant_keyframes(probs[:n])
        res[f"matches_oracle_{n}"] = all(arr[k].n_removed == want[k]["n_removed"] for k in range(n))
        oarr, okeep = mapping.pack_cull_problems(probs[:n])
        res[f"cpu_{n}_1thread_ms"] = median_ms(lambda: [CO.lib().cull_oracle(C.byref(oarr[k])) for k in range(n)], max(3, a.reps // 4))
    L.b200_matcher_destroy(h)
    print(json.dumps(res), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
