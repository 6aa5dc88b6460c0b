"""Time the landmark creation of the mapping module on one GPU: the device chain (b200_create_new_landmarks), the per-neighbour path
(b200_match_pairs + b200_triangulate_pairs, valid rows updated on the host between neighbours) and the single-thread CPU restatement
(tests/mapping_oracle.c + oracle/pairs_oracle.c, the stand-in for the reference's serial loop).  16 current keyframes x 10 neighbours x
2000 keypoints, monocular and stereo.  The GPU figures are END-TO-END HOST-CALL times of the Python entry points: ctypes packing of the
keyframes, upload, kernels, download and the synchronisation inside the call (CUDA events on the matcher's stream around the call, which
synchronises, so they equal the wall time); not kernel time.  The CPU restatement is timed twice.  Prints the card and power limit, and
the SM clock sampled by nvidia-smi (read-only query) while the timed calls run.

    python tools/mapping_time.py [--keyframes 16] [--neighbours 10] [--keypoints 2000] [--reps 20]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import mapping_oracle as MO  # noqa: E402
from stella_vslam_b200 import _lib, mapping  # noqa: E402
from stella_vslam_b200.match import PAIRS_TRIANGULATION, _matcher, match_pairs_batch  # noqa: E402
from workloads import synth  # noqa: E402


def gpu_info():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], text=True)
        return out.strip()
    except Exception as e:  # noqa: BLE001
        return f"unavailable ({e})"


class ClockSampler:
    """SM clock of GPU 0 every ~0.2 s while the timed calls run (nvidia-smi --query-gpu, read-only)."""

    def __init__(self):
        self.samples, self._stop = [], threading.Event()
        self._t = threading.Thread(target=self._run, daemon=True)

    def _run(self):
        while not self._stop.is_set():
            try:
                out = subprocess.check_output(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i", "0"], text=True)
                self.samples.append(float(out.strip()))
            except Exception:  # noqa: BLE001
                return
            self._stop.wait(0.2)

    def __enter__(self):
        self._t.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join()


def per_neighbour(items):
    for cur, nb in items:
        free = cur["no_landmark"].copy()
        for ngh in nb:
            pr = MO.triangulation_problem(cur, ngh, mapping.RESIDUAL_RAD_THR, False, free)
            mo, _ = match_pairs_batch([pr], PAIRS_TRIANGULATION, 0.95, False)[0]
            i1 = np.flatnonzero(mo >= 0)
            pairs = np.stack([i1, mo[i1]], 1).astype(np.int32)
            _, ok = mapping.triangulate_pairs_batch([(cur, ngh, pairs, 1.0)])[0]
            free[pairs[ok][:, 0]] = 0


def timed(fn, stream, reps):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ms, wall = [], []
    for _ in range(reps):
        t = time.perf_counter()
        ev[0].record(stream)
        fn()
        ev[1].record(stream)
        ev[1].synchronize()
        wall.append((time.perf_counter() - t) * 1e3)
        ms.append(ev[0].elapsed_time(ev[1]))
    return float(np.median(ms)), float(np.median(wall))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keyframes", type=int, default=16)
    ap.add_argument("--neighbours", type=int, default=10)
    ap.add_argument("--keypoints", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    stream = torch.cuda.current_stream()
    _lib.check(_lib.lib().b200_matcher_set_stream(_matcher(0), C.c_void_p(stream.cuda_stream), 0))
    print("gpu:", gpu_info())
    for stereo in (False, True):
        items = [synth.make_mapping_problem(100 + k, a.neighbours, a.keypoints, stereo=stereo) for k in range(a.keyframes)]
        chain = lambda: mapping.create_new_landmarks_batch(items)  # noqa: E731
        res = chain()
        for _ in range(2):  # warm-up
            chain()
            per_neighbour(items)
        with ClockSampler() as clk:
            chain_ms, chain_wall = timed(chain, stream, a.reps)
            pn_ms, pn_wall = timed(lambda: per_neighbour(items), stream, a.reps)
        cpu_ms = []
        for _ in range(2):
            t = time.perf_counter()
            for cur, nb in items:
                MO.create_new_landmarks(cur, nb)
            cpu_ms.append(round((time.perf_counter() - t) * 1e3, 1))
        print(json.dumps(dict(stereo=stereo, keyframes=a.keyframes, neighbours=a.neighbours, keypoints=a.keypoints,
                              landmarks=int(sum(len(r["rank"]) for r in res)), chain_host_call_ms=round(chain_ms, 3),
                              chain_wall_ms=round(chain_wall, 3), per_neighbour_host_call_ms=round(pn_ms, 3),
                              per_neighbour_wall_ms=round(pn_wall, 3), cpu_oracle_ms_runs=cpu_ms,
                              sm_clock_mhz_during=dict(min=min(clk.samples, default=None), max=max(clk.samples, default=None),
                                                       n=len(clk.samples)))))
    _lib.check(_lib.lib().b200_matcher_set_stream(_matcher(0), None, 1))


if __name__ == "__main__":
    main()
