"""Stereo rectification timing: device time of b200_stereo_rectify_device per batch of 64 pairs (EuRoC 752x480 perspective, TUM-VI
512x512 fisheye; 1 and 3 channels), host-call time of b200_stereo_rectify for one pair, and single-thread cv2.remap of both eyes in the
same run when cv2 imports.  Bandwidth counts the algorithmic bytes of a batch: the fixed-point table once (8 B per pixel and eye) plus
2 W H C read and 2 W H C written per pair, against the H100 SXM data-sheet 3.35 TB/s.  Prints the card name and power limit read in
the same run.  Usage: python tools/rectify_time.py"""
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from stella_vslam_b200 import feature  # noqa: E402
from stella_vslam_b200._lib import check, lib  # noqa: E402
from workloads import synth  # noqa: E402

PEAK_GBS = 3350.0
B = 64


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def median_ms(fn, reps=20):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    ts = []
    for _ in range(reps):
        flush.zero_()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2]


def main():
    print(f"card: {card()}")
    try:
        import cv2
        cv2.setNumThreads(1)
    except ImportError:
        cv2 = None
    for name, cal in (("EuRoC", synth.EUROC_STEREO), ("TUM-VI", synth.TUM_VI_STEREO)):
        W, H = cal["cols"], cal["rows"]
        rect = feature.stereo_rectifier(cal["model"], W, H, cal["K_rect"], cal["K"][0], cal["D"][0], cal["R"][0], cal["K"][1], cal["D"][1], cal["R"][1])
        rect.set_stream(torch.cuda.current_stream())
        for ch in (1, 3):
            shape = (B, H, W) + (() if ch == 1 else (ch,))
            src_l = torch.randint(0, 256, shape, dtype=torch.uint8, device="cuda")
            src_r = torch.randint(0, 256, shape, dtype=torch.uint8, device="cuda")
            out = torch.empty((2 * B,) + shape[1:], dtype=torch.uint8, device="cuda")
            run = lambda: rect.rectify_device(src_l, src_r, out[0::2], out[1::2])  # noqa: E731
            for _ in range(5):
                run()
            ms = median_ms(run)
            gb = (2 * W * H * 8 + B * 4 * W * H * ch) / 1e9
            print(f"{name} {W}x{H} {ch}ch: {ms:.3f} ms per {B} pairs on the device ({ms / B * 1e3:.1f} us per pair), "
                  f"{gb / ms * 1e3:.0f} GB/s = {gb / ms * 1e3 / PEAK_GBS:.2f} of {PEAK_GBS:.0f} GB/s")
        rect.set_stream(None)
        l, r = synth.make_raw_stereo_pair(cal, seed=5)
        rect.rectify(l, r)
        ts = []
        for _ in range(20):
            t = time.perf_counter()
            rect.rectify(l, r)
            ts.append(time.perf_counter() - t)
        print(f"{name} host call b200_stereo_rectify (1 pair, 1ch, uploads + downloads): {sorted(ts)[10] * 1e3:.3f} ms")
        if cv2 is not None:
            maps = [rect.maps(e) for e in range(2)]
            ts = []
            for _ in range(20):
                t = time.perf_counter()
                a = cv2.remap(l, maps[0][0], maps[0][1], cv2.INTER_LINEAR)
                b = cv2.remap(r, maps[1][0], maps[1][1], cv2.INTER_LINEAR)
                ts.append(time.perf_counter() - t)
            ok = all(np.array_equal(x, y) for x, y in zip((a, b), rect.rectify(l, r)))
            print(f"{name} cv2.remap both eyes, 1 thread: {sorted(ts)[10] * 1e3:.3f} ms (identical output: {ok})")
        rect.close()


if __name__ == "__main__":
    main()
