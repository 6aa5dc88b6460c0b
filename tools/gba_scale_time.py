"""Global-BA timing beyond the on-chip Cholesky: one LM iteration (one build, one trial) of b200_global_ba_solve on the multi-lap
maps of tests/gba_scale.py at 1 000, 2 000 and 4 000 free keyframes (n = 6 000 / 12 000 / 24 000 keyframe unknowns), with the
device time per stage from the profiling mode (an event after every launch, b200_lba_enable_profile / b200_lba_kernel_ms), beside
the card name and power limit.  The "cholesky" stage is every gchol_panel_kernel / gchol_trail_kernel launch and gchol_finish_kernel.
usage: python tools/gba_scale_time.py [free keyframe counts ...]"""
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np  # noqa: E402

import gba_scale as G  # noqa: E402
from stella_vslam_b200 import optimize  # noqa: E402

NAMES = ["plan", "landmark_build", "pose_rows", "schur", "cholesky", "backsub+trial", "(unused)", "tail"]


def main():
    sizes = [int(a) for a in sys.argv[1:]] or [1000, 2000, 4000]
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(f"device: {card}", flush=True)
    for kf in sizes:
        pr = G.multi_lap_map(kf + 1, 15 * kf, seed=kf)
        gba = optimize.global_bundle_adjuster(1)
        L = gba._L
        L.b200_lba_enable_profile.argtypes = [C.c_void_p, C.c_int]
        L.b200_lba_kernel_ms.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_int)]
        gba.optimize(pr, gain_threshold=0.0)                                # warm-up: module load, arena allocation
        out = gba.optimize(pr, gain_threshold=0.0)
        L.b200_lba_enable_profile(gba._h, 1)
        prof = gba.optimize(pr, gain_threshold=0.0)
        L.b200_lba_enable_profile(gba._h, 0)
        parts = []
        for k, nm in enumerate(NAMES):
            v, n = C.c_float(), C.c_int()
            L.b200_lba_kernel_ms(gba._h, k, C.byref(v), C.byref(n))
            if n.value:
                parts.append(f"{nm} {v.value:.1f} ms")
        n = 6 * int((pr["pose_fixed"] == 0).sum())
        print(f"global BA {kf} free keyframes (n = {n}, {len(pr['points'])} landmarks, {len(pr['e_pose'])} edges), one iteration: "
              f"{out['gpu_ms']:.1f} ms on the stream, {out['launches']} launches; M {8 * (n + 1) * (n + 2) / 1e9:.2f} GB", flush=True)
        print(f"   per stage (profiling mode, {prof['gpu_ms']:.1f} ms): " + ", ".join(parts), flush=True)
        gba.close()
        del pr
        assert np.isfinite(out["chi2"])


if __name__ == "__main__":
    main()
