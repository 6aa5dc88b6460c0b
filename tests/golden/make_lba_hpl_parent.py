#!/usr/bin/env python3
"""lba_hpl_parent.npz: the local bundle adjuster's GPU results before the Hpl records were factored (kHplStride 20, the full 6x3
block per edge), on one window per edge model.  tests/test_lba_hpl_record.py solves the same windows with the factored records
(A = ww Jpi^T Ji and pc, kHplStride 12) and holds them to these results.

Run it on an H100 from the root of a checkout of the commit to pin (it imports the stella_vslam_b200 package two directories up):
    python tests/golden/make_lba_hpl_parent.py <out.npz>
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

# name -> make_ba_problem arguments; "stereo" is the bench's window
WINDOWS = {
    "stereo": dict(n_poses=50, n_fixed=10, n_points=10000, seed=0, model="stereo"),
    "mono": dict(n_poses=30, n_fixed=6, n_points=3000, seed=5, model="mono"),
    "equirect": dict(n_poses=20, n_fixed=4, n_points=2000, seed=3, model="equirect"),
}


def solve_windows(optimize, synth):
    out = {}
    ba = optimize.local_bundle_adjuster()
    for name, kw in WINDOWS.items():
        got = ba.optimize(synth.make_ba_problem(**kw))
        out[f"{name}_iterations"] = np.asarray(got["iterations"], np.int64)
        out[f"{name}_outliers"] = np.asarray(got["outliers"], np.uint8)
        out[f"{name}_pose_cw"] = np.asarray(got["pose_cw"], np.float64)
        out[f"{name}_points"] = np.asarray(got["points"], np.float64)
        out[f"{name}_chi2"] = np.asarray(got["chi2"], np.float64)
    ba.close()
    return out


def main(path):
    sys.path.insert(0, ROOT)
    from stella_vslam_b200 import optimize
    from workloads import synth
    np.savez_compressed(path, **solve_windows(optimize, synth))
    print("wrote", path)


if __name__ == "__main__":
    main(sys.argv[1])
