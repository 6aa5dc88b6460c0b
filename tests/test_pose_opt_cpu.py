"""optimize::pose_optimizer oracle (oracle/lba_oracle.c: orc_pose_optimize, pose_optimizer_g2o.cc:38-175).  No reference test or
golden exists; each LM step is pinned instead against the independent high-precision reference of tests/pose_reference.py (its
lambda_init, the lambda of later steps, the classification between rounds and the re-posed later rounds:
tests/test_pose_precision_cpu.py, and on the device tests/test_pose_precision_gpu.py).  Here: protocol properties and agreement
with ground truth on synthetic frames."""
import numpy as np
import pytest

from oracle import pyoracle as O
from workloads import synth


def _pose_err(a, b):
    dR = a[:3, :3] @ b[:3, :3].T
    ang = np.degrees(np.arccos(np.clip((np.trace(dR) - 1) / 2, -1, 1)))
    ca, cb = -a[:3, :3].T @ a[:3, 3], -b[:3, :3].T @ b[:3, 3]
    return ang, np.linalg.norm(ca - cb)


@pytest.mark.parametrize("model", ["mono", "stereo", "equirect"])
def test_pose_optimizer_recovers_pose_and_outliers(model):
    pr = synth.make_pose_problem(3, n_obs=800, model=model)
    n, pose, flags = O.pose_optimize(pr)
    ang0, tr0 = _pose_err(pr["pose_cw"][0], pr["gt_pose_cw"])
    ang, tr = _pose_err(pose, pr["gt_pose_cw"])
    assert ang < 0.1 * ang0 and tr < 0.2 * tr0 + 0.02
    assert n == (~flags).sum()
    assert flags[pr["gt_outlier"]].mean() > 0.95            # gross outliers are rejected
    assert flags[~pr["gt_outlier"]].mean() < 0.15           # 5 % chi-square tail (+ level noise)


def test_pose_optimizer_protocol_edges():
    pr = synth.make_pose_problem(4, n_obs=4)                 # fewer than 5 observations: untouched pose, 0 (:116-118)
    n, pose, flags = O.pose_optimize(pr)
    assert n == 0 and np.array_equal(pose, pr["pose_cw"][0]) and not flags.any()
    pr = synth.make_pose_problem(5, n_obs=300, outlier_frac=0.0)
    a = O.pose_optimize(pr, 2, 2, 10)
    b = O.pose_optimize(pr, 0, 4, 10)                        # no robust trials: the kernel is dropped from the start (:123-127)
    c = O.pose_optimize(pr, 4, 0, 10)                        # num_trials_ == 0: Huber stays on in every trial (:164)
    for r in (a, b, c):
        assert _pose_err(r[1], pr["gt_pose_cw"])[0] < 0.05
    assert not np.array_equal(a[1], b[1])
    # idempotence: starting from the optimum nothing moves beyond numerical noise and the flags are unchanged
    pr2 = dict(pr, pose_cw=a[1][None])
    a2 = O.pose_optimize(pr2)
    assert np.allclose(a2[1], a[1], atol=1e-6) and np.array_equal(a2[2], a[2])
