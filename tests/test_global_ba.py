"""optimize::global_bundle_adjuster (global_bundle_adjuster.cc): one LM round over a whole map.
CPU: the oracle's single-round solve against its own two-round local solve and against ground truth; GPU: CUDA vs oracle within 1e-5
on a small map (on-chip Cholesky) and on maps whose reduced system exceeds the on-chip limit (panel-by-panel Cholesky from HBM)."""
import numpy as np
import pytest

from oracle import pyoracle as O
from workloads import synth

REL = 1e-5


def test_oracle_single_round_equals_first_round_of_local_ba():
    pr = synth.make_ba_problem(10, 1, 300, seed=7, model="stereo")
    g = O.global_ba_solve(pr, num_iter=5)
    l = O.lba_solve(pr, iters1=5, iters2=0)
    # same first round: same iteration count, chi2 and lambda; the local solve then marks outliers, which moves nothing with 0 iterations
    assert g["iterations"] == l["iterations"][0] and abs(g["chi2"] - l["chi2"][0]) <= 1e-9 * l["chi2"][0]
    assert np.allclose(g["pose_cw"], l["pose_cw"], rtol=0, atol=1e-12) and np.allclose(g["points"], l["points"], rtol=0, atol=1e-12)


def test_oracle_gain_threshold_controls_the_stop():
    pr = synth.make_ba_problem(8, 1, 200, seed=2, model="mono")
    loose = O.global_ba_solve(pr, num_iter=50, gain_threshold=0.5)
    tight = O.global_ba_solve(pr, num_iter=50, gain_threshold=1e-9)
    assert loose["iterations"] < tight["iterations"] <= 50 and tight["chi2"] <= loose["chi2"]


def _check(got, ref, pr):
    assert got["iterations"] == ref["iterations"], (got["iterations"], ref["iterations"])
    ps = max(1.0, np.abs(ref["points"]).max())
    assert np.abs(got["points"] - ref["points"]).max() <= REL * ps
    assert np.abs(got["pose_cw"] - ref["pose_cw"]).max() <= REL * max(1.0, np.abs(ref["pose_cw"]).max())
    assert abs(got["chi2"] - ref["chi2"]) <= 1e-6 * max(1.0, abs(ref["chi2"]))
    assert abs(got["lambda_init"] - ref["lambda_init"]) <= 1e-9 * ref["lambda_init"]
    fixed = pr["pose_fixed"].astype(bool)
    assert np.array_equal(got["pose_cw"][fixed], pr["pose_cw"][fixed])


@pytest.mark.gpu
@pytest.mark.parametrize("model,K,L,seed", [("stereo", 30, 2000, 1), ("mono", 40, 1500, 2), ("equirect", 20, 800, 3)])
def test_small_map_vs_oracle(model, K, L, seed):
    from stella_vslam_b200 import optimize
    pr = synth.make_ba_problem(K, 1 if model != "mono" else 2, L, seed=seed, model=model)     # spanning root fixed (mono: gauge needs two)
    gba = optimize.global_bundle_adjuster(10)
    _check(gba.optimize(pr), O.global_ba_solve(pr, 10), pr)
    nh = optimize.global_bundle_adjuster(10, use_huber_kernel=False)
    pr2 = dict(pr, e_robust=np.zeros(len(pr["e_pose"]), np.uint8))
    _check(nh.optimize(pr), O.global_ba_solve(pr2, 10), pr)


@pytest.mark.gpu
@pytest.mark.parametrize("K,L,seed", [(180, 4000, 11), (260, 6000, 12)])
def test_large_map_off_chip_cholesky(K, L, seed):
    # 179 / 259 free keyframes: 1074 / 1554 unknowns in the reduced system, beyond the on-chip factorisation (1000)
    from stella_vslam_b200 import optimize
    pr = synth.make_ba_problem(K, 1, L, seed=seed, model="stereo")
    gba = optimize.global_bundle_adjuster(6)
    got = gba.optimize(pr)
    _check(got, O.global_ba_solve(pr, 6), pr)
    assert got["launches"] > 2 * (6 * (K - 1) // 24)          # the panel-by-panel path ran
    with pytest.raises(RuntimeError):                           # the local-BA entry point keeps its documented limit
        optimize.local_bundle_adjuster().optimize(pr)


def _free_columns(pr):
    """The reduced system's keyframe column of every edge (-1: fixed keyframe), numbered as the host plan numbers them."""
    fixed = pr["pose_fixed"].astype(bool)
    col = np.where(fixed, -1, np.cumsum(~fixed) - 1)
    return col[pr["e_pose"]]


@pytest.mark.gpu
@pytest.mark.parametrize("Kf", [64, 65, 128, 129, 166, 167, 192, 193, 257])
def test_free_keyframe_count_thresholds(Kf, monkeypatch):
    # The plan keeps one 64-bit mask word per 64 free keyframe columns for every landmark (lba_kernels.cu:2153: mask_words =
    # ceil(Kf / 64)); these counts sit on both sides of each word boundary.  6 * Kf <= kCholOnChipMax (1000, :1350) is factored on
    # chip, above that panel by panel (:2340: `large = max_n > kCholOnChipMax`): 166 and 167 straddle that switch.
    from stella_vslam_b200 import optimize
    pr = synth.make_ba_problem(Kf + 1, 1, 3000, seed=100 + Kf, model="stereo")
    assert (pr["pose_fixed"] == 0).sum() == Kf
    col = _free_columns(pr)
    for b in range(64, Kf, 64):                                 # a landmark seen on both sides of every word boundary
        lo = np.zeros(len(pr["points"]), bool)
        hi = np.zeros(len(pr["points"]), bool)
        lo[pr["e_point"][(col >= 0) & (col < b)]] = True
        hi[pr["e_point"][col >= b]] = True
        assert (lo & hi).sum() > 10, (b, (lo & hi).sum())
    got = optimize.global_bundle_adjuster(4).optimize(pr)
    _check(got, O.global_ba_solve(pr, 4), pr)
    if 6 * Kf > 1000:
        assert got["launches"] > 2 * (6 * Kf // 24)             # the panel-by-panel path ran
    else:                                                       # the on-chip path ran: forcing the panels adds their launches
        monkeypatch.setenv("B200_LBA_FORCE_OFFCHIP", "1")
        off = optimize.global_bundle_adjuster(4).optimize(pr)
        assert off["iterations"] == got["iterations"] and off["launches"] > got["launches"]


@pytest.mark.gpu
def test_force_stop_protocol():
    from stella_vslam_b200 import optimize
    pr = synth.make_ba_problem(12, 1, 400, seed=5, model="stereo")
    gba = optimize.global_bundle_adjuster(50)
    flag = np.array([1], np.uint8)
    assert gba.optimize(pr, flag) is None                       # raised by the caller: "aborted"
    flag = np.array([0], np.uint8)
    got = gba.optimize(pr, flag)                                # the gain stop raises the flag too, but that is a normal return
    rflag = np.array([0], np.uint8)
    ref = O.global_ba_solve(pr, 50, force_stop=rflag)
    assert got is not None and flag[0] == rflag[0] == 1 and got["iterations"] == ref["iterations"] < 50
    _check(got, ref, pr)
    got2 = gba.optimize(pr, None, gain_threshold=0.3)           # optimize_for_initialization's own threshold
    ref2 = O.global_ba_solve(pr, 50, gain_threshold=0.3)
    assert got2["iterations"] == ref2["iterations"] < got["iterations"]


@pytest.mark.gpu
def test_off_chip_cholesky_equals_on_chip_on_small_systems(monkeypatch):
    """The panel-by-panel factorisation (global BA) forced onto systems the on-chip kernel also solves: same panels, same tile arithmetic,
    same backward solve -> the same states up to the last bits of one reduction (computeScale's sum runs in a different thread count)."""
    from stella_vslam_b200 import optimize
    for model, K, L, seed in [("stereo", 30, 2000, 1), ("mono", 25, 900, 4)]:
        pr = synth.make_ba_problem(K, 2, L, seed=seed, model=model)
        monkeypatch.delenv("B200_LBA_FORCE_OFFCHIP", raising=False)
        on = optimize.global_bundle_adjuster(8).optimize(pr)
        monkeypatch.setenv("B200_LBA_FORCE_OFFCHIP", "1")
        gba = optimize.global_bundle_adjuster(8)
        off = gba.optimize(pr)
        lba = optimize.local_bundle_adjuster().optimize(pr)               # the local-BA protocol through the same path
        monkeypatch.delenv("B200_LBA_FORCE_OFFCHIP")
        assert off["launches"] > on["launches"] and off["iterations"] == on["iterations"]
        assert np.allclose(off["pose_cw"], on["pose_cw"], rtol=1e-11, atol=1e-13) and np.allclose(off["points"], on["points"], rtol=1e-11, atol=1e-13)
        ref = O.lba_solve(pr)
        assert lba["iterations"] == ref["iterations"] and np.array_equal(lba["outliers"], ref["outliers"])
        assert np.abs(lba["points"] - ref["points"]).max() <= REL * max(1.0, np.abs(ref["points"]).max())
