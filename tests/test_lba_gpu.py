"""GPU parity tests for the local bundle adjuster: CUDA (through the C ABI) vs the CPU oracle.
Tolerance: 1e-5 relative on poses and landmarks (BASELINE.json north_star); iteration counts, outlier flags and the
abort protocol must be identical."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

REL = 1e-5


@pytest.fixture(scope="module")
def mods():
    from oracle import pyoracle as O
    from stella_vslam_b200 import optimize
    from workloads import synth
    return O, optimize, synth


def check_same(got, ref, pr, same_iterations=True):
    if same_iterations:
        assert got["iterations"] == ref["iterations"], (got["iterations"], ref["iterations"])
    assert np.array_equal(got["outliers"], ref["outliers"])
    assert got["n_outliers"] == ref["n_outliers"]
    ps = max(1.0, np.abs(ref["points"]).max())
    assert np.abs(got["points"] - ref["points"]).max() <= REL * ps
    assert np.abs(got["pose_cw"] - ref["pose_cw"]).max() <= REL * max(1.0, np.abs(ref["pose_cw"]).max())
    # per-element relative check where the magnitude allows it
    big = np.abs(ref["points"]) > 1e-2
    assert (np.abs(got["points"] - ref["points"])[big] / np.abs(ref["points"])[big]).max() <= 10 * REL
    for a, b in zip(got["chi2"], ref["chi2"]):
        assert abs(a - b) <= 1e-6 * max(1.0, abs(b))
    assert abs(got["lambda_init"] - ref["lambda_init"]) <= 1e-9 * ref["lambda_init"]
    fixed = pr["pose_fixed"].astype(bool)
    assert np.array_equal(got["pose_cw"][fixed], pr["pose_cw"][fixed])


@pytest.mark.parametrize("model,K,F,L,seed", [("mono", 12, 3, 600, 1), ("stereo", 12, 3, 600, 2), ("equirect", 10, 2, 400, 3),
                                              ("stereo", 4, 1, 60, 4), ("mono", 30, 6, 3000, 5)])
def test_vs_oracle(mods, model, K, F, L, seed):
    O, optimize, synth = mods
    pr = synth.make_ba_problem(K, F, L, seed=seed, model=model)
    ba = optimize.local_bundle_adjuster()
    check_same(ba.optimize(pr), O.lba_solve(pr), pr)
    ba.close()


def test_full_size_kitti_window(mods):
    # BASELINE config 4: 50 keyframes (10 fixed) / 10 000 landmarks
    O, optimize, synth = mods
    pr = synth.make_ba_problem(50, 10, 10000, seed=0, model="stereo")
    ba = optimize.local_bundle_adjuster()
    got = ba.optimize(pr)
    check_same(got, O.lba_solve(pr), pr)
    assert got["launches"] > 20 and got["gpu_ms"] > 0
    # size-independent property: re-optimising the optimum changes (almost) nothing and removes no further inliers
    pr2 = dict(pr)
    pr2["pose_cw"], pr2["points"] = got["pose_cw"], got["points"]
    keep = got["outliers"] == 0
    for k in ("e_pose", "e_point", "e_cam", "e_obs", "e_inv_sigma_sq", "e_delta"):
        pr2[k] = pr[k][keep]
    again = ba.optimize(pr2)
    assert again["chi2"][1] <= got["chi2"][1] * (1 + 1e-6)
    assert again["n_outliers"] <= 0.01 * keep.sum()


def test_force_stop_protocol(mods):
    O, optimize, synth = mods
    pr = synth.make_ba_problem(8, 3, 200, seed=2, model="mono")
    ba = optimize.local_bundle_adjuster()
    flag = np.array([1], np.uint8)
    assert ba.optimize(pr, flag) is None                       # local_bundle_adjuster_g2o.cc:308-310
    ba2 = optimize.local_bundle_adjuster(50, 10)
    flag = np.array([0], np.uint8)
    got = ba2.optimize(pr, flag)
    rflag = np.array([0], np.uint8)
    ref = O.lba_solve(pr, iters1=50, iters2=10, force_stop=rflag)
    assert flag[0] == rflag[0] == 1 and got["iterations"] == ref["iterations"] and got["iterations"][1] == 0
    check_same(got, ref, pr)


def test_fixed_points_markers_and_plain_edges(mods):
    O, optimize, synth = mods
    pr = synth.make_ba_problem(6, 2, 80, seed=9, model="mono")
    pf = np.zeros(80, np.uint8)
    pf[:10] = 1
    pr["point_fixed"] = pf
    marker = np.isin(pr["e_point"], np.arange(10))
    pr["e_can_be_outlier"] = (~marker).astype(np.uint8)
    pr["e_robust"] = (~marker).astype(np.uint8)               # use_huber_loss = false for marker edges (:297-299)
    ba = optimize.local_bundle_adjuster()
    got = ba.optimize(pr)
    check_same(got, O.lba_solve(pr), pr)
    assert np.array_equal(got["points"][:10], pr["points"][:10])


def test_degenerate_inputs(mods):
    O, optimize, synth = mods
    ba = optimize.local_bundle_adjuster()
    pr = synth.make_ba_problem(3, 3, 20, seed=4, model="mono")   # every keyframe fixed: landmarks only
    # (converges to machine precision within a few steps; after that the accept/terminate decisions hinge on the last
    #  bit of chi2, so only the results are compared, not the number of no-op iterations)
    check_same(ba.optimize(pr), O.lba_solve(pr), pr, same_iterations=False)
    pr = synth.make_ba_problem(4, 1, 10, seed=5, model="stereo")
    for k in ("e_pose", "e_point", "e_cam", "e_obs", "e_inv_sigma_sq", "e_delta"):
        pr[k] = pr[k][:0]
    got = ba.optimize(pr)                                           # no edges at all
    assert got["n_outliers"] == 0 and np.array_equal(got["points"], pr["points"])


def test_factory():
    from stella_vslam_b200 import optimize
    with pytest.raises(RuntimeError):
        optimize.create({"backend": "gtsam"})                       # local_bundle_adjuster_factory.h:26,30
    assert optimize.create({"backend": "b200", "num_first_iter": 3}).num_first_iter_ == 3


# ---- b200_lba_solve_batch: many windows per launch sequence --------------------------------------------------------------------

def test_batch_vs_oracle_and_single(mods):
    """Windows of different size / model / iteration count advance in lockstep; every one must equal the oracle, and (same code path,
    deterministic reductions) the batch-of-one result bit for bit."""
    O, optimize, synth = mods
    specs = [("stereo", 12, 3, 600, 11), ("mono", 8, 2, 300, 12), ("equirect", 10, 2, 400, 13), ("stereo", 4, 1, 60, 14),
             ("mono", 30, 6, 3000, 15), ("stereo", 3, 3, 20, 16)]
    prs = [synth.make_ba_problem(K, F, L, seed=s, model=m) for m, K, F, L, s in specs]
    ba = optimize.local_bundle_adjuster()
    got = ba.optimize_batch(prs)
    assert len(got) == len(prs)
    assert got[0]["launches"] < 200, got[0]["launches"]          # one launch sequence for all six windows
    for i, (g, pr) in enumerate(zip(got, prs)):
        ref = O.lba_solve(pr)
        check_same(g, ref, pr, same_iterations=(i != 5))           # (window 5: every keyframe fixed, see test_degenerate_inputs)
        one = ba.optimize(pr)
        assert np.array_equal(one["pose_cw"], g["pose_cw"]) and np.array_equal(one["points"], g["points"])
        assert np.array_equal(one["outliers"], g["outliers"]) and one["iterations"] == g["iterations"]
    ba.close()


def test_batch_of_identical_full_size_windows(mods):
    # 8 x BASELINE config 4 in one launch sequence: same result for every copy, launch count independent of the batch size
    O, optimize, synth = mods
    pr = synth.make_ba_problem(50, 10, 10000, seed=0, model="stereo")
    ba = optimize.local_bundle_adjuster()
    one = ba.optimize(pr)
    got = ba.optimize_batch([pr] * 8)
    for g in got:
        assert np.array_equal(g["pose_cw"], one["pose_cw"]) and np.array_equal(g["points"], one["points"])
        assert np.array_equal(g["outliers"], one["outliers"]) and g["iterations"] == one["iterations"]
    assert got[0]["launches"] <= one["launches"] + 24
    check_same(got[3], O.lba_solve(pr), pr)


def test_no_flag_runs_second_round_after_gain_stop(mods):
    # ADVICE r1: with force_stop == NULL the gain stop of round 1 lands in g2o's auxiliary flag, which optimize() resets:
    # round 2 must run (local_bundle_adjuster_g2o.cc:317-321 only tests the CALLER's flag)
    O, optimize, synth = mods
    pr = synth.make_ba_problem(8, 3, 200, seed=2, model="mono")
    ba = optimize.local_bundle_adjuster(50, 10)
    got = ba.optimize(pr)
    ref = O.lba_solve(pr, iters1=50, iters2=10)
    assert ref["iterations"][0] < 50 and ref["iterations"][1] > 0     # round 1 ended on the gain threshold, round 2 ran
    check_same(got, ref, pr)
    pr = synth.make_ba_problem(20, 5, 1500, seed=21, model="stereo")
    got = ba.optimize(pr)
    check_same(got, O.lba_solve(pr, iters1=50, iters2=10), pr)


def test_many_fixed_keyframes(mods):
    # ADVICE r1: only FREE keyframes enter the reduced system; windows with well over 166 keyframes in total must be solved
    O, optimize, synth = mods
    pr = synth.make_ba_problem(200, 180, 1500, seed=31, model="stereo")
    ba = optimize.local_bundle_adjuster()
    check_same(ba.optimize(pr), O.lba_solve(pr), pr)
    big = synth.make_ba_problem(170, 0, 200, seed=32, model="mono")     # 170 free keyframes: documented limit
    with pytest.raises(RuntimeError):
        ba.optimize(big)


def test_on_chip_limit_alone_and_in_a_batch(mods):
    # 166 free keyframes is the largest window the on-chip Cholesky takes (6 * Kf <= kCholOnChipMax = 1000, lba_kernels.cu): n = 996,
    # the largest dynamic shared-memory plan.  Alone it runs in a cluster of 8 CTAs, in a batch of three windows in clusters of 4
    # (lba_kernels.cu: `nw <= 2 ? 8 : 4`); 167 free keyframes is refused.
    O, optimize, synth = mods
    pr = synth.make_ba_problem(176, 10, 3000, seed=51, model="stereo")
    assert (pr["pose_fixed"] == 0).sum() == 166
    ba = optimize.local_bundle_adjuster()
    one = ba.optimize(pr)
    check_same(one, O.lba_solve(pr), pr)
    small = [synth.make_ba_problem(12, 3, 600, seed=52, model="mono"), synth.make_ba_problem(8, 2, 300, seed=53, model="stereo")]
    got = ba.optimize_batch([small[0], pr, small[1]])
    assert np.array_equal(got[1]["pose_cw"], one["pose_cw"]) and np.array_equal(got[1]["points"], one["points"])
    assert np.array_equal(got[1]["outliers"], one["outliers"]) and got[1]["iterations"] == one["iterations"]
    for g, p in zip((got[0], got[2]), small):
        check_same(g, O.lba_solve(p), p)
    with pytest.raises(RuntimeError):
        ba.optimize(synth.make_ba_problem(177, 10, 400, seed=54, model="stereo"))


def test_batch_force_stop_flags_and_bad_edges(mods):
    O, optimize, synth = mods
    prs = [synth.make_ba_problem(8, 3, 200, seed=2, model="mono"), synth.make_ba_problem(6, 2, 100, seed=3, model="stereo"),
           synth.make_ba_problem(8, 3, 200, seed=2, model="mono")]
    ba = optimize.local_bundle_adjuster(50, 10)
    flags = [np.array([0], np.uint8), np.array([1], np.uint8), None]
    got = ba.optimize_batch(prs, flags)
    assert got[1] is None and flags[1][0] == 1                         # set on entry: that window is not touched (:308-310)
    rflag = np.array([0], np.uint8)
    ref0 = O.lba_solve(prs[0], iters1=50, iters2=10, force_stop=rflag)
    assert flags[0][0] == rflag[0] == 1 and got[0]["iterations"] == ref0["iterations"] and got[0]["iterations"][1] == 0
    check_same(got[0], ref0, prs[0])
    check_same(got[2], O.lba_solve(prs[2], iters1=50, iters2=10), prs[2])   # same window without a flag: second round runs
    bad = dict(prs[1])
    bad["e_point"] = prs[1]["e_point"].copy()
    bad["e_point"][7] = 10 ** 6
    with pytest.raises(RuntimeError):
        ba.optimize(bad)
    check_same(ba.optimize_batch([prs[1]])[0], O.lba_solve(prs[1], iters1=50, iters2=10), prs[1])  # the handle is still usable


def test_unsorted_edge_order(mods):
    # the ABI accepts the observations in any order; the device plan sorts them by landmark and reports outliers in the caller's order
    O, optimize, synth = mods
    pr = synth.make_ba_problem(12, 3, 600, seed=41, model="stereo")
    perm = np.random.default_rng(5).permutation(len(pr["e_pose"]))
    pr2 = dict(pr)
    for k in ("e_pose", "e_point", "e_cam", "e_obs", "e_inv_sigma_sq", "e_delta"):
        pr2[k] = np.ascontiguousarray(pr[k][perm])
    ba = optimize.local_bundle_adjuster()
    check_same(ba.optimize(pr2), O.lba_solve(pr2), pr2)


def test_batch_of_32_mixed_windows(mods):
    # SURVEY 8d: >= 32 independent problems per launch sequence; mixed models / sizes, every window against the oracle
    O, optimize, synth = mods
    rng = np.random.default_rng(77)
    specs = [(("mono", "stereo", "equirect")[i % 3], int(rng.integers(4, 14)), int(rng.integers(1, 4)), int(rng.integers(60, 500)), 200 + i) for i in range(32)]
    prs = [synth.make_ba_problem(K, min(F, K - 1) if m != "mono" else min(max(F, 2), K - 1), L, seed=s, model=m) for m, K, F, L, s in specs]
    ba = optimize.local_bundle_adjuster()
    got = ba.optimize_batch(prs)
    assert len(got) == 32 and got[0]["launches"] < 200
    for g, pr in zip(got, prs):
        check_same(g, O.lba_solve(pr), pr)
