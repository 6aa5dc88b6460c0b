"""GPU parity: b200_twoview_ransac (solve::homography_solver / fundamental_solver::find_via_ransac) against the CPU restatement, bit for
bit, over mixed H / F batches, every synthetic case, both recompute settings, the early returns and each SVD path at its threshold."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import twoview_oracle as O  # noqa: E402

from workloads import synth  # noqa: E402

pytestmark = pytest.mark.gpu

CASES = [None, "pure_rotation", "collinear", "duplicated", "n7", "n8", "inliers5", "inliers9", "inliers10"]


def _problem(seed, n, model, recompute, scene="general", case=None, max_num_iter=100, inlier_frac=None, camera="euroc"):
    from stella_vslam_b200 import solve
    frac = np.random.default_rng(seed).uniform(0.4, 0.9) if inlier_frac is None else inlier_frac
    p = synth.make_twoview_problem(seed, n, frac, scene, case=case, camera=camera)
    m, k = len(p["matches_12"]), 4 if model == "H" else 8
    ms = solve.draw_min_sets(m, max_num_iter, solve.mt19937((seed,)), set_size=k) if m >= 8 else np.zeros((0, k), np.int32)
    return dict(model=model, keypts_1=p["keypts_1"], keypts_2=p["keypts_2"], matches_12=p["matches_12"], min_sets=ms,
                recompute=recompute), p


def _oracle(pr):
    return O.twoview_ransac(pr["model"], pr["keypts_1"], pr["keypts_2"], pr["matches_12"], pr["min_sets"], pr.get("sigma", 1.0),
                            pr["recompute"])


def _assert_same(dev, ref):
    assert dev["status"] == (-1 if ref["status"] & O.STATUS_SVD else 0)
    for k in ("valid", "best_iter", "num_inliers"):
        assert dev[k] == ref[k], k
    assert dev["best_cost"].tobytes() == ref["best_cost"].tobytes()
    if ref["inlier_flags"] is None:
        assert dev["inlier_flags"] is None
    else:
        np.testing.assert_array_equal(dev["inlier_flags"], ref["inlier_flags"])
    if ref["valid"]:
        assert dev["M_21"].tobytes() == ref["M_21"].tobytes()


@pytest.mark.parametrize("recompute", [False, True])
@pytest.mark.parametrize("scene", ["planar", "general"])
def test_single_problems_match_oracle(scene, recompute):
    from stella_vslam_b200 import solve
    for seed in range(3):
        for model in ("H", "F"):
            pr, _ = _problem(seed, 1000, model, recompute, scene, camera="kitti" if seed == 2 else "euroc")
            ref = _oracle(pr)
            assert ref["valid"]
            _assert_same(solve.twoview_ransac_batch([pr])[0], ref)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("scene", ["planar", "general"])
def test_synth_cases_in_mixed_batches_match_oracle(case, scene):
    """Each case in one call with H and F problems interleaved, with and without the recompute."""
    from stella_vslam_b200 import solve
    prs = []
    for seed in range(4):
        for model in ("H", "F"):
            prs.append(_problem(200 + seed, 300, model, bool(seed % 2), scene, case=case)[0])
    for dev, pr in zip(solve.twoview_ransac_batch(prs), prs):
        _assert_same(dev, _oracle(pr))


@pytest.mark.parametrize("model,case,rows", [("H", "inliers5", 10), ("F", "inliers9", 9), ("F", "inliers10", 10)])
def test_recompute_svd_paths_at_their_thresholds(model, case, rows):
    """A winner with exactly 5 inliers (H: the tall path at 10 rows), 9 (F: square) or 10 (F: tall) goes into the recompute."""
    from stella_vslam_b200 import solve
    target = rows // 2 if model == "H" else rows
    found = 0
    for seed in range(200):
        for scene in ("planar", "general"):
            if model == "H" and scene == "general":
                continue
            pr, _ = _problem(seed, 0, model, True, scene, case=case, max_num_iter=300)
            ref = _oracle(pr)
            if not ref["valid"] or ref["num_inliers"] != target:
                continue
            _assert_same(solve.twoview_ransac_batch([pr])[0], ref)
            found += 1
        if found >= 3:
            break
    assert found >= 3


def test_degenerate_minimal_sets_are_skipped_identically():
    """On the collinear scene most H minimal sets lose rank: the oracle skips some iterations, and the device skips the same ones."""
    from stella_vslam_b200 import solve
    pr, _ = _problem(31, 200, "H", False, "planar", case="collinear", max_num_iter=200)
    n1, _, _, _ = O.normalize(pr["keypts_1"])
    n2, _, _, _ = O.normalize(pr["keypts_2"])
    mt = pr["matches_12"]
    skipped = sum(O.estimate("H", n1[mt[s, 0]], n2[mt[s, 1]])[0] is None for s in pr["min_sets"])
    assert skipped > 20
    _assert_same(solve.twoview_ransac_batch([pr])[0], _oracle(pr))


def test_batch_of_256_equals_single_calls():
    from stella_vslam_b200 import solve
    rng = np.random.default_rng(13)
    sizes = np.concatenate([[8, 9, 10, 2000], rng.integers(8, 2001, 252)])
    prs = []
    for i, n in enumerate(sizes):
        prs.append(_problem(3000 + i, int(n), "H" if i % 2 else "F", bool(i % 3), "planar" if i % 4 < 2 else "general",
                            max_num_iter=50)[0])
    batch = solve.twoview_ransac_batch(prs)
    for i, pr in enumerate(prs):
        alone = solve.twoview_ransac_batch([pr])[0]
        _assert_same(batch[i], dict(alone, status=O.STATUS_SVD if alone["status"] else 0))
    for i in range(0, len(prs), 8):
        _assert_same(batch[i], _oracle(prs[i]))


def test_both_models_of_one_attempt_in_one_call():
    """initialize::perspective's attempt: an H and an F problem on the same pair, recompute off, 100 iterations, 64 pairs in one call.
    Both models explain most of a planar scene's inliers (F is not unique there); on a general scene only F does, and rel_cost_H =
    cost_H / (cost_H + cost_F) in float is above 0.5.  With 0.5 px noise a few true inliers exceed the 5.991 px^2 threshold, and the
    winner of 100 iterations without the recompute keeps more than 90 % of them.  On a noisy planar scene the reference's cost (the errors of the inliers plus the threshold for the
    outliers) does not favour H: its transfer error is two-dimensional and symmetric, the Sampson distance one-dimensional."""
    from stella_vslam_b200 import solve
    prs, probs = [], []
    for seed in range(32):
        for scene in ("planar", "general"):
            for model in ("H", "F"):
                pr, p = _problem(500 + seed, 800, model, False, scene, inlier_frac=0.8)
                prs.append(pr)
                probs.append(p)
    res = solve.twoview_ransac_batch(prs)
    for k in range(0, len(res), 2):
        rh, rf, gt = res[k], res[k + 1], probs[k]["gt_inlier"]
        assert rh["valid"] and rf["valid"]
        rel = np.float32(rh["best_cost"] / np.float32(rh["best_cost"] + rf["best_cost"]))
        if (k // 2) % 2 == 0:
            assert rh["inlier_flags"][gt].mean() > 0.9 and rf["num_inliers"] > 0.8 * gt.sum()
        else:
            assert rf["inlier_flags"][gt].mean() > 0.9
            assert rel > 0.5 and rh["num_inliers"] < 0.5 * gt.sum()
    for k in range(0, len(prs), 16):
        _assert_same(res[k], _oracle(prs[k]))


def test_invalid_input_writes_nothing():
    from stella_vslam_b200 import solve
    from stella_vslam_b200._lib import B200Error
    pr, _ = _problem(3, 50, "H", True, max_num_iter=10)
    bad_index = dict(pr, min_sets=np.where(pr["min_sets"] == pr["min_sets"][0, 0], 50, pr["min_sets"]))
    mt = pr["matches_12"].copy()
    mt[3, 1] = len(pr["keypts_2"])
    bad_match = dict(pr, matches_12=mt)
    for bad in (bad_index, bad_match):
        keep = []
        arr = (solve.TwoviewProblem * 2)()
        arr[0], fl0 = solve._pack_twoview(pr, keep)
        arr[1], _ = solve._pack_twoview(bad, keep)
        for S in arr:
            S.status, S.valid, S.best_iter, S.num_inliers, S.best_cost = 77, 77, 77, 77, 7.0
        fl0[:] = 9
        assert solve._L().b200_twoview_ransac(solve._handle(0), 2, arr) == -1
        for S in arr:
            assert (S.status, S.valid, S.best_iter, S.num_inliers, S.best_cost) == (77, 77, 77, 77, 7.0)
        assert (fl0 == 9).all()
    keep = []
    arr = (solve.TwoviewProblem * 1)()
    arr[0], _ = solve._pack_twoview(pr, keep)
    arr[0].model = 2
    assert solve._L().b200_twoview_ransac(solve._handle(0), 1, arr) == -1
    arr[0].model = 0
    arr[0].matches_12 = None
    assert solve._L().b200_twoview_ransac(solve._handle(0), 1, arr) == -1
    arr[0], _ = solve._pack_twoview(pr, keep)
    arr[0].n_keypts_1 = -1
    assert solve._L().b200_twoview_ransac(solve._handle(0), 1, arr) == -1
    with pytest.raises(B200Error):
        solve.twoview_ransac_batch([bad_index])
    assert solve._L().b200_twoview_ransac(solve._handle(0), -1, None) == -1
    assert solve._L().b200_twoview_ransac(solve._handle(0), 0, None) == 0


@pytest.mark.parametrize("cls,model", [("homography_solver", "H"), ("fundamental_solver", "F")])
def test_python_solvers_match_oracle_and_continue_their_engines(cls, model):
    from stella_vslam_b200 import solve
    p = synth.make_twoview_problem(21, 400, 0.6, "planar" if model == "H" else "general")
    s = getattr(solve, cls)(p["keypts_1"], p["keypts_2"], p["matches_12"], 1.0, use_fixed_seed=True)
    eng = solve.mt19937()
    for _ in range(2):  # the second call continues the engine
        s.find_via_ransac(100, False)
        ms = solve.draw_min_sets(400, 100, eng, set_size=4 if model == "H" else 8)
        ref = O.twoview_ransac(model, p["keypts_1"], p["keypts_2"], p["matches_12"], ms, 1.0, False)
        assert s.solution_is_valid() == ref["valid"] and ref["valid"]
        assert s.get_best_cost().tobytes() == ref["best_cost"].tobytes()
        M = s.get_best_H_21() if model == "H" else s.get_best_F_21()
        assert M.tobytes() == ref["M_21"].tobytes()
        assert s.get_inlier_matches() == [bool(v) for v in ref["inlier_flags"]]
