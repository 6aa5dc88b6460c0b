"""GPU parity: b200_essential_ransac (solve::essential_solver::find_via_ransac, five-point) against the CPU restatement, bit for bit, and
the tracker's robust-matching fallback chain (brute-force match, then the essential RANSAC) on a synthetic keyframe pair."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import essential_oracle as O  # noqa: E402

from workloads import synth  # noqa: E402

pytestmark = pytest.mark.gpu

CASES = [None, "pure_rotation", "planar", "duplicated", "n5", "inliers8", "inliers9", "inliers10"]


def _problem(seed, n, model, recompute, case=None, max_num_iter=200, inlier_frac=None):
    from stella_vslam_b200 import solve
    frac = np.random.default_rng(seed).uniform(0.3, 0.9) if inlier_frac is None else inlier_frac
    p = synth.make_essential_problem(seed, n, frac, model, case=case)
    m = len(p["bearings_1"])
    ms = solve.draw_min_sets(m, max_num_iter, solve.mt19937((seed,)), set_size=5) if m >= 5 else np.zeros((0, 5), np.int32)
    return dict(bearings_1=p["bearings_1"], bearings_2=p["bearings_2"], min_sets=ms, recompute=recompute), p


def _assert_same(dev, ref):
    assert dev["status"] == (-1 if ref["status"] & (O.STATUS_SCHUR | O.STATUS_SVD) else 0)
    for k in ("valid", "best_iter", "best_candidate", "num_inliers"):
        assert dev[k] == ref[k], k
    assert dev["best_cost"].tobytes() == ref["best_cost"].tobytes()
    if ref["inlier_flags"] is None:
        assert dev["inlier_flags"] is None
    else:
        np.testing.assert_array_equal(dev["inlier_flags"], ref["inlier_flags"])
    if ref["valid"]:
        assert dev["E_21"].tobytes() == ref["E_21"].tobytes()


def _oracle(pr):
    return O.essential_ransac(pr["bearings_1"], pr["bearings_2"], pr["min_sets"], pr["recompute"])


@pytest.mark.parametrize("recompute", [False, True])
@pytest.mark.parametrize("model", ["perspective", "equirect"])
def test_single_problem_matches_oracle(model, recompute):
    from stella_vslam_b200 import solve
    for seed in range(3):
        pr, _ = _problem(seed, 500, model, recompute, max_num_iter=1000 if seed == 0 else 100)
        dev = solve.essential_ransac_batch([pr])[0]
        ref = _oracle(pr)
        assert ref["valid"]
        _assert_same(dev, ref)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("model", ["perspective", "equirect"])
def test_synth_cases_match_oracle(case, model):
    from stella_vslam_b200 import solve
    prs, refs = [], []
    for seed in range(4):
        pr, _ = _problem(100 + seed, 300, model, True, case=case)
        prs.append(pr)
        refs.append(_oracle(pr))
    for dev, ref in zip(solve.essential_ransac_batch(prs), refs):
        _assert_same(dev, ref)


@pytest.mark.parametrize("target", [8, 9, 10])
def test_recompute_svd_paths_at_their_thresholds(target):
    """A winner with exactly 8 (wide), 9 (square) or >= 10 (tall, ColPivHouseholderQR) inliers goes into the recompute."""
    from stella_vslam_b200 import solve
    case = {8: "inliers8", 9: "inliers9", 10: "inliers10"}[target]
    found = 0
    for seed in range(200):
        for model in ("perspective", "equirect"):
            pr, _ = _problem(seed, 0, model, True, case=case, max_num_iter=300)
            ref = _oracle(pr)
            if not ref["valid"] or (ref["num_inliers"] != target if target < 10 else ref["num_inliers"] < 10):
                continue
            _assert_same(solve.essential_ransac_batch([pr])[0], ref)
            found += 1
        if found >= 3:
            break
    assert found >= 3


def test_batch_of_1024_is_permutation_invariant_and_matches_oracle():
    from stella_vslam_b200 import solve
    rng = np.random.default_rng(11)
    sizes = np.concatenate([[5, 6, 7, 8, 2000], rng.integers(5, 2001, 1019)])
    prs = []
    for i, n in enumerate(sizes):
        pr, _ = _problem(1000 + i, int(n), "equirect" if i % 3 == 0 else "perspective", bool(i % 2), max_num_iter=16)
        prs.append(pr)
    a = solve.essential_ransac_batch(prs)
    perm = rng.permutation(len(prs))
    b = solve.essential_ransac_batch([prs[i] for i in perm])
    for k, i in enumerate(perm):
        _assert_same(b[k], dict(a[i], status=0 if a[i]["status"] == 0 else O.STATUS_SCHUR))
    for i in range(0, len(prs), 4):  # every fourth against the oracle
        _assert_same(a[i], _oracle(prs[i]))


def test_invalid_input_writes_nothing():
    import ctypes as C
    from stella_vslam_b200 import solve
    from stella_vslam_b200._lib import B200Error
    pr, _ = _problem(3, 50, "perspective", True, max_num_iter=10)
    bad_index = dict(pr, min_sets=np.where(pr["min_sets"] == pr["min_sets"][0, 0], 50, pr["min_sets"]))
    bad_size = dict(pr, min_set_size=8, min_sets=np.zeros((10, 8), np.int32))
    for bad in (bad_index, bad_size):
        keep = []
        arr = (solve.EssentialProblem * 2)()
        arr[0], fl0 = solve._pack_essential(pr, keep)
        arr[1], fl1 = solve._pack_essential(bad, keep)
        for S in arr:
            S.status, S.valid, S.best_iter, S.num_inliers, S.best_cost = 77, 77, 77, 77, 7.0
        fl0[:] = 9
        rc = solve._L().b200_essential_ransac(solve._handle(0), 2, arr)
        assert rc == -1
        for S in arr:
            assert (S.status, S.valid, S.best_iter, S.num_inliers, S.best_cost) == (77, 77, 77, 77, 7.0)
        assert (fl0 == 9).all()
    with pytest.raises(B200Error):
        solve.essential_ransac_batch([bad_index])
    assert solve._L().b200_essential_ransac(solve._handle(0), -1, None) == -1
    assert solve._L().b200_essential_ransac(solve._handle(0), 0, None) == 0
    del C


def test_python_solver_matches_oracle_and_continues_its_engine():
    from stella_vslam_b200 import solve
    p = synth.make_essential_problem(21, 400, 0.5, "equirect")
    rng = np.random.default_rng(0)
    n1 = 450
    b1 = rng.standard_normal((n1, 3))
    b2 = rng.standard_normal((n1 + 30, 3))
    i1, i2 = rng.permutation(n1)[:400], rng.permutation(n1 + 30)[:400]
    b1[i1], b2[i2] = p["bearings_1"], p["bearings_2"]
    s = solve.essential_solver(b1, b2, np.stack([i1, i2], 1), use_fixed_seed=True)
    eng = solve.mt19937()
    for _ in range(2):  # the second call continues the engine
        s.find_via_ransac(300, True)
        ms = solve.draw_min_sets(400, 300, eng, set_size=5)
        ref = O.essential_ransac(p["bearings_1"], p["bearings_2"], ms, True)
        assert s.solution_is_valid() == ref["valid"] and ref["valid"]
        assert s.get_best_cost().tobytes() == ref["best_cost"].tobytes()
        assert s.get_best_E_21().tobytes() == ref["E_21"].tobytes()
        assert s.get_inlier_matches() == [bool(v) for v in ref["inlier_flags"]]


def _decompose(E):
    U, _, Vt = np.linalg.svd(E)
    W = np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1.0]])
    Rs = [U @ W @ Vt, U @ W.T @ Vt]
    return [R * np.sign(np.linalg.det(R)) for R in Rs], U[:, 2] / np.linalg.norm(U[:, 2])


def test_tracking_fallback_chain_recovers_the_relative_pose():
    from stella_vslam_b200 import match, solve
    k1, k2, g = synth.make_keyframe_pair(5, n1=1500, n2=1500)
    pairs = match.robust(0.8, True).brute_force_match(k1["desc"], k1["angle"], k2["desc"], k2["angle"])
    assert len(pairs) > 100
    s = solve.essential_solver(k1["bearings"], k2["bearings"], pairs, use_fixed_seed=True)
    s.find_via_ransac(1000, True)
    assert s.solution_is_valid() and s.status_ == 0
    ms = solve.draw_min_sets(len(pairs), 1000, solve.mt19937(), set_size=5)
    ref = O.essential_ransac(k1["bearings"][pairs[:, 0]], k2["bearings"][pairs[:, 1]], ms, True)
    assert s.get_best_E_21().tobytes() == ref["E_21"].tobytes()
    E, E_true = s.get_best_E_21(), g["E_12"].T
    Rs, t = _decompose(E)
    Rs_true, t_true = _decompose(E_true)
    rot_err = min(np.arccos(np.clip((np.trace(R.T @ Q) - 1) / 2, -1, 1)) for R in Rs for Q in Rs_true)
    t_err = np.arccos(np.clip(abs(t @ t_true), -1, 1))
    # the reference's unnormalised eight-point recompute over the 1 deg inliers constrains the translation direction of this mostly
    # forward motion far more loosely than the rotation: 0.12 rad here, 0.10 rad on the true correspondences (DESIGN.md section 8)
    assert rot_err < 1e-2 and t_err < 0.2
    # the injected epipolar violations (geometry["wrong"]) among the matched pairs.  The injected perturbation is isotropic, so about
    # half of it lies along the epipolar plane: even the true E rejects only about half of the injected set at the reference's 1 deg
    # threshold (52 % on this pair), so no estimate can flag 90 % of the whole set.  The check is on the injected violations more than
    # 3 deg off their plane, which any estimate close to the truth must reject.
    truth = {(int(a), int(b)): bool(w) for a, b, w in zip(g["perm1"], g["perm2"], g["wrong"])}
    injected = np.array([truth.get((int(a), int(b)), False) for a, b in pairs])
    b1, b2 = k1["bearings"][pairs[:, 0]], k2["bearings"][pairs[:, 1]]
    epi = b2 @ g["E_12"].T  # E_12 b2
    far = np.abs(np.sum(b1 * epi, 1)) / np.linalg.norm(epi, axis=1) > np.sin(np.deg2rad(3.0))
    flags = np.array(s.get_inlier_matches())
    assert injected.sum() > 30 and (injected & far).sum() > 10
    assert (~flags[injected & far]).mean() >= 0.9
