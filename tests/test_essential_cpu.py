"""solve::essential_solver on the CPU: the oracle's stages against numpy / scipy, the RANSAC rules and check_inliers' NaN handling."""
import os
import subprocess
import tempfile

import numpy as np
import pytest
import scipy.linalg

import essential_oracle as eo
from workloads import synth


def _unit(a):
    return a / np.linalg.norm(a, axis=-1, keepdims=True)


def _same_up_to_scale(A, B):
    a, b = A.reshape(-1) / np.linalg.norm(A), B.reshape(-1) / np.linalg.norm(B)
    return min(np.abs(a - b).max(), np.abs(a + b).max())


def _five(seed, model="perspective"):
    p = synth.make_essential_problem(seed, n=5, model=model, case="n5")
    return p["bearings_1"], p["bearings_2"], p["E_21"]


def _action_matrix(b1, b2):
    basis, _ = eo.nullspace5(b1, b2)
    M = eo.constraint_matrix(basis)
    X, _ = eo.lu_solve10(M[:, :10], M[:, 10:])
    A = np.zeros((10, 10))
    A[:3] = X[:3]
    A[3], A[4], A[5] = X[4], X[5], X[7]
    A[6, 0] = A[7, 1] = A[8, 3] = A[9, 6] = -1.0
    return A


@pytest.mark.parametrize("seed", range(6))
def test_nullspace_spans_scipy_null_space(seed):
    rng = np.random.default_rng(seed)
    b1, b2 = _unit(rng.standard_normal((5, 3))), _unit(rng.standard_normal((5, 3)))
    basis, wide = eo.nullspace5(b1, b2)
    assert basis is not None and not wide
    A = np.zeros((9, 9))
    for i in range(5):
        A[i] = np.concatenate([b2[i, 0] * b1[i], b2[i, 1] * b1[i], b2[i, 2] * b1[i]])
    ref = scipy.linalg.null_space(A)
    assert ref.shape[1] == 4
    assert np.max(scipy.linalg.subspace_angles(basis, ref)) < 1e-12


def test_lu_kernel_of_rank_deficient_matrix():
    rng = np.random.default_rng(1)
    A = rng.standard_normal((9, 9))
    A[3:] = 0.0
    A[2] = A[0]  # rank 2: a kernel of seven columns
    K = eo.lu_kernel(A)
    assert K.shape == (9, 7)
    assert np.abs(A @ K).max() < 1e-12
    assert np.linalg.matrix_rank(K) == 7


def test_duplicated_bearings_take_the_first_four_kernel_columns():
    b1, b2, _ = _five(2)
    b1[4], b2[4] = b1[1], b2[1]
    basis, wide = eo.nullspace5(b1, b2)
    assert wide and basis is not None
    A = np.zeros((9, 9))
    for i in range(5):
        A[i] = np.concatenate([b2[i, 0] * b1[i], b2[i, 1] * b1[i], b2[i, 2] * b1[i]])
    assert np.abs(A @ basis).max() < 1e-12
    _, fl = eo.minimal(b1, b2)
    assert fl & eo.STATUS_WIDE_KER


def test_lu_solve_matches_numpy_and_handles_rank_deficiency():
    rng = np.random.default_rng(3)
    A, B = rng.standard_normal((10, 10)), rng.standard_normal((10, 10))
    X, r = eo.lu_solve10(A, B)
    assert r == 10
    np.testing.assert_allclose(X, np.linalg.solve(A, B), rtol=0, atol=1e-10)
    A[7] = A[2] + A[5]
    B = A @ rng.standard_normal((10, 10))  # consistent right-hand sides
    X, r = eo.lu_solve10(A, B)
    assert r == 9
    assert np.abs(A @ X - B).max() < 1e-10


@pytest.mark.parametrize("seed", range(8))
@pytest.mark.parametrize("model", ["perspective", "equirect"])
def test_real_eigenvalues_match_numpy(seed, model):
    b1, b2, _ = _five(seed, model)
    A = _action_matrix(b1, b2)
    ev, V = eo.eigen10(A)
    ref = np.linalg.eigvals(A)
    mine = np.sort(ev[ev.imag == 0].real)
    theirs = np.sort(ref[np.abs(ref.imag) <= 1e-9 * np.maximum(1.0, np.abs(ref.real))].real)
    assert len(mine) == len(theirs)
    np.testing.assert_allclose(mine, theirs, rtol=0, atol=1e-9 * max(1.0, np.abs(theirs).max()))
    for s in np.flatnonzero(ev.imag == 0):  # unit eigenvectors
        v = V[:, s]
        assert abs(np.linalg.norm(v) - 1.0) < 1e-12
        assert np.abs(A @ v - ev[s].real * v).max() < 1e-8 * max(1.0, np.abs(A).max())


@pytest.mark.parametrize("seed", range(10))
@pytest.mark.parametrize("model", ["perspective", "equirect"])
def test_true_essential_among_minimal_candidates(seed, model):
    b1, b2, E = _five(seed, model)
    cands, fl = eo.minimal(b1, b2)
    assert fl == 0 and len(cands) >= 1
    assert min(_same_up_to_scale(C, E) for C in cands) < 1e-8
    for C in cands:  # every candidate satisfies the five epipolar constraints
        assert np.abs(np.einsum("ij,jk,ik->i", b2, C / np.linalg.norm(C), b1)).max() < 1e-9


@pytest.mark.parametrize("m", [8, 9, 50])
def test_eight_point_recompute_matches_numpy(m):
    rng = np.random.default_rng(m)
    p = synth.make_essential_problem(10 + m, n=m, inlier_frac=1.0, noise=2e-3)
    b1, b2 = p["bearings_1"], p["bearings_2"]
    E, st = eo.nonminimal(b1, b2)
    assert st == 0
    A = np.stack([np.concatenate([y[0] * x, y[1] * x, y[2] * x]) for x, y in zip(b1, b2)])
    v = np.linalg.svd(A)[2][-1] if m >= 9 else scipy.linalg.null_space(A)[:, 0]
    U, s, Vt = np.linalg.svd(v.reshape(3, 3))
    ref = U @ np.diag([s[0], s[1], 0.0]) @ Vt
    assert _same_up_to_scale(E, ref) < 1e-10
    assert abs(np.linalg.norm(E) - np.linalg.norm(ref)) < 1e-10
    assert abs(np.linalg.det(E)) < 1e-12
    del rng


def _ransac_py(b1, b2, min_sets, recompute=True):
    """The reference's find_via_ransac control flow over the oracle's stages."""
    best, best_E, best_num, best_it, best_k = np.float32(np.finfo(np.float32).max), None, 0, -1, -1
    for it, s in enumerate(min_sets):
        cands, _ = eo.minimal(b1[s], b2[s])
        for k, C in enumerate(cands):
            num, _, cost = eo.check_inliers(b1, b2, C)
            if num > 5 and best > cost:
                best, best_E, best_num, best_it, best_k = cost, C, num, it, k
    valid = best < np.finfo(np.float32).max
    if not valid:
        return dict(valid=False, best_cost=best)
    _, flags, _ = eo.check_inliers(b1, b2, best_E)
    if recompute and best_num >= 8:
        best_E, _ = eo.nonminimal(b1[flags], b2[flags])
        _, flags, best = eo.check_inliers(b1, b2, best_E)
    return dict(valid=True, best_cost=best, E_21=best_E, num_inliers=best_num, best_iter=best_it, best_candidate=best_k, inlier_flags=flags)


@pytest.mark.parametrize("recompute", [False, True])
@pytest.mark.parametrize("case", [None, "planar", "duplicated"])
def test_ransac_follows_the_reference_rules(recompute, case):
    p = synth.make_essential_problem(5, n=60, inlier_frac=0.5, case=case, noise=1e-3)
    rng = np.random.default_rng(0)
    ms = np.array([rng.choice(60, 5, replace=False) for _ in range(40)], np.int32)
    r = eo.essential_ransac(p["bearings_1"], p["bearings_2"], ms, recompute)
    ref = _ransac_py(p["bearings_1"], p["bearings_2"], ms, recompute)
    assert r["valid"] == ref["valid"]
    assert r["best_cost"].tobytes() == np.float32(ref["best_cost"]).tobytes()
    if ref["valid"]:
        assert (r["best_iter"], r["best_candidate"], r["num_inliers"]) == (ref["best_iter"], ref["best_candidate"], ref["num_inliers"])
        assert r["E_21"].tobytes() == np.asarray(ref["E_21"]).tobytes()
        assert (r["inlier_flags"] == ref["inlier_flags"]).all()


def test_first_of_equal_costs_wins_and_recompute_needs_eight_inliers():
    p = synth.make_essential_problem(7, n=40, inlier_frac=0.6, noise=1e-3)
    b1, b2 = p["bearings_1"], p["bearings_2"]
    inl = np.flatnonzero(p["gt_inlier"])
    s = inl[:5].astype(np.int32)
    r = eo.essential_ransac(b1, b2, np.stack([s, s, s]), recompute=False)
    assert r["valid"] and r["best_iter"] == 0  # the repeats score the same: only a strictly lower cost replaces the winner
    cands, _ = eo.minimal(b1[s], b2[s])
    assert r["E_21"].tobytes() == cands[r["best_candidate"]].tobytes()
    # a winner with 6 or 7 inliers is kept as it is: no recompute below 8
    q = synth.make_essential_problem(8, n=14, inlier_frac=0.5, noise=0.0)
    qi = np.flatnonzero(q["gt_inlier"])[:5].astype(np.int32)
    rr = eo.essential_ransac(q["bearings_1"], q["bearings_2"], qi[None], recompute=True)
    if rr["valid"] and rr["num_inliers"] < 8:
        cands, _ = eo.minimal(q["bearings_1"][qi], q["bearings_2"][qi])
        assert rr["E_21"].tobytes() == cands[rr["best_candidate"]].tobytes()
    assert rr["valid"] and 5 < rr["num_inliers"] < 8


def test_strictly_more_than_five_inliers():
    p = synth.make_essential_problem(4, n=5, case="n5")
    r = eo.essential_ransac(p["bearings_1"], p["bearings_2"], [[0, 1, 2, 3, 4]] * 3)
    assert not r["valid"] and r["best_cost"] == np.finfo(np.float32).max
    assert not r["inlier_flags"].any()


def test_early_return_writes_nothing():
    b = _unit(np.random.default_rng(0).standard_normal((4, 3)))
    r = eo.essential_ransac(b, b, np.zeros((0, 5), np.int32))
    assert not r["valid"] and r["inlier_flags"] is None and r["best_cost"] == 0.0


def _check_inliers_numpy(b1, b2, E):
    thr = eo.cos_angle_thr()
    e2, e1 = b1 @ E.T, b2 @ E
    with np.errstate(invalid="ignore", divide="ignore"):
        c2 = (np.linalg.norm(np.cross(e2, b2), axis=1) / np.linalg.norm(e2, axis=1)).astype(np.float32)
        c1 = (np.linalg.norm(np.cross(e1, b1), axis=1) / np.linalg.norm(e1, axis=1)).astype(np.float32)
    worst = np.where(c2 < c1, c2, c1)  # std::min(cos_in_1, cos_in_2)
    flags = thr < worst
    cost = np.float32(0.0)
    for j in range(len(b1)):
        cost = np.float32(np.float64(cost) + (1.0 - np.float64(worst[j] if flags[j] else thr)))
    return flags, cost


def test_nan_terms_stay_outliers():
    rng = np.random.default_rng(5)
    b1, b2 = _unit(rng.standard_normal((12, 3))), _unit(rng.standard_normal((12, 3)))
    num, flags, cost = eo.check_inliers(b1, b2, np.zeros((3, 3)))  # 0/0 on both sides
    assert num == 0 and not flags.any()
    assert cost == _check_inliers_numpy(b1, b2, np.zeros((3, 3)))[1]
    # a rank-one E whose left null space holds some of view 2's bearings: cos_in_1 is 0/0 there and std::min keeps the NaN
    u, w = _unit(rng.standard_normal(3)), _unit(rng.standard_normal(3))
    E = np.outer(u, w)
    b2[:4] = _unit(np.cross(u, rng.standard_normal((4, 3))))
    num, flags, cost = eo.check_inliers(b1, b2, E)
    ref_flags, ref_cost = _check_inliers_numpy(b1, b2, E)
    assert not flags[:4].any()
    assert (flags == ref_flags).all() and cost.tobytes() == ref_cost.tobytes()


@pytest.mark.parametrize("seed", range(4))
def test_check_inliers_matches_numpy(seed):
    p = synth.make_essential_problem(seed, n=200, model="equirect", noise=1e-3)
    E = p["E_21"] + 1e-3 * np.random.default_rng(seed).standard_normal((3, 3))
    num, flags, cost = eo.check_inliers(p["bearings_1"], p["bearings_2"], E)
    ref_flags, ref_cost = _check_inliers_numpy(p["bearings_1"], p["bearings_2"], E)
    assert (flags == ref_flags).all() and num == ref_flags.sum()
    assert cost.tobytes() == ref_cost.tobytes()


def test_solver_early_return_draws_nothing():
    from stella_vslam_b200 import solve
    b = _unit(np.random.default_rng(0).standard_normal((4, 3)))
    s = solve.essential_solver(b, b, [(i, i) for i in range(4)], use_fixed_seed=True)
    before = bytes(s.random_engine_)
    s.find_via_ransac(1000, True)
    assert not s.solution_is_valid() and s.get_best_cost() == 0.0 and s.get_inlier_matches() == []
    assert bytes(s.random_engine_) == before
    with pytest.raises(ValueError):
        s.find_via_ransac(10, True, 8)


def test_problem_struct_layout():
    import ctypes as C
    from stella_vslam_b200 import solve
    S = solve.EssentialProblem
    names = [f[0] for f in S._fields_]
    d = tempfile.mkdtemp(prefix="b200_layout_")
    src, exe = os.path.join(d, "l.c"), os.path.join(d, "l")
    inc = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "include")
    with open(src, "w") as f:
        f.write("#include <stddef.h>\n#include <stdio.h>\n#include \"b200vslam.h\"\nint main(void) {\n")
        for nm in names:
            f.write(f'    printf("%zu\\n", offsetof(b200_essential_problem_t, {nm}));\n')
        f.write('    printf("%zu\\n", sizeof(b200_essential_problem_t));\n    return 0;\n}\n')
    subprocess.check_call([os.environ.get("CC", "gcc"), "-std=c11", "-I", inc, "-o", exe, src])
    ref = [int(v) for v in subprocess.check_output([exe]).split()]
    assert [getattr(S, nm).offset for nm in names] + [C.sizeof(S)] == ref
