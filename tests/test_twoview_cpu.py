"""CPU checks of the two-view RANSAC restatement (csrc/twoview_core.h compiled as C by tests/twoview_oracle.c) against numpy: solve::normalize,
the DLT / eight-point null vectors and JacobiSVD rank, the transfer and Sampson errors, and recovery of the true H / F; plus the ctypes
layout of b200_twoview_problem_t.  No GPU needed."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import twoview_oracle as O  # noqa: E402

from workloads import synth  # noqa: E402


def _unit(M):
    """M scaled to unit Frobenius norm with its largest entry positive (a projective matrix up to sign and scale)."""
    M = np.asarray(M, np.float64)
    M = M / np.linalg.norm(M)
    return M * np.sign(M.flat[np.argmax(np.abs(M))])


def test_normalize_matches_the_float_recipe():
    rng = np.random.default_rng(0)
    pts = np.stack([rng.uniform(0, 752, 301), rng.uniform(0, 480, 301)], 1).astype(np.float32)
    out, mean, l1, T = O.normalize(pts)
    f = np.float32
    sx, sy = f(0), f(0)
    for x, y in pts:  # std::accumulate: float adds in order
        sx, sy = f(sx + x), f(sy + y)
    m = np.array([f(np.float64(sx) / len(pts)), f(np.float64(sy) / len(pts))], np.float32)  # Point2f / double: in double, then float
    lx, ly = f(0), f(0)
    for x, y in pts:
        lx, ly = f(lx + abs(f(x - m[0]))), f(ly + abs(f(y - m[1])))
    d = np.array([f(np.float64(lx) / len(pts)), f(np.float64(ly) / len(pts))], np.float32)
    assert mean.tobytes() == m.tobytes() and l1.tobytes() == d.tobytes()
    np.testing.assert_array_equal(out, ((pts - m) / d).astype(np.float32))
    ref_T = np.array([[1 / np.float64(d[0]), 0, -np.float64(m[0]) / np.float64(d[0])],
                      [0, 1 / np.float64(d[1]), -np.float64(m[1]) / np.float64(d[1])], [0, 0, 1]])
    assert T.tobytes() == ref_T.tobytes()
    # the normalised points have zero mean and unit mean absolute deviation up to float rounding
    assert np.abs(out.astype(np.float64).mean(0)).max() < 1e-5
    np.testing.assert_allclose(np.abs(out.astype(np.float64)).mean(0), 1.0, rtol=1e-5)


@pytest.mark.parametrize("m", [8, 9, 10, 18])
def test_svd_n9_null_vector_and_rank(m):
    """The wide (8 rows), square (9) and tall (>= 10) paths: V's last column against numpy's, the singular values, rank()."""
    rng = np.random.default_rng(m)
    A = rng.standard_normal((m, 9))
    v, sv, rank, st = O.svd_n9(A)
    assert st == 0
    _, s_np, Vt = np.linalg.svd(A)
    np.testing.assert_allclose(sv, s_np[:min(m, 9)], rtol=1e-12, atol=1e-13)
    assert rank == min(m, 9)
    if m == 8:  # a wide matrix has an exact null vector; numpy's last right singular vector spans it
        assert np.linalg.norm(A @ v) < 1e-12
    np.testing.assert_allclose(v * np.sign(v @ Vt[-1]), Vt[-1], atol=1e-10)
    B = A.copy()
    B[:, 4] = B[:, 2] + B[:, 3]  # two dependent columns less: rank min(m, 9) - 1
    B[:, 5] = 2 * B[:, 1]
    assert O.svd_n9(B)[2] == min(m, 9) - 2 if m > 8 else O.svd_n9(B)[2] == 7


def _dlt_h(p1, p2):
    rows = []
    for (x1, y1), (x2, y2) in zip(p1.astype(np.float64), p2.astype(np.float64)):
        rows.append([0, 0, 0, -x1, -y1, -1, y2 * x1, y2 * y1, y2])
        rows.append([x1, y1, 1, 0, 0, 0, -x2 * x1, -x2 * y1, -x2])
    return np.array(rows)


def _dlt_f(p1, p2):
    return np.array([[x2 * x1, x2 * y1, x2, y2 * x1, y2 * y1, y2, x1, y1, 1] for (x1, y1), (x2, y2) in
                     zip(p1.astype(np.float64), p2.astype(np.float64))])


@pytest.mark.parametrize("m", [4, 5, 12])
def test_compute_H_21_is_the_dlt_null_vector(m):
    p = synth.make_twoview_problem(3, 60, 1.0, "planar", noise=0.0)
    mt = p["matches_12"][:m]
    n1, _, _, _ = O.normalize(p["keypts_1"])
    n2, _, _, _ = O.normalize(p["keypts_2"])
    q1, q2 = n1[mt[:, 0]], n2[mt[:, 1]]
    H, st = O.estimate("H", q1, q2)
    assert st == 0 and H is not None
    A = _dlt_h(q1, q2)
    _, _, Vt = np.linalg.svd(A)
    np.testing.assert_allclose(_unit(H), _unit(Vt[-1].reshape(3, 3)), atol=1e-9)


@pytest.mark.parametrize("m", [8, 9, 20])
def test_compute_F_21_is_the_rank2_projection_of_the_null_vector(m):
    p = synth.make_twoview_problem(4, 60, 1.0, "general", noise=0.0)
    mt = p["matches_12"][:m]
    n1, _, _, _ = O.normalize(p["keypts_1"])
    n2, _, _, _ = O.normalize(p["keypts_2"])
    q1, q2 = n1[mt[:, 0]], n2[mt[:, 1]]
    F, st = O.estimate("F", q1, q2)
    assert st == 0
    _, _, Vt = np.linalg.svd(_dlt_f(q1, q2))
    U, s, Wt = np.linalg.svd(Vt[-1].reshape(3, 3))
    ref = U @ np.diag([s[0], s[1], 0.0]) @ Wt
    np.testing.assert_allclose(_unit(F), _unit(ref), atol=1e-9)
    assert abs(np.linalg.det(F)) < 1e-14 * np.linalg.norm(F) ** 3


def test_collinear_and_duplicated_minimal_sets_are_degenerate_for_H():
    rng = np.random.default_rng(5)
    q1 = rng.standard_normal((4, 2)).astype(np.float32)
    q2 = rng.standard_normal((4, 2)).astype(np.float32)
    assert O.estimate("H", q1, q2)[0] is not None
    c1, c2 = q1.copy(), q2.copy()
    c1[3], c2[3] = c1[2], c2[2]  # a repeated correspondence: six independent equations
    assert O.estimate("H", c1, c2)[0] is None
    s = np.array([-1.0, 0.0, 0.5, 1.5], np.float32)
    l1 = np.stack([s, 2 * s], 1).astype(np.float32)  # four points on one line in both frames
    l2 = np.stack([s, 0.5 - s], 1).astype(np.float32)
    assert O.estimate("H", l1, l2)[0] is None


def test_inverse33_and_errors_against_numpy():
    rng = np.random.default_rng(6)
    M = rng.standard_normal((3, 3))
    np.testing.assert_allclose(O.inverse33(M), np.linalg.inv(M), rtol=1e-12, atol=1e-12)
    H = np.array([[1.02, 0.01, 3.0], [-0.02, 0.99, -2.0], [1e-5, -2e-5, 1.0]])
    for _ in range(20):
        k1 = rng.uniform(0, 700, 2).astype(np.float32)
        k2 = rng.uniform(0, 700, 2).astype(np.float32)
        a, b = np.append(k1.astype(np.float64), 1), np.append(k2.astype(np.float64), 1)
        t1, t2 = H @ a, np.linalg.inv(H) @ b
        ref = max(np.sum((b - t1 / t1[2]) ** 2), np.sum((a - t2 / t2[2]) ** 2))
        np.testing.assert_allclose(O.error("H", H, k1, k2), ref, rtol=1e-6)
        F = rng.standard_normal((3, 3))
        Fa, bF = F @ a, b @ F
        ref = (b @ F @ a) ** 2 / (Fa[0] ** 2 + Fa[1] ** 2 + bF[0] ** 2 + bF[1] ** 2)
        np.testing.assert_allclose(O.error("F", F, k1, k2), ref, rtol=1e-12)


def test_check_inliers_cost_is_the_float_sum_in_match_order():
    p = synth.make_twoview_problem(7, 200, 0.6, "planar")
    num, fl, cost = O.check_inliers("H", p["keypts_1"], p["keypts_2"], p["matches_12"], p["H_21"])
    f = np.float32
    thr = f(f(5.991) * f(1.0))
    c = f(0)
    k1, k2 = p["keypts_1"][p["matches_12"][:, 0]], p["keypts_2"][p["matches_12"][:, 1]]
    for j in range(len(k1)):
        e = f(O.error("H", p["H_21"], k1[j], k2[j]))
        assert bool(fl[j]) == (np.float64(thr) > np.float64(e))
        c = f(c + (e if fl[j] else thr))
    assert cost.tobytes() == c.tobytes() and num == fl.sum()
    assert (fl == p["gt_inlier"]).mean() > 0.95


def _ransac(p, model, n_iter=200, recompute=True, seed=0):
    from_engine = np.random.default_rng(seed)
    n, k = len(p["matches_12"]), 4 if model == "H" else 8
    ms = np.array([from_engine.choice(n, k, replace=False) for _ in range(n_iter)], np.int32) if n >= k else np.zeros((0, k), np.int32)
    return O.twoview_ransac(model, p["keypts_1"], p["keypts_2"], p["matches_12"], ms, recompute=recompute)


def test_noise_free_recovery_of_H_and_F():
    """The keypoints are float (cv::KeyPoint), so noise-free data still carries a float rounding of the pixel coordinates: the estimates
    agree with the truth to about 1e-6 relative, not to double precision."""
    p = synth.make_twoview_problem(8, 300, 1.0, "planar", noise=0.0)
    r = _ransac(p, "H")
    assert r["valid"] and r["inlier_flags"].all()
    np.testing.assert_allclose(_unit(r["M_21"]), _unit(p["H_21"]), atol=1e-6)
    p = synth.make_twoview_problem(9, 300, 1.0, "general", noise=0.0)
    r = _ransac(p, "F")
    assert r["valid"] and r["inlier_flags"].all()
    np.testing.assert_allclose(_unit(r["M_21"]), _unit(p["F_21"]), atol=1e-6)


@pytest.mark.parametrize("model", ["H", "F"])
def test_early_return_below_eight_matches(model):
    p7 = synth.make_twoview_problem(10, case="n7")
    r = _ransac(p7, model)
    assert (r["valid"], r["best_iter"], r["best_cost"], r["inlier_flags"]) == (False, -1, np.float32(0.0), None)
    p8 = synth.make_twoview_problem(10, case="n8", noise=0.0)
    r = _ransac(p8, model, n_iter=20)
    assert r["inlier_flags"] is not None
    if model == "F":  # eight matches cannot give more than eight inliers: no winner, the cost stays FLT_MAX
        assert not r["valid"] and r["best_cost"] == np.finfo(np.float32).max and not r["inlier_flags"].any()


def test_recovery_with_outliers_selects_the_true_inliers():
    p = synth.make_twoview_problem(11, 400, 0.6, "planar")
    r = _ransac(p, "H", recompute=True)
    assert r["valid"] and (r["inlier_flags"] == p["gt_inlier"]).mean() > 0.97
    p = synth.make_twoview_problem(12, 400, 0.6, "general")
    r = _ransac(p, "F", recompute=True)
    assert r["valid"] and (r["inlier_flags"][p["gt_inlier"]]).mean() > 0.97


def test_problem_struct_layout():
    import ctypes as C
    from stella_vslam_b200 import solve
    S = solve.TwoviewProblem
    names = [f[0] for f in S._fields_]
    d = tempfile.mkdtemp(prefix="b200_layout_")
    src, exe = os.path.join(d, "l.c"), os.path.join(d, "l")
    inc = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "include")
    with open(src, "w") as f:
        f.write("#include <stddef.h>\n#include <stdio.h>\n#include \"b200vslam.h\"\nint main(void) {\n")
        for nm in names:
            f.write(f'    printf("%zu\\n", offsetof(b200_twoview_problem_t, {nm}));\n')
        f.write('    printf("%zu\\n", sizeof(b200_twoview_problem_t));\n    return 0;\n}\n')
    subprocess.check_call([os.environ.get("CC", "gcc"), "-std=c11", "-I", inc, "-o", exe, src])
    ref = [int(v) for v in subprocess.check_output([exe]).split()]
    assert [getattr(S, nm).offset for nm in names] + [C.sizeof(S)] == ref
