"""optimize::graph_optimizer without a GPU: the oracle's g2o::Sim3 algebra against 4x4 similarity matrices (scipy expm / logm), the
edge and its numeric Jacobian, the LM against scipy.optimize.least_squares, the write-back rules, build_essential_graph's edge
selection, the library's host-side ordering, and the ctypes mirrors of the new structs."""
import ctypes as C
import os

import numpy as np
import pytest
import scipy.linalg as sl
import scipy.optimize as so

import pgo_oracle as O
import test_abi_layout as ABI

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _hat(u):
    w, v, s = u[:3], u[3:6], u[6]
    M = np.zeros((4, 4))
    M[:3, :3] = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]) + s * np.eye(3)
    M[:3, 3] = v
    return M


def _mat(g):
    """4x4 similarity [s R | t] of a Sim3 8-vector."""
    x, y, z, w = g[:4]
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    M = np.eye(4)
    M[:3, :3] = g[7] * R
    M[:3, 3] = g[4:7]
    return M


# omega norm and sigma on both sides of each eps = 1e-5 branch, away from the boundary, and sigma = 0.  Inside |sigma| < 1e-5 g2o takes
# C = 1 (and A = 1/2, B = 1/6 for small omega): first-order terms whose error is about sigma / 2, so the 1e-12 comparison with expm uses
# sigma below 1e-12 there; the round trip through log (same approximations) is checked at sigma = 4e-6 as well.  For small omega g2o
# writes R = I + Omega + Omega^2, whose error is |omega|^2 / 2, so the small-angle cases use |omega| = 3e-8.
CASES = [(3e-8, 0.0), (3e-8, 5e-13), (3e-8, 0.2), (3e-8, -0.3), (0.4, 0.0), (0.4, -5e-13), (0.4, 0.25), (1.3, -0.4), (2.5, 0.1)]
LOG_CASES = CASES + [(3e-7, 4e-6), (3e-7, 0.2), (0.4, -3e-6)]


@pytest.mark.parametrize("theta,sigma", CASES)
def test_exp_matches_expm(theta, sigma):
    rng = np.random.default_rng(int(theta * 1e3) + int(abs(sigma) * 1e3) + 7)
    ax = rng.standard_normal(3)
    u = np.concatenate([theta * ax / np.linalg.norm(ax), rng.uniform(-2, 2, 3), [sigma]])
    np.testing.assert_allclose(_mat(O.exp(u)), sl.expm(_hat(u)), rtol=0, atol=1e-12)


@pytest.mark.parametrize("theta,sigma", LOG_CASES)
def test_log_inverts_exp(theta, sigma):
    rng = np.random.default_rng(11)
    ax = rng.standard_normal(3)
    u = np.concatenate([theta * ax / np.linalg.norm(ax), rng.uniform(-2, 2, 3), [sigma]])
    # the small-angle branch of log approximates theta / (2 sin theta) by 1/2: exact to O(theta^2)
    np.testing.assert_allclose(O.log(O.exp(u)), u, rtol=0, atol=1e-9)


def _rand_sim3(rng, scale=True):
    return O.exp(np.concatenate([rng.uniform(-1, 1, 3), rng.uniform(-5, 5, 3), [rng.uniform(-0.5, 0.5) if scale else 0.0]]))


def test_mul_inverse_map_match_matrices():
    rng = np.random.default_rng(3)
    for _ in range(20):
        a, b = _rand_sim3(rng), _rand_sim3(rng)
        np.testing.assert_allclose(_mat(O.mul(a, b)), _mat(a) @ _mat(b), atol=1e-12)
        np.testing.assert_allclose(_mat(O.inverse(a)), np.linalg.inv(_mat(a)), atol=1e-12)
        p = rng.uniform(-10, 10, 3)
        np.testing.assert_allclose(O.map(a, p), (_mat(a) @ np.append(p, 1))[:3], atol=1e-12)


def test_edge_error_zero_on_consistent_graph():
    rng = np.random.default_rng(4)
    for _ in range(10):
        v1, v2 = _rand_sim3(rng), _rand_sim3(rng)
        meas = O.mul(v2, O.inverse(v1))                    # Sim3_21 = Sim3_2w * Sim3_w1
        assert np.abs(O.edge_error(meas, v1, v2)).max() < 1e-12


def _err_matrix(meas, v1, v2):
    return np.real(sl.logm(_mat(meas) @ _mat(v1) @ np.linalg.inv(_mat(v2))))


def _vee(M):
    return np.array([M[2, 1], M[0, 2], M[1, 0], M[0, 3], M[1, 3], M[2, 3], (M[0, 0] + M[1, 1] + M[2, 2]) / 3])


@pytest.mark.parametrize("fix_scale", [False, True])
def test_numeric_jacobian_matches_independent_difference(fix_scale):
    rng = np.random.default_rng(5)
    for _ in range(4):
        v1, v2 = _rand_sim3(rng, not fix_scale), _rand_sim3(rng, not fix_scale)
        meas = O.mul(O.exp(rng.uniform(-0.05, 0.05, 7)), O.mul(v2, O.inverse(v1)))
        for side in (0, 1):
            J = O.edge_jacobian(meas, v1, v2, side, fix_scale)
            Jr = np.zeros((7, 7))
            for d in range(7 if not fix_scale else 6):
                du = np.zeros(7)
                du[d] = 1e-6
                ep = [sl.expm(_hat(du)) @ _mat(v) if k == side else _mat(v) for k, v in enumerate((v1, v2))]
                em = [sl.expm(_hat(-du)) @ _mat(v) if k == side else _mat(v) for k, v in enumerate((v1, v2))]
                fp = _vee(np.real(sl.logm(_mat(meas) @ ep[0] @ np.linalg.inv(ep[1]))))
                fm = _vee(np.real(sl.logm(_mat(meas) @ em[0] @ np.linalg.inv(em[1]))))
                Jr[:, d] = (fp - fm) / 2e-6
            np.testing.assert_allclose(J, Jr, rtol=0, atol=1e-5 * max(1.0, np.abs(Jr).max()))
            if fix_scale:
                assert np.array_equal(J[:, 6], np.zeros(7))


def _loop_graph(n=14, seed=6, fix_scale=False):
    from workloads import synth
    return synth.make_pose_graph(n, seed=seed, fix_scale=fix_scale, laps=1.0, lm_per_keyframe=2)


@pytest.mark.parametrize("n,fix_scale", [(14, False), (14, True), (40, False)])
def test_lm_optimum_matches_least_squares(n, fix_scale):
    g = _loop_graph(n, fix_scale=fix_scale)
    ref = O.graph_optimize(g, max_iter=200, gain_threshold=1e-12)
    early = O.graph_optimize(g)                                        # gain 1e-3 stops earlier
    assert early["iterations"] < ref["iterations"]
    free = np.nonzero(g["fixed"] == 0)[0]
    est0 = np.asarray(g["estimate"])
    dim = 6 if fix_scale else 7

    def poses(x):
        est = est0.copy()
        for k, v in enumerate(free):
            u = np.zeros(7)
            u[:dim] = x[dim * k:dim * k + dim]
            est[v] = O.mul(O.exp(u), est0[v])
        return est

    def resid(x):
        est = poses(x)
        return np.concatenate([O.edge_error(m, est[a], est[b]) for m, a, b in zip(g["e_meas"], g["e_v1"], g["e_v2"])])

    sol = so.least_squares(resid, np.zeros(dim * len(free)), xtol=1e-15, ftol=1e-15, gtol=1e-15, method="lm")
    want = poses(sol.x)
    for v in free:
        np.testing.assert_allclose(_mat(ref["estimate"][v]), _mat(want[v]), rtol=0, atol=1e-6 * max(1.0, np.abs(_mat(want[v])).max()))
    assert abs(ref["chi2_final"] - 2 * sol.cost) <= 1e-6 * 2 * sol.cost
    fixed = g["fixed"].astype(bool)
    assert np.array_equal(ref["estimate"][fixed], est0[fixed]) and np.array_equal(early["estimate"][fixed], est0[fixed])


def test_writeback_float_scale():
    g = _loop_graph()
    g = dict(g, estimate=np.asarray(g["estimate"]).copy())
    g["estimate"][:, 7] = 1.0 + 1e-4 * np.arange(len(g["estimate"]))         # scales whose float rounding changes t / s
    r = O.graph_optimize(g)
    for v in range(len(g["estimate"])):
        s64 = r["estimate"][v, 7]
        s32 = float(np.float32(s64))
        M = _mat(r["estimate"][v])
        want_t = r["estimate"][v, 4:7] / s32                             # pose_cw = [R | t / (float)s], R = sR / s
        np.testing.assert_allclose(r["pose_cw"][v, :3, :3], M[:3, :3] / s64, rtol=0, atol=1e-15)
        assert np.array_equal(r["pose_cw"][v, :3, 3], want_t)
        np.testing.assert_array_equal(r["pose_cw"][v, 3], [0, 0, 0, 1])
    diff = [not np.array_equal(r["estimate"][v, 4:7] / r["estimate"][v, 7], r["pose_cw"][v, :3, 3]) for v in range(len(g["estimate"]))]
    assert any(diff)                                                      # float and double scale give different t / s


def test_landmark_correction_honours_found_reference():
    from workloads import synth
    g, d = synth.make_pose_graph(40, seed=12, return_description=True)
    r = O.graph_optimize(g)
    vidx = {k: i for i, k in enumerate(g["vertex_ids"])}
    found = d["found_lm_to_ref_keyfrm_id"]
    assert found
    for k, (lid, pos_w, ref) in enumerate(d["landmarks"]):
        v = vidx[found.get(lid, ref)]
        # corrected_Sim3_wc[ref] (the inverse of the optimised Sim3_cw) after Sim3_cw[ref] before, as 4x4 similarity matrices
        want = (np.linalg.inv(_mat(r["estimate"][v])) @ _mat(g["estimate"][v]) @ np.append(pos_w, 1))[:3]
        np.testing.assert_allclose(r["points"][k], want, rtol=0, atol=1e-9 * max(1.0, np.abs(want).max()))
    moved = [lid for lid in found if found[lid] != d["landmarks"][lid][2]]
    assert moved                                                          # the re-referenced landmarks take the loop keyframe's correction


def test_workload_honours_found_lm_to_ref_keyfrm_id():
    from workloads import synth
    g, d = synth.make_pose_graph(60, seed=12, return_description=True)
    vidx = {k: i for i, k in enumerate(g["vertex_ids"])}
    assert d["found_lm_to_ref_keyfrm_id"]
    for k, (lid, _, ref) in enumerate(d["landmarks"]):
        assert g["point_ref"][k] == vidx[d["found_lm_to_ref_keyfrm_id"].get(lid, ref)]


# ---------------- build_essential_graph: one hand-built case per selection rule ----------------
def _kf(i, parent, children=(), loop_edges=(), covis=(), erased=False):
    return dict(id=i, rot_cw=np.eye(3), trans_cw=np.array([float(i), 0.0, 0.0]), erased=erased, parent=parent, children=list(children),
                loop_edges=list(loop_edges), covisibilities=list(covis))


def _edges(g):
    ids = g["vertex_ids"]
    return [(ids[a], ids[b]) for a, b in zip(g["e_v1"], g["e_v2"])]


def test_builder_parent_loop_and_covisibility_rules():
    from stella_vslam_b200.optimize import build_essential_graph
    kfs = [_kf(0, None, [1], covis=[(1, 300), (3, 200)]),
           _kf(1, 0, [2], covis=[(0, 300), (2, 250)]),
           _kf(2, 1, [3], covis=[(1, 250), (3, 120), (0, 100)]),
           _kf(3, 2, [4], loop_edges=[0], covis=[(2, 120), (0, 200), (4, 150), (1, 99)]),
           _kf(4, 3, [], covis=[(3, 150), (5, 300), (2, 101)]),
           _kf(5, 4, [], erased=True, covis=[(4, 300)])]
    g = build_essential_graph(kfs, curr_id=4, loop_id=0, loop_connections=[], min_num_shared_lms=100)
    assert g["vertex_ids"] == [0, 1, 2, 3, 4]                          # erased keyframes are no vertices
    assert list(g["fixed"]) == [1, 0, 0, 0, 1]                         # root, loop and current keyframes are fixed
    # per keyframe: parent edge, loop edges (id1 > id2), covisibilities >= threshold, not parent/child/loop edge/erased, id1 > id2, new
    assert _edges(g) == [(1, 0), (2, 1), (2, 0), (3, 2), (3, 0), (4, 3), (4, 2)]


def test_builder_loop_connections_threshold_and_current_loop_pair():
    from stella_vslam_b200.optimize import build_essential_graph
    kfs = [_kf(0, None, [1], covis=[(3, 50)]), _kf(1, 0, [2], covis=[(3, 150)]), _kf(2, 1, [3]), _kf(3, 2, [], covis=[(0, 50), (1, 150)])]
    lc = [(3, [0, 1]), (2, [0])]
    g = build_essential_graph(kfs, curr_id=3, loop_id=0, loop_connections=lc, min_num_shared_lms=100)
    # (3, 0) is kept below the threshold (current <-> loop), (3, 1) by its 150 shared landmarks, (2, 0) dropped (0 shared)
    assert _edges(g)[:2] == [(3, 0), (3, 1)]
    assert _edges(g)[2:] == [(1, 0), (2, 1), (3, 2)]


def test_builder_duplicates_and_measurements():
    from stella_vslam_b200.optimize import build_essential_graph, sim3_from_rts, sim3_inverse, sim3_mul
    kfs = [_kf(0, None, [1]), _kf(1, 0, [2], covis=[(0, 500)]), _kf(2, 1, [], covis=[(0, 400), (1, 300)])]
    pre = {2: sim3_from_rts(np.eye(3), [5.0, 1.0, 0.0], 0.9)}
    non = {2: sim3_from_rts(np.eye(3), [2.5, 0.0, 0.0], 1.0)}
    lc = [(2, [0])]
    g = build_essential_graph(kfs, curr_id=2, loop_id=0, loop_connections=lc, non_corrected_Sim3s=non, pre_corrected_Sim3s=pre,
                              min_num_shared_lms=100)
    # the loop connection inserted (2, 0) first, so the covisibility (2, 0) is a duplicate and skipped
    assert _edges(g) == [(2, 0), (1, 0), (2, 1)]
    S = {k: sim3_from_rts(np.eye(3), [float(k), 0.0, 0.0], 1.0) for k in (0, 1)}
    S[2] = pre[2]
    np.testing.assert_array_equal(g["estimate"][2], pre[2])
    # loop connections measure from the (pre-corrected) estimates, the other edges from non_corrected where present
    np.testing.assert_array_equal(g["e_meas"][0], sim3_mul(S[0], sim3_inverse(S[2])))
    np.testing.assert_array_equal(g["e_meas"][1], sim3_mul(S[0], sim3_inverse(S[1])))
    np.testing.assert_array_equal(g["e_meas"][2], sim3_mul(S[1], sim3_inverse(non[2])))


def test_builder_parent_with_larger_id_skips_the_keyframe():
    from stella_vslam_b200.optimize import build_essential_graph
    # keyframe 2 was reparented to its sibling 4 (graph_node::recover_spanning_connections): the reference's `continue` skips its
    # loop and covisibility edges as well, not only the parent edge
    kfs = [_kf(0, None, [1, 3]), _kf(1, 0, [], covis=[(0, 300)]), _kf(2, 4, [], loop_edges=[0], covis=[(1, 300), (0, 200)]),
           _kf(3, 0, [4], covis=[(2, 150)]), _kf(4, 3, [2], covis=[(2, 400), (1, 120)])]
    g = build_essential_graph(kfs, curr_id=4, loop_id=0, loop_connections=[], min_num_shared_lms=100)
    assert _edges(g) == [(1, 0), (3, 0), (3, 2), (4, 3), (4, 1)]


def test_builder_sim3_matches_oracle():
    from stella_vslam_b200.optimize import sim3_from_rts, sim3_inverse, sim3_mul
    rng = np.random.default_rng(13)
    for _ in range(20):
        a, b = _rand_sim3(rng), _rand_sim3(rng)
        assert np.array_equal(sim3_mul(a, b), O.mul(a, b))
        assert np.array_equal(sim3_inverse(a), O.inverse(a))
        R = sl.expm(_hat(np.concatenate([rng.uniform(-3, 3, 3), np.zeros(4)])))[:3, :3]
        t = rng.uniform(-5, 5, 3)
        assert np.array_equal(sim3_from_rts(R, t), O.from_rts(R, t))


def test_library_ordering_matches_oracle():
    from workloads import synth
    from stella_vslam_b200 import optimize
    for n, laps in ((50, 1.0), (400, 2.5)):
        g = synth.make_pose_graph(n, seed=n, laps=laps)
        order, env = optimize.pgo_envelope(g)
        o2, env2 = O.rcm(g)
        assert np.array_equal(order, o2) and env == env2


def test_ctypes_mirrors_match_the_header(tmp_path):
    from stella_vslam_b200 import optimize
    ABI._check(tmp_path, os.path.join(ROOT, "include"), "b200vslam.h",
               {"b200_sim3_t": optimize.Sim3, "b200_pose_graph_t": optimize.PoseGraph, "b200_pgo_stats_t": optimize.PgoStats})
