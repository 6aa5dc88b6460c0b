"""The method of tests/test_lba_precision_gpu.py, pinned without a GPU: the reference of tests/lba_reference.py against finite
differences of itself and against the CPU oracle edge by edge (orc_lba_linearize), and the oracle's own one-step states judged by
it.  The oracle's exact Schur route (dense Cholesky of the reduced system) must sit at the readback floor, its lambda_init must be
1e-5 max diag(H_ref), its chi2 the reference chi2 at its output state, and its lambda_final the rho prediction of an accepted first
trial; otherwise the reference, not the device, would be what the GPU file judges."""
import numpy as np
import pytest

import ba_windows as BW
import lba_reference as R
from oracle import pyoracle as O
from workloads import synth

WINDOWS = ("three_cams", "kitti_euroc", "equirect_persp", "two_view_mono")


def _fd(pr, h_rot, h_rel):
    """Fourth-order central difference of the reference residual, per edge: (Jp (E,3,6), Jl (E,3,3)).  Every keyframe is moved by
    exp(h e_j) and every landmark by h e_j at once (each residual depends on one of each); translation and landmark steps scale with
    the edge's distance from its camera."""
    T0, P0 = np.asarray(pr["pose_cw"], np.float64), np.asarray(pr["points"], np.float64)
    _, pc = R.residuals(pr, T0, P0)
    dist = np.linalg.norm(pc, axis=1)
    # every edge gets its own copy of its keyframe and landmark, so one sweep per coordinate differentiates every edge at once
    E = len(pc)
    ep, el = np.asarray(pr["e_pose"]), np.asarray(pr["e_point"])
    one = dict(pr, e_pose=np.arange(E, dtype=np.int32), e_point=np.arange(E, dtype=np.int32), pose_fixed=np.zeros(E, np.uint8))
    Te, Pe = T0[ep], P0[el]
    Jp, Jl = np.zeros((E, 3, 6)), np.zeros((E, 3, 3))
    for j in range(6):
        h = np.full(E, h_rot) if j < 3 else h_rel * dist
        cols = []
        for s in (2, 1, -1, -2):
            T = np.stack([R.exp_oplus(Te[e], s * h[e] * np.eye(6)[j]) for e in range(E)])
            cols.append(R.residuals(one, T, Pe)[0])
        Jp[:, :, j] = (-cols[0] + 8 * cols[1] - 8 * cols[2] + cols[3]) / (12 * h[:, None])
    for j in range(3):
        h = h_rel * dist
        cols = [R.residuals(one, Te, Pe + s * h[:, None] * np.eye(3)[j])[0] for s in (2, 1, -1, -2)]
        Jl[:, :, j] = (-cols[0] + 8 * cols[1] - 8 * cols[2] + cols[3]) / (12 * h[:, None])
    return Jp, Jl


def _block_rel(J, Jref):
    m = np.abs(Jref).reshape(len(Jref), -1).max(1)
    return (np.abs(J - Jref).reshape(len(J), -1).max(1) / m)


@pytest.mark.parametrize("name", WINDOWS)
def test_jacobians_against_fourth_order_difference(name):
    pr = BW.window(name)
    Jp, Jl = R.jacobians(pr, pr["pose_cw"], pr["points"])
    Fp, Fl = _fd(pr, 1e-4, 1e-4)
    ep = _block_rel(Jp, Fp)
    el = _block_rel(Jl, Fl)
    kinds = np.asarray(pr["kinds"])[pr["e_point"]]
    equi = np.array([pr["cams"][c]["model"] == 1 for c in pr["e_cam"]])
    print(f"{name}: pose {ep.max():.2e} landmark {el.max():.2e}; pole {ep[kinds == 'pole'].max(initial=0):.2e} "
          f"seam {ep[kinds == 'seam'].max(initial=0):.2e}")
    if name in ("three_cams", "equirect_persp"):                     # polar and seam edges of the equirectangular model
        assert ((kinds == "pole") & equi).any() and ((kinds == "seam") & equi).any()
    assert ep.max() <= 1e-7 and el.max() <= 1e-7, (ep.max(), el.max())


def _linearize_cases():
    out = []
    for name in WINDOWS:
        out.append((name, BW.window(name)))
    out.append(("stereo", synth.make_ba_problem(12, 2, 600, seed=4, model="stereo")))
    out.append(("equirect", synth.make_ba_problem(10, 1, 400, seed=5, model="equirect")))
    return out


@pytest.mark.parametrize("round2", [False, True])
def test_edges_match_oracle_linearize(round2):
    for name, pr in _linearize_cases():
        T, P = pr["pose_cw"], pr["points"]
        level, rob = R.second_round_masks(pr, T, P) if round2 else R.first_round_masks(pr)
        lin = O.lba_linearize(pr, T, P, level.astype(np.uint8), rob.astype(np.uint8))
        err, _ = R.residuals(pr, T, P)
        Jp, Jl = R.jacobians(pr, T, P)
        _, _, ww = R.edge_costs(pr, err, rob)
        a = ~level
        assert lin["n_active"] == a.sum()
        assert not lin["err"][level].any() and not lin["Jj"][level].any() and not lin["weight"][level].any()
        scale = lambda v: np.abs(v[a]).reshape(a.sum(), -1).max(1)
        d_err = (np.abs(err[a] - lin["err"][a]).max(1) / np.maximum(scale(err), 1.0)).max()
        d_w = (np.abs(ww[a] - lin["weight"][a]) / ww[a]).max()
        d_p = (np.abs(Jp[a] - lin["Jj"][a]).reshape(a.sum(), -1).max(1) / scale(Jp)).max()
        d_l = (np.abs(Jl[a] - lin["Ji"][a]).reshape(a.sum(), -1).max(1) / scale(Jl)).max()
        print(f"{name} round {2 if round2 else 1}: {a.sum()} edges, err {d_err:.1e} weight {d_w:.1e} Jp {d_p:.1e} Jl {d_l:.1e}")
        assert max(d_err, d_w, d_p, d_l) <= 2e-12, (name, d_err, d_w, d_p, d_l)
        if round2:
            assert level.any() and not rob[a].any()


ORACLE_CASES = {
    "three_cams": lambda: (BW.window("three_cams"), "local"),
    "two_view_mono": lambda: (BW.window("two_view_mono"), "local"),
    "stereo_window": lambda: (synth.make_ba_problem(30, 5, 3000, seed=21, model="stereo"), "local"),
    "global_stereo_huber": lambda: (synth.make_ba_problem(30, 1, 2000, seed=1, model="stereo"), "global"),
    "global_mono_no_huber": lambda: (synth.make_ba_problem(40, 2, 1500, seed=2, model="mono"), "global_nohuber"),
    "global_equirect_huber": lambda: (synth.make_ba_problem(20, 1, 800, seed=3, model="equirect"), "global"),
    "round2_three_cams": lambda: (BW.window("three_cams"), "round2"),
    "round2_gross": lambda: (R.gross_landmarks(synth.make_ba_problem(30, 5, 3000, seed=23, model="stereo"), 20, seed=23), "round2"),
}


@pytest.mark.parametrize("name", list(ORACLE_CASES))
def test_oracle_step_at_readback_floor(name):
    pr, kind = ORACLE_CASES[name]()
    if kind == "global_nohuber":
        pr = dict(pr, e_robust=np.zeros(len(pr["e_pose"]), np.uint8))
    if kind == "round2":
        level, rob = R.second_round_masks(pr, pr["pose_cw"], pr["points"])
        BW.assert_clear_of_thresholds(pr, pr["pose_cw"], pr["points"])
        S = R.system(pr, level=level, robust=rob)
        o = O.lba_solve(pr, iters1=0, iters2=1)
        assert o["iterations"] == [0, 1]
        lam, lam_rep, chi, lam_fin = R.lambda_init(S), None, o["chi2"][1], o["lambda_final"][1]
        assert level.any()
        if name == "round2_gross":
            assert (S["pt_col"] < 0).sum() >= 20                    # the landmarks whose every edge left are out of the system
    else:
        S = R.system(pr)
        if kind == "local":
            o = O.lba_solve(pr, iters1=1, iters2=0)
            lam_rep, chi, lam_fin = o["lambda_init"], o["chi2"][0], o["lambda_final"][0]
        else:
            o = O.global_ba_solve(pr, num_iter=1, gain_threshold=0.0)
            lam_rep, chi, lam_fin = o["lambda_init"], o["chi2"], o["lambda_final"]
        lam = lam_rep
    J = R.check_step(S, lam, lam_rep, chi, lam_fin, o["pose_cw"], o["points"], pr)
    print(f"{name}: omega_orc {J['omega']:.2e} (keyframe rows {J['omega_kf']:.2e}) floor {J['floor']:.2e} ({J['floor_kf']:.2e}) "
          f"kappa_bound {J['kappa_bound']:.2e} forward {J['forward']:.2e}")
    # the oracle solves its own system exactly: at the readback floor, within rounding of the floor itself
    assert J["omega"] <= 4 * J["floor"] + 1e-15 and J["omega_kf"] <= 4 * J["floor_kf"] + 1e-15, J
    assert J["forward"] <= J["kappa_bound"] * J["omega"]
