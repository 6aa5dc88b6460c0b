"""Monocular initialisation without a GPU: the b200_init_problem_t mirror against the header, and the CPU restatement of the
reconstruction (tests/initialize_oracle.c on csrc/initialize_core.h) against numpy and against a plain transcription of
find_most_plausible_pose; every rejection of initialize() reached by a constructed input."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest

import initialize_oracle as O
from stella_vslam_b200 import initialize as I

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rot(ang):
    th = np.linalg.norm(ang)
    k = ang / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def test_struct_fields_follow_the_header():
    with open(os.path.join(ROOT, "include", "b200vslam.h")) as f:
        src = f.read()
    body = src[src.index("typedef struct b200_init_problem {"):src.index("} b200_init_problem_t;")]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";")[:-1]:
        decl = decl.split("{", 1)[-1].strip()
        typ_and_names = re.sub(r"\[\d+\]", "", decl)
        for part in typ_and_names.split(","):
            names.append(part.strip().split()[-1].lstrip("*"))
    assert names == [n for n, _ in I.InitProblem._fields_]
    arr_sizes = dict(re.findall(r"(\w+)\[(\d+)\]", body))
    for n, t in I.InitProblem._fields_:
        if n in arr_sizes:
            assert t._length_ == int(arr_sizes[n]), n
    assert C.sizeof(I.InitProblem) == 632  # x86-64, as the C compiler lays it out


def test_svd33_against_numpy():
    rng = np.random.default_rng(0)
    for k in range(50):
        A = rng.standard_normal((3, 3)) * (10.0 ** rng.integers(-3, 4))
        U, s, V, st = O.svd33(A)
        assert st == 0
        assert np.allclose(s, np.linalg.svd(A, compute_uv=False), rtol=1e-13, atol=0)
        assert np.all(np.diff(s) <= 0) and np.all(s >= 0)
        assert np.allclose(U @ np.diag(s) @ V.T, A, rtol=0, atol=1e-13 * np.abs(A).max())
        assert np.allclose(U.T @ U, np.eye(3), atol=1e-14) and np.allclose(V.T @ V, np.eye(3), atol=1e-14)


def test_decompose_H_recovers_the_true_motion():
    rng = np.random.default_rng(1)
    K = np.array([[458.654, 0, 367.215], [0, 457.296, 248.375], [0, 0, 1.0]])
    for k in range(20):
        R = _rot(0.05 * rng.standard_normal(3))
        t = rng.standard_normal(3)
        n = np.array([0.1 * rng.standard_normal(), 0.1 * rng.standard_normal(), 1.0])
        n /= np.linalg.norm(n)
        d = 5.0
        H = K @ (R + np.outer(t, n) / d) @ np.linalg.inv(K)
        H *= rng.uniform(0.5, 2.0)
        Rs, ts, ns = O.decompose_H(H, K, K)
        # the reference's intermediates are float: agreement to float precision
        hit = [i for i in range(8) if np.allclose(Rs[i], R, atol=1e-5) and np.allclose(ts[i], t / np.linalg.norm(t), atol=1e-5)
               and np.allclose(ns[i], n, atol=1e-5)]
        assert hit, k
        for i in range(8):
            # sin and cos are float in the reference: orthogonal to float precision
            assert np.allclose(Rs[i] @ Rs[i].T, np.eye(3), atol=1e-6) and abs(np.linalg.norm(ts[i]) - 1) < 1e-12


def test_decompose_E_is_numpys_set():
    rng = np.random.default_rng(2)
    for k in range(20):
        R = _rot(0.3 * rng.standard_normal(3))
        t = rng.standard_normal(3)
        tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
        E = tx @ R
        Rs, ts = O.decompose_E(E)
        U, _, Vt = np.linalg.svd(E)
        W = np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1.0]])
        cand = []
        for Rc in (U @ W @ Vt, U @ W.T @ Vt):
            Rc = -Rc if np.linalg.det(Rc) < 0 else Rc
            for tc in (U[:, 2], -U[:, 2]):
                cand.append((Rc, tc))
        for i in range(4):
            assert sum(np.allclose(Rs[i], Rc, atol=1e-10) and np.allclose(ts[i], tc, atol=1e-10) for Rc, tc in cand) == 1
        assert any(np.allclose(Rs[i], R, atol=1e-10) and np.allclose(ts[i], t / np.linalg.norm(t), atol=1e-10) for i in range(4))


def test_midpoint_against_numpy():
    rng = np.random.default_rng(3)
    for k in range(50):
        R = _rot(0.1 * rng.standard_normal(3))
        t = rng.standard_normal(3)
        X = rng.uniform(-2, 2, 3) + np.array([0, 0, 6.0])
        b1 = X / np.linalg.norm(X)
        b2 = R @ X + t + 1e-3 * rng.standard_normal(3)
        b2 /= np.linalg.norm(b2)
        c2 = -R.T @ t
        d2 = R.T @ b2
        A = np.stack([b1, -d2], 1)
        lam = np.linalg.lstsq(A, c2, rcond=None)[0]
        want = (lam[0] * b1 + lam[1] * d2 + c2) / 2.0
        assert np.allclose(O.midpoint(b1, b2, R, t), want, rtol=1e-9, atol=1e-12)


def _plain_select(nv, nt, pc, p):
    """base.cc:63-87 transcribed."""
    b = int(np.argmax(nv))
    if nv[b] < p["min_num_valid_pts"]:
        return O.STAGE_MIN_VALID, b
    if sum(0.8 * nv[b] < v for v in nv) > 1:
        return O.STAGE_AMBIGUOUS, b
    if float(pc[b]) > math.cos(p["parallax_deg_thr"] / 180.0 * math.pi):
        return O.STAGE_PARALLAX, b
    if nt[b] < p["min_num_triangulated"]:
        return O.STAGE_MIN_TRIANGULATED, b
    return O.STAGE_SUCCEEDED, b


@pytest.mark.parametrize("kind", ["euroc", "kitti", "planar", "equirect"])
def test_find_most_plausible_pose_matches_a_plain_transcription(kind):
    if kind == "equirect":
        p = O.equirect_problem(seed=1)
    else:
        p = O.perspective_problem(seed=502, n=800, camera="kitti" if kind == "kitti" else "euroc",
                                  **(dict(scene="planar", inlier_frac=0.3, noise=0.0) if kind == "planar" else {}))
    model, s = O.choose(O.ransac(p))
    assert model == {"planar": "H", "equirect": "E"}.get(kind, "F")
    M = s["E_21"] if model == "E" else s["M_21"]
    if model == "H":
        Rs, ts, _ = O.decompose_H(M, O.K_of(p["cam_ref"]), O.K_of(p["cam_cur"]))
    else:
        Rs, ts = O.decompose_E(M if model == "E" else O.essential_of_F(M, O.K_of(p["cam_ref"]), O.K_of(p["cam_cur"])))
    tri = [O.triangulate(p, Rs[i], ts[i], s["inlier_flags"], model != "E") for i in range(len(Rs))]
    nv, nt, pc = [r[0] for r in tri], [r[1] for r in tri], [r[2] for r in tri]
    rec = O.reconstruct(p, model, M, s["inlier_flags"])
    assert list(rec["nums_valid"]) == nv and list(rec["num_triangulated"]) == nt
    assert np.array_equal(rec["parallax_cos"], np.array(pc, np.float32))
    stage, b = _plain_select(nv, nt, pc, O.DEFAULTS)
    assert rec["stage"] == stage
    if stage == O.STAGE_SUCCEEDED:
        assert np.array_equal(rec["rot_ref_to_cur"], Rs[b]) and np.array_equal(rec["trans_ref_to_cur"], ts[b])
        assert np.array_equal(rec["triangulated_pts"], tri[b][3]) and np.array_equal(rec["triangulated_flags"], tri[b][4])
    else:
        assert not rec["rot_ref_to_cur"].any() and not rec["trans_ref_to_cur"].any()


def test_rank_test_rejects_a_pure_rotation():
    K = np.array([[458.654, 0, 367.215], [0, 457.296, 248.375], [0, 0, 1.0]])
    H = K @ _rot(np.array([0.01, 0.02, -0.03])) @ np.linalg.inv(K)
    assert O.decompose_H(H, K, K) is None


def test_choose_H_rule():
    assert O.choose_H(1.0, 3.0, True) and not O.choose_H(1.0, 3.0, False) and not O.choose_H(3.0, 1.0, True)
    assert not O.choose_H(0.0, 0.0, True)  # NaN: the F path runs
    assert not O.choose_H(1.0, 1.0, True)


# constructed inputs for every stage of initialize() (shared with the GPU tests)
STAGE_CASES = {
    "succeeded_F": (lambda: O.perspective_problem(seed=500, n=800), O.STAGE_SUCCEEDED),
    "succeeded_E": (lambda: O.equirect_problem(seed=1), O.STAGE_SUCCEEDED),
    "min_valid": (lambda: O.perspective_problem(seed=500, n=800, min_num_valid_pts=100000), O.STAGE_MIN_VALID),
    "n_valid_0": (lambda: O.perspective_problem(seed=500, n=800, reproj_err_thr=0.0), O.STAGE_MIN_VALID),
    "ambiguous_H": (lambda: O.perspective_problem(seed=502, n=800, scene="planar", inlier_frac=0.3, noise=0.0), O.STAGE_AMBIGUOUS),
    "parallax": (lambda: O.perspective_problem(seed=500, n=800, parallax_deg_thr=30.0), O.STAGE_PARALLAX),
    "min_triangulated": (lambda: O.perspective_problem(seed=500, n=800, min_num_triangulated=100000), O.STAGE_MIN_TRIANGULATED),
    "few_valid": (lambda: O.perspective_problem(seed=500, n=60, min_num_valid_pts=10, min_num_triangulated=10), None),
    "fewer_than_8": (lambda: O.perspective_problem(seed=500, case="n7"), O.STAGE_NO_MODEL),
    "pure_rotation_F": (lambda: O.perspective_problem(seed=500, n=800, case="pure_rotation", noise=0.0), O.STAGE_AMBIGUOUS),
    "succeeded_H": (lambda: O.plane_problem(seed=0), O.STAGE_SUCCEEDED),
    "succeeded_H_2": (lambda: O.plane_problem(seed=2), O.STAGE_SUCCEEDED),
    "decompose": (lambda: O.plane_problem(seed=3, inlier_frac=0.2, tilt=0.6, t_norm=0.0), O.STAGE_DECOMPOSE),
    "decompose_2": (lambda: O.plane_problem(seed=6, inlier_frac=0.2, tilt=0.6, t_norm=0.0), O.STAGE_DECOMPOSE),
}


@pytest.mark.parametrize("case", sorted(STAGE_CASES))
def test_each_stage_is_reached(case):
    make, stage = STAGE_CASES[case]
    p = make()
    r = O.initialize(p)
    if stage is not None:
        assert r["stage"] == stage, (r["stage"], r["model"], r["nums_valid"])
    if case == "fewer_than_8":
        assert r["cost_H"] == 0 and r["cost_F"] == 0 and not r["valid_F"]  # both costs 0: NaN rel_cost_H, the F path, no model
    if case == "n_valid_0":
        assert (r["nums_valid"] == 0).all() and (r["parallax_cos"] == 1.0).all()
    if case.startswith(("succeeded_H", "decompose")):
        assert r["model"] == "H"
    if case.startswith("succeeded_H"):  # the true motion, up to the scale of t
        R, t = p["truth"]["R"], p["truth"]["t"]
        assert np.allclose(r["rot_ref_to_cur"], R, atol=1e-3) and np.allclose(r["trans_ref_to_cur"], t / np.linalg.norm(t), atol=1e-3)
    if case == "few_valid":
        assert 0 < r["nums_valid"].max() <= 51
    if r["stage"] >= O.STAGE_MIN_VALID:
        assert r["rot_ref_to_cur"] is not None
        if r["stage"] != O.STAGE_SUCCEEDED:
            assert not r["rot_ref_to_cur"].any()
    else:
        assert r["rot_ref_to_cur"] is None
