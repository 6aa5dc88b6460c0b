"""b200_initialize against the CPU restatement (tests/initialize_oracle.py): every integer and flag output, the model and the stage bit
for bit; R, t and the points bit for bit on the perspective path and within 1e-12 relative on the equirectangular one (asin / atan2 of
CUDA's libm).  The chain also equals the stage-by-stage path (b200_twoview_ransac / b200_essential_ransac, then the CPU
reconstruction), and a mixed batch equals one-problem calls."""
import numpy as np
import pytest

import initialize_oracle as O
from stella_vslam_b200 import _lib, initialize as I, solve
from test_initialize_cpu import STAGE_CASES

pytestmark = pytest.mark.gpu

INTS = ("succeeded", "model", "stage", "n_matches", "valid_H", "valid_F", "valid_E", "num_inliers_H", "num_inliers_F", "num_inliers_E",
        "n_hypotheses")


def _close(a, b, exact):
    if a is None or b is None:
        return a is None and b is None
    if exact:
        return np.array_equal(a, b)
    return np.allclose(a, b, rtol=1e-12, atol=1e-12 * max(1.0, float(np.abs(b).max())))


def _same(got, want, exact=True):
    for k in INTS:
        assert got[k] == want[k], (k, got[k], want[k])
    assert (got["status"] != 0) == (want["status"] != 0)
    for k in ("cost_H", "cost_F", "cost_E"):
        assert np.float32(got[k]).tobytes() == np.float32(want[k]).tobytes(), k
    for k in ("nums_valid", "num_triangulated", "parallax_cos"):
        assert np.array_equal(got[k], want[k]), (k, got[k], want[k])
    for k in ("triangulated_flags", "inlier_flags"):
        assert (got[k] is None) == (want[k] is None) and (got[k] is None or np.array_equal(got[k], want[k])), k
    for k in ("rot_ref_to_cur", "trans_ref_to_cur", "triangulated_pts"):
        assert _close(got[k], want[k], exact), k


CASES = {
    "euroc_F": lambda: O.perspective_problem(seed=500, n=800),
    "kitti_F": lambda: O.perspective_problem(seed=501, n=800, camera="kitti"),
    "planar_H_30": lambda: O.perspective_problem(seed=502, n=800, scene="planar", inlier_frac=0.3, noise=0.0),
    "planar_H_30_noise": lambda: O.perspective_problem(seed=507, n=800, scene="planar", inlier_frac=0.3, noise=0.25),
    "planar_H_succeeds": lambda: O.plane_problem(seed=0),
    "planar_H_succeeds_2": lambda: O.plane_problem(seed=15, inlier_frac=0.3),
    "planar_H_20": lambda: O.perspective_problem(seed=503, n=800, scene="planar", inlier_frac=0.2, noise=0.25),
    "fisheye": lambda: O.perspective_problem(seed=504, n=800, model="fisheye"),
    "radial_division": lambda: O.perspective_problem(seed=505, n=800, model="radial_division"),
    "equirect_E": lambda: O.equirect_problem(seed=1),
    "equirect_E_seeded": lambda: O.equirect_problem(seed=2, inlier_frac=0.5, draw_seed=7),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_chain_matches_the_oracle(case):
    p = CASES[case]()
    got = I.initialize_batch([p])[0]
    want = O.initialize(p)
    _same(got, want, exact=case.startswith("equirect") is False)
    if case.startswith("planar"):
        assert got["model"] == "H"
        assert got["succeeded"] == case.startswith("planar_H_succeeds")
    elif case.startswith("equirect"):
        assert got["model"] == "E" and got["succeeded"]
    else:
        assert got["model"] == "F" and got["succeeded"]


@pytest.mark.parametrize("case", sorted(STAGE_CASES))
def test_every_stage_matches_the_oracle(case):
    make, stage = STAGE_CASES[case]
    p = make()
    got = I.initialize_batch([p])[0]
    _same(got, O.initialize(p), exact=not case.endswith("_E"))
    if stage is not None:
        assert got["stage"] == stage
    if stage == O.STAGE_DECOMPOSE:  # the rank test rejects before find_most_plausible_pose: no hypotheses, R and t untouched
        assert got["model"] == "H" and got["n_hypotheses"] == 0 and got["rot_ref_to_cur"] is None


def test_chain_equals_the_stage_by_stage_path():
    for p in (CASES["euroc_F"](), CASES["planar_H_30"](), CASES["planar_H_succeeds"](), CASES["equirect_E"]()):
        got = I.initialize_batch([p])[0]
        mt = O.matches_of(p["ref_matches_with_cur"])
        if got["model"] == "E":
            s = solve.essential_ransac_batch([dict(bearings_1=p["bearings_ref"][mt[:, 0]], bearings_2=p["bearings_cur"][mt[:, 1]],
                                                   min_sets=p["min_sets_E"], recompute=False)])[0]
            model, M = "E", s["E_21"]
        else:
            h, f = solve.twoview_ransac_batch([dict(model=k, keypts_1=p["undist_ref"], keypts_2=p["undist_cur"], matches_12=mt,
                                                    min_sets=p["min_sets_" + k], recompute=False) for k in ("H", "F")])
            s, model = (h, "H") if O.choose_H(h["best_cost"], f["best_cost"], h["valid"]) else (f, "F")
            M = s["M_21"]
            assert np.float32(got["cost_H"]) == h["best_cost"] and np.float32(got["cost_F"]) == f["best_cost"]
        assert got["model"] == model and np.array_equal(got["inlier_flags"], s["inlier_flags"])
        rec = O.reconstruct(p, model, M, s["inlier_flags"])
        for k in ("stage", "n_hypotheses"):
            assert got[k] == rec[k]
        for k in ("nums_valid", "num_triangulated", "parallax_cos"):
            assert np.array_equal(got[k], rec[k])
        for k in ("rot_ref_to_cur", "trans_ref_to_cur", "triangulated_pts"):
            assert _close(got[k], rec[k], model != "E"), k


def test_mixed_batch_equals_single_calls():
    makers = list(CASES.values()) + [m for m, _ in STAGE_CASES.values()]
    probs = [makers[i % len(makers)]() for i in range(64)]
    batch = I.initialize_batch(probs)
    for p, got in zip(probs, batch):
        _same(got, I.initialize_batch([p])[0])


def test_mirror_classes():
    p = CASES["euroc_F"]()
    ref = dict(camera=p["cam_ref"], img_bounds=p["bounds_ref"], undist_keypts=p["undist_ref"], bearings=p["bearings_ref"])
    cur = dict(camera=p["cam_cur"], img_bounds=p["bounds_cur"], undist_keypts=p["undist_cur"], bearings=p["bearings_cur"])
    ini = I.perspective(ref, use_fixed_seed=True)
    assert ini.initialize(cur, p["ref_matches_with_cur"])
    want = O.initialize(O.with_min_sets(p))  # default engines: what use_fixed_seed draws
    assert np.array_equal(ini.get_rotation_ref_to_cur(), want["rot_ref_to_cur"])
    assert np.array_equal(ini.get_translation_ref_to_cur(), want["trans_ref_to_cur"])
    assert np.array_equal(ini.get_triangulated_pts(), want["triangulated_pts"])
    assert ini.get_triangulated_flags() == list(want["triangulated_flags"])
    with pytest.raises(ValueError):
        I.bearing_vector(ref)


def test_invalid_inputs_write_nothing():
    import ctypes as C
    p = CASES["euroc_F"]()
    bad = [dict(p, ref_matches_with_cur=np.where(np.arange(len(p["undist_ref"])) == 3, len(p["undist_cur"]), p["ref_matches_with_cur"])),
           dict(p, cam_cur=dict(model="equirectangular", cols=752.0, rows=480.0)),
           dict(p, cam_ref=dict(p["cam_ref"], model="fisheye", k1=float("nan"))),
           dict(p, min_sets_H=None),
           dict(p, min_sets_F=np.full_like(p["min_sets_F"], 100000))]
    for b in bad:
        keep = []
        S, (pts, tri, inl) = I._pack(b, keep)
        S.status, S.stage, S.succeeded, S.n_hypotheses = 77, 77, 77, 77
        S.rot_ref_to_cur[:] = [5.0] * 9
        pts[:], tri[:], inl[:] = 7.0, 9, 9
        rc = I._L().b200_initialize(solve._handle(0), 1, C.byref(S))
        assert rc == _lib.ERR_INVALID
        assert (S.status, S.stage, S.succeeded, S.n_hypotheses) == (77, 77, 77, 77) and list(S.rot_ref_to_cur) == [5.0] * 9
        assert (pts == 7.0).all() and (tri == 9).all() and (inl == 9).all()
