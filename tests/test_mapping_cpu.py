"""CPU checks of the landmark-creation restatement (tests/mapping_oracle.c): the Jacobi SVD against numpy, the triangulation against
the true point and the stereo closed form, the distance of every workload decision from its threshold, and the ctypes layouts."""
import os

import numpy as np
import pytest

import mapping_oracle as MO
from stella_vslam_b200 import mapping
from test_abi_layout import _check
from workloads import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = [("perspective", False), ("perspective", True), ("equirectangular", False)]


def _linear_system(cur, ngh, i1, i2):
    b1, b2 = cur["bearings"][i1], ngh["bearings"][i2]
    P1, P2 = np.asarray(cur["pose_cw"]), np.asarray(ngh["pose_cw"])
    return np.stack([b1[0] * P1[2] - b1[2] * P1[0], b1[1] * P1[2] - b1[2] * P1[1], b2[0] * P2[2] - b2[2] * P2[0], b2[1] * P2[2] - b2[2] * P2[1]])


@pytest.mark.parametrize("model,stereo", CASES)
def test_svd_null_vector_matches_numpy(model, stereo):
    cur, nb = synth.make_mapping_problem(5, 3, 1000, model=model, stereo=stereo)
    n = 0
    for ngh in nb:
        m = MO.create_new_landmarks(cur, [ngh])["match_out"][0]
        i1s = np.flatnonzero(m >= 0)
        _, ok = MO.triangulate_pairs(cur, ngh, np.stack([i1s, m[i1s]], 1))
        for i1 in i1s[ok]:
            if stereo and (cur["x_right"][i1] >= 0 or ngh["x_right"][m[i1]] >= 0):
                continue  # accepted linear-triangulation pairs only (a stereo side may have taken the stereo branch)
            A = _linear_system(cur, ngh, i1, m[i1])
            v, sweeps = MO.jacobi_svd4_null(A)
            assert 0 < sweeps <= 12
            w = np.linalg.svd(A)[2][3]
            p, q = v[:3] / v[3], w[:3] / w[3]
            assert np.all(np.abs(p - q) <= 1e-9 * np.abs(q).max()), (p, q)
            n += 1
    assert n > 100


def test_linear_triangulation_recovers_the_true_point():
    rng = np.random.default_rng(0)
    cur, nb = synth.make_mapping_problem(6, 1, 50)
    ngh = nb[0]
    for _ in range(200):
        X = np.array([rng.uniform(-3, 3), rng.uniform(-2, 2), rng.uniform(3, 20)])
        kfs = []
        for kf in (cur, ngh):
            P = np.asarray(kf["pose_cw"])
            xc = P[:3, :3] @ X + P[:3, 3]
            k = dict(kf)
            k["bearings"] = (xc / np.linalg.norm(xc))[None]
            k["x"] = np.array([kf["fx"] * xc[0] / xc[2] + kf["cx"]], np.float32)
            k["y"] = np.array([kf["fy"] * xc[1] / xc[2] + kf["cy"]], np.float32)
            k["octave"] = np.zeros(1, np.int32)
            k["x_right"] = k["depth"] = None
            kfs.append(k)
        pos, ok = MO.triangulate_pairs(kfs[0], kfs[1], np.array([[0, 0]]))
        cos = float(np.dot(kfs[0]["bearings"][0] @ np.asarray(cur["pose_cw"])[:3, :3], kfs[1]["bearings"][0] @ np.asarray(ngh["pose_cw"])[:3, :3]))
        if cos < np.cos(np.deg2rad(1.0)):
            assert ok[0]
            assert np.abs(pos[0] - X).max() <= 1e-9 * np.abs(X).max()


def test_stereo_triangulation_closed_form():
    cur, nb = synth.make_mapping_problem(7, 1, 800, stereo=True)
    ngh = nb[0]
    # a stereo keypoint whose ray has (almost) no parallax with its partner takes the stereo branch of its own side
    st = np.flatnonzero(cur["x_right"] >= 0)[:50]
    k2 = dict(ngh)
    k2["pose_cw"], k2["pose_wc"] = cur["pose_cw"], cur["pose_wc"]
    k2["bearings"], k2["x"], k2["y"], k2["octave"] = cur["bearings"], cur["x"], cur["y"], cur["octave"]
    k2["x_right"], k2["depth"] = np.full(len(cur["x"]), -1, np.float32), None
    pos, ok = MO.triangulate_pairs(cur, k2, np.stack([st, st], 1))
    W = np.asarray(cur["pose_wc"])
    for k, i in enumerate(st):
        d = np.float32(cur["depth"][i])
        ux = np.float32((np.float64(cur["x"][i]) - cur["cx"]) * np.float64(d) * cur["fx_inv"])
        uy = np.float32((np.float64(cur["y"][i]) - cur["cy"]) * np.float64(d) * cur["fy_inv"])
        want = W[:3, :3] @ np.array([ux, uy, d], np.float64) + W[:3, 3]
        assert np.abs(pos[k] - want).max() <= 1e-12 * max(1.0, np.abs(want).max())


@pytest.mark.parametrize("model,stereo", CASES)
def test_workload_decisions_are_not_at_their_thresholds(model, stereo):
    """No linear-branch parallax test of the workloads sits within 1e-12 (relative) of its threshold, so CUDA's libm (1-2 ulp from
    glibc, used for the stereo parallax and the equirectangular reprojection) cannot flip a decision (DESIGN.md section 4)."""
    for seed in (11, 21, 31):
        cur, nb = synth.make_mapping_problem(seed, 6, 1500, model=model, stereo=stereo)
        for ngh in nb:
            cos_thr, _ = MO.constants(cur, ngh)
            R1, R2 = np.asarray(cur["pose_cw"])[:3, :3], np.asarray(ngh["pose_cw"])[:3, :3]
            rw1, rw2 = cur["bearings"] @ R1, ngh["bearings"] @ R2
            m = MO.create_new_landmarks(cur, [ngh])["match_out"][0]
            i1 = np.flatnonzero(m >= 0)
            c = np.sum(rw1[i1] * rw2[m[i1]], 1)
            thr = [np.float64(cos_thr)]
            for kf, idx in ((cur, i1), (ngh, m[i1])):
                if kf.get("depth") is not None:
                    d = kf["depth"][idx].astype(np.float64)
                    thr.append(np.cos(2.0 * np.arctan2(kf["true_baseline"] / 2.0, d)))
            for t in thr:
                assert np.all(np.abs(c - t) > 1e-12 * np.maximum(np.abs(t), 1e-300))


def test_ctypes_mirrors_match_the_header(tmp_path):
    mirrors = {"b200_tri_keyframe_t": mapping.TriKeyframe, "b200_triangulate_problem_t": mapping.TriangulateProblem,
               "b200_new_landmarks_neighbour_t": mapping.NewLandmarksNeighbour, "b200_new_landmarks_problem_t": mapping.NewLandmarksProblem}
    _check(tmp_path, os.path.join(ROOT, "include"), "b200vslam.h", mirrors)


def test_oracle_keyframe_layout_matches_the_header(tmp_path):
    """The oracle reads the same TriKeyframe struct: its C declaration must have the header's layout."""
    src = open(os.path.join(ROOT, "tests", "mapping_oracle.c")).read()
    decl = src[src.index("typedef struct {\n    double pose_cw[16]"):src.index("} orc_tri_keyframe_t;") + len("} orc_tri_keyframe_t;")]
    (tmp_path / "orc_tri.h").write_text("#include <stdint.h>\n" + decl + "\n")
    _check(tmp_path, str(tmp_path), "orc_tri.h", {"orc_tri_keyframe_t": mapping.TriKeyframe})


# ---- a deliberately literal walk of two_view_triangulator.{h,cc}, written from the reference and not from mapping_oracle.c ----------
# Python floats are IEEE doubles evaluated one operation at a time (no contraction); np.float32 scalars where the reference uses float.
f32 = np.float32
DBL_MIN, DBL_EPS = np.finfo(np.float64).tiny, np.finfo(np.float64).eps


def _eigen_jacobi_svd_V(A):
    """Eigen::JacobiSVD<Mat44_t>(A, ComputeFullU | ComputeFullV).matrixV() for a square matrix (no QR preconditioner)."""
    scale = 0.0
    for r in range(4):
        for c in range(4):
            if abs(A[r][c]) > scale:
                scale = abs(A[r][c])
    if scale == 0.0:
        scale = 1.0
    W = [[A[r][c] / scale for c in range(4)] for r in range(4)]
    V = [[1.0 if r == c else 0.0 for c in range(4)] for r in range(4)]

    def apply_rotation_in_the_plane(get, put, p, q, c, s, size=4):
        if c == 1.0 and s == 0.0:
            return
        for i in range(size):
            xi, yi = get(p, i), get(q, i)
            put(p, i, c * xi + s * yi)
            put(q, i, -s * xi + c * yi)

    max_diag = max(abs(W[i][i]) for i in range(4))
    finished, sweeps = False, 0
    while not finished:
        sweeps += 1
        assert sweeps <= 64
        finished = True
        for p in range(1, 4):
            for q in range(p):
                threshold = max(DBL_MIN, (2.0 * DBL_EPS) * max_diag)
                if abs(W[p][q]) > threshold or abs(W[q][p]) > threshold:
                    finished = False
                    # real_2x2_jacobi_svd
                    m = [[W[p][p], W[p][q]], [W[q][p], W[q][q]]]
                    t, d = m[0][0] + m[1][1], m[1][0] - m[0][1]
                    if abs(d) < DBL_MIN:
                        s1, c1 = 0.0, 1.0
                    else:
                        u = t / d
                        tmp = np.sqrt(1.0 + u * u)
                        s1, c1 = 1.0 / tmp, u / tmp
                    apply_rotation_in_the_plane(lambda r, i: m[r][i], lambda r, i, v: m[r].__setitem__(i, v), 0, 1, c1, s1, 2)
                    x, y, z = m[0][0], m[0][1], m[1][1]  # makeJacobi(m, 0, 1)
                    deno = 2.0 * abs(y)
                    if deno < DBL_MIN:
                        cr, sr = 1.0, 0.0
                    else:
                        tau = (x - z) / deno
                        w = float(np.sqrt(tau * tau + 1.0))
                        tt = 1.0 / (tau + w) if tau > 0.0 else 1.0 / (tau - w)
                        sign_t = 1.0 if tt > 0.0 else -1.0
                        n = 1.0 / float(np.sqrt(tt * tt + 1.0))
                        sr = -sign_t * (y / abs(y)) * abs(tt) * n
                        cr = n
                    cl, sl = c1 * cr - s1 * -sr, c1 * -sr + s1 * cr  # rot1 * j_right.transpose()
                    apply_rotation_in_the_plane(lambda r, i: W[r][i], lambda r, i, v: W[r].__setitem__(i, v), p, q, cl, sl)
                    apply_rotation_in_the_plane(lambda c, i: W[i][c], lambda c, i, v: W[i].__setitem__(c, v), p, q, cr, -sr)
                    apply_rotation_in_the_plane(lambda c, i: V[i][c], lambda c, i, v: V[i].__setitem__(c, v), p, q, cr, -sr)
                    max_diag = max(max_diag, max(abs(W[p][p]), abs(W[q][q])))
    sv = [abs(W[i][i]) * scale for i in range(4)]
    for i in range(4):
        pos = max(range(i, 4), key=lambda k: (sv[k], -k))
        if sv[pos] == 0.0:
            break
        if pos != i:
            sv[i], sv[pos] = sv[pos], sv[i]
            for r in range(4):
                V[r][i], V[r][pos] = V[r][pos], V[r][i]
    return V


def _mat_vec(M, v):  # Eigen's 3x3 * 3 in index order
    return [M[r][0] * v[0] + M[r][1] * v[1] + M[r][2] * v[2] for r in range(3)]


def _walk(k1, k2, idx_1, idx_2, deg=1.0):
    """two_view_triangulator(k1, k2, deg).triangulate(idx_1, idx_2).  Returns (ok, pos_w, reason, margins): reason names the branch /
    test that decided, margins the (value, threshold) of every comparison fed by libm."""
    P1 = [[float(v) for v in row] for row in np.asarray(k1["pose_cw"])]
    P2 = [[float(v) for v in row] for row in np.asarray(k2["pose_cw"])]
    rot_1w, rot_2w = [r[:3] for r in P1[:3]], [r[:3] for r in P2[:3]]
    rot_w1, rot_w2 = [list(c) for c in zip(*rot_1w)], [list(c) for c in zip(*rot_2w)]
    trans_1w, trans_2w = [P1[r][3] for r in range(3)], [P2[r][3] for r in range(3)]
    W1, W2 = np.asarray(k1["pose_wc"]), np.asarray(k2["pose_wc"])
    cam_center_1, cam_center_2 = [float(W1[r][3]) for r in range(3)], [float(W2[r][3]) for r in range(3)]
    ratio_factor = f32(2.0) * max(f32(k1["scale_factor"]), f32(k2["scale_factor"]))
    cos_rays_parallax_thr = f32(np.cos(f32(deg) * np.pi / 180.0))
    margins = []

    x_right_1 = f32(-1.0) if k1.get("x_right") is None else f32(k1["x_right"][idx_1])
    x_right_2 = f32(-1.0) if k2.get("x_right") is None else f32(k2["x_right"][idx_2])
    is_stereo_1, is_stereo_2 = 0 <= x_right_1, 0 <= x_right_2
    ray_c_1, ray_c_2 = [float(v) for v in k1["bearings"][idx_1]], [float(v) for v in k2["bearings"][idx_2]]
    ray_w_1, ray_w_2 = _mat_vec(rot_w1, ray_c_1), _mat_vec(rot_w2, ray_c_2)
    cos_rays_parallax = ray_w_1[0] * ray_w_2[0] + ray_w_1[1] * ray_w_2[1] + ray_w_1[2] * ray_w_2[2]
    depth_1 = f32(-1.0) if k1.get("depth") is None else f32(k1["depth"][idx_1])
    depth_2 = f32(-1.0) if k2.get("depth") is None else f32(k2["depth"][idx_2])
    cos_sp_1 = float(np.cos(2.0 * np.arctan2(k1["true_baseline"] / 2.0, float(depth_1)))) if is_stereo_1 else 2.0
    cos_sp_2 = float(np.cos(2.0 * np.arctan2(k2["true_baseline"] / 2.0, float(depth_2)))) if is_stereo_2 else 2.0
    cos_stereo_parallax = min(cos_sp_1, cos_sp_2)
    if is_stereo_1 or is_stereo_2:
        margins += [(cos_rays_parallax, cos_stereo_parallax)]
        if is_stereo_1 and is_stereo_2:
            margins += [(cos_sp_1, cos_sp_2)]
    two = ((not is_stereo_1 and not is_stereo_2) and 0.0 < cos_rays_parallax and cos_rays_parallax < float(cos_rays_parallax_thr)) \
        or ((is_stereo_1 or is_stereo_2) and 0.0 < cos_rays_parallax and cos_rays_parallax < cos_stereo_parallax)

    def triangulate_stereo(k, idx):
        depth = f32(-1.0) if k.get("depth") is None else f32(k["depth"][idx])
        if not 0.0 < depth:
            return [0.0, 0.0, 0.0]
        ux = f32((float(f32(k["x"][idx])) - k["cx"]) * float(depth) * k["fx_inv"])
        uy = f32((float(f32(k["y"][idx])) - k["cy"]) * float(depth) * k["fy_inv"])
        W = np.asarray(k["pose_wc"])
        rot_wc, trans_wc = [[float(v) for v in W[r][:3]] for r in range(3)], [float(W[r][3]) for r in range(3)]
        p = _mat_vec(rot_wc, [float(ux), float(uy), float(depth)])
        return [p[r] + trans_wc[r] for r in range(3)]

    if two:
        b1, b2 = ray_c_1, ray_c_2
        A = [[b1[0] * P1[2][j] - b1[2] * P1[0][j] for j in range(4)], [b1[1] * P1[2][j] - b1[2] * P1[1][j] for j in range(4)],
             [b2[0] * P2[2][j] - b2[2] * P2[0][j] for j in range(4)], [b2[1] * P2[2][j] - b2[2] * P2[1][j] for j in range(4)]]
        V = _eigen_jacobi_svd_V(A)
        pos_w, reason = [V[r][3] / V[3][3] for r in range(3)], "linear"
    elif is_stereo_1 and cos_sp_1 < cos_sp_2:
        pos_w, reason = triangulate_stereo(k1, idx_1), "stereo_1"
    elif is_stereo_2 and cos_sp_2 < cos_sp_1:
        pos_w, reason = triangulate_stereo(k2, idx_2), "stereo_2"
    else:
        return False, [0.0, 0.0, 0.0], "reject_no_branch", margins

    def depth_is_positive(rot_cw, trans_cw, k):
        pos_z = (rot_cw[2][0] * pos_w[0] + rot_cw[2][1] * pos_w[1] + rot_cw[2][2] * pos_w[2]) + trans_cw[2]
        return int(k["model"]) == 1 or 0 < pos_z

    if not depth_is_positive(rot_1w, trans_1w, k1) or not depth_is_positive(rot_2w, trans_2w, k2):
        return False, pos_w, "reject_depth", margins

    def reprojection_ok(rot_cw, trans_cw, k, idx, x_right, sigma_sq, is_stereo):
        pc = _mat_vec(rot_cw, pos_w)
        pc = [pc[r] + trans_cw[r] for r in range(3)]
        if int(k["model"]) == 1:
            n2 = pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2]
            b = [v / float(np.sqrt(n2)) for v in pc] if n2 > 0.0 else pc
            latitude, longitude = -float(np.arcsin(b[1])), float(np.arctan2(b[0], b[2]))
            reproj = [k["cols"] * (0.5 + longitude / (2.0 * np.pi)), k["rows"] * (0.5 - latitude / np.pi)]
            x_right_in_cur = f32(0.0)
        else:
            z_inv = 1.0 / pc[2]
            reproj = [k["fx"] * pc[0] * z_inv + k["cx"], k["fy"] * pc[1] * z_inv + k["cy"]]
            x_right_in_cur = f32(reproj[0] - k["focal_x_baseline"] * z_inv)
        e = [reproj[0] - float(f32(k["x"][idx])), reproj[1] - float(f32(k["y"][idx]))]
        if is_stereo:
            err_xr = f32(x_right_in_cur - x_right)
            val, thr = (e[0] * e[0] + e[1] * e[1]) + float(f32(err_xr * err_xr)), float(f32(7.81473) * sigma_sq)
        else:
            val, thr = e[0] * e[0] + e[1] * e[1], float(f32(5.99146) * sigma_sq)
        if int(k["model"]) == 1:
            margins.append((val, thr))
        return not (thr < val)

    if not reprojection_ok(rot_1w, trans_1w, k1, idx_1, x_right_1, f32(k1["level_sigma_sq"][k1["octave"][idx_1]]), is_stereo_1) \
            or not reprojection_ok(rot_2w, trans_2w, k2, idx_2, x_right_2, f32(k2["level_sigma_sq"][k2["octave"][idx_2]]), is_stereo_2):
        return False, pos_w, "reject_reprojection", margins
    v1 = [pos_w[r] - cam_center_1[r] for r in range(3)]
    v2 = [pos_w[r] - cam_center_2[r] for r in range(3)]
    d1, d2 = float(np.sqrt(v1[0] * v1[0] + v1[1] * v1[1] + v1[2] * v1[2])), float(np.sqrt(v2[0] * v2[0] + v2[1] * v2[1] + v2[2] * v2[2]))
    if d1 == 0 or d2 == 0:
        return False, pos_w, "reject_zero_distance", margins
    ratio_dists = d2 / d1
    ratio_octave = f32(k1["scale_factors"][k1["octave"][idx_1]]) / f32(k2["scale_factors"][k2["octave"][idx_2]])
    if not (float(ratio_octave) / ratio_dists < float(ratio_factor) and ratio_dists / float(ratio_octave) < float(ratio_factor)):
        return False, pos_w, "reject_scale", margins
    return True, pos_w, reason, margins


def _walk_pairs(cur, ngh, seed=3, n_random=600):
    m = MO.create_new_landmarks(cur, [ngh])["match_out"][0]
    i1 = np.flatnonzero(m >= 0)
    rng = np.random.default_rng(seed)
    rnd = np.stack([rng.integers(0, len(cur["x"]), n_random), rng.integers(0, len(ngh["x"]), n_random)], 1)
    return np.concatenate([np.stack([i1, m[i1]], 1), rnd]).astype(np.int32)


@pytest.mark.parametrize("model,stereo", CASES)
def test_oracle_equals_literal_walk(model, stereo):
    """ok flags and every pos_w of the C restatement equal the literal walk; every branch and reject reason the workload can reach is
    exercised (stereo workloads hold mono/mono, stereo/stereo and mixed pairs)."""
    cur, nb = synth.make_mapping_problem(11, 3, 800, model=model, stereo=stereo)
    seen, kinds = set(), set()
    for ngh in nb:
        pairs = _walk_pairs(cur, ngh)
        pos, ok = MO.triangulate_pairs(cur, ngh, pairs)
        for k, (i1, i2) in enumerate(pairs):
            w_ok, w_pos, reason, _ = _walk(cur, ngh, int(i1), int(i2))
            assert ok[k] == w_ok, (k, reason)
            assert np.array_equal(pos[k], np.asarray(w_pos)) or np.all(np.abs(pos[k] - w_pos) <= 1e-12 * np.maximum(np.abs(w_pos), 1.0)), reason
            seen.add(reason if not w_ok else "accepted_" + reason)
            if stereo:
                kinds.add((bool(cur["x_right"][i1] >= 0), bool(ngh["x_right"][i2] >= 0)))
    want = {"accepted_linear", "reject_no_branch", "reject_reprojection", "reject_scale"}
    if model != "equirectangular":
        want.add("reject_depth")  # an equirectangular camera skips the depth test (two_view_triangulator.h:88-91)
    if stereo:
        want |= {"accepted_stereo_1", "accepted_stereo_2"}
        assert kinds == {(False, False), (False, True), (True, False), (True, True)}
    assert want <= seen, want - seen


def test_composition_with_row_claims_equals_literal_walk():
    """mapping_module::create_new_landmarks: neighbours in order, matches by ascending idx_1, every created landmark closes its row."""
    from oracle import pyoracle as O
    cur, nb = synth.make_mapping_problem(13, 4, 600, stereo=True)
    want = MO.create_new_landmarks(cur, nb)
    free = cur["no_landmark"].copy()
    created = []
    for r, ngh in enumerate(nb):
        mo, _ = O.match_pairs(MO.triangulation_problem(cur, ngh, 0.2 * np.pi / 180.0, False, free.copy()), 1, 0.95, False)
        for i1 in range(len(mo)):
            if mo[i1] < 0:
                continue
            ok, pos, _, _ = _walk(cur, ngh, i1, int(mo[i1]))
            if ok:
                created.append((r, i1, int(mo[i1]), pos))
                free[i1] = 0
    assert [c[0] for c in created] == list(want["rank"])
    assert [(c[1], c[2]) for c in created] == [tuple(v) for v in want["idx"]]
    assert np.all(np.abs(np.array([c[3] for c in created]) - want["pos_w"]) <= 1e-12 * np.maximum(np.abs(want["pos_w"]), 1.0))


@pytest.mark.parametrize("model,stereo", CASES)
def test_libm_fed_decisions_are_not_at_their_thresholds(model, stereo):
    """Every comparison fed by atan2 / cos (stereo parallax, stereo branch choice) or asin / atan2 (equirectangular chi-square) over the
    pairs the GPU tests triangulate (matched and random) is farther than 1e-12 (relative) from its threshold, so CUDA's libm (1-2 ulp
    from glibc) cannot flip one."""
    cur, nb = synth.make_mapping_problem(11, 3, 800, model=model, stereo=stereo)
    n = 0
    for ngh in nb:
        for i1, i2 in _walk_pairs(cur, ngh):
            for val, thr in _walk(cur, ngh, int(i1), int(i2))[3]:
                assert abs(val - thr) > 1e-12 * max(abs(thr), 1e-300), (val, thr)
                n += 1
    assert n > 0 or (model == "perspective" and not stereo)


def test_python_mirror_epipolar_geometry_matches_the_oracles():
    for model in ("perspective", "equirectangular"):
        cur, nb = synth.make_mapping_problem(14, 6, 50, model=model)
        for ngh in nb:
            E1, e1, v1 = mapping.epipolar_geometry(cur, ngh)
            E2, e2, v2 = MO.epipolar_geometry(cur, ngh)
            assert np.allclose(E1, E2, rtol=0, atol=1e-12) and np.allclose(e1, e2, rtol=0, atol=1e-12) and v1 == v2
