"""The factored Hpl record of the local bundle adjuster (lba_kernels.cu, kHplStride).

Each edge stores A = ww Jpi^T Ji (3x3) and the camera-frame point pc instead of the 6x3 block Hpl = ww Jj^T Ji, which the Schur
complement rebuilds as [[pc]x A ; A] and the back-substitution uses as Hpl^T [w; v] = A^T (v + w x pc).
CPU: a numpy restatement of edge_jacobians for the three edge models checks both identities on random poses and points.
GPU: the windows of tests/golden/make_lba_hpl_parent.py are solved and held to the results of the unfactored 160-byte records
(tests/golden/lba_hpl_parent.npz): identical iteration counts and outlier flags, poses, points and chi2 within 1e-9 relative."""
import os

import numpy as np
import pytest

from workloads.synth import KITTI

EQUI = dict(cols=3840.0, rows=1920.0)


def _edge_jacobians(model, cam, R, pc, stereo):
    """Ji (3x3, landmark) and Jj (3x6, pose, rotation first) as lba_kernels.cu's edge_jacobians forms them; unused rows zero."""
    x, y, z = pc
    Ji, Jj = np.zeros((3, 3)), np.zeros((3, 6))
    if model == 1:
        L = np.sqrt(x * x + y * y + z * z)
        dx = [0, z, -y, 1, 0, 0, *R[0]]
        dy = [-z, 0, x, 0, 1, 0, *R[1]]
        dz = [y, -x, 0, 0, 0, 1, *R[2]]
        k0 = -(cam["cols"] / (2 * np.pi)) * (1.0 / (x * x + z * z))
        k1 = -(cam["rows"] / np.pi) * (1.0 / (L * np.sqrt(x * x + z * z)))
        for j in range(9):
            dL = (1.0 / L) * (x * dx[j] + y * dy[j] + z * dz[j])
            j0 = k0 * (z * dx[j] - x * dz[j])
            j1 = k1 * (L * dy[j] - y * dL)
            if j < 6:
                Jj[0, j], Jj[1, j] = j0, j1
            else:
                Ji[0, j - 6], Ji[1, j - 6] = j0, j1
        return Ji, Jj
    fx, fy, zz = cam["fx"], cam["fy"], z * z
    for j in range(3):
        Ji[0, j] = -fx * R[0, j] / z + fx * x * R[2, j] / zz
        Ji[1, j] = -fy * R[1, j] / z + fy * y * R[2, j] / zz
    Jj[0] = [x * y / zz * fx, -(1.0 + x * x / zz) * fx, y / z * fx, -1.0 / z * fx, 0.0, x / zz * fx]
    Jj[1] = [(1.0 + y * y / zz) * fy, -x * y / zz * fy, -x / z * fy, 0.0, -1.0 / z * fy, y / zz * fy]
    if stereo:  # oxr >= 0
        fxb = cam["fxb"]
        Ji[2] = Ji[0] - fxb * R[2] / zz
        Jj[2] = [Jj[0, 0] - fxb * y / zz, Jj[0, 1] + fxb * x / zz, Jj[0, 2], Jj[0, 3], 0.0, Jj[0, 5] - fxb / zz]
    return Ji, Jj


def _skew(p):
    return np.array([[0, -p[2], p[1]], [p[2], 0, -p[0]], [-p[1], p[0], 0]])


def _random_rotation(rng):
    q = rng.standard_normal(4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _cases(rng, model):
    """(R, t, P) with pc = R P + t; a quarter of them near-degenerate (depth 1e-3..1e-2, or next to the equirectangular pole)."""
    for i in range(400):
        R, t = _random_rotation(rng), rng.uniform(-5, 5, 3)
        pc = rng.uniform(-20, 20, 3)
        if model == 1:
            if i % 4 == 0:
                pc[[0, 2]] = rng.uniform(-1e-3, 1e-3, 2)   # next to the pole, where the longitude's derivative blows up
        else:
            pc[2] = rng.uniform(1e-3, 1e-2) if i % 4 == 0 else rng.uniform(0.5, 80)
        yield R, t, R.T @ (pc - t)


@pytest.mark.parametrize("model,stereo", [(0, False), (0, True), (1, False)], ids=["mono", "stereo", "equirect"])
def test_hpl_factors_through_pc(model, stereo):
    rng = np.random.default_rng(11 + 2 * model + stereo)
    cam = EQUI if model == 1 else KITTI
    for R, t, P in _cases(rng, model):
        pc = R @ P + t
        Ji, Jj = _edge_jacobians(model, cam, R, pc, stereo)
        ww = rng.uniform(0.01, 2.0)
        H = ww * Jj.T @ Ji
        A = ww * Jj[:, 3:].T @ Ji
        H_rec = np.vstack([_skew(pc) @ A, A])
        scale = np.abs(H).max()
        assert scale > 0
        assert np.abs(H - H_rec).max() <= 1e-12 * scale
        # back-substitution form:  Hpl^T [w; v] = A^T (v + w x pc)
        x = rng.standard_normal(6)
        g = H.T @ x
        assert np.abs(g - A.T @ (x[3:] + np.cross(x[:3], pc))).max() <= 1e-12 * scale * np.abs(x).max() * max(1.0, np.abs(pc).max())


REL = 1e-9


@pytest.mark.gpu
def test_windows_match_unfactored_records(golden_dir):
    from golden.make_lba_hpl_parent import WINDOWS, solve_windows
    from stella_vslam_b200 import optimize
    from workloads import synth
    ref = np.load(os.path.join(golden_dir, "lba_hpl_parent.npz"))
    got = solve_windows(optimize, synth)
    for name in WINDOWS:
        assert np.array_equal(got[f"{name}_iterations"], ref[f"{name}_iterations"]), name
        assert np.array_equal(got[f"{name}_outliers"], ref[f"{name}_outliers"]), name
        for k in ("pose_cw", "points"):
            a, b = got[f"{name}_{k}"], ref[f"{name}_{k}"]
            assert np.abs(a - b).max() <= REL * max(1.0, np.abs(b).max()), (name, k, np.abs(a - b).max())
        a, b = got[f"{name}_chi2"], ref[f"{name}_chi2"]
        assert np.all(np.abs(a - b) <= REL * np.maximum(1.0, np.abs(b))), (name, a, b)
