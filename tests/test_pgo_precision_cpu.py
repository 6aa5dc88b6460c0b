"""The precision method of tests/test_pgo_precision_gpu.py, pinned without a GPU: the reference system of tests/pgo_reference.py (a
fourth-order central difference at delta 1e-4) against an independent matrix difference, the size of the noise in g2o's delta-1e-9
Jacobian, and the CPU oracle's one-iteration LM step judged by its backward error against the reference system (the control the
device is compared with).

Measured (oracle, first LM step at lambda_init, trials == 1; kappa_bound = ||H + lambda I||_inf / lambda, an upper bound on the
condition number):
  graph                    units    omega_orc   kappa_bound   forward error
  loop500                  1        1.25e-7     1.39e5        6.3e-6
  loop500                  1/1000   1.29e-7     2.06e5        4.2e-7
  loop2000                 1        1.22e-7     1.28e5        2.4e-5
  loop2000                 1/1000   1.80e-8     1.87e5        1.5e-7
  loop4000_fixed_scale     1        8.34e-8     1.81e5        2.5e-5
  loop4000_fixed_scale     1/1000   5.42e-8     2.57e5        1.2e-7
  loop4000                 1        5.89e-8     1.37e5        1.9e-5
  loop4000                 1/1000   4.79e-8     2.48e5        1.7e-7
  revisit1200              1        1.99e-7     1.37e5        1.1e-5
  revisit1200              1/1000   3.37e-8     2.09e5        7.4e-8
  chain_pad0               1        2.62e-6     1.91e5        9.5e-4
  chain_pad0               1/1000   9.96e-9     2.02e5        3.4e-7
  chain_pad31              1        4.60e-6     1.91e5        5.9e-4
  chain_pad31              1/1000   9.08e-9     2.02e5        4.9e-7
  chain_pad1               1        4.24e-6     1.92e5        1.7e-3
  chain_pad1               1/1000   8.06e-9     2.02e5        7.6e-7
  grid96x40                1        5.73e-7     2.01e5        3.2e-6
  grid96x40                1/1000   1.17e-11    2.00e5        1.4e-9
eigsh's condition number on loop500 is 1.00e5 (own units) and 8.3e2 (1/1000), on chain_pad0 1.36e5 and 1.44e5.  The forward errors
stay 60x .. 1e5x under kappa_bound * omega.  The fixed-scale 4 000-keyframe loop's first step turns six vertices by more than pi
(up to 7.7 rad); read back through log alone it showed a backward error of 4.5e-5, read back on the branch nearest the reference step
it shows 8.3e-8 like the other loops.  g2o's Jacobian differs from the reference by up to 2e-4 of a
block's largest entry at the 4 000-keyframe graph's own units (|t| up to about 640 m) and by about 1e-6 at 1/1000 of them."""
import numpy as np
import pytest
import scipy.linalg as sl

import pgo_oracle as O
import pgo_reference as R
from test_pgo_cpu import _hat, _mat, _vee

UNITS = (1.0, 1e-3)


def _graph(name, f):
    g = R.CASES[name]()
    return g if f == 1.0 else R.scaled(g, f)


def test_reference_jacobian_matches_matrix_difference():
    """J_ref and each edge's H blocks J_s^T J_t against the expm / logm central difference of 4x4 similarity matrices."""
    g = R.CASES["loop500"]()
    err, J = O.graph_linearize(g, R.DELTA, R.STENCIL)
    est = np.asarray(g["estimate"])
    fixed = np.asarray(g["fixed"]).astype(bool)
    for k in (0, 17, 250, len(err) - 1):
        m, v = g["e_meas"][k], (est[g["e_v1"][k]], est[g["e_v2"][k]])
        np.testing.assert_allclose(err[k], O.edge_error(m, *v), rtol=0, atol=0)
        Jr = np.zeros((2, 7, 7))
        for side in (0, 1):
            if fixed[(g["e_v1"][k], g["e_v2"][k])[side]]:
                assert not J[k, side].any()
                continue
            for d in range(7):
                du = np.zeros(7)
                du[d] = 1e-6
                f = []
                for sgn in (1, -1):
                    M = [sl.expm(_hat(sgn * du)) @ _mat(x) if i == side else _mat(x) for i, x in enumerate(v)]
                    f.append(_vee(np.real(sl.logm(_mat(m) @ M[0] @ np.linalg.inv(M[1])))))
                Jr[side, :, d] = (f[0] - f[1]) / 2e-6
        tol = 1e-5 * np.abs(Jr).max()
        np.testing.assert_allclose(J[k], Jr, rtol=0, atol=tol)
        for s in (0, 1):
            for t in (0, 1):
                np.testing.assert_allclose(J[k, s].T @ J[k, t], Jr[s].T @ Jr[t], rtol=0, atol=3 * tol * np.abs(Jr).max())


@pytest.mark.parametrize("f", UNITS)
def test_reference_jacobian_two_steps_agree(f):
    """The fourth-order stencil at delta 1e-4 and 2e-4 agree to 1e-8 of each block's largest entry on the 4 000-keyframe graph."""
    g = _graph("loop4000", f)
    _, J1 = O.graph_linearize(g, 1e-4, 4)
    _, J2 = O.graph_linearize(g, 2e-4, 4)
    assert R.block_error(J2, J1) <= 1e-8


def test_g2o_jacobian_noise_grows_with_translation():
    """g2o's delta-1e-9 central difference (the oracle's and the device's Jacobian) carries rounding of edge_error (about eps |t|)
    divided by the 1e-9 step: 1e-4 .. 1e-3 of a block's largest entry at the 4 000-keyframe graph's own units, under 3e-6 at 1/1000 of
    them (measured 2.0e-4 on 150 edges and about 1e-6)."""
    got = {}
    for f in UNITS:
        g = _graph("loop4000", f)
        _, Jg = O.graph_linearize(g, 1e-9, 2)
        _, Jr = O.graph_linearize(g, R.DELTA, R.STENCIL)
        got[f] = R.block_error(Jg, Jr)
        k = np.flatnonzero(np.asarray(g["fixed"])[g["e_v1"]] == 0)[5]
        est = np.asarray(g["estimate"])
        assert np.array_equal(Jg[k, 0], O.edge_jacobian(g["e_meas"][k], est[g["e_v1"][k]], est[g["e_v2"][k]], 0))
    assert 1e-4 <= got[1.0] <= 1e-3, got
    assert got[1e-3] <= 3e-6, got
    assert got[1.0] >= 30 * got[1e-3], got


def test_kappa_bound_is_tight():
    """||H + lambda I||_inf / lambda bounds the condition number from above; on the 500-keyframe graph it is within 1.5x of eigsh's."""
    g = R.CASES["loop500"]()
    S = R.system(g)
    lam = 1e-5 * S["H"].diagonal().max()
    A = R.damped(S["H"], lam)
    k, kb = R.kappa(A), R.kappa_bound(A, lam)
    assert k <= kb <= 1.5 * k, (k, kb)


@pytest.mark.parametrize("f", UNITS)
@pytest.mark.parametrize("name", [n for n in R.CASES if n != "grid96x576"])
def test_oracle_step_backward_error(name, f):
    """The oracle's exact profile-Cholesky solve of its own (noisy) system is a step whose backward error against the reference system
    stays under 5e-7 at 1/1000 units and 1e-5 at the graphs' own units, and whose forward error against the reference step stays under
    0.1 kappa_bound * omega (kappa_bound * omega overstates it by 60x .. 1e5x)."""
    g = _graph(name, f)
    S = R.system(g)
    orc = O.graph_optimize(g, max_iter=1, gain_threshold=0.0)
    assert orc["iterations"] == 1 and orc["trials"] == 1, orc
    lam = orc["lambda_init"]
    assert abs(lam - 1e-5 * S["H"].diagonal().max()) <= (1e-4 if f == 1.0 else 1e-5) * lam
    assert abs(orc["chi2_init"] - S["chi2"]) <= 1e-12 * S["chi2"]
    A = R.damped(S["H"], lam)
    xr = R.exact_step(A, S["b"])
    x = R.step(g, orc["estimate"], S["order"], near=xr)
    omega, kb, fwd = R.backward_error(A, x, S["b"]), R.kappa_bound(A, lam), R.rel(x, xr)
    print(f"{name} units {f:g}: omega_orc {omega:.3e} kappa_bound {kb:.3e} forward {fwd:.3e}")
    assert omega <= (5e-7 if f < 1 else 1e-5), omega
    assert fwd <= 0.1 * kb * omega, (fwd, kb, omega)
