"""b200_graph_optimize's first LM step judged against the high-precision reference system of tests/pgo_reference.py, with the CPU
oracle's step as the control (tests/test_pgo_precision_cpu.py pins the method without a GPU).

Per graph, at its own units and with every translation scaled by 1/1000 (the same topology, order and envelope, and g2o's delta-1e-9
Jacobian about 100x less noisy), one iteration with trials == 1: chi2_init equals the reference chi2 (math.fsum) to 1e-12; lambda_init
equals 1e-5 max diag(H_ref) to 1e-5 (1e-4 at the graph's own units, where the Jacobian noise reaches the diagonal); the device step's
normwise backward error against H_ref + lambda I is at most 2x the oracle's (measured: equal to 1 %) (the oracle's profile Cholesky is an exact solve of its
own Jacobian), and at most 1e-6 at 1/1000 units; its forward error against the reference step is under kappa * omega; fixed vertices
are bit-unchanged.  A missed or misplaced tile update, a wrong tile offset or active row, or a lambda on the wrong entries gives a
backward error orders of magnitude above the oracle's even where the step still lowers chi2.  The 96 x 576 grid, whose envelope is
within 0.1 % of B200_PGO_MAX_ENVELOPE_DOUBLES, is too large for the CPU oracle: its backward error is bounded absolutely.

Measured on an H100 80GB HBM3: the device's backward error equals the oracle's to two or more digits on every graph (1.2e-7 on the
500- and 2 000-keyframe loops, 5.9e-8 and 8.3e-8 on the 4 000-keyframe loops, free and fixed scale, at their own units; 1e-11 ..
1.3e-7 at 1/1000 units; 4.2e-9 on the 96 x 576 grid at 1/1000), so the discrepancy between the two on large graphs is Jacobian noise
times kappa, not the tiled solve."""
import numpy as np
import pytest

import pgo_oracle as O
import pgo_reference as R

UNITS = (1.0, 1e-3)


CASES = [(n, f) for n in R.CASES for f in UNITS]


@pytest.mark.gpu
@pytest.mark.parametrize("name,f", CASES)
def test_first_step_backward_error(name, f):
    from stella_vslam_b200 import optimize
    g0 = R.CASES[name]()
    g = g0 if f == 1.0 else R.scaled(g0, f)
    S = R.system(g)
    dev = optimize.graph_optimizer(max_iter=1, gain_threshold=0.0).optimize(g)
    assert dev["iterations"] == 1 and dev["trials"] == 1, (dev["iterations"], dev["trials"])
    env = O.rcm(g0)[1]
    assert dev["envelope_doubles"] == env == O.rcm(g)[1]
    if name == "grid96x576":
        assert 0.9 * optimize.PGO_MAX_ENVELOPE_DOUBLES <= env <= optimize.PGO_MAX_ENVELOPE_DOUBLES
    assert abs(dev["chi2_init"] - S["chi2"]) <= 1e-12 * S["chi2"]
    lam = dev["lambda_init"]
    assert abs(lam - 1e-5 * S["H"].diagonal().max()) <= (1e-4 if f == 1.0 else 1e-5) * lam
    fixed = np.asarray(g["fixed"]).astype(bool)
    assert np.array_equal(dev["estimate"][fixed], np.asarray(g["estimate"])[fixed])

    A = R.damped(S["H"], lam)
    xr = R.exact_step(A, S["b"])
    x = R.step(g, dev["estimate"], S["order"], near=xr)
    omega = R.backward_error(A, x, S["b"])
    kb = R.kappa_bound(A, lam)
    fwd = R.rel(x, xr)
    omega_orc = None
    if name != "grid96x576":
        orc = O.graph_optimize(g, max_iter=1, gain_threshold=0.0)
        assert orc["trials"] == 1
        xo = R.step(g, orc["estimate"], S["order"], near=xr)
        omega_orc = R.backward_error(R.damped(S["H"], orc["lambda_init"]), xo, S["b"])
    print(f"{name} units {f:g}: omega_dev {omega:.3e} omega_orc {omega_orc if omega_orc is None else f'{omega_orc:.3e}'} "
          f"kappa_bound {kb:.3e} forward {fwd:.3e}")
    if omega_orc is None:  # the CPU oracle's step on this grid: 6.2e-7 at its own units (85 s of profile Cholesky)
        assert omega <= (6.2e-6 if f == 1.0 else 1e-6), omega
    else:
        assert omega <= 2 * omega_orc, (omega, omega_orc)
    if f < 1.0:
        assert omega <= 1e-6, omega
    # kappa_bound * omega overstates the forward error by 60x .. 1e5x on these graphs (largest measured ratio 1.7e-2): C = 0.1
    assert fwd <= 0.1 * kb * omega, (fwd, kb, omega)


# LM run to convergence (gain 1e-12, at most 200 iterations) against the reference optimum: Gauss-Newton on the reference system,
# from the graph's estimate at 1/1000 units and from the oracle's converged estimate at the graph's own units (undamped steps diverge
# from the drifted estimate there).  At 1/1000 units both LMs reach the optimum (measured: the oracle 1.9e-11 above it after 8
# iterations).  At the graph's own units g2o's noisy Jacobian moves LM's fixed point: the oracle's chi2 history flattens 2.5e-8 above
# the optimum after 53 iterations, where the reference gradient J^T e is still 0.12 (not 0).  The device, with its own realisation of
# that noise, must stall no further off than 10x the oracle's gap.
@pytest.mark.gpu
@pytest.mark.parametrize("f", UNITS)
def test_converged_chi2_against_reference_optimum(f):
    from stella_vslam_b200 import optimize
    g0 = R.CASES["loop2000"]()
    g = g0 if f == 1.0 else R.scaled(g0, f)
    dev = optimize.graph_optimizer(max_iter=200, gain_threshold=1e-12).optimize(g)
    orc = O.graph_optimize(g, max_iter=200, gain_threshold=1e-12)
    _, chi_opt = R.gauss_newton(g, None if f < 1.0 else orc["estimate"])
    gap_dev, gap_orc = dev["chi2_final"] / chi_opt - 1, orc["chi2_final"] / chi_opt - 1
    hist = orc["chi2_history"]
    print(f"loop2000 units {f:g}: chi2_opt {chi_opt:.10e} gap_dev {gap_dev:.3e} ({dev['iterations']} it) gap_orc {gap_orc:.3e} "
          f"({orc['iterations']} it) oracle history gaps {[f'{c / chi_opt - 1:.2e}' for c in hist[-4:]]}")
    assert gap_dev >= -1e-9 and gap_orc >= -1e-9          # nothing below the optimum
    if f < 1.0:
        assert gap_dev <= 1e-6 and gap_orc <= 1e-6
    else:
        # the oracle's stall: its last iterations change chi2 by under 1e-9 while it sits above the optimum
        assert abs(hist[-1] - hist[-2]) <= 1e-9 * chi_opt and gap_orc > 1e-10
        assert gap_dev <= 10 * gap_orc + 1e-9, (gap_dev, gap_orc)
