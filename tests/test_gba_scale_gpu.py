"""Each LM step of global BA's panel-by-panel Cholesky (gchol_panel_kernel, gchol_trail_kernel, gchol_finish_kernel) on multi-lap
maps from 500 free keyframes to the 4 000-free-keyframe limit of b200_global_ba_solve, judged against the high-precision reference
of tests/lba_reference.py with the exact step of tests/gba_scale.py (the method is pinned without a GPU by test_gba_scale_cpu.py).

Every keyframe of these maps shares landmarks with the keyframes that revisit its place a lap earlier and later, so the reduced
matrix has nonzero blocks far from the diagonal, and the sizes reach what only large systems exercise: trailing-update tile ids past
ten million (the tile row recovered from a double sqrt), a trailing-update grid past 65 535 CTAs (n > 23 191: 3 866 free keyframes
and more), full and partial last panels (n % 24 == 0 or not), and M rebuilt over the previous iteration's factor on every step.
Per case, as test_lba_precision_gpu.py judges a step:
  - lambda_init equals 1e-5 max diag(H_ref) to 1e-12 relative (first steps);
  - the reported chi2 equals the reference chi2 at the device's output state to 1e-11;
  - lambda_final equals the rho prediction of an accepted first trial to 1e-8;
  - the normwise backward error of the step read back from the output state against H_ref + lambda I, and the largest one of a
    keyframe's block rows, are at most 2 max(omega_floor, 4 u); where the CPU oracle runs (500 free keyframes) its step, an exact
    Schur solve of its own system read back the same way, is one more realisation of that floor: 2 max(omega_orc, omega_floor, 4 u)
    as in test_lba_precision_gpu.py;
  - the forward error against the exact step is at most kappa_bound * omega;
  - the fixed keyframes are bit-unchanged, and the launch count shows that the panel path ran.

Measured on an H100 80GB HBM3: see DESIGN.md section 4."""
import ctypes as C

import numpy as np
import pytest

import gba_scale as G
import lba_reference as R
from oracle import pyoracle as O
from workloads import synth

pytestmark = pytest.mark.gpu

ROUNDOFF = 4 * 2.0 ** -53
HUBER_MARGIN = 1e-12        # no Huber decision of a judged state within this of its threshold (device and reference must agree)


@pytest.fixture(scope="module")
def cache():
    """The maps of gba_scale.MAPS, each built once, and the device's one-step results with Huber (the state before step 2)."""
    return dict(maps={}, first={})


def _map(cache, name):
    if name not in cache["maps"]:
        cache["maps"][name] = G.named_map(name)
    return cache["maps"][name]


def _n(pr):
    return 6 * int((np.asarray(pr["pose_fixed"]) == 0).sum())


def _need_memory(pr):
    """Skip when the device has less free memory than the dense reduced system M ((n + 1) (n + 2) doubles) plus 1 GiB."""
    import torch
    n = _n(pr)
    need = 8 * (n + 1) * (n + 2) + (1 << 30)
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"{free} bytes of device memory free, {need} needed for n = {n}")


def _solve(pr, num_iter, huber):
    from stella_vslam_b200 import optimize
    dev = optimize.global_bundle_adjuster(num_iter, use_huber_kernel=huber).optimize(pr, gain_threshold=0.0)
    assert dev["iterations"] == num_iter
    assert dev["launches"] > 2 * (_n(pr) // 24)                 # the panel-by-panel path ran
    return dev


def _judge(label, pr, S, lam, lam_rep, dev, orc=None):
    assert G.huber_margin(pr, S["pose_cw"], S["points"]) > HUBER_MARGIN
    x_exact, omegas = G.exact_step(S, lam)
    J = R.check_step(S, lam, lam_rep, dev["chi2"], dev["lambda_final"], dev["pose_cw"], dev["points"], pr, x_exact=x_exact)
    ratio = J["forward"] / (J["kappa_bound"] * J["omega"])
    line = (f"{label}: omega_dev {J['omega']:.2e} floor {J['floor']:.2e} | keyframe rows dev {J['omega_kf']:.2e} floor "
            f"{J['floor_kf']:.2e} | kappa_bound {J['kappa_bound']:.2e} forward {J['forward']:.2e} (forward / kappa omega {ratio:.1e}) "
            f"| exact step {omegas[-1]:.1e} after {len(omegas) - 1} refinements | gpu_ms {dev['gpu_ms']:.1f} launches {dev['launches']}")
    bound, bound_kf = max(J["floor"], ROUNDOFF), max(J["floor_kf"], ROUNDOFF)
    if orc is not None:
        Jo = R.judge(S, orc["lambda_init"], orc["pose_cw"], orc["points"], x_exact=x_exact)
        line += f" | omega_orc {Jo['omega']:.2e} keyframe rows {Jo['omega_kf']:.2e}"
        bound, bound_kf = max(bound, Jo["omega"]), max(bound_kf, Jo["omega_kf"])
    print(line)
    assert J["omega"] <= 2 * bound, (J["omega"], J["floor"])
    assert J["omega_kf"] <= 2 * bound_kf, (J["omega_kf"], J["floor_kf"])
    assert J["forward"] <= J["kappa_bound"] * J["omega"], (J["forward"], J["kappa_bound"], J["omega"])


FIRST = [(m, h) for m in ("free500", "free1000", "free2047", "free3333", "free4000") for h in (True, False)] + \
        [("mono998", True), ("equirect1001", True)]


@pytest.mark.parametrize("name,huber", FIRST)
def test_first_step(name, huber, cache):
    pr = _map(cache, name)
    _need_memory(pr)
    pr_h = pr if huber else dict(pr, e_robust=np.zeros(len(pr["e_pose"]), np.uint8))
    dev = _solve(pr, 1, huber)
    if huber:
        cache["first"][name] = dev
    orc = None
    if name == "free500":                                       # the existing tests' control, at a size the C oracle factors in seconds
        orc = O.global_ba_solve(pr_h, num_iter=1, gain_threshold=0.0)
        assert orc["iterations"] == 1
    S = R.system(pr_h)
    _judge(f"{name} huber {huber} step 1", pr_h, S, dev["lambda_init"], dev["lambda_init"], dev, orc)


@pytest.mark.parametrize("name", ["free1000", "free4000"])
def test_later_steps(name, cache):
    """Steps 2 and 3 (step 1 is test_first_step's Huber case): num_iter = k, judged at the state and lambda the device's own run of
    k - 1 iterations left (the device is run-to-run deterministic).  M holds the previous step's factor when it is rebuilt, so every
    block -- those no landmark pair touches included -- must be rewritten on every build."""
    pr = _map(cache, name)
    _need_memory(pr)
    prev = cache["first"].get(name) or _solve(pr, 1, True)
    for k in (2, 3):
        dev = _solve(pr, k, True)
        assert dev["lambda_init"] == prev["lambda_init"]
        S = R.system(pr, prev["pose_cw"], prev["points"])
        _judge(f"{name} step {k} lambda {prev['lambda_final']:.3e}", pr, S, prev["lambda_final"], None, dev)
        prev = dev


def test_limit_straddle(cache):
    """4 000 free keyframes are accepted (test_first_step's free4000 cases); the same map with its root unfixed, 4 001 free keyframes,
    is refused with B200_ERR_INVALID before anything is allocated or launched, and the output buffers are not written."""
    import torch
    from stella_vslam_b200 import _lib, optimize
    pr = _map(cache, "free4000")
    pr4001 = dict(pr, pose_fixed=np.zeros(len(pr["pose_cw"]), np.uint8))
    assert _n(pr) == 24000 and _n(pr4001) == 24006
    gba = optimize.global_bundle_adjuster(3)
    small = synth.make_ba_problem(12, 1, 400, seed=5)
    assert gba.optimize(small)["launches"] > 0                  # the handle's last launch count is not zero before the refusal
    L = gba._L
    P, keep = optimize.pack_problem(pr4001)
    pose_out = np.full((P.n_poses, 4, 4), 7.25)
    pts_out = np.full((P.n_points, 3), -3.5)
    st = optimize.LbaStats()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    rc = L.b200_global_ba_solve(gba._h, C.byref(P), 3, 0.0, None, _lib.ptr(pose_out), _lib.ptr(pts_out), C.byref(st))
    free1 = torch.cuda.mem_get_info()[0]
    msg = L.b200_last_error().decode()
    print(f"4001 free keyframes: rc {rc}, '{msg}', device memory free {free0} -> {free1}")
    assert rc == _lib.ERR_INVALID
    assert "4001 free keyframes" in msg and "limit of this entry point is 4000" in msg, msg
    assert (pose_out == 7.25).all() and (pts_out == -3.5).all()
    ms, launches = C.c_float(), C.c_int()
    L.b200_lba_last_profile(gba._h, C.byref(ms), C.byref(launches))
    assert launches.value == 0 and ms.value == 0.0
    assert free0 - free1 < 256 << 20                            # M alone would be (n + 1) (n + 2) doubles = 4.6 GB
