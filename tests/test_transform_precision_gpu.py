"""b200_transform_optimize judged one LM step at a time against the high-precision reference of tests/transform_reference.py, with
the CPU oracle's steps as the control (tests/test_transform_precision_cpu.py pins the method without a GPU).

How a step is isolated: num_iter sets round 2 only, round 1 always runs five iterations.  The num_iter = 0 run exports the state
round 1 leaves, and its keep flags are exactly round 1's survivors (the inlier test runs at the state the outlier test did).  Round-2
step k is the difference of the num_iter = k - 1 and k runs, judged where trials[1] == iterations[1] == k.  Its lambda is
lambda_init[1] for k = 1; for k >= 2 it is the value the reference's rho predicts, judged only where every earlier rho sits on the
1/3 or 2/3 clamp with margin (the skipped steps are counted and printed).

Per case and units (1, and every translation times 1e-3, where g2o's delta-1e-9 translation columns are 1000x less noisy):
  - lambda_init[0] equals 1e-5 max diag of the reference's robust H at the caller's Sim3 over every pair.  Round 2's active edges are
    inside the Huber zone by construction (the outlier threshold is delta^2), so the robust branch of H is judged here and through
    the replay of round 1.  lambda_init[1] is judged the same way at the round-1 state over the survivors;
  - each judged step: its normwise backward error omega_dev against H_ref + lambda I is at most max(16 omega_orc, floor, 4 u), and
    at most 1e-6 on the steps where omega_orc <= 1e-6 ("sharp"); its forward error is at most 2 kappa_bound omega; chi2[1] equals
    the reference's robust chi2 at the exported state to 1e-10; under fix_scale the scale is bit-unchanged;
  - round 1 as a whole: the device's round-1 state is within max(10x the oracle's tangent distance, floor) of the reference LM's,
    and its iteration count equals the reference's when no step failed; its trial count equals the reference's wherever the
    oracle's does, on all but MAX_TRIALS_DIFFER cases;
  - every keep flag whose chi2 is clear of chi_sq by a relative 1e-6 equals the reference's test at the exported state;
  - at units 1e-3, 50 iterations reach the reference Gauss-Newton optimum over the survivors; at units 1 the device's chi2 gap to
    it is at most 10x the oracle's;
  - all cases in one ragged call are bit-identical to their single calls.

The number of edges beyond the Huber delta at each judged state is printed (round 1 starts with many, round 2 with none).
Thresholds: see DESIGN.md section 4 for the values measured on an H100 80GB HBM3."""
import functools

import numpy as np
import pytest

import transform_oracle as O
import transform_reference as R
from workloads import synth

CHI_SQ = 10.0
UNITS = (1.0, 1e-3)
K = 5                    # round-2 steps judged per case
FLAG_MARGIN = 1e-6       # relative distance of a chi2 from chi_sq below which a keep flag is not judged
SHARP = 1e-6
MODELS = {"pp": ("perspective", "perspective"), "ee": ("equirect", "equirect"), "pe": ("perspective", "equirect"),
          "ep": ("equirect", "perspective")}


# ---------------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------------
def _rebuilt(pr, pc1, seed, outlier_frac=0.0):
    """pr with its pairs rebuilt from points pc1 (n, 3) given in keyframe 1's camera frame, through the true Sim3, with the noise
    and octave weights of the first n pairs of pr and gross errors of 20-80 px on one observation of a fraction outlier_frac."""
    rng = np.random.default_rng(seed)
    n = len(pc1)
    X = (pc1 - pr["trans_1w"]) @ pr["rot_1w"]
    Gi = np.linalg.inv(R.mat(pr["gt_sim3_12"]))
    pc2 = pc1 @ Gi[:3, :3].T + Gi[:3, 3]                                 # keyframe 2's frame, at the drifted scale
    w1, w2 = np.asarray(pr["inv_sigma_sq_1"][:n], np.float32), np.asarray(pr["inv_sigma_sq_2"][:n], np.float32)
    o1 = R.project(pr["cam_1"], pc1) + rng.standard_normal((n, 2)) / np.sqrt(w1.astype(np.float64))[:, None]
    o2 = R.project(pr["cam_2"], pc2) + rng.standard_normal((n, 2)) / np.sqrt(w2.astype(np.float64))[:, None]
    bad = rng.random(n) < outlier_frac
    side = rng.integers(0, 2, n)
    for o, s in ((o1, 0), (o2, 1)):
        sel = bad & (side == s)
        o[sel] += rng.choice([-1, 1], (sel.sum(), 2)) * rng.uniform(20, 80, (sel.sum(), 2))
    return dict(pr, n_matches=n, obs_1=o1.astype(np.float32), obs_2=o2.astype(np.float32), inv_sigma_sq_1=w1, inv_sigma_sq_2=w2,
                pos_w_1=X, pos_w_2=(pc2 - pr["trans_2w"]) @ pr["rot_2w"], gt_outlier=bad)


def _far(seed):
    """Points 30-40 m from keyframe 1 in its image: the scale is weakly observed, kappa is large."""
    pr = synth.make_sim3_pair(seed, 300, outlier_frac=0.0)
    rng = np.random.default_rng(seed)
    cam = pr["cam_1"]
    d = rng.uniform(30, 40, 300)
    u, v = rng.uniform(100, cam["cols"] - 100, 300), rng.uniform(60, cam["rows"] - 60, 300)
    return _rebuilt(pr, np.stack([(u - cam["cx"]) / cam["fx"] * d, (v - cam["cy"]) / cam["fy"] * d, d], 1), seed, 0.2)


def _seam_pole(seed):
    """Equirectangular pair whose points crowd the +-pi seam (within 0.03-0.1 rad of it) and both poles (0.06-0.15 rad from them)."""
    pr = synth.make_sim3_pair(seed, 400, models=MODELS["ee"], outlier_frac=0.0)
    rng = np.random.default_rng(seed)
    m = 100
    th = np.pi + rng.choice([-1, 1], m) * rng.uniform(0.03, 0.1, m)
    ph = rng.uniform(-0.6, 0.6, m)
    seam = np.stack([np.sin(th) * np.cos(ph), np.sin(ph), np.cos(th) * np.cos(ph)], 1)
    ph = rng.choice([-1, 1], m) * (np.pi / 2 - rng.uniform(0.06, 0.15, m))
    th = rng.uniform(-np.pi, np.pi, m)
    pole = np.stack([np.sin(th) * np.cos(ph), np.sin(ph), np.cos(th) * np.cos(ph)], 1)
    pc1 = np.concatenate([seam, pole, np.asarray(R.camera_points(pr)[1][:2 * m])]) * rng.uniform(4, 20, 4 * m)[:, None]
    return _rebuilt(pr, pc1, seed, 0.2)


def _near_optimum(seed, f):
    """A clean pair started 1e-7 (tangent) from the reference optimum over every pair."""
    pr = R.scaled(synth.make_sim3_pair(seed, 300, outlier_frac=0.0, pixel_sigma=0.5), f)
    S, _ = R.gauss_newton(pr, pr["gt_sim3_12"])
    u = np.random.default_rng(seed).standard_normal(7)
    u[3:6] *= f
    return dict(pr, sim3_12=R.oplus(S, 1e-7 * u / np.abs(u).max()))


def _pair(seed, n, models="pp", fix_scale=False, outlier_frac=0.3, **kw):
    return lambda: synth.make_sim3_pair(seed, n, models=MODELS[models], fix_scale=fix_scale, outlier_frac=outlier_frac, **kw)


CASES = {f"{m}_{'fixed' if fs else 'free'}": _pair(10 + 2 * i + fs, 300, m, fs) for i, m in enumerate(MODELS) for fs in (False, True)}
CASES.update({
    "pp_clean": _pair(20, 300, outlier_frac=0.0),
    "ee_clean": _pair(21, 300, "ee", outlier_frac=0.0),
    "wide_start": _pair(22, 300, outlier_frac=0.3, init_noise=(0.1, 0.2, 0.05)),
    "far": lambda: _far(23),
    "seam_pole": lambda: _seam_pole(24),
    "n10": _pair(25, 10, outlier_frac=0.0, pixel_sigma=0.5),
    **{f"n{n}": _pair(26 + k, n, outlier_frac=0.2) for k, n in enumerate((255, 256, 257, 512, 513, 2000))},
    "n15168": _pair(33, 15400, "ee", outlier_frac=0.2),       # trimmed to 15 168 after the guard
    "near_optimum": None,
})
NAMES = list(CASES)


@functools.lru_cache(maxsize=None)
def case(name, f):
    if name == "near_optimum":
        return _near_optimum(34, f)
    pr = CASES[name]()
    pr = pr if f == 1.0 else R.scaled(pr, f)
    # no equirectangular stencil may reach the seam or a pole, at the start or at the truth
    seam, pole = R.guard(pr, pr["sim3_12"], pr["fix_scale"])
    seam_t, pole_t = R.guard(pr, pr["gt_sim3_12"], pr["fix_scale"])
    ok = ~(seam | pole | seam_t | pole_t)
    if not ok.all():
        pr = dict(R._subset(pr, ok), n_matches=int(ok.sum()), gt_outlier=np.asarray(pr["gt_outlier"])[ok])
    if name == "n15168":            # the pair count of a 3840 x 1920 golden frame
        keep = np.arange(len(pr["obs_1"])) < 15168
        pr = dict(R._subset(pr, keep), n_matches=15168, gt_outlier=np.asarray(pr["gt_outlier"])[keep])
        assert len(pr["obs_1"]) == 15168
    return pr


# ---------------------------------------------------------------------------------------------------------------------
# judging
# ---------------------------------------------------------------------------------------------------------------------
def device_runs(pr, ks):
    from stella_vslam_b200 import optimize
    return {k: optimize.transform_optimizer(pr["fix_scale"], num_iter=k).optimize(pr, CHI_SQ) for k in ks}


def oracle_runs(pr, ks):
    return {k: O.transform_optimize(pr, CHI_SQ, k) for k in ks}


def round2_steps(pr, runs):
    """The judged round-2 steps of one implementation's runs {num_iter: result}: [dict(k, lam, Sys, J, chi2)], and the number of
    steps not judged because a rho was off the clamp."""
    fs = pr["fix_scale"]
    active = runs[0]["keep"].astype(bool)
    lam = runs[1]["lambda_init"][1]
    out, skipped = [], 0
    for k in range(1, K + 1):
        o = runs[k]
        if not (o["iterations"][1] == k and o["trials"][1] == k):
            break
        Sys = R.system(pr, runs[k - 1]["sim3_12"], active, fs, CHI_SQ)
        J = R.judge(Sys, lam, o["sim3_12"])
        chi_new = R.robust_chi2(pr, o["sim3_12"], active, CHI_SQ)
        out.append(dict(k=k, lam=lam, Sys=Sys, J=J, chi2=chi_new))
        r = R.gain_ratio(Sys, lam, J["x"], chi_new)
        if not R.on_clamp(r):
            skipped = K - k
            break
        lam *= R.lambda_factor(r)
    return out, skipped


def check_flags(pr, S, keep, active=None):
    """keep equals the reference's test at S on every pair whose chi2 are clear of chi_sq; returns the number not judged."""
    c = R.edge_chi2(pr, S)
    act = np.ones(len(c), bool) if active is None else np.asarray(active, bool)
    want = act & (c < CHI_SQ).all(1) if active is None else act & (c <= CHI_SQ).all(1)
    clear = (np.abs(c - CHI_SQ) > FLAG_MARGIN * CHI_SQ).all(1) | ~act
    bad = np.nonzero(clear & (np.asarray(keep, bool) != want))[0]
    assert len(bad) == 0, (bad[:10], len(bad))
    return int((~clear).sum())


def _tag(name, f):
    return f"{name} units {f:g}"


# ---------------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def judged(name, f):
    """Everything test_steps asserts on for one case, computed once per session (test_coverage reads it for every case)."""
    pr = case(name, f)
    n, fs = len(pr["obs_1"]), pr["fix_scale"]
    ks = list(range(K + 1))
    dev, orc = device_runs(pr, ks), oracle_runs(pr, ks)
    d0 = dev[0]

    # lambda at the start of both rounds: the robust branch of H (round 1 starts with every pair, outliers beyond delta included)
    S_init = R.system(pr, pr["sim3_12"], None, fs, CHI_SQ)
    active = d0["keep"].astype(bool)
    S_r1 = R.system(pr, d0["sim3_12"], active, fs, CHI_SQ)
    lam_ref = (R.lambda_init(S_init), R.lambda_init(S_r1))
    lam_err = [abs(d0["lambda_init"][0] / lam_ref[0] - 1), abs(dev[1]["lambda_init"][1] / lam_ref[1] - 1)]
    lam_err_orc = [abs(orc[0]["lambda_init"][0] / lam_ref[0] - 1), abs(orc[1]["lambda_init"][1] / lam_ref[1] - 1)]

    # round 1 replayed with exact solves
    ref1 = R.lm_round(pr, pr["sim3_12"], 5, None, fs, CHI_SQ)
    dist_dev = R.tangent_distance(d0["sim3_12"], ref1["S"], fs)
    dist_orc = R.tangent_distance(orc[0]["sim3_12"], ref1["S"], fs)
    floor1 = 16 * R.U * (1 + np.abs(ref1["S"][4:7]).max())

    steps, skipped = round2_steps(pr, dev)
    steps_o, _ = round2_steps(pr, orc)
    equi = pr["cam_1"]["model"] == 1 or pr["cam_2"]["model"] == 1
    print(f"{_tag(name, f)}: n {n} outliers1 {d0['n_outliers_round1']} beyond-delta at start {S_init['n_beyond']} at round-1 state "
          f"{S_r1['n_beyond']} | lambda_init rel err dev {lam_err[0]:.1e} {lam_err[1]:.1e} orc {lam_err_orc[0]:.1e} {lam_err_orc[1]:.1e} | "
          f"round 1 dist dev {dist_dev:.2e} orc {dist_orc:.2e} floor {floor1:.1e} it {d0['iterations'][0]}/{ref1['iterations']} "
          f"trials dev {d0['trials'][0]} orc {orc[0]['trials'][0]} ref {ref1['trials']} | judged {len(steps)} skipped {skipped}")
    rows = []
    for st in steps:
        J, k = st["J"], st["k"]
        so = next((s for s in steps_o if s["k"] == k), None)
        om_orc = so["J"]["omega"] if so is not None else None
        chi_err = abs(dev[k]["chi2"][1] / st["chi2"] - 1)
        fw = J["forward"] / max(J["kappa_bound"] * J["omega"], 1e-300)
        rows.append(dict(k=k, omega=J["omega"], omega_orc=om_orc, floor=J["floor"], kappa_bound=J["kappa_bound"], forward=J["forward"],
                         chi_err=chi_err))
        print(f"  step {k}: omega_dev {J['omega']:.2e} omega_orc {om_orc if om_orc is None else f'{om_orc:.2e}'} floor "
              f"{J['floor']:.2e} kappa_bound {J['kappa_bound']:.2e} forward {J['forward']:.2e} ({fw:.1e} of kappa omega) chi2 rel "
              f"{chi_err:.1e} ({'equirect' if equi else 'perspective'}) beyond-delta {st['Sys']['n_beyond']}")
    return dict(pr=pr, dev=dev, orc=orc, active=active, lam_err=lam_err, ref1=ref1, dist_dev=dist_dev, dist_orc=dist_orc,
                floor1=floor1, rows=rows, equi=equi)


@pytest.mark.gpu
@pytest.mark.parametrize("f", UNITS)
@pytest.mark.parametrize("name", NAMES)
def test_steps(name, f):
    c = judged(name, f)
    pr, dev, d0, ref1 = c["pr"], c["dev"], c["dev"][0], c["ref1"]
    n, fs = len(pr["obs_1"]), pr["fix_scale"]

    # the num_iter = 0 run: round 1's state and survivors
    assert int(d0["keep"].sum()) == n - d0["n_outliers_round1"] == d0["num_inliers"], (d0["keep"].sum(), d0["n_outliers_round1"])
    assert d0["iterations"][1] == 0 and n - d0["n_outliers_round1"] >= 10
    assert c["lam_err"][0] <= LAM_TOL[f == 1.0], c["lam_err"]
    assert c["lam_err"][1] <= LAM_TOL[f == 1.0], c["lam_err"]
    assert c["dist_dev"] <= max(DIST_RATIO * c["dist_orc"], c["floor1"]), (c["dist_dev"], c["dist_orc"])
    if not ref1["failed"]:
        assert d0["iterations"][0] == ref1["iterations"]
        check_flags(pr, d0["sim3_12"], d0["keep"])
    # the first round-2 trial of a small or converged problem can be rejected on g2o's noise: nothing to judge there
    assert len(c["rows"]) >= 1 or f == 1.0 or name == "near_optimum"
    for r in c["rows"]:
        k, om, om_orc = r["k"], r["omega"], r["omega_orc"]
        # omega_orc is None where the oracle's trial of that step was rejected (measured: converged steps at units 1, omega_dev
        # 2e-4 .. 8e-4, the size of g2o's Jacobian noise): no control, so no backward-error bound there
        if om_orc is not None:
            assert om <= max(OMEGA_RATIO * om_orc, r["floor"], R.ROUNDOFF), (k, om, om_orc, r["floor"])
            if om_orc <= SHARP:
                assert om <= SHARP, (k, om)
        if name != "near_optimum":     # there the reference step is smaller than the Jacobian noise of b
            assert r["forward"] <= FWD_C * r["kappa_bound"] * max(om, r["floor"]), (k, r["forward"], r["kappa_bound"], om)
        assert r["chi_err"] <= CHI_TOL, (k, r["chi_err"])
        if fs:
            assert dev[k]["sim3_12"][7] == dev[k - 1]["sim3_12"][7]
        check_flags(pr, dev[k]["sim3_12"], dev[k]["keep"], c["active"])


@pytest.mark.gpu
def test_coverage():
    """Over every case: enough sharp steps judged on the device, and round 1's trial count equal to the replay's wherever the
    oracle's is (a late round-1 trial rejected on g2o's noisy Jacobian adds trials, the oracle's as well as the device's)."""
    sharp, judged_steps, same_orc, differ = 0, 0, 0, []
    for name in NAMES:
        for f in UNITS:
            c = judged(name, f)
            judged_steps += len(c["rows"])
            sharp += sum(r["omega_orc"] is not None and r["omega_orc"] <= SHARP for r in c["rows"])
            t_dev, t_orc, t_ref = c["dev"][0]["trials"][0], c["orc"][0]["trials"][0], c["ref1"]["trials"]
            if not c["ref1"]["failed"] and t_orc == t_ref:
                same_orc += 1
                if t_dev != t_ref:
                    differ.append((_tag(name, f), t_dev, t_ref))
    print(f"judged steps {judged_steps}, sharp {sharp}; round-1 trials: oracle equal to the replay on {same_orc} cases, "
          f"device different on {differ}")
    assert sharp >= MIN_SHARP, sharp
    assert len(differ) <= MAX_TRIALS_DIFFER, differ


# Measured on an H100 80GB HBM3 (the 44 cases, 169 judged steps): lambda_init against the reference up to 3.4e-8 at units 1 and
# 3.7e-9 at 1e-3; omega_dev / omega_orc up to 12.2 over the 165 steps the oracle also took (two realisations of g2o's delta-1e-9
# noise); the round-1 distance ratio up to 5.7; chi2[1] against the reference up to 3.7e-11 with perspective cameras and 2.2e-11
# with an equirectangular one (the oracle's own chi2 is 6e-12 off: the reference maps points through a rotation matrix, the
# kernel through a quaternion, and e = obs - u loses three digits to cancellation), so one bound for both.
LAM_TOL = {True: 1e-7, False: 1e-8}
OMEGA_RATIO = 16.0
DIST_RATIO = 10.0
FWD_C = 2.0             # measured: forward error up to 0.99 kappa_bound omega
CHI_TOL = 1e-10
MIN_SHARP = 120         # measured: 170 judged steps, 132 of them sharp
MAX_TRIALS_DIFFER = 2   # measured: the oracle's trial count equals the replay's on 38 cases, the device's differs on 1 (n10 units 1)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["pp_free", "ee_free", "pp_clean", "far"])
def test_converged(name):
    """50 round-2 iterations against the reference Gauss-Newton optimum over the survivors."""
    out = []
    for f in UNITS:
        pr = case(name, f)
        fs = pr["fix_scale"]
        dev = device_runs(pr, [0, 50])
        orc = oracle_runs(pr, [50])[50]
        active = dev[0]["keep"].astype(bool)
        S_opt, chi_opt = R.gauss_newton(pr, dev[50]["sim3_12"], active, fs, CHI_SQ)
        H = np.asarray(R.system(pr, S_opt, active, fs, CHI_SQ)["H"], np.float64)[:6 if fs else 7, :6 if fs else 7]
        d = 1 / np.sqrt(np.diag(H))
        kappa = float(np.linalg.cond(d[:, None] * H * d[None, :]))     # of the equilibrated H: the same at every units
        d_dev, d_orc = R.tangent_distance(dev[50]["sim3_12"], S_opt, fs), R.tangent_distance(orc["sim3_12"], S_opt, fs)
        chi_dev, chi_orc = R.robust_chi2(pr, dev[50]["sim3_12"], active, CHI_SQ), R.robust_chi2(pr, orc["sim3_12"], active, CHI_SQ)
        gap_dev, gap_orc = chi_dev / chi_opt - 1, chi_orc / chi_opt - 1
        print(f"{_tag(name, f)}: dist dev {d_dev:.2e} orc {d_orc:.2e} kappa {kappa:.2e} (dist / kappa noise: dev "
              f"{d_dev / (kappa * JAC_NOISE):.1e} orc {d_orc / (kappa * JAC_NOISE):.1e}) gap dev {gap_dev:.2e} orc {gap_orc:.2e} "
              f"it {dev[50]['iterations']} {orc['iterations']}")
        out.append((f, d_dev, d_orc, gap_dev, gap_orc, kappa))
    for f, d_dev, d_orc, gap_dev, gap_orc, kappa in out:
        assert gap_dev >= -1e-12 and gap_orc >= -1e-12
        if f < 1.0:
            assert d_dev <= CONV_C * kappa * JAC_NOISE and gap_dev <= 1e-12, (d_dev, kappa, gap_dev)
        else:
            assert gap_dev <= 10 * gap_orc + 1e-13, (gap_dev, gap_orc)


# LM's fixed point is where g2o's noisy gradient vanishes: it sits off the optimum by about kappa times the Jacobian's relative
# noise (JAC_NOISE: the delta-1e-9 difference's rotation columns at units 1e-3, tests/test_transform_precision_cpu.py).
JAC_NOISE = 3e-7
CONV_C = 1.0             # measured: the distance is 1.6e-5 .. 5.1e-2 of kappa JAC_NOISE for the device, up to 0.19 for the oracle


@pytest.mark.gpu
def test_ragged_batch_equals_single_calls():
    from stella_vslam_b200 import optimize
    for fs in (False, True):
        probs = [case(n, f) for n in NAMES for f in UNITS if case(n, f)["fix_scale"] == fs]
        batch = optimize.transform_optimizer(fs, num_iter=K).optimize_batch(probs, CHI_SQ)
        for pr, b in zip(probs, batch):
            a = device_runs(pr, [K])[K]
            for k in ("sim3_12", "keep", "chi2", "lambda_init"):
                assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k
            for k in ("num_inliers", "n_outliers_round1", "iterations", "trials"):
                assert a[k] == b[k], k
