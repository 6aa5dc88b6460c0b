"""The multi-lap maps and the exact step of tests/gba_scale.py, pinned without a GPU: the maps couple every keyframe with the keyframes
a lap away (so the far tiles of the off-chip trailing update are not zero), and the Schur-route exact step agrees with SuperLU on the
full system where SuperLU runs and reaches a few unit roundoffs of backward error at 24 000 keyframe unknowns."""
import numpy as np
import pytest

import gba_scale as G
import lba_reference as R
from workloads import synth

TILE = 32                   # keyframes per tile of the block pattern


@pytest.fixture(scope="module")
def map4000():
    return G.named_map("free4000")


@pytest.mark.parametrize("name", ["free500", "free4000"])
def test_every_keyframe_couples_a_lap_away(name, map4000):
    pr = map4000 if name == "free4000" else G.named_map(name)
    i, j, Kf = G.keyframe_blocks(pr)
    lap = Kf / pr["laps"]
    far = np.zeros(Kf, bool)
    d = np.abs(j - i)
    far[i[d >= lap - 2]] = True
    far[j[d >= lap - 2]] = True
    print(f"{name}: {Kf} free keyframes, {len(i)} nonzero blocks, farthest {d.max()}")
    assert far.all(), np.nonzero(~far)[0][:10]
    # the block pattern at 32 x 32-keyframe tiles: every tile row has a nonzero tile next to the diagonal and one a lap away
    ti, tj = np.concatenate([i, j]) // TILE, np.concatenate([j, i]) // TILE
    n_t = -(-Kf // TILE)
    near_t, far_t = np.zeros(n_t, bool), np.zeros(n_t, bool)
    near_t[ti[np.abs(ti - tj) <= 1]] = True
    far_t[ti[np.abs(ti - tj) * TILE >= lap - 2 * TILE]] = True
    assert near_t.all() and far_t.all(), (np.nonzero(~near_t)[0], np.nonzero(~far_t)[0])


def test_map_shape(map4000):
    """Keyframe i and i + K/laps, i + 2K/laps stand within a few decimetres of each other; every landmark is observed at least twice,
    3..8 times per lap; no Huber decision of any map of the GPU file lies within 1e-12 of its threshold at the initial state."""
    pr = map4000
    K, P = len(pr["pose_cw"]), pr["places"]
    c = -np.einsum("kji,kj->ki", pr["gt_pose_cw"][:, :3, :3], pr["gt_pose_cw"][:, :3, 3])
    gap = np.linalg.norm(c[P:] - c[:K - P], axis=1)
    assert gap.max() < 0.5 and np.linalg.norm(c[1:P] - c[:P - 1], axis=1).min() > 0.5
    deg = np.bincount(pr["e_point"])
    print(f"free4000: {len(deg)} landmarks, {len(pr['e_pose'])} edges, observations per landmark {deg.min()}..{deg.max()} "
          f"(mean {deg.mean():.1f})")
    assert deg.min() >= 2 and 10 <= deg.mean() <= 24 and deg.max() <= 24
    assert len(deg) >= 59000
    for name in G.MAPS:
        m = map4000 if name == "free4000" else G.named_map(name)
        margin = G.huber_margin(m, m["pose_cw"], m["points"])
        assert margin > 1e-12, (name, margin)
        assert np.bincount(m["e_pose"], minlength=len(m["pose_cw"])).min() > 50, name


SMALL = {
    "small_stereo": lambda: synth.make_ba_problem(30, 1, 2000, seed=1),
    "map180": lambda: synth.make_ba_problem(180, 1, 4000, seed=11),
    "free500": lambda: G.named_map("free500"),
}


@pytest.mark.parametrize("huber", [True, False])
@pytest.mark.parametrize("name", list(SMALL))
def test_exact_step_agrees_with_superlu(name, huber):
    """The Schur-route step against sparse_lm.exact_step (SuperLU on the full system, one refinement): forward difference within
    kappa_bound u, backward error within 2x.  On the multi-lap map SuperLU's own fill-reducing order takes minutes, so its factor
    eliminates the landmarks first there."""
    pr = SMALL[name]()
    if not huber:
        pr = dict(pr, e_robust=np.zeros(len(pr["e_pose"]), np.uint8))
    S = R.system(pr)
    lam = R.lambda_init(S)
    A = R.damped(S["H"], lam)
    x, omegas = G.exact_step(S, lam)
    lu = G.LandmarksFirstLU(A, S["n_pose"]) if name == "free500" else None
    x_lu = R.exact_step(A, S["b"], lu)
    om, om_lu = R.backward_error(A, x.astype(R.LD), S["b"]), R.backward_error(A, x_lu.astype(R.LD), S["b"])
    kb = R.kappa_bound(A, lam)
    print(f"{name} huber {huber}: n {A.shape[0]} (keyframes {S['n_pose']}), omega schur {om:.1e} (refinements {omegas}) superlu "
          f"{om_lu:.1e}, rel {R.rel(x, x_lu):.1e}, kappa_bound u {kb * G.U:.1e}")
    assert R.rel(x, x_lu) <= kb * G.U
    assert om <= 2 * om_lu


def test_exact_step_at_the_limit(map4000):
    """24 000 keyframe unknowns and 180 000 landmark unknowns: at most 4 u of backward error after at most four refinements."""
    S = R.system(map4000)
    assert S["n_pose"] == 24000
    lam = R.lambda_init(S)
    x, omegas = G.exact_step(S, lam, target=4 * G.U)
    print(f"free4000: backward error per refinement {omegas}")
    assert len(omegas) - 1 <= 4 and omegas[-1] <= 4 * G.U
    assert omegas[-1] == pytest.approx(R.backward_error(R.damped(S["H"], lam), x.astype(R.LD), S["b"]), rel=1e-6)
