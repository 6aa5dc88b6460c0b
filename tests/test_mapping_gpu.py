"""b200_triangulate_pairs and b200_create_new_landmarks against the CPU restatement (tests/mapping_oracle.c with
oracle.pyoracle's match_for_triangulation), and the chain against the stage-by-stage GPU path."""
import numpy as np
import pytest

import mapping_oracle as MO
from stella_vslam_b200 import _lib, mapping
from stella_vslam_b200.match import PAIRS_TRIANGULATION, match_pairs_batch
from workloads import synth

pytestmark = pytest.mark.gpu

CASES = [("perspective", False), ("perspective", True), ("equirectangular", False)]


def _close(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape
    if a.size:
        same = (a == b) | (np.isnan(a) & np.isnan(b))  # rejected far pairs may carry inf / nan (v(3) = 0)
        assert np.all(same | (np.abs(a - b) <= 1e-12 * np.maximum(np.abs(b), 1.0))), np.abs(a - b)[~same].max()


def _all_pairs(cur, ngh, rng, n=3000):
    return np.stack([rng.integers(0, len(cur["x"]), n), rng.integers(0, len(ngh["x"]), n)], 1).astype(np.int32)


@pytest.mark.parametrize("model,stereo", CASES)
def test_triangulate_pairs_matches_oracle(model, stereo):
    cur, nb = synth.make_mapping_problem(11, 3, 1500, model=model, stereo=stereo)
    rng = np.random.default_rng(3)
    problems, want = [], []
    for ngh in nb:
        # true correspondences (via the chain's matches) plus random pairs, which exercise every reject branch
        m = MO.create_new_landmarks(cur, [ngh])["match_out"][0]
        i1 = np.flatnonzero(m >= 0)
        pairs = np.concatenate([np.stack([i1, m[i1]], 1), _all_pairs(cur, ngh, rng)]).astype(np.int32)
        problems.append((cur, ngh, pairs, 1.0))
        want.append(MO.triangulate_pairs(cur, ngh, pairs, 1.0))
    got = mapping.triangulate_pairs_batch(problems)
    n_ok = 0
    for (gp, gok), (wp, wok) in zip(got, want):
        assert np.array_equal(gok, wok)
        _close(gp, wp)  # every match: the point before the tests (rejected branches included), zeros without a branch
        n_ok += int(wok.sum())
    assert n_ok > 100


@pytest.mark.parametrize("bow", [False, True])
@pytest.mark.parametrize("model,stereo", CASES)
def test_create_new_landmarks_matches_oracle(model, stereo, bow):
    cur, nb = synth.make_mapping_problem(21, 6, 1500, model=model, stereo=stereo)
    got = mapping.create_new_landmarks_batch([(cur, nb)], bow=bow, return_matches=True)[0]
    want = MO.create_new_landmarks(cur, nb, bow=bow)
    for g, w in zip(got["match_out"], want["match_out"]):
        assert np.array_equal(g, w)
    assert np.array_equal(got["n_matches"], want["n_matches"])
    assert np.array_equal(got["n_created"], want["n_created"])
    assert np.array_equal(got["rank"], want["rank"]) and np.array_equal(got["idx"], want["idx"])
    _close(got["pos_w"], want["pos_w"])
    assert len(got["rank"]) > 100


def test_chain_equals_stage_by_stage_gpu_path():
    cur, nb = synth.make_mapping_problem(31, 8, 2000, stereo=True)
    chain = mapping.create_new_landmarks_batch([(cur, nb)], return_matches=True)[0]
    free = cur["no_landmark"].copy()
    ranks, idx, pos, claimed_then_matched = [], [], [], 0
    for r, ngh in enumerate(nb):
        pr = MO.triangulation_problem(cur, ngh, mapping.RESIDUAL_RAD_THR, False, free.copy())
        mo, n = match_pairs_batch([pr], PAIRS_TRIANGULATION, 0.95, False)[0]
        assert np.array_equal(mo, chain["match_out"][r]) and n == chain["n_matches"][r]
        # would a row already claimed by an earlier rank have matched here?
        pr_open = MO.triangulation_problem(cur, ngh, mapping.RESIDUAL_RAD_THR, False, cur["no_landmark"].copy())
        mo_open, _ = match_pairs_batch([pr_open], PAIRS_TRIANGULATION, 0.95, False)[0]
        claimed_then_matched += int(np.sum((free == 0) & (cur["no_landmark"] == 1) & (mo_open >= 0)))
        i1 = np.flatnonzero(mo >= 0)
        pairs = np.stack([i1, mo[i1]], 1).astype(np.int32)
        p, ok = mapping.two_view_triangulator(cur, ngh).triangulate(pairs)
        ranks += [r] * int(ok.sum())
        idx.append(pairs[ok])
        pos.append(p[ok])
        free[pairs[ok][:, 0]] = 0
    assert np.array_equal(chain["rank"], np.array(ranks))
    assert np.array_equal(chain["idx"], np.concatenate(idx))
    assert np.array_equal(chain["pos_w"], np.concatenate(pos))
    assert claimed_then_matched > 0


def test_ragged_batches():
    items = [synth.make_mapping_problem(40 + k, 1 + k % 4, 600 + 50 * k, stereo=k % 2 == 1) for k in range(16)]
    items = [(c, n) for c, n in items]
    items[3] = (items[3][0], [])                                        # no neighbours
    empty = dict(items[5][1][0])
    for f in ("x", "y", "octave", "node", "no_landmark", "angle", "x_right", "depth"):
        if empty.get(f) is not None:
            empty[f] = empty[f][:0]
    empty["bearings"], empty["desc"] = empty["bearings"][:0], empty["desc"][:0]
    items[5] = (items[5][0], [items[5][1][0], empty] + items[5][1][1:])  # a neighbour without keypoints
    full = dict(items[7][0])
    full["no_landmark"] = np.zeros_like(full["no_landmark"])             # every row already carries a landmark
    items[7] = (full, items[7][1])
    batch = mapping.create_new_landmarks_batch(items, return_matches=True)
    for k, (cur, nb) in enumerate(items):
        want = MO.create_new_landmarks(cur, nb)
        single = mapping.create_new_landmarks_batch([(cur, nb)], return_matches=True)[0]
        for got in (batch[k], single):
            assert np.array_equal(got["rank"], want["rank"]) and np.array_equal(got["idx"], want["idx"])
            assert np.array_equal(got["n_matches"], want["n_matches"]) and np.array_equal(got["n_created"], want["n_created"])
            _close(got["pos_w"], want["pos_w"])
        assert np.array_equal(batch[k]["pos_w"], single["pos_w"])
    assert len(batch[3]["rank"]) == 0 and len(batch[7]["rank"]) == 0 and batch[5]["n_matches"][1] == 0


def test_errors():
    cur, nb = synth.make_mapping_problem(50, 2, 1500)
    # a neighbour listing every keypoint twice: each matchable row keeps at least two gated candidates
    dup = {f: (np.concatenate([v, v]) if isinstance(v, np.ndarray) and f not in ("pose_cw", "pose_wc", "scale_factors", "level_sigma_sq")
               else v) for f, v in nb[0].items()}
    with pytest.raises(_lib.B200Error) as e:
        mapping.create_new_landmarks_batch([(cur, [dup])], max_candidates=1)
    assert e.value.code == _lib.ERR_CAPACITY
    assert len(mapping.create_new_landmarks_batch([(cur, [dup])], max_candidates=256)[0]["rank"]) > 0
    bad = dict(cur, octave=cur["octave"].copy())
    bad["octave"][0] = 8
    for args in ([(bad, nb[0], np.array([[0, 0]]), 1.0)], [(cur, nb[0], np.array([[len(cur["x"]), 0]]), 1.0)]):
        with pytest.raises(_lib.B200Error) as e:
            mapping.triangulate_pairs_batch(args)
        assert e.value.code == _lib.ERR_INVALID
    eq, enb = synth.make_mapping_problem(51, 1, 300, model="equirectangular")
    eq = dict(eq, x_right=np.full(len(eq["x"]), -1, np.float32), depth=np.full(len(eq["x"]), -1, np.float32))
    eq["x_right"][4] = 10.0
    with pytest.raises(_lib.B200Error) as e:
        mapping.triangulate_pairs_batch([(eq, enb[0], np.array([[4, 0]]), 1.0)])
    assert e.value.code == _lib.ERR_INVALID
    with pytest.raises(_lib.B200Error) as e:
        mapping.create_new_landmarks_batch([(eq, enb)])
    assert e.value.code == _lib.ERR_INVALID
