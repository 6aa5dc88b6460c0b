"""GPU parity of keyframe culling (b200_remove_redundant_keyframes) with the C restatement (tests/cull_oracle.c) and, through the
reference-side adapter's protocol, with the transcription of local_map_cleaner::remove_redundant_keyframes (tests/cull_reference.py):
the named cases, a mixed batch of 64 maps against the oracle and against each map run alone, a 30 x 4 000-keypoint map, and the
rejection of inconsistent tables with the outputs untouched."""
import copy
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cull_oracle as CO  # noqa: E402
import cull_reference as CR  # noqa: E402

pytestmark = pytest.mark.gpu
FIELDS = ("skipped", "n_valid", "n_redundant", "removed")


@pytest.fixture(scope="module")
def mods():
    from stella_vslam_b200 import _lib, mapping
    from workloads import synth
    return _lib, mapping, synth


def _same(got, want):
    assert got["n_removed"] == want["n_removed"] and got["status"] == 0
    for f in FIELDS:
        assert got[f].tolist() == want[f].tolist(), f


@pytest.mark.parametrize("name", sorted(CR.named_cases()))
def test_named_case(mods, name):
    _, mapping, synth = mods
    m, thr, top_n = CR.named_cases()[name]
    prob = synth.gather_cull_problem(m, None, thr)
    _same(mapping.remove_redundant_keyframes([prob])[0], CO.remove_redundant_keyframes([prob])[0])
    want_map, got_map = copy.deepcopy(m), copy.deepcopy(m)
    n_want, want = CR.remove_redundant_keyframes(want_map, thr, top_n)
    n_got, got, calls = CR.remove_with_device_protocol(got_map, thr, top_n, mapping.remove_redundant_keyframes)
    assert (n_got, got) == (n_want, want)
    assert calls == (2 if name == "unerasable" else 1)
    assert [lm["num_observations"] for lm in got_map["landmarks"]] == [lm["num_observations"] for lm in want_map["landmarks"]]


def _mixed_batch(synth, n=64, seed=7):
    rng = np.random.default_rng(seed)
    probs = []
    for k in range(n):
        m = synth.make_cull_map(rng, n_covisibilities=int(rng.integers(0, 40)), n_keypoints=int(rng.integers(1, 2500)),
                                observers=int(rng.integers(2, 12)), redundant_frac=float(rng.uniform(0.0, 1.0)),
                                stereo_frac=float(rng.uniform(0.0, 1.0)), erased_frac=float(rng.uniform(0.0, 0.1)),
                                cur_id=int(rng.integers(300, 1 << 32)))
        probs.append(synth.gather_cull_problem(m, None, float(rng.choice([0.9, 0.9, 0.8, 0.95, 0.0, 1.0]))))
    return probs


def test_mixed_batch_of_64_maps(mods):
    _, mapping, synth = mods
    probs = _mixed_batch(synth)
    got = mapping.remove_redundant_keyframes(probs)
    want = CO.remove_redundant_keyframes(probs)
    for g, w in zip(got, want):
        _same(g, w)
    assert sum(w["n_removed"] for w in want) > 0
    for k in range(0, 64, 7):  # each problem alone equals its result inside the batch
        _same(mapping.remove_redundant_keyframes([probs[k]])[0], got[k])


def test_large_map(mods):
    _, mapping, synth = mods
    prob = synth.gather_cull_problem(synth.make_cull_map(np.random.default_rng(11), n_covisibilities=30, n_keypoints=4000, stereo_frac=0.5))
    got, want = mapping.remove_redundant_keyframes([prob])[0], CO.remove_redundant_keyframes([prob])[0]
    _same(got, want)
    assert want["n_removed"] > 0


def _corruptions(p):
    """(name, problem) pairs each breaking one rule of the input check."""
    def cp():
        q = dict(p, covisibilities=[dict(c) for c in p["covisibilities"]])
        for f in ("obs_offsets", "obs_rank", "obs_octave", "obs_weight"):
            q[f] = np.array(p[f])
        for c in q["covisibilities"]:
            c["kp_landmark"] = np.array(c["kp_landmark"])
        return q
    listed = [(r, i) for r, c in enumerate(p["covisibilities"]) for i in np.flatnonzero(c["kp_landmark"] >= 0)]
    r0, i0 = listed[0]
    out = []
    q = cp(); q["obs_rank"][0] = len(p["covisibilities"]); out.append(("rank out of range", q))
    q = cp(); q["obs_rank"][0] = -2; out.append(("rank below -1", q))
    q = cp(); q["obs_weight"][0] = 3; out.append(("weight", q))
    q = cp(); q["covisibilities"][r0]["kp_landmark"][i0] = len(p["obs_offsets"]) - 1; out.append(("landmark out of range", q))
    q = cp(); q["covisibilities"][r0]["kp_landmark"][i0] = -1; out.append(("listed landmark missing", q))
    q = cp(); q["obs_offsets"][1:] = q["obs_offsets"][1:][::-1]; out.append(("descending offsets", q))
    # an observation by a rank whose keypoints do not list that landmark
    q = cp(); q["obs_rank"][np.flatnonzero(q["obs_rank"] == -1)[0]] = r0; out.append(("unlisted observation", q))
    # two keypoints of one rank listing the same landmark
    q = cp(); kl = q["covisibilities"][r0]["kp_landmark"]; free = np.flatnonzero(kl < 0); kl[free[0]] = kl[i0]; out.append(("listed twice", q))
    return out


def test_inconsistent_tables_are_rejected_untouched(mods):
    _lib, mapping, synth = mods
    good = synth.gather_cull_problem(synth.make_cull_map(np.random.default_rng(3), n_covisibilities=6, n_keypoints=200))
    for name, bad in _corruptions(good):
        probs = [good, bad]
        arr, _keep = mapping.pack_cull_problems(probs)
        for k in range(2):
            arr[k].n_removed, arr[k].status = -7, -7
            for r in range(arr[k].n_covisibilities):
                K = arr[k].covisibilities[r]
                K.n_valid = K.n_redundant = K.skipped = K.removed = -7
        mapping._setup()
        rc = _lib.lib().b200_remove_redundant_keyframes(mapping._matcher(0), 2, arr)
        assert rc == _lib.ERR_INVALID, name
        for k in range(2):
            assert (arr[k].n_removed, arr[k].status) == (-7, -7), name
            for r in range(arr[k].n_covisibilities):
                K = arr[k].covisibilities[r]
                assert (K.n_valid, K.n_redundant, K.skipped, K.removed) == (-7, -7, -7, -7), name
    _same(mapping.remove_redundant_keyframes([good])[0], CO.remove_redundant_keyframes([good])[0])  # the handle still works


def test_empty_calls(mods):
    _, mapping, _ = mods
    assert mapping.remove_redundant_keyframes([]) == []
    empty = dict(cur_id=5, redundant_obs_ratio_thr=0.9, covisibilities=[], obs_offsets=[0], obs_rank=[], obs_octave=[], obs_weight=[])
    _same(mapping.remove_redundant_keyframes([empty])[0], dict(n_removed=0, **{f: np.zeros(0) for f in FIELDS}))
