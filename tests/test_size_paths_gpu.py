"""The host picks a different code path, memory placement or launch shape from the problem size in several places; these tests run
both sides of each such switch against the oracle.  Every threshold is derived here from the formula the host uses (cited), so a
change of the formula shows up as a case that no longer straddles it.  Also: results must not depend on what earlier calls, on the
same handle or in the same process, left behind in scratch buffers or in the context's local memory."""
import ctypes as C

import numpy as np
import pytest

from oracle import pyoracle as O
from workloads import synth

pytestmark = pytest.mark.gpu


# ---- brute force: resolve_kernel's state placement ----------------------------------------------------------------------------

def bf_resolve_mode(max_n1):
    """Matcher::run (match_kernels.cu:1318-1320): 2 = state and frame descriptors in shared memory, 1 = state only, 0 = global scratch."""
    taken_words = -(-max_n1 // 32)
    state_bytes = 4 * (taken_words + 2 * max_n1)      # taken bitmap, idx_1 -> idx_2 table, claim table
    stage_bytes = 4 * 9 * max_n1                      # 8 descriptor words + 1 angle per frame keypoint
    if state_bytes + stage_bytes <= 200 * 1024:
        return 2
    return 1 if state_bytes <= 200 * 1024 else 0


def test_brute_force_thresholds_straddled():
    # the sizes test_match_gpu.py::test_brute_force_vs_oracle and the cases below use
    assert [bf_resolve_mode(n) for n in (4641, 4642, 25206, 25207)] == [2, 1, 1, 0]
    assert bf_resolve_mode(15168) == 1               # the 3840x1920 golden frame (BASELINE config 3)


def _collision_problem(n1, seed):
    """test_match_gpu.py::test_brute_force_collisions_force_exact_fallback's construction -- 480 keyframe keypoints compete for 36
    frame keypoints, so candidate lists are exhausted by taken entries and rows fall back to the exact scan -- with the 36 scattered
    among far-away random frame descriptors up to n1."""
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (12, 32), dtype=np.uint8)
    near = np.repeat(base, 3, axis=0)
    near[1::3, 0] ^= 1
    near[2::3, 1] ^= 3
    d2 = np.repeat(base, 40, axis=0)
    flips = rng.integers(0, 256, (480,))
    for i, b in enumerate(flips):
        d2[i, b >> 3] ^= np.uint8(1 << (b & 7))
    d1 = rng.integers(0, 256, (n1, 32), dtype=np.uint8)
    far = np.unpackbits(d1[:, None, :] ^ base[None, :, :], axis=2).sum(2).min(1) > 80
    assert far.all()                                   # random descriptors lie ~128 bits from the base: never a candidate
    d1[np.sort(rng.choice(n1, 36, replace=False))] = near
    return d1, np.zeros(n1, np.float32), d2, np.zeros(480, np.float32)


@pytest.mark.parametrize("n1", [4641, 15168, 25207])
def test_brute_force_exact_fallback_in_every_mode(n1):
    from stella_vslam_b200 import match
    d1, a1, d2, a2 = _collision_problem(n1, seed=n1)
    for lowe in (0.6, 1.0):
        got = match.robust(lowe, False).brute_force_match(d1, a1, d2, a2)
        ref = O.brute_force_match(d1, a1, d2, a2, None, lowe, False)
        assert np.array_equal(got, ref) and len(ref) > 0


def test_brute_force_batch_mode_follows_the_largest_problem():
    # the mode is chosen from max_n1 over the whole batch: one 25 207-keypoint frame puts every problem on the global-scratch path
    from stella_vslam_b200 import match
    probs = [synth.make_descriptor_pair(n1, n2, seed=60 + i) for i, (n1, n2) in enumerate([(300, 400), (25207, 2000), (1200, 900), (1, 1)])]
    d1, a1, d2, a2 = _collision_problem(600, seed=64)
    probs.append((d1, a1, d2, a2, None))
    assert bf_resolve_mode(max(len(p[0]) for p in probs)) == 0
    got = match.robust(0.8, True).brute_force_match_batch(probs)
    for g, (d1, a1, d2, a2, v2) in zip(got, probs):
        assert np.array_equal(g, O.brute_force_match(d1, a1, d2, a2, v2, 0.8, True))


def _upload_batch(probs):
    import torch
    dev = torch.device("cuda", 0)
    cnt1 = np.array([len(p[0]) for p in probs], np.int32)
    cnt2 = np.array([len(p[2]) for p in probs], np.int32)
    t = dict(d1=np.concatenate([p[0] for p in probs]), a1=np.concatenate([p[1] for p in probs]).astype(np.float32),
             d2=np.concatenate([p[2] for p in probs]), a2=np.concatenate([p[3] for p in probs]).astype(np.float32),
             off1=np.concatenate([[0], np.cumsum(cnt1)[:-1]]).astype(np.int32), cnt1=cnt1,
             off2=np.concatenate([[0], np.cumsum(cnt2)[:-1]]).astype(np.int32), cnt2=cnt2)
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in t.items()}
    n1, n2 = int(cnt1.max()), int(cnt2.max())
    t["pairs"] = torch.full((len(probs), n1, 2), -7, dtype=torch.int32, device=dev)
    t["n_pairs"] = torch.full((len(probs),), -7, dtype=torch.int32, device=dev)
    return t, n1, n2


def _bf_device(L, hm, t, n1, n2, lowe=0.8, ori=1):
    from stella_vslam_b200._lib import check
    p = lambda k: C.c_void_p(t[k].data_ptr())   # noqa: E731
    check(L.b200_match_bruteforce_device(hm, len(t["cnt1"]), p("d1"), p("a1"), 4, p("off1"), p("cnt1"), p("d2"), p("a2"), 4, None,
                                         p("off2"), p("cnt2"), n1, n2, lowe, ori, p("pairs"), n1, p("n_pairs")))


def _pairs_of(t):
    pn, nn = t["pairs"].cpu().numpy(), t["n_pairs"].cpu().numpy()
    return [pn[i, :nn[i]] for i in range(len(nn))]


@pytest.mark.parametrize("async_resolve", [1, 0])
def test_device_batches_back_to_back_and_scratch_reuse(async_resolve):
    """Two device-path batches of different sizes on one handle, the second growing its scratch while the first one's resolve may
    still run on the side stream, then join: both equal the oracle.  A small batch after the large one equals it on a fresh handle."""
    import torch
    from stella_vslam_b200._lib import check, lib
    L = lib()
    small = [synth.make_descriptor_pair(n1, n2, seed=70 + i) for i, (n1, n2) in enumerate([(3000, 2500), (500, 1300)])]
    large = [synth.make_descriptor_pair(n1, n2, seed=72 + i) for i, (n1, n2) in enumerate([(15168, 15168), (40, 3000)])]
    refs = [[O.brute_force_match(d1, a1, d2, a2, None, 0.8, True) for d1, a1, d2, a2, _ in b] for b in (small, large)]
    s = torch.cuda.current_stream().cuda_stream
    hms = []
    for _ in range(2):
        hm = C.c_void_p()
        check(L.b200_matcher_create(0, C.byref(hm)))
        check(L.b200_matcher_set_stream(hm, C.c_void_p(s), 0))
        check(L.b200_matcher_set_async_resolve(hm, async_resolve))
        hms.append(hm)
    try:
        hm, fresh = hms
        ta, na1, na2 = _upload_batch(small)
        tb, nb1, nb2 = _upload_batch(large)
        _bf_device(L, hm, ta, na1, na2)
        _bf_device(L, hm, tb, nb1, nb2)
        check(L.b200_matcher_join(hm))                # stream-ordered: the copies below run after both resolves
        for t, ref in ((ta, refs[0]), (tb, refs[1])):
            for g, r in zip(_pairs_of(t), ref):
                assert np.array_equal(g, r)
        tc, nc1, nc2 = _upload_batch(small)
        td, _, _ = _upload_batch(small)
        _bf_device(L, hm, tc, nc1, nc2)               # after the large batch: grown scratch with its contents
        _bf_device(L, fresh, td, nc1, nc2)
        check(L.b200_matcher_join(hm))
        check(L.b200_matcher_join(fresh))
        for g, f, r in zip(_pairs_of(tc), _pairs_of(td), refs[0]):
            assert np.array_equal(g, f) and np.array_equal(g, r)
    finally:
        for h in hms:
            check(L.b200_matcher_sync(h))
            check(L.b200_matcher_destroy(h))


# ---- guided_resolve_kernel's claim / state table: guided, all-pairs, track chain and new-landmark matchers -----------------------

def resolve_table_side(n):
    """rs_bytes = 6 * max(n, 1) + 16, computed by each caller of guided_resolve_kernel from its own largest keypoint count
    (match_kernels.cu:1627 b200_match_guided, :1853 b200_track_local_map, :2104 b200_match_pairs, :2739 b200_create_new_landmarks):
    default shared memory up to 48 KiB, opt-in above (:1712, :1987, :2154, :2898), B200_ERR_CAPACITY above 200 KiB."""
    rs = 6 * max(n, 1) + 16
    return "default" if rs <= 48 * 1024 else ("opt-in" if rs <= 200 * 1024 else "capacity")


def test_resolve_table_thresholds_straddled():
    assert [resolve_table_side(n) for n in (8189, 8190, 34130, 34131)] == ["default", "opt-in", "opt-in", "capacity"]


def _guided(n_train, seed):
    # a 3840x1920 frame keeps the keypoint density of the 640x480 default problem (2000 keypoints) at up to 34 130 keypoints
    return synth.make_guided_problem(seed, n_train=n_train, n_queries=3000, mode=0, width=3840, height=1920)


def _bow(n2, seed):
    k1, k2, _ = synth.make_keyframe_pair(seed, n1=2000, n2=n2)
    return dict(desc1=k1["desc"], angle1=k1["angle"], valid1=k1["has_landmark"], node1=k1["node"], desc2=k2["desc"], angle2=k2["angle"],
                node2=k2["node"], valid2=k2["has_landmark"])


@pytest.mark.parametrize("n", [8189, 8190, 34130])
def test_guided_resolve_table_sizes(n):
    from stella_vslam_b200 import match
    pr = _guided(n, seed=n)
    got, occ, cnt = match.match_guided_batch([pr], 0, 100, 0.8, True)[0]
    want, occ_want, n_want = O.match_guided(pr, 0, thr=100, lowe_ratio=0.8, check_orientation=True)
    assert np.array_equal(got, want) and cnt == n_want > 300
    assert np.array_equal(occ, occ_want)


@pytest.mark.parametrize("n", [8189, 8190, 34130])
def test_pairs_resolve_table_sizes(n):
    from stella_vslam_b200 import match
    pr = _bow(n, seed=n)
    got, cnt = match.match_pairs_batch([pr], match.PAIRS_BOW, 0.6, True)[0]
    want, n_want = O.match_pairs(pr, match.PAIRS_BOW, 0.6, True)
    assert np.array_equal(got, want) and cnt == n_want > 100


def test_resolve_table_capacity_leaves_outputs_untouched():
    from stella_vslam_b200 import match
    from stella_vslam_b200._lib import ERR_CAPACITY, GuidedProblem, PairsProblem, lib, pack_guided_problem, pack_pairs_problem
    hm = match._matcher(0)
    S, keep = pack_guided_problem(_guided(34131, seed=5))
    occ0 = keep["t_occupied"].copy()
    arr = (GuidedProblem * 1)(S)
    arr[0].n_matches = -5
    assert lib().b200_match_guided(hm, 1, arr, 0, 100, 0.8, 1, 0) == ERR_CAPACITY
    assert (keep["match_out"] == -2).all() and arr[0].n_matches == -5 and np.array_equal(keep["t_occupied"], occ0)
    S, keep = pack_pairs_problem(_bow(34131, seed=6))
    arr = (PairsProblem * 1)(S)
    arr[0].n_matches = -5
    assert lib().b200_match_pairs(hm, 1, arr, match.PAIRS_BOW, 0.6, 1, 0) == ERR_CAPACITY
    assert (keep["match_out"] == -2).all() and arr[0].n_matches == -5


EQUIRECT_3840 = dict(model="equirectangular", cols=3840.0, rows=1920.0, fxb=0.0, setup="monocular")   # BASELINE config 3's camera


def _extractor_holding(n, seed):
    """An extractor whose last results are one frame of `n` synthetic keypoints over a 3840x1920 image, in buffers bound with a
    keypoint stride of n: b200_track_local_map sizes its table from that stride (match_kernels.cu:1853, kc = stride).  A small
    frame is extracted into the bound buffers first (the chain needs the extractor to hold results), then overwritten."""
    import torch
    from stella_vslam_b200 import feature
    from stella_vslam_b200._lib import KP_DTYPE, check, lib
    L = lib()
    ex = feature.orb_extractor(feature.orb_params(), 800, max_batch=1)
    w, h = 320, 240
    assert L.b200_orb_max_keypoints(ex._h, w, h) <= n          # the bound stride must hold the small frame's keypoint bound
    dev = torch.device("cuda", 0)
    bufs = dict(kps=torch.zeros((1, n, 6), dtype=torch.float32, device=dev), desc=torch.zeros((1, n, 32), dtype=torch.uint8, device=dev),
                counts=torch.zeros(1, dtype=torch.int32, device=dev), img=torch.from_numpy(synth.make_frame(w, h, seed=seed)).to(dev))
    p = lambda k: C.c_void_p(bufs[k].data_ptr())   # noqa: E731
    check(L.b200_orb_set_stream(ex._h, C.c_void_p(torch.cuda.current_stream().cuda_stream), 0))
    check(L.b200_orb_bind_outputs(ex._h, p("kps"), p("desc"), p("counts"), n))
    check(L.b200_orb_extract_device(ex._h, p("img"), w, h, w, w * h, 1, None, 0))
    rng = np.random.default_rng(seed)
    sf = np.asarray(ex.orb_params_.scale_factors_, np.float32)
    kps = np.zeros(n, KP_DTYPE)
    kps["x"] = rng.uniform(0, 3840, n)
    kps["y"] = rng.uniform(0, 1920, n)
    kps["octave"] = rng.choice(8, n, p=np.array([.3, .22, .16, .12, .08, .06, .04, .02]))
    kps["size"] = 31.0 * sf[kps["octave"]]
    kps["angle"] = rng.uniform(0, 360, n)
    kps["response"] = rng.uniform(1, 100, n)
    desc = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    bufs["kps"][0] = torch.from_numpy(kps.view(np.float32).reshape(n, 6)).to(dev)
    bufs["desc"][0] = torch.from_numpy(desc).to(dev)
    bufs["counts"].fill_(n)
    torch.cuda.synchronize()
    ex._keep = bufs
    return ex, kps, desc


@pytest.mark.parametrize("n", [8189, 8190, 34130])
def test_track_chain_resolve_table_sizes(n):
    from stella_vslam_b200 import tracking
    ex, kps, desc = _extractor_holding(n, seed=n)
    prm = ex.orb_params_
    fr = dict(synth.make_tracking_frame(kps, desc, EQUIRECT_3840, prm.scale_factors_, seed=n + 1, pixel_sigma=0.7), frame=0)
    g = tracking.local_map_tracker(ex, EQUIRECT_3840).track([fr], kp_cap=n)[0]
    ref = O.track_local_map(EQUIRECT_3840, kps, desc, fr, prm.scale_factors_, prm.inv_level_sigma_sq_, prm.log_scale_factor_, monocular=True)
    assert g["n_keypoints"] == ref["n_keypoints"] == n
    assert np.array_equal(g["observable"], ref["observable"]) and np.array_equal(g["kp_landmark"], ref["kp_landmark"])
    assert g["n_matches"] == ref["n_matches"] > 0.3 * n and g["n_valid"] == ref["n_valid"]
    assert np.array_equal(g["kp_outlier"], ref["kp_outlier"])
    assert np.abs(g["pose_cw"] - ref["pose_cw"]).max() <= 1e-5 * max(1.0, np.abs(ref["pose_cw"]).max())   # test_track_gpu.py's tolerance


@pytest.mark.parametrize("n", [8189, 8190, 34130])
def test_new_landmarks_resolve_table_sizes(n):
    # the table covers the neighbour's keypoints (max_n2, match_kernels.cu:2739); BoW nodes keep the oracle's row scans short
    import mapping_oracle as MO
    from stella_vslam_b200 import mapping
    cur, nb = synth.make_mapping_problem(n, 1, n)
    assert len(nb[0]["x"]) == n
    got = mapping.create_new_landmarks_batch([(cur, nb)], bow=True, max_candidates=256, return_matches=True)[0]
    want = MO.create_new_landmarks(cur, nb, bow=True)
    assert np.array_equal(got["match_out"][0], want["match_out"][0])
    assert np.array_equal(got["n_matches"], want["n_matches"]) and want["n_matches"][0] > 0.1 * n
    assert np.array_equal(got["n_created"], want["n_created"])
    assert np.array_equal(got["rank"], want["rank"]) and np.array_equal(got["idx"], want["idx"])
    same = got["pos_w"] == want["pos_w"]                        # test_mapping_gpu.py's tolerance
    assert np.all(same | (np.abs(got["pos_w"] - want["pos_w"]) <= 1e-12 * np.maximum(np.abs(want["pos_w"]), 1.0)))


class _OutputsWatch:
    """Stands in for the library in stella_vslam_b200.mapping: fills every output of b200_create_new_landmarks with a byte pattern
    before the call and records whether the call changed any of it."""

    def __init__(self, real):
        self.real, self.touched = real, None

    def __getattr__(self, name):
        return getattr(self.real, name)

    def b200_create_new_landmarks(self, h, n_kf, probs, *rest):
        views = []
        for k in range(n_kf):
            P = probs[k]
            n1 = max(P.keyfrm.contents.n_keypoints, 1)
            for addr, nbytes in ((P.created_rank, 4 * n1), (P.created_idx, 8 * n1), (P.created_pos_w, 24 * n1)):
                views.append(np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(addr)))
            for r in range(P.n_neighbours):
                N = P.neighbours[r]
                views.append(np.ctypeslib.as_array((C.c_uint8 * (4 * n1)).from_address(N.match_out)))
                N.n_matches = N.n_created = -5
            P.n_created = -5
        for v in views:
            v[:] = 0xA5
        rc = self.real.b200_create_new_landmarks(h, n_kf, probs, *rest)
        self.touched = any((v != 0xA5).any() for v in views) or any(
            probs[k].n_created != -5 or any(probs[k].neighbours[r].n_matches != -5 or probs[k].neighbours[r].n_created != -5
                                            for r in range(probs[k].n_neighbours)) for k in range(n_kf))
        return rc


def test_track_chain_and_new_landmarks_capacity_leave_outputs_untouched(monkeypatch):
    from stella_vslam_b200 import mapping, tracking
    from stella_vslam_b200._lib import ERR_CAPACITY, B200Error, lib
    n = 34131
    ex, kps, desc = _extractor_holding(n, seed=7)
    tr = tracking.local_map_tracker(ex, EQUIRECT_3840)
    fr = dict(synth.make_tracking_frame(kps, desc, EQUIRECT_3840, ex.orb_params_.scale_factors_, seed=8), frame=0)
    arr, keep, outs = tr.pack([fr], n)
    o = outs[0]
    o["observable"][:], o["kp_landmark"][:], o["kp_outlier"][:] = 7, -5, 9
    arr[0].n_keypoints = arr[0].n_matches = -5
    with pytest.raises(B200Error) as e:
        tr.run_packed((arr, keep, outs))
    assert e.value.code == ERR_CAPACITY
    assert (o["observable"] == 7).all() and (o["kp_landmark"] == -5).all() and (o["kp_outlier"] == 9).all()
    assert arr[0].n_keypoints == arr[0].n_matches == -5 and not any(arr[0].pose_cw_out)
    cur, nb = synth.make_mapping_problem(9, 1, n)
    watch = _OutputsWatch(lib())
    monkeypatch.setattr(mapping, "lib", lambda: watch)
    with pytest.raises(B200Error) as e:
        mapping.create_new_landmarks_batch([(cur, nb)], bow=True, return_matches=True)
    assert e.value.code == ERR_CAPACITY and watch.touched is False


# ---- bundle adjustment: independence from earlier work ------------------------------------------------------------------------

def _same(a, b):
    assert a["iterations"] == b["iterations"] and a["chi2"] == b["chi2"]
    assert np.array_equal(a["pose_cw"], b["pose_cw"]) and np.array_equal(a["points"], b["points"])


def test_global_ba_independent_of_earlier_kernels_and_calls():
    """A map with more than 192 free keyframes (four landmark-mask words per landmark in the plan) solved on a fresh handle, again
    after the pose optimiser and the PnP kernels ran in this process (local memory belongs to the context and those kernels leave
    large non-zero stack frames in it), and again on a new handle: bit-identical, and equal to the oracle.  A small map solved
    on the grown handle equals it on a fresh one."""
    from stella_vslam_b200 import optimize, solve
    from test_global_ba import _check
    pr = synth.make_ba_problem(200, 1, 3000, seed=81, model="stereo")
    assert (pr["pose_fixed"] == 0).sum() > 192
    gba = optimize.global_bundle_adjuster(4)
    first = gba.optimize(pr)
    po = optimize.pose_optimizer()
    po.optimize_batch([synth.make_pose_problem(s, n_obs=1500, model=m) for s, m in enumerate(("stereo", "mono", "stereo", "mono"))])
    po.close()
    probs = []
    for seed in range(64):
        p = synth.make_pnp_problem(seed, 300, 0.5, "perspective")
        probs.append(dict(bearings=p["bearings"], points=p["points"], octaves=p["octaves"], scale_factors=p["scale_factors"], recompute=True,
                          min_num_inliers=10, gauss_newton_num_iter=10, min_sets=solve.draw_min_sets(300, 100, solve.mt19937((seed,)))))
    assert sum(r["valid"] for r in solve.pnp_ransac_batch(probs)) > 32
    again = gba.optimize(pr)
    other = optimize.global_bundle_adjuster(4)
    new = other.optimize(pr)
    _same(first, again)
    _same(first, new)
    _check(first, O.global_ba_solve(pr, 4), pr)
    sm = synth.make_ba_problem(20, 1, 800, seed=82, model="mono")
    _same(gba.optimize(sm), optimize.global_bundle_adjuster(4).optimize(sm))
    gba.close()
    other.close()


def test_local_ba_small_window_after_large_one():
    # the handle keeps the scratch a 166-free-keyframe window grew; a small window afterwards must not read what it left
    from stella_vslam_b200 import optimize
    big = synth.make_ba_problem(170, 4, 2000, seed=83, model="stereo")
    sm = synth.make_ba_problem(12, 3, 600, seed=84, model="mono")
    ba = optimize.local_bundle_adjuster()
    ba.optimize(big)
    got = ba.optimize(sm)
    fresh = optimize.local_bundle_adjuster().optimize(sm)
    assert got["iterations"] == fresh["iterations"] and np.array_equal(got["outliers"], fresh["outliers"])
    assert np.array_equal(got["pose_cw"], fresh["pose_cw"]) and np.array_equal(got["points"], fresh["points"])
    ba.close()
