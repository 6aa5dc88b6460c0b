#!/usr/bin/env python3
"""Small instances of every kernel family of libb200vslam.so, each checked against the oracle, meant to be run UNDER
compute-sanitizer:

    compute-sanitizer --tool memcheck  python tests/sanitize_cases.py
    compute-sanitizer --tool racecheck python tests/sanitize_cases.py
    compute-sanitizer --tool synccheck python tests/sanitize_cases.py

The full `pytest -m gpu` suite is 50-100x slower under the sanitizer than the GPU budget allows; these cases keep every kernel,
the claim tables of the resolve kernels, the last-CTA control kernels of the local BA and the cluster barrier of the Cholesky in
play at sizes that finish in minutes.  Select families with argv (orb match guided pairs stereo lba global_ba track pose); default = all."""
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import pyoracle as O  # noqa: E402
from stella_vslam_b200 import feature, match, optimize  # noqa: E402
from workloads import synth  # noqa: E402


def case_orb():
    img = synth.make_frame(320, 240, seed=3)
    ex = feature.orb_extractor(feature.orb_params(), 400, max_batch=2)
    kps, desc = ex.extract(img)
    ref = O.orb_extract(img, min_area=400)
    assert np.array_equal(kps, ref["kps"]) and np.array_equal(desc, ref["desc"]) and len(kps) > 50
    mask = np.full(img.shape, 255, np.uint8)
    mask[:60] = 0
    kb, db = ex.extract_batch(np.stack([img, img[::-1].copy()]), mask)
    ref = O.orb_extract(img, mask=mask, min_area=400)
    assert np.array_equal(kb[0], ref["kps"]) and np.array_equal(db[0], ref["desc"])
    return len(kps)


def case_match():
    total = 0
    # (15000, 64): resolve state in shared memory, descriptors from L2; (26000, 64): state in global scratch (Matcher::run)
    for n1, n2, seed in [(300, 280, 1), (129, 517, 2), (15000, 64, 4), (26000, 64, 5), (1, 1, 3)]:
        d1, a1, d2, a2, v2 = synth.make_descriptor_pair(n1, n2, seed=seed)
        m = match.robust(0.8, True)
        got = m.brute_force_match(d1, a1, d2, a2, v2)
        want = O.brute_force_match(d1, a1, d2, a2, v2, 0.8, True)
        assert np.array_equal(got, want), (n1, n2)
        total += len(got)
    D = match.hamming_matrix(d1, d2)
    assert D.shape == (len(d1), len(d2))
    return total


def case_guided():
    total = 0
    for mode in (0, 1, 3, 4):
        pr = synth.make_guided_problem(40 + mode, n_train=400, n_queries=300, mode=mode, stereo=bool(mode & 1))
        thr = 100 if mode < 2 else 50
        got, occ, n = match.match_guided_batch([pr], mode, thr, 0.8, True)[0]
        want, occ_want, n_want = O.match_guided(pr, mode, thr=thr, lowe_ratio=0.8, check_orientation=True)
        assert np.array_equal(got, want) and n == n_want, mode
        total += n
    pr = synth.make_guided_problem(9, n_train=64, n_queries=600, mode=0)        # contention: the claim table decides
    got, _, n = match.match_guided_batch([pr], 0, 100, 0.9, True)[0]
    want, _, n_want = O.match_guided(pr, 0, thr=100, lowe_ratio=0.9, check_orientation=True)
    assert np.array_equal(got, want)
    return total + n


def case_pairs():
    k1, k2, g = synth.make_keyframe_pair(11, n1=400, n2=380)
    thr = 0.2 * np.pi / 180.0
    total = 0
    for nodes in (False, True):
        pr = match._triangulation_problem(k1, k2, g["E_12"], g["epiplane_in_keyfrm_2"], True, thr, nodes)
        got, n = match.match_pairs_batch([pr], match.PAIRS_TRIANGULATION, 0.6, True)[0]
        want, n_want = O.match_pairs(pr, match.PAIRS_TRIANGULATION, 0.6, True)
        assert np.array_equal(got, want) and n == n_want
        total += n
    pr = dict(desc1=k1["desc"], angle1=k1["angle"], valid1=k1["has_landmark"], node1=k1["node"], desc2=k2["desc"], angle2=k2["angle"],
              node2=k2["node"], valid2=k2["has_landmark"])
    got, n = match.match_pairs_batch([pr], match.PAIRS_BOW, 0.75, True)[0]
    want, n_want = O.match_pairs(pr, match.PAIRS_BOW, 0.75, True)
    assert np.array_equal(got, want) and n == n_want
    return total + n


def case_stereo():
    left, right = synth.make_stereo_pair(320, 240, seed=21, disparities=(5, 17))
    fxb, bl = 435.2 * 0.11, 0.11
    a = O.orb_extract(left, min_area=400, want_pyramid=True)
    b = O.orb_extract(right, min_area=400, want_pyramid=True)
    xr_want, dep_want, n_want = O.stereo_compute(a["pyramid"], b["pyramid"], a["kps"], a["desc"], b["kps"], b["desc"], fxb, bl)
    ex = feature.orb_extractor(feature.orb_params(), 400, max_batch=2)
    kps, descs = ex.extract_batch(np.stack([left, right]))
    st = match.stereo(ex, ex, kps[0], kps[1], descs[0], descs[1], fxb, bl, frame_left=0, frame_right=1)
    xr, dep = st.compute()
    assert np.array_equal(xr, xr_want) and np.array_equal(dep, dep_want) and st.num_matched_ == n_want
    return n_want


def case_lba():
    specs = [("stereo", 6, 2, 120, 11), ("mono", 5, 2, 80, 12), ("equirect", 5, 1, 90, 13), ("stereo", 3, 3, 20, 16)]
    prs = [synth.make_ba_problem(K, F, L, seed=s, model=m) for m, K, F, L, s in specs]
    ba = optimize.local_bundle_adjuster(4, 3)
    got = ba.optimize_batch(prs)                                    # lockstep batch: cluster-per-window Cholesky, last-CTA tails
    for i, (g, pr) in enumerate(zip(got, prs)):
        ref = O.lba_solve(pr, iters1=4, iters2=3)
        assert np.array_equal(g["outliers"], ref["outliers"]), i
        assert np.abs(g["points"] - ref["points"]).max() <= 1e-5 * max(1.0, np.abs(ref["points"]).max()), i
        assert np.abs(g["pose_cw"] - ref["pose_cw"]).max() <= 1e-5 * max(1.0, np.abs(ref["pose_cw"]).max()), i
    one = ba.optimize(prs[0])                                       # batch of one: 8-CTA cluster
    assert np.array_equal(one["points"], got[0]["points"])
    return len(prs)


def case_global_ba():
    os.environ["B200_LBA_FORCE_OFFCHIP"] = "1"           # the panel-by-panel Cholesky of the global bundle adjuster on a small map
    try:
        pr = synth.make_ba_problem(8, 1, 150, seed=21, model="stereo")
        got = optimize.global_bundle_adjuster(4).optimize(pr)
        ref = O.global_ba_solve(pr, 4)
        assert got["iterations"] == ref["iterations"]
        assert np.abs(got["points"] - ref["points"]).max() <= 1e-5 * max(1.0, np.abs(ref["points"]).max())
    finally:
        os.environ.pop("B200_LBA_FORCE_OFFCHIP", None)
    return got["iterations"]


def case_track():
    from stella_vslam_b200 import tracking
    imgs = np.stack([synth.make_frame(320, 240, seed=3), synth.make_frame(320, 240, seed=4)])
    ex = feature.orb_extractor(feature.orb_params(), 400, max_batch=2)
    kps, descs = ex.extract_batch(imgs)
    cam = dict(model="perspective", fx=300.0, fy=300.0, cx=160.0, cy=120.0, fxb=30.0, cols=320.0, rows=240.0, setup="stereo")
    frames = [dict(synth.make_tracking_frame(kps[i], descs[i], cam, ex.orb_params_.scale_factors_, seed=9 + i, stereo=True), frame=i) for i in range(2)]
    got = tracking.local_map_tracker(ex, cam).track(frames)
    prm = ex.orb_params_
    for i, (fr, g) in enumerate(zip(frames, got)):
        ref = O.track_local_map(cam, kps[i], descs[i], fr, prm.scale_factors_, prm.inv_level_sigma_sq_, prm.log_scale_factor_, monocular=False)
        assert np.array_equal(g["kp_landmark"], ref["kp_landmark"]) and np.array_equal(g["kp_outlier"], ref["kp_outlier"]) and g["n_valid"] == ref["n_valid"]
    return sum(g["n_matches"] for g in got)


def case_pose():
    pp = synth.make_pose_problem(1, n_obs=200, model="stereo")
    n_valid, pose, flags = optimize.pose_optimizer().optimize(pp)
    n_ref, pose_ref, flags_ref = O.pose_optimize(pp)
    assert n_valid == n_ref and np.array_equal(flags, flags_ref) and np.allclose(pose, pose_ref, rtol=1e-5, atol=1e-7)
    return n_valid


CASES = dict(orb=case_orb, match=case_match, guided=case_guided, pairs=case_pairs, stereo=case_stereo, lba=case_lba, global_ba=case_global_ba,
             track=case_track, pose=case_pose)

if __name__ == "__main__":
    names = sys.argv[1:] or list(CASES)
    for nm in names:
        t0 = time.time()
        r = CASES[nm]()
        print(f"[sanitize_cases] {nm}: OK ({r}) in {time.time() - t0:.1f} s", flush=True)
    print("[sanitize_cases] all OK")
