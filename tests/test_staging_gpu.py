"""One staging arena per handle serves every host-buffer entry point that runs on it.  On one matcher handle and on one local-BA
handle, calls of growing and then shrinking size, interleaved across those entry points, must give bit for bit what the same call
gives on a fresh handle.  The tracking chains also share the matcher's arena, and each keeps its own stage timer and parameter checks."""
import contextlib
import ctypes as C

import numpy as np
import pytest

from stella_vslam_b200 import _lib, feature, mapping, match, optimize, solve, tracking
from workloads import synth

pytestmark = pytest.mark.gpu

THR = 0.2 * np.pi / 180.0


def _same(a, b):
    if isinstance(a, dict):
        assert a.keys() == b.keys()
        for k in a:
            _same(a[k], b[k])
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            _same(x, y)
    elif isinstance(a, np.ndarray):
        assert a.dtype == b.dtype and np.array_equal(a, b)
    else:
        assert a == b or (a is None and b is None)


@contextlib.contextmanager
def _matcher_handle(h=None):
    """Routes the match and mapping wrappers to h, or to a fresh handle that is destroyed afterwards."""
    own = h is None
    if own:
        h = C.c_void_p()
        _lib.check(_lib.lib().b200_matcher_create(0, C.byref(h)))
    saved = getattr(match._tls, "matchers", None)
    match._tls.matchers = {0: h}
    try:
        yield h
    finally:
        match._tls.matchers = saved
        if own:
            _lib.lib().b200_matcher_destroy(h)


@contextlib.contextmanager
def _lba_handle(h=None):
    """Routes the solve wrappers to h, or to a fresh handle that is destroyed afterwards."""
    L = optimize._bind()
    own = h is None
    if own:
        h = C.c_void_p()
        _lib.check(L.b200_lba_create(0, C.byref(h)))
    saved = solve._HANDLES.get(0)
    solve._HANDLES[0] = h
    try:
        yield h
    finally:
        if saved is None:
            del solve._HANDLES[0]
        else:
            solve._HANDLES[0] = saved
        if own:
            L.b200_lba_destroy(h)


def _matcher_calls():
    d1, a1, d2, a2, v2 = synth.make_descriptor_pair(6000, 6000, seed=3)
    s1, sa1, s2, sa2, sv2 = synth.make_descriptor_pair(300, 200, seed=4)
    guided = [synth.make_guided_problem(21, mode=0), synth.make_guided_problem(22, n_train=300, n_queries=200, mode=1, stereo=True)]
    rng = np.random.default_rng(5)
    lm_descs = [rng.integers(0, 256, (int(k), 32), dtype=np.uint8) for k in rng.integers(1, 12, 40)]
    k1, k2, g = synth.make_keyframe_pair(11, n1=2000, n2=2000)
    pairs = [match._triangulation_problem(k1, k2, g["E_12"], g["epiplane_in_keyfrm_2"], True, THR, True)]
    cur, nb = synth.make_mapping_problem(11, 2, 1500)
    tri = [(cur, ngh, np.stack([rng.integers(0, len(cur["x"]), 2000), rng.integers(0, len(ngh["x"]), 2000)], 1).astype(np.int32), 1.0)
           for ngh in nb]
    large = [(d1, a1, d2, a2, v2), (d2[:4000], a2[:4000], d1[:5000], a1[:5000], v2[:5000])]
    return [
        lambda: match.robust(0.8, True).brute_force_match_batch(large),
        lambda: match.match_guided_batch(guided, 0, 100, 0.8, True),
        lambda: match.landmark_descriptors(lm_descs),
        lambda: match.match_pairs_batch(pairs, match.PAIRS_TRIANGULATION, 0.6, True),
        lambda: mapping.triangulate_pairs_batch(tri),
        lambda: match.robust(0.8, True).brute_force_match_batch([(s1, sa1, s2, sa2, sv2)]),
    ]


def test_matcher_arena_shared_across_entry_points():
    calls = _matcher_calls()
    want = []
    for call in calls:
        with _matcher_handle():
            want.append(call())
    with _matcher_handle() as h:
        for _ in range(2):  # the second pass starts from the arena the first one grew
            for call, w in zip(calls, want):
                with _matcher_handle(h):
                    _same(call(), w)
        for call, w in zip(reversed(calls), reversed(want)):
            with _matcher_handle(h):
                _same(call(), w)


def _lba_calls():
    L = optimize._bind()
    ba = synth.make_ba_problem(20, 5, 3000, seed=5, model="stereo")
    pnp = synth.make_pnp_problem(80, 300, 0.5, "perspective")
    graph = synth.make_pose_graph(300, seed=10)
    sim3 = [synth.make_sim3_pair(seed=s, n_matches=200) for s in range(4)]
    epnp = [dict(bearings=pnp["bearings"][pnp["gt_inlier"]], points=pnp["points"][pnp["gt_inlier"]])]

    def lba_solve():
        P, keep = optimize.pack_problem(ba)
        out = (np.zeros((P.n_poses, 4, 4)), np.zeros((P.n_points, 3)), np.zeros(P.n_edges, np.uint8))
        _lib.check(L.b200_lba_solve(solve._handle(0), C.byref(P), 5, 10, None, *[optimize.ptr(o) for o in out], None))
        return out

    def pnp_ransac():
        s = solve.pnp_solver(pnp["bearings"], pnp["octaves"], pnp["points"], pnp["scale_factors"], use_fixed_seed=True)
        s.find_via_ransac(30, True)
        return s.get_best_cam_pose(), s.get_inlier_flags()

    def graph_optimize():
        G, keep = optimize.pack_pose_graph(graph)
        st = optimize.PgoStats()
        _lib.check(L.b200_graph_optimize(solve._handle(0), C.byref(G), 50, 1e-3, C.byref(st)))
        return keep["estimate_out"], keep["pose_cw_out"], keep["points_out"], st.chi2_final, st.trials

    def transform_optimize():
        packed = [optimize.pack_transform_problem(pr, False) for pr in sim3]
        arr = (optimize.TransformProblem * len(packed))(*[pk[0] for pk in packed])
        _lib.check(L.b200_transform_optimize(solve._handle(0), len(packed), arr, 10.0, 10))
        return [optimize._transform_result(arr[i], pk[1]) for i, pk in enumerate(packed)]

    return [lba_solve, pnp_ransac, graph_optimize, transform_optimize, lambda: solve.compute_pose_batch(epnp)]


def test_lba_arena_shared_across_entry_points():
    calls = _lba_calls()
    want = []
    for call in calls:
        with _lba_handle():
            want.append(call())
    with _lba_handle() as h:
        for _ in range(2):
            for call, w in zip(calls, want):
                with _lba_handle(h):
                    _same(call(), w)
        for call, w in zip(reversed(calls), reversed(want)):
            with _lba_handle(h):
                _same(call(), w)


KITTI = dict(model="perspective", fx=718.856, fy=718.856, cx=607.1928, cy=185.2157, fxb=386.1448, cols=1241.0, rows=376.0, setup="stereo")


@pytest.fixture(scope="module")
def chains():
    """64 extracted KITTI-sized stereo frames with a local map, a last-frame table and a reference keyframe each, and the trackers."""
    ex = feature.orb_extractor(feature.orb_params(), 2000, max_batch=64)
    imgs = [synth.make_frame(1241, 376, seed=s) for s in range(200, 208)]
    kps, descs = ex.extract_batch(np.stack([imgs[i % 8] for i in range(64)]))
    sf = ex.orb_params_.scale_factors_
    local = [dict(synth.make_tracking_frame(kps[i], descs[i], KITTI, sf, seed=70 + i, stereo=True), frame=i) for i in range(64)]
    motion = [dict(synth.make_motion_frame(kps[i], descs[i], KITTI, sf, seed=170 + i, stereo=True), frame=i) for i in range(64)]
    robust = [dict(synth.make_robust_frame(kps[i], descs[i], KITTI, seed=300 + i, stereo=True), frame=i) for i in range(64)]
    return dict(ex=ex, local=local, motion=motion, robust=robust, lm=tracking.local_map_tracker(ex, KITTI),
                ft=tracking.frame_tracker(ex, KITTI, use_fixed_seed=True))


def _robust_frames(c, n):
    # a fresh engine per call: the draws depend only on the frame
    return [dict(fr, engine=solve.mt19937([i, 7])) for i, fr in enumerate(c["robust"][:n])]


def _chain_calls(c):
    calls = []
    for n in (1, 8, 64, 2):
        calls += [lambda n=n: c["lm"].track(c["local"][:n]), lambda n=n: c["ft"].motion_based_track(c["motion"][:n]),
                  lambda n=n: c["ft"].robust_match_based_track(_robust_frames(c, n))]
    return calls


def test_tracking_chains_share_the_matcher_arena(chains):
    calls = _chain_calls(chains)
    want = []
    for call in calls:
        with _matcher_handle():
            want.append(call())
    assert sum(r["tracked"] for r in want[-4]) >= 32  # the 64-frame robust call tracks
    with _matcher_handle() as h:
        for call, w in zip(calls, want):
            with _matcher_handle(h):
                _same(call(), w)
        for call, w in zip(reversed(calls), reversed(want)):
            with _matcher_handle(h):
                _same(call(), w)


def test_chain_stage_timers_are_separate(chains):
    c = chains
    lm, ft = c["lm"], c["ft"]
    runs = dict(local=lambda: lm.track(c["local"][:2]), motion=lambda: ft.motion_based_track(c["motion"][:2]),
                robust=lambda: ft.robust_match_based_track(_robust_frames(c, 2)))
    timers = dict(local=lm.stage_ms, motion=ft.stage_ms, robust=ft.robust_stage_ms)
    with _matcher_handle():
        started = set()
        for name in ("local", "motion", "robust"):
            for other in timers:
                if other not in started:  # a chain's timer is unset until its own first call
                    with pytest.raises(_lib.B200Error):
                        timers[other]()
            runs[name]()
            started.add(name)
        for name in runs:
            read = timers[name]()
            assert len(read) == 7
            for other in runs:
                if other != name:
                    runs[other]()
            assert timers[name]() == read, name


def test_chain_parameter_checks(chains):
    c = chains
    ex = c["ex"]
    with _matcher_handle():
        for grid in ((0, 48), (64, 0)):
            with pytest.raises(_lib.B200Error):
                tracking.local_map_tracker(ex, KITTI, grid=grid).track(c["local"][:1])
            with pytest.raises(_lib.B200Error):
                tracking.frame_tracker(ex, KITTI, grid=grid).motion_based_track(c["motion"][:1])
        # the robust chain runs no guided search: it reads neither the grid nor max_candidates
        free = tracking.frame_tracker(ex, KITTI, grid=(0, 0), max_candidates=-1, use_fixed_seed=True)
        _same(free.robust_match_based_track(_robust_frames(c, 2)), c["ft"].robust_match_based_track(_robust_frames(c, 2)))
        with pytest.raises(_lib.B200Error):
            tracking.frame_tracker(ex, KITTI, true_baseline=float("nan")).motion_based_track(c["motion"][:1])
        nan_ratio = tracking.frame_tracker(ex, KITTI, use_fixed_seed=True)
        nan_ratio._prm.lowe_ratio = float("nan")
        with pytest.raises(_lib.B200Error):
            nan_ratio.robust_match_based_track(_robust_frames(c, 1))
        _same(nan_ratio.motion_based_track(c["motion"][:2]), c["ft"].motion_based_track(c["motion"][:2]))  # the motion chain does not read it
