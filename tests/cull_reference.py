"""Literal Python transcription of keyframe culling on object-graph maps (workloads.synth.make_cull_map): local_map_cleaner::
remove_redundant_keyframes and count_redundant_observations (module/local_map_cleaner.cc:68-193), keyframe::prepare_for_erasing
(data/keyframe.cc:613-660) and landmark::erase_observation (data/landmark.cc:124-160), erasing in place.  The descriptor / geometry
refresh and the covisibility-graph repair decide nothing here and are left out.

  remove_redundant_keyframes(m, thr, top_n)          the reference loop; returns (num_removed, per-rank dicts)
  remove_with_device_protocol(m, thr, top_n, call)   the reference-side adapter's protocol around a flat-table call (the C oracle or
                                                     the device): gather, call, apply prepare_for_erasing in rank order, and gather
                                                     and call again after a removed keyframe that could not be erased
"""
import numpy as np

from workloads import synth

NUM_BETTER_OBS_THR = 3
WINDOW_SIZE_NOT_TO_REMOVE = 2
U32 = 0xFFFFFFFF


def erase_observation(m, lm, kf):
    idx = lm["observations"][kf["id"]]
    if kf["x_right"] is not None and 0 <= kf["x_right"][idx]:
        lm["num_observations"] -= 2
    else:
        lm["num_observations"] -= 1
    del lm["observations"][kf["id"]]
    if not lm["observations"]:
        lm["will_be_erased"] = True  # landmark::prepare_for_erasing: no observer is left to detach


def prepare_for_erasing(m, kf):
    if kf["is_root"] or kf["cannot_be_erased"]:
        return
    kf["will_be_erased"] = True
    for li in kf["landmarks"]:
        if li < 0:
            continue
        lm = m["landmarks"][li]
        if lm["will_be_erased"]:
            continue
        erase_observation(m, lm, kf)


def count_redundant_observations(m, kf):
    num_valid_obs = num_redundant_obs = 0
    for idx, li in enumerate(kf["landmarks"]):
        if li < 0:
            continue
        lm = m["landmarks"][li]
        if lm["will_be_erased"]:
            continue
        if kf["depth"] is not None:
            depth = float(kf["depth"][idx])
            if depth < 0.0 or kf["depth_thr"] < depth:
                continue
        num_valid_obs += 1
        if lm["num_observations"] <= NUM_BETTER_OBS_THR:
            continue
        scale_level = int(kf["octave"][idx])
        obs_by_keyfrm_is_redundant = False
        num_better_obs = 0
        for ngh_id, ngh_idx in lm["observations"].items():
            if ngh_id == kf["id"]:
                continue
            ngh_scale_level = int(m["keyframes"][ngh_id]["octave"][ngh_idx])
            if ngh_scale_level <= scale_level + 1:
                num_better_obs += 1
                if NUM_BETTER_OBS_THR <= num_better_obs:
                    obs_by_keyfrm_is_redundant = True
                    break
        if obs_by_keyfrm_is_redundant:
            num_redundant_obs += 1
    return num_valid_obs, num_redundant_obs


def _ratio(num_redundant_obs, num_valid_obs):
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(np.float32(num_redundant_obs) / np.float32(num_valid_obs))


def remove_redundant_keyframes(m, redundant_obs_ratio_thr=0.9, top_n=30):
    if redundant_obs_ratio_thr < 0.0 or top_n <= 0:
        return 0, []
    num_removed = 0
    ranks = []
    cur_id = m["cur_id"]
    for kid in m["covisibilities"][:top_n]:
        kf = m["keyframes"][kid]
        rec = dict(id=kid, skipped=0, n_valid=0, n_redundant=0, removed=0)
        ranks.append(rec)
        if kf["is_root"]:
            rec["skipped"] = 1
            continue
        if kid <= cur_id and cur_id <= (kid + WINDOW_SIZE_NOT_TO_REMOVE) & U32:
            rec["skipped"] = 2
            continue
        rec["n_valid"], rec["n_redundant"] = count_redundant_observations(m, kf)
        if redundant_obs_ratio_thr <= _ratio(rec["n_redundant"], rec["n_valid"]):
            num_removed += 1
            rec["removed"] = 1
            prepare_for_erasing(m, kf)
    return num_removed, ranks


def remove_with_device_protocol(m, redundant_obs_ratio_thr, top_n, call):
    """call(list of flat problems) -> list of result dicts (mapping.remove_redundant_keyframes or cull_oracle's).  Returns
    (num_removed, per-rank dicts of the call that decided each rank, number of calls)."""
    if redundant_obs_ratio_thr < 0.0 or top_n <= 0:
        return 0, [], 0
    covs = m["covisibilities"][:top_n]
    start, num_removed, ranks, calls = 0, 0, [], 0
    while start < len(covs):
        res = call([synth.gather_cull_problem(m, covs[start:], redundant_obs_ratio_thr)])[0]
        calls += 1
        restart = None
        for r in range(len(covs) - start):
            ranks.append(dict(id=covs[start + r], **{f: int(res[f][r]) for f in ("skipped", "n_valid", "n_redundant", "removed")}))
            if not res["removed"][r]:
                continue
            num_removed += 1
            kf = m["keyframes"][covs[start + r]]
            prepare_for_erasing(m, kf)
            if not kf["will_be_erased"]:  # pinned: the call's later ranks assumed it was erased
                restart = start + r + 1
                break
        if restart is None:
            break
        start = restart
    return num_removed, ranks, calls


# ---- hand-built maps -------------------------------------------------------------------------------------------------------------------------
def make_map(cur_id, keyframes, landmarks, covisibilities):
    """An object-graph map in make_cull_map's shape from specs.  keyframes: dicts of id, n (keypoints), octave (scalar or list), and
    optionally x_right / depth (lists), depth_thr, is_root, cannot_be_erased.  landmarks: lists of (keyframe id, keypoint index)."""
    kfs = {}
    for s in keyframes:
        n = s["n"]
        kfs[s["id"]] = dict(id=s["id"], is_root=bool(s.get("is_root", False)), octave=np.broadcast_to(np.asarray(s.get("octave", 0), np.int32), (n,)).copy(),
                            x_right=None if s.get("x_right") is None else np.asarray(s["x_right"], np.float32),
                            depth=None if s.get("depth") is None else np.asarray(s["depth"], np.float32), depth_thr=float(s.get("depth_thr", 5.0)),
                            landmarks=np.full(n, -1, np.int64), will_be_erased=False, cannot_be_erased=bool(s.get("cannot_be_erased", False)))
    lms = []
    for li, obs in enumerate(landmarks):
        num = 0
        for kid, idx in obs:
            kf = kfs[kid]
            assert kf["landmarks"][idx] < 0
            kf["landmarks"][idx] = li
            num += 2 if kf["x_right"] is not None and 0 <= kf["x_right"][idx] else 1
        lms.append(dict(observations={kid: idx for kid, idx in obs}, num_observations=num, will_be_erased=False))
    return dict(cur_id=cur_id, keyframes=kfs, landmarks=lms, covisibilities=list(covisibilities))


OTHERS = (10, 11, 12, 13)  # observers outside the covisibility list


def _others(n=10, octave=0):
    return [dict(id=o, n=4 * n, octave=octave) for o in OTHERS]


class _slots:
    """Next free keypoint index of each keyframe."""

    def __init__(self):
        self.next = {}

    def __call__(self, kid):
        i = self.next.get(kid, 0)
        self.next[kid] = i + 1
        return (kid, i)


def _redundant_rows(slot, kid, n, n_others=3):
    """n landmarks each seen by `kid` and by n_others of OTHERS at octave 0: redundant for `kid` at octave >= 0."""
    return [[slot(kid)] + [slot(o) for o in OTHERS[:n_others]] for _ in range(n)]


def named_cases():
    """name -> (map, redundant_obs_ratio_thr, top_n)."""
    cases = {}
    # the spanning root is never removed, even when redundant
    s = _slots()
    cases["root"] = (make_map(100, [dict(id=1, n=10, is_root=True), dict(id=50, n=10)] + _others(),
                              _redundant_rows(s, 1, 10) + _redundant_rows(s, 50, 10), [1, 50]), 0.9, 30)
    # the recent window: cur - 2 is skipped, cur - 3 and ids above cur are not
    s = _slots()
    cases["recent"] = (make_map(100, [dict(id=k, n=10) for k in (98, 97, 101, 99)] + _others(n=40),
                                sum((_redundant_rows(s, k, 10) for k in (98, 97, 101, 99)), []), [98, 97, 101, 99]), 0.9, 30)
    # unsigned arithmetic: id + 2 wraps, so cur = 2^32 - 1 does not protect id = 2^32 - 2
    s = _slots()
    cases["recent_wrap"] = (make_map(U32, [dict(id=U32 - 1, n=10), dict(id=U32 - 3, n=10)] + _others(n=20),
                                     _redundant_rows(s, U32 - 1, 10) + _redundant_rows(s, U32 - 3, 10), [U32 - 1, U32 - 3]), 0.9, 30)
    # num_observations exactly 3 and exactly 4, the stereo weight making up the count: keypoint 0 mono + stereo observer (3),
    # keypoint 1 stereo + stereo observer (4, one other observer), keypoints 2..9 mono with three mono observers (4)
    s = _slots()
    st = dict(id=20, n=10, x_right=[5.0] * 10)
    rows = [[s(60), s(20)], [s(60), s(20)]] + _redundant_rows(s, 60, 8)
    cases["num_observations_3_4"] = (make_map(100, [dict(id=60, n=10, x_right=[-1.0, 3.0] + [-1.0] * 8), st] + _others(), rows, [60]), 0.5, 30)
    # depths: below 0 and above depth_thr are not valid, exactly depth_thr is
    s = _slots()
    d = [-0.5, 5.0, 5.0 * 1.0000001, 5.5, 1.0, 2.0, 3.0, 4.0, 5.0, 0.0]
    cases["depth"] = (make_map(100, [dict(id=70, n=10, x_right=[-1.0] * 10, depth=d, depth_thr=5.0)] + _others(), _redundant_rows(s, 70, 10), [70]), 0.9, 30)
    # n_valid = 0: 0 / 0 is NaN and removes nothing, even at a threshold of 0
    s = _slots()
    cases["no_valid"] = (make_map(100, [dict(id=71, n=4, x_right=[-1.0] * 4, depth=[-1.0] * 4), dict(id=72, n=4)] + _others(),
                                  _redundant_rows(s, 71, 4), [71, 72]), 0.0, 30)
    # 9 redundant of 10: 0.9f < 0.9, kept; 10 of 10 removed
    s = _slots()
    cases["ratio_9_10"] = (make_map(100, [dict(id=73, n=10)] + _others(), _redundant_rows(s, 73, 9) + [[s(73), s(10)]], [73]), 0.9, 30)
    s = _slots()
    cases["ratio_1"] = (make_map(100, [dict(id=74, n=10)] + _others(), _redundant_rows(s, 74, 10), [74]), 0.9, 30)
    # a cascade: rank 0 and rank 1 share landmarks seen by two others; erasing rank 0 leaves rank 1's landmarks 3 observations
    s = _slots()
    casc_kfs = [dict(id=80, n=10), dict(id=81, n=10)] + _others()
    casc_rows = [[s(80), s(81), s(10), s(11)] for _ in range(10)]
    cases["cascade"] = (make_map(100, casc_kfs, casc_rows, [80, 81]), 0.9, 30)
    # a landmark discarded when its last observer is erased: D is seen by ranks 0 and 1 only, and both are removed
    s = _slots()
    rows = _redundant_rows(s, 82, 10) + _redundant_rows(s, 83, 10) + [[s(82), s(83)]]
    cases["discard"] = (make_map(100, [dict(id=82, n=11), dict(id=83, n=11), dict(id=84, n=10)] + _others(n=30), rows + _redundant_rows(s, 84, 10),
                                 [82, 83, 84]), 0.9, 30)
    # the cascade with rank 0 pinned (set_not_to_be_erased): the reference counts it removed but does not erase it, so rank 1 stays
    # redundant; a single call that assumed the erasure would keep rank 1
    s = _slots()
    kfs = [dict(casc_kfs[0], cannot_be_erased=True)] + casc_kfs[1:]
    rows = [[s(80), s(81), s(10), s(11)] for _ in range(10)] + _redundant_rows(s, 85, 10)
    cases["unerasable"] = (make_map(100, kfs + [dict(id=85, n=10)], rows, [80, 81, 85]), 0.9, 30)
    return cases
