"""Keyframe culling on the CPU: the C restatement (tests/cull_oracle.c), driven by the reference-side adapter's protocol, equals a literal
transcription of local_map_cleaner::remove_redundant_keyframes with in-place erasure (tests/cull_reference.py) on hand-built and random
maps; and the ctypes mirrors match include/b200vslam.h."""
import copy
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cull_oracle as CO  # noqa: E402
import cull_reference as CR  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = CR.named_cases()
FIELDS = ("skipped", "n_valid", "n_redundant", "removed")


def _agree(m, thr, top_n, call=CO.remove_redundant_keyframes):
    """Runs the transcription and the protocol around `call` on copies of m; asserts they agree and returns (transcribed map,
    protocol map, ranks, number of calls)."""
    want_map, got_map = copy.deepcopy(m), copy.deepcopy(m)
    n_want, want = CR.remove_redundant_keyframes(want_map, thr, top_n)
    n_got, got, calls = CR.remove_with_device_protocol(got_map, thr, top_n, call)
    assert n_got == n_want
    assert got == want
    assert [kf["will_be_erased"] for kf in got_map["keyframes"].values()] == [kf["will_be_erased"] for kf in want_map["keyframes"].values()]
    assert [lm["num_observations"] for lm in got_map["landmarks"]] == [lm["num_observations"] for lm in want_map["landmarks"]]
    assert [lm["will_be_erased"] for lm in got_map["landmarks"]] == [lm["will_be_erased"] for lm in want_map["landmarks"]]
    return want_map, got_map, want, calls


@pytest.mark.parametrize("name", sorted(CASES))
def test_named_case_matches_transcription(name):
    m, thr, top_n = CASES[name]
    _, _, ranks, calls = _agree(m, thr, top_n)
    assert calls == (2 if name == "unerasable" else 1)
    got = [tuple(r[f] for f in FIELDS) for r in ranks]
    expect = {
        "root": [(1, 0, 0, 0), (0, 10, 10, 1)],
        "recent": [(2, 0, 0, 0), (0, 10, 10, 1), (0, 10, 10, 1), (2, 0, 0, 0)],
        "recent_wrap": [(0, 10, 10, 1), (0, 10, 10, 1)],
        "num_observations_3_4": [(0, 10, 8, 1)],
        "depth": [(0, 7, 7, 1)],
        "no_valid": [(0, 0, 0, 0), (0, 0, 0, 0)],
        "ratio_9_10": [(0, 10, 9, 0)],
        "ratio_1": [(0, 10, 10, 1)],
        "cascade": [(0, 10, 10, 1), (0, 10, 0, 0)],
        "discard": [(0, 11, 10, 1), (0, 11, 10, 1), (0, 10, 10, 1)],
        "unerasable": [(0, 10, 10, 1), (0, 10, 10, 1), (0, 10, 10, 1)],
    }[name]
    assert got == expect


def test_discarded_landmark_and_cascade_state():
    m, thr, top_n = CASES["discard"]
    want_map, _, _, _ = _agree(m, thr, top_n)
    assert want_map["landmarks"][-11]["will_be_erased"] and not want_map["landmarks"][-11]["observations"]  # D: both observers erased
    m, thr, top_n = CASES["cascade"]
    alone = CO.remove_redundant_keyframes([CR.synth.gather_cull_problem(m, [81], thr)])[0]
    assert alone["removed"].tolist() == [1]  # rank 1 is redundant on the untouched map; only rank 0's erasure keeps it


def test_unerasable_needs_the_second_call():
    m, thr, _ = CASES["unerasable"]
    single = CO.remove_redundant_keyframes([CR.synth.gather_cull_problem(m, None, thr)])[0]
    assert single["removed"].tolist() == [1, 0, 1]  # the call assumed rank 0 was erased


def test_early_return():
    m, _, _ = CASES["ratio_1"]
    for thr, top_n in ((-0.1, 30), (0.9, 0)):
        assert CR.remove_redundant_keyframes(copy.deepcopy(m), thr, top_n) == (0, [])
        assert CR.remove_with_device_protocol(copy.deepcopy(m), thr, top_n, None) == (0, [], 0)


@pytest.mark.parametrize("seed", range(12))
def test_random_maps_match_transcription(seed):
    from workloads import synth
    rng = np.random.default_rng(seed)
    m = synth.make_cull_map(rng, n_covisibilities=int(rng.integers(1, 36)), n_keypoints=int(rng.integers(50, 400)),
                            observers=int(rng.integers(3, 11)), redundant_frac=float(rng.uniform(0.2, 0.8)),
                            stereo_frac=float(rng.uniform(0.0, 1.0)), cur_id=int(rng.integers(200, 1 << 32)) if seed % 3 else 500)
    thr = float(rng.choice([0.9, 0.9, 0.8, 0.95, 0.0, 1.0]))
    top_n = int(rng.choice([30, 30, 10, 60]))
    _agree(m, thr, top_n)


def test_random_maps_remove_and_cascade():
    """The workload exercises what it is built for: removed and kept ranks, and ranks decided differently than on the untouched map."""
    from workloads import synth
    removed = kept = cascades = 0
    for seed in range(8):
        m = synth.make_cull_map(np.random.default_rng(100 + seed), n_keypoints=300)
        res = CO.remove_redundant_keyframes([synth.gather_cull_problem(m)])[0]
        alone = CO.remove_redundant_keyframes([synth.gather_cull_problem(m, [k]) for k in m["covisibilities"]])
        removed += int(res["removed"].sum())
        kept += int(((res["removed"] == 0) & (res["skipped"] == 0)).sum())
        cascades += sum(int(a["removed"][0]) != int(res["removed"][r]) for r, a in enumerate(alone))
    assert removed > 0 and kept > 0 and cascades > 0


# ---- ctypes mirrors --------------------------------------------------------------------------------------------------------------------------
def test_ctypes_layout(tmp_path):
    from stella_vslam_b200 import mapping
    mirrors = {"b200_cull_keyframe_t": mapping.CullKeyframe, "b200_cull_problem_t": mapping.CullProblem}
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "b200vslam.h"', "int main(void) {"]
    for cname, T in mirrors.items():
        lines.append(f'  printf("{cname} __sizeof__ %zu\\n", sizeof({cname}));')
        for fname, _ in T._fields_:
            lines.append(f'  printf("{cname} {fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ["  return 0;", "}"]
    src, exe = tmp_path / "probe.c", tmp_path / "probe.exe"
    src.write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    want = {}
    for ln in subprocess.check_output([str(exe)], text=True).splitlines():
        parts = ln.split()
        want[(parts[0], parts[1])] = int(parts[2])
    for cname, T in mirrors.items():
        assert C.sizeof(T) == want[(cname, "__sizeof__")]
        for fname, _ in T._fields_:
            assert getattr(T, fname).offset == want[(cname, fname)], (cname, fname)
