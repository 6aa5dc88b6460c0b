"""GPU parity tests for the Hamming matchers (match/base.h, match/robust.cc:232-328) against the oracle."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mods():
    from oracle import pyoracle as O
    from stella_vslam_b200 import match
    from workloads import synth
    return O, match, synth


def test_hamming_kat(mods, golden_dir):
    # test/stella_vslam/match/base.cc:11-57
    O, match, synth = mods
    g = np.load(os.path.join(golden_dir, "hamming_kat.npz"))
    for a, b, d in zip(g["a"], g["b"], g["dist"]):
        assert match.compute_descriptor_distance_32(a, b) == d
        assert match.compute_descriptor_distance_64(a, b) == d


def test_hamming_matrix_vs_oracle(mods):
    O, match, synth = mods
    rng = np.random.default_rng(1)
    a = rng.integers(0, 256, (70, 32), dtype=np.uint8)
    b = rng.integers(0, 256, (133, 32), dtype=np.uint8)
    m = match.hamming_matrix(a, b)
    ref = np.unpackbits(a[:, None, :] ^ b[None, :, :], axis=2).sum(2)
    assert np.array_equal(m, ref)
    assert m[3, 7] == O.hamming_32(a[3], b[7])


@pytest.mark.parametrize("n1,n2,lowe,ori,seed", [(2000, 2000, 0.8, True, 7), (2000, 2000, 0.95, False, 8), (500, 1300, 0.7, True, 9),
                                                 (1, 1, 0.8, True, 10), (37, 5, 0.6, False, 11), (3000, 2500, 0.75, True, 12),
                                                 # both sides of resolve_kernel's two placement switches (4641 | 4642, 25206 | 25207,
                                                 # test_size_paths_gpu.bf_resolve_mode) and the 3840x1920 golden frame's 15 168
                                                 (4641, 4641, 0.8, True, 13), (4642, 4642, 0.8, True, 14), (15168, 15168, 0.8, True, 15),
                                                 (25206, 25206, 0.8, True, 16), (25207, 25207, 0.8, True, 17)])
def test_brute_force_vs_oracle(mods, n1, n2, lowe, ori, seed):
    O, match, synth = mods
    d1, a1, d2, a2, v2 = synth.make_descriptor_pair(n1, n2, seed=seed)
    m = match.robust(lowe, ori)
    got = m.brute_force_match(d1, a1, d2, a2, v2)
    ref = O.brute_force_match(d1, a1, d2, a2, v2, lowe, ori)
    assert np.array_equal(got, ref)
    if n1 >= 500:
        assert len(ref) > 50


def test_brute_force_collisions_force_exact_fallback(mods):
    # many keyframe keypoints compete for few frame keypoints: candidate lists get exhausted by "taken" entries
    O, match, synth = mods
    rng = np.random.default_rng(3)
    base = rng.integers(0, 256, (12, 32), dtype=np.uint8)
    d1 = np.repeat(base, 3, axis=0)                       # 36 frame descriptors, triplicates
    d1[1::3, 0] ^= 1
    d1[2::3, 1] ^= 3
    d2 = np.repeat(base, 40, axis=0)                      # 480 keyframe descriptors hitting the same 36
    flips = rng.integers(0, 256, (480,))
    for i, b in enumerate(flips):
        d2[i, b >> 3] ^= np.uint8(1 << (b & 7))
    a1 = np.zeros(36, np.float32)
    a2 = np.zeros(480, np.float32)
    for lowe in (0.6, 0.8, 1.0):
        got = match.robust(lowe, False).brute_force_match(d1, a1, d2, a2)
        ref = O.brute_force_match(d1, a1, d2, a2, None, lowe, False)
        assert np.array_equal(got, ref)


def test_identical_descriptors_tie_break(mods):
    # all distances tie: the reference's strict '<' keeps the first frame keypoint in index order
    O, match, synth = mods
    d1 = np.zeros((50, 32), np.uint8)
    d2 = np.zeros((20, 32), np.uint8)
    a = np.zeros(50, np.float32)
    got = match.robust(1.0, True).brute_force_match(d1, a, d2, a[:20])
    ref = O.brute_force_match(d1, a, d2, a[:20], None, 1.0, True)
    assert np.array_equal(got, ref)


def test_batch_and_empty_problems(mods):
    O, match, synth = mods
    probs = []
    for s, (n1, n2) in enumerate([(300, 400), (0, 10), (10, 0), (1200, 900)]):
        d1, a1, d2, a2, v2 = synth.make_descriptor_pair(max(n1, 1), max(n2, 1), seed=40 + s)
        probs.append((d1[:n1], a1[:n1], d2[:n2], a2[:n2], v2[:n2]))
    m = match.robust(0.8, True)
    got = m.brute_force_match_batch(probs)
    for g, (d1, a1, d2, a2, v2) in zip(got, probs):
        assert np.array_equal(g, O.brute_force_match(d1, a1, d2, a2, v2, 0.8, True))


def test_orientation_gate_boundaries(mods):
    O, match, synth = mods
    d = np.zeros((4, 32), np.uint8)
    a1 = np.array([0.0, 30.0, 30.000002, 359.0], np.float32)
    for q in (0.0, 329.0, 330.0, 180.0, 59.999996):
        a2 = np.array([q], np.float32)
        got = match.robust(1.0, True).brute_force_match(d, a1, d[:1], a2)
        ref = O.brute_force_match(d, a1, d[:1], a2, None, 1.0, True)
        assert np.array_equal(got, ref)


def test_device_path_with_bound_outputs(mods):
    """Extractor writing into torch-owned buffers + the device matcher on (offset, count) views == oracle."""
    import ctypes as C

    import torch

    O, match, synth = mods
    from stella_vslam_b200 import feature
    from stella_vslam_b200._lib import check, lib
    L = lib()
    B, w, h = 3, 640, 480
    frames = np.stack([synth.make_frame(w, h, seed=50, shift=(4 * i, 3 * i)) for i in range(B)])
    ex = feature.orb_extractor(feature.orb_params(), 800, max_batch=B)
    stride = L.b200_orb_max_keypoints(ex._h, w, h)
    dev = torch.device("cuda", 0)
    kps = torch.zeros((B, stride, 6), dtype=torch.float32, device=dev)
    desc = torch.zeros((B, stride, 32), dtype=torch.uint8, device=dev)
    counts = torch.zeros(B, dtype=torch.int32, device=dev)
    s = torch.cuda.current_stream().cuda_stream
    check(L.b200_orb_set_stream(ex._h, C.c_void_p(s), 0))
    check(L.b200_orb_bind_outputs(ex._h, C.c_void_p(kps.data_ptr()), C.c_void_p(desc.data_ptr()), C.c_void_p(counts.data_ptr()), stride))
    fd = torch.from_numpy(frames).to(dev)
    check(L.b200_orb_extract_device(ex._h, C.c_void_p(fd.data_ptr()), w, h, w, w * h, B, None, 0))
    hm = C.c_void_p()
    check(L.b200_matcher_create(0, C.byref(hm)))
    check(L.b200_matcher_set_stream(hm, C.c_void_p(s), 0))
    off = (torch.arange(B, dtype=torch.int32, device=dev) * stride).contiguous()
    pairs = torch.zeros((B - 1, stride, 2), dtype=torch.int32, device=dev)
    npairs = torch.zeros(B - 1, dtype=torch.int32, device=dev)
    ang = kps.data_ptr() + 12
    check(L.b200_match_bruteforce_device(hm, B - 1, C.c_void_p(desc.data_ptr()), C.c_void_p(ang), 24, C.c_void_p(off[1:].data_ptr()),
                                         C.c_void_p(counts[1:].data_ptr()), C.c_void_p(desc.data_ptr()), C.c_void_p(ang), 24, None,
                                         C.c_void_p(off.data_ptr()), C.c_void_p(counts.data_ptr()), stride, stride, 0.8, 1,
                                         C.c_void_p(pairs.data_ptr()), stride, C.c_void_p(npairs.data_ptr())))
    torch.cuda.synchronize()
    cn, kn, dn = counts.cpu().numpy(), kps.cpu().numpy(), desc.cpu().numpy()
    refs = [O.orb_extract(frames[f]) for f in range(B)]
    for f in range(B):
        assert cn[f] == len(refs[f]["kps"])
        assert np.array_equal(dn[f, :cn[f]], refs[f]["desc"])
        assert np.array_equal(kn[f, :cn[f], 3], refs[f]["kps"]["angle"])
    pn, nn = pairs.cpu().numpy(), npairs.cpu().numpy()
    for p in range(B - 1):
        a, b = refs[p + 1], refs[p]
        ref = O.brute_force_match(a["desc"], a["kps"]["angle"], b["desc"], b["kps"]["angle"], None, 0.8, True)
        assert np.array_equal(pn[p, :nn[p]], ref) and len(ref) > 20
    check(L.b200_matcher_destroy(hm))
