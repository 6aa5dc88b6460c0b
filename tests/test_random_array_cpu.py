"""The minimal-set sampler of the RANSAC solvers on the CPU: std::mt19937 and util::create_random_array against libstdc++."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest


def test_engine_raw_stream_is_mt19937():
    from stella_vslam_b200 import solve
    e = solve.mt19937()
    mine = np.array([solve._L().b200_mt19937_next(C.byref(e)) for _ in range(2000)], np.uint64)
    bg = np.random.MT19937()
    bg._legacy_seeding(5489)
    np.testing.assert_array_equal(mine, bg.random_raw(2000))


_SAMPLER = r"""
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>
// util::create_random_array (src/stella_vslam/util/random_array.cc) restated with the standard library it relies on
static std::vector<unsigned> create_random_array(size_t size, unsigned lo, unsigned hi, std::mt19937& e) {
    std::uniform_int_distribution<unsigned> d(lo, hi);
    const auto make_size = static_cast<size_t>(size * 1.2);
    std::vector<unsigned> v;
    v.reserve(size);
    while (v.size() != size) {
        while (v.size() < make_size) v.push_back(d(e));
        std::sort(v.begin(), v.end());
        auto u = std::unique(v.begin(), v.end());
        if (size < static_cast<size_t>(std::distance(v.begin(), u))) u = std::next(v.begin(), size);
        v.erase(u, v.end());
    }
    std::shuffle(v.begin(), v.end(), e);
    return v;
}
int main(int argc, char** argv) {
    const unsigned size = atoi(argv[1]), n = atoi(argv[2]), iters = atoi(argv[3]), nseed = atoi(argv[4]);
    std::mt19937 e;
    if (nseed) {
        std::vector<std::uint_least32_t> w;
        for (unsigned k = 0; k < nseed; ++k) w.push_back((unsigned)strtoul(argv[5 + k], nullptr, 10));
        std::seed_seq s(w.begin(), w.end());
        e = std::mt19937(s);
    }
    for (unsigned it = 0; it < iters; ++it)
        for (unsigned x : create_random_array(size, 0u, n - 1, e)) printf("%u\n", x);
    printf("%u\n", (unsigned)e());
}
"""


@pytest.fixture(scope="module")
def sampler_exe():
    d = tempfile.mkdtemp(prefix="b200_sampler_")
    src, exe = os.path.join(d, "s.cc"), os.path.join(d, "s")
    with open(src, "w") as f:
        f.write(_SAMPLER)
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O1", "-std=c++17", "-o", exe, src])
    return exe


# n: each set size's smallest two counts (4, 5 / 5, 6 / 8, 9) and larger ones up to 123457, under PnP's (4), the essential solver's
# (5) and the two-view solvers' (4, 8) set sizes; set sizes above n are not drawn
@pytest.mark.parametrize("seed", [None, (1, 2, 3), (7, 0xFFFFFFFF, 12345, 99, 5, 6, 7, 8, 9, 10), tuple(range(10, 20)), (4294967295, 0, 17)])
@pytest.mark.parametrize("n", [4, 5, 6, 7, 8, 9, 10, 37, 50, 300, 1000, 1500, 123457])
def test_draw_min_sets_matches_libstdcxx(sampler_exe, n, seed):
    from stella_vslam_b200 import solve
    L = solve._L()
    words = [] if seed is None else list(seed)
    for set_size in [k for k in (4, 5, 8) if k <= n]:
        iters = 40 if n <= set_size + 1 else 300
        out = subprocess.check_output([sampler_exe, str(set_size), str(n), str(iters), str(len(words))] + [str(w) for w in words])
        ref = np.array(out.split(), np.uint64)
        e = solve.mt19937(words or None)
        got = solve.draw_min_sets(n, iters, e, set_size=set_size)
        assert got.shape == (iters, set_size)
        np.testing.assert_array_equal(got.reshape(-1).astype(np.uint64), ref[:-1])
        if set_size == 4:  # PnP's entry point draws the same sets and leaves the engine in the same state
            e4 = solve.mt19937(words or None)
            pnp = np.zeros((iters, 4), np.int32)
            assert L.b200_pnp_draw_min_sets(C.byref(e4), C.c_uint32(n), C.c_uint32(iters), pnp.ctypes.data_as(C.POINTER(C.c_int32))) == 0
            np.testing.assert_array_equal(pnp, got)
            assert bytes(e4) == bytes(e)
        assert L.b200_mt19937_next(e) == int(ref[-1])  # the engine continues where the reference's does


def test_min_sets_distinct_and_continuing():
    from stella_vslam_b200 import solve
    e = solve.mt19937((7, 8))
    a, b = solve.draw_min_sets(9, 10, e), solve.draw_min_sets(9, 20, e)
    whole = solve.draw_min_sets(9, 30, solve.mt19937((7, 8)))
    np.testing.assert_array_equal(np.concatenate([a, b]), whole)
    assert all(len(set(r)) == 4 and r.min() >= 0 and r.max() < 9 for r in whole)
    with pytest.raises(Exception):
        solve.draw_min_sets(3, 1)


def test_draw_min_sets_rejects_too_few_matches():
    from stella_vslam_b200 import solve
    from stella_vslam_b200._lib import B200Error
    with pytest.raises(B200Error):
        solve.draw_min_sets(4, 3, solve.mt19937(), set_size=5)
