// random_array.cu -- the minimal-set sampler of the RANSAC solvers, on the host: std::mt19937 and util::create_random_array
// (src/stella_vslam/util/random_array.cc) as libstdc++ evaluates them.  The solvers draw their minimal sets here, in draw order, and
// pass them to b200_pnp_ransac, b200_essential_ransac and b200_twoview_ransac.
#include <cstdint>
#include <vector>

#include "common.cuh"

namespace b200 {
namespace {

void mt_twist(b200_mt19937_t* e) {
    uint32_t* x = e->state;
    for (int k = 0; k < 624; ++k) {
        const uint32_t y = (x[k] & 0x80000000u) | (x[(k + 1) % 624] & 0x7fffffffu);
        x[k] = x[(k + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    }
    e->index = 0;
}

uint32_t mt_next(b200_mt19937_t* e) {
    if (e->index >= 624) mt_twist(e);
    uint32_t y = e->state[e->index++];
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= y >> 18;
    return y;
}

// uniform_int_distribution{0, range - 1} on a 32-bit engine: Lemire's nearly divisionless method (libstdc++ _S_nd)
uint32_t uniform_below(b200_mt19937_t* e, uint32_t range) {
    uint64_t product = (uint64_t)mt_next(e) * range;
    uint32_t low = (uint32_t)product;
    if (low < range) {
        const uint32_t threshold = (uint32_t)(0u - range) % range;
        while (low < threshold) {
            product = (uint64_t)mt_next(e) * range;
            low = (uint32_t)product;
        }
    }
    return (uint32_t)(product >> 32);
}

// util::create_random_array(set_size, 0, n - 1, engine): make_size = size_t(set_size * 1.2) draws of uniform_int_distribution<unsigned>,
// sort + unique (truncated to set_size), repeated until set_size remain, then std::shuffle.
void create_random_array(b200_mt19937_t* e, uint32_t set_size, uint32_t n, uint32_t* v, int32_t* out) {
    const size_t make_size = (size_t)(set_size * 1.2);
    size_t size = 0;
    while (size != set_size) {
        while (size < make_size) v[size++] = uniform_below(e, n);
        for (size_t i = 1; i < size; ++i)
            for (size_t j = i; j > 0 && v[j - 1] > v[j]; --j) {
                const uint32_t t = v[j];
                v[j] = v[j - 1];
                v[j - 1] = t;
            }
        size_t u = 0;
        for (size_t i = 0; i < size; ++i)
            if (u == 0 || v[u - 1] != v[i]) v[u++] = v[i];
        size = u < set_size ? u : set_size;
    }
    // std::shuffle: with a 32-bit engine and set_size^2 <= 2^32 - 1, swap positions come in pairs from one draw
    uint32_t t;
    size_t i = 1;
    if (set_size % 2 == 0) {
        const uint32_t d = uniform_below(e, 2);
        t = v[i], v[i] = v[d], v[d] = t;
        ++i;
    }
    while (i < set_size) {
        const uint32_t r = (uint32_t)i + 1;
        const uint32_t x = uniform_below(e, r * (r + 1));
        t = v[i], v[i] = v[x / (r + 1)], v[x / (r + 1)] = t;
        ++i;
        t = v[i], v[i] = v[x % (r + 1)], v[x % (r + 1)] = t;
        ++i;
    }
    for (uint32_t k = 0; k < set_size; ++k) out[k] = (int32_t)v[k];
}

}  // namespace
}  // namespace b200

extern "C" {

int b200_mt19937_seed(b200_mt19937_t* e, const uint32_t* seed_seq, int n_seed) {
    if (!e || n_seed < 0 || (n_seed > 0 && !seed_seq)) return B200_ERR_INVALID;
    uint32_t* x = e->state;
    if (n_seed == 0) {
        x[0] = 5489u;
        for (uint32_t i = 1; i < 624; ++i) x[i] = 1812433253u * (x[i - 1] ^ (x[i - 1] >> 30)) + i;
    } else {  // std::seed_seq::generate over 624 words, then mersenne_twister_engine::seed(seed_seq&)
        const uint32_t n = 624, s = (uint32_t)n_seed, t = 11, p = (n - t) / 2, q = p + t, m = (s + 1 > n) ? s + 1 : n;
        for (uint32_t k = 0; k < n; ++k) x[k] = 0x8b8b8b8bu;
        auto T = [](uint32_t v) { return v ^ (v >> 27); };
        for (uint32_t k = 0; k < m; ++k) {
            const uint32_t r1 = 1664525u * T(x[k % n] ^ x[(k + p) % n] ^ x[(k + n - 1) % n]);
            const uint32_t r2 = r1 + (k == 0 ? s : (k <= s ? k % n + seed_seq[k - 1] : k % n));
            x[(k + p) % n] += r1;
            x[(k + q) % n] += r2;
            x[k % n] = r2;
        }
        for (uint32_t k = m; k < m + n; ++k) {
            const uint32_t r3 = 1566083941u * T(x[k % n] + x[(k + p) % n] + x[(k + n - 1) % n]);
            const uint32_t r4 = r3 - k % n;
            x[(k + p) % n] ^= r3;
            x[(k + q) % n] ^= r4;
            x[k % n] = r4;
        }
        bool zero = (x[0] & 0x80000000u) == 0;
        for (uint32_t i = 1; i < n && zero; ++i) zero = x[i] == 0;
        if (zero) x[0] = 0x80000000u;
    }
    e->index = 624;
    return B200_OK;
}

uint32_t b200_mt19937_next(b200_mt19937_t* e) { return e ? b200::mt_next(e) : 0u; }

int b200_draw_min_sets(b200_mt19937_t* e, uint32_t set_size, uint32_t n_matches, uint32_t max_num_iter, int32_t* out) {
    // set_size <= 65535 keeps set_size^2 within the engine's range (the paired shuffle) and the products below in 32 bits
    if (!e || set_size < 1 || set_size > 65535u || n_matches < set_size || (max_num_iter > 0 && !out)) return B200_ERR_INVALID;
    std::vector<uint32_t> v((size_t)(set_size * 1.2) + set_size);
    for (uint32_t it = 0; it < max_num_iter; ++it) b200::create_random_array(e, set_size, n_matches, v.data(), out + (size_t)set_size * it);
    return B200_OK;
}

int b200_pnp_draw_min_sets(b200_mt19937_t* e, uint32_t n_matches, uint32_t max_num_iter, int32_t* out) {
    return b200_draw_min_sets(e, 4, n_matches, max_num_iter, out);
}

}  // extern "C"
