// random_array.cuh -- std::mt19937 and util::create_random_array (src/stella_vslam/util/random_array.cc) as libstdc++ evaluates them,
// for the host (b200_draw_min_sets) and for one warp on the device (the minimal-set sampler of b200_robust_match_based_track).  One
// implementation: on the device every lane of the warp runs the same draws on the engine state in shared memory (the values and
// branches are the same in every lane), and the lanes share the twist.
#pragma once

#include <cstddef>
#include <cstdint>

namespace b200 {
namespace rnd {

// An engine's state words (host memory or the warp's shared memory) and its index; `lanes` threads of one warp run the calls together,
// `lane` is this thread's (host: lane 0 of 1).
struct MtRef {
    uint32_t* x;
    uint32_t index;
    unsigned lane, lanes;
};

__host__ __device__ __forceinline__ void mt_sync() {
#ifdef __CUDA_ARCH__
    __syncwarp();
#endif
}

// The twist in three ranges: a new word of [0, 227) reads old words only, one of [227, 454) reads words of the first range, one of
// [454, 624) words of the second (and word 623 the new word 0).  Within a range the lanes read before any of them writes.
__host__ __device__ inline void mt_twist(MtRef& e) {
    uint32_t* x = e.x;
    const int bounds[4] = {0, 227, 454, 624};
    for (int p = 0; p < 3; ++p)
        for (int k0 = bounds[p]; k0 < bounds[p + 1]; k0 += (int)e.lanes) {
            const int k = k0 + (int)e.lane;
            uint32_t nv = 0;
            if (k < bounds[p + 1]) {
                const uint32_t y = (x[k] & 0x80000000u) | (x[(k + 1) % 624] & 0x7fffffffu);
                nv = x[(k + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
            }
            mt_sync();
            if (k < bounds[p + 1]) x[k] = nv;
            mt_sync();
        }
    e.index = 0;
}

__host__ __device__ inline uint32_t mt_next(MtRef& e) {
    if (e.index >= 624) mt_twist(e);
    uint32_t y = e.x[e.index++];
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= y >> 18;
    return y;
}

// uniform_int_distribution{0, range - 1} on a 32-bit engine: Lemire's nearly divisionless method (libstdc++ _S_nd)
__host__ __device__ inline uint32_t uniform_below(MtRef& e, uint32_t range) {
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

// Scratch entries create_random_array needs in v
__host__ __device__ constexpr size_t scratch_size(uint32_t set_size) { return (size_t)(set_size * 1.2) + set_size; }
// Largest set size of the device sampler (its scratch lives in registers)
constexpr uint32_t kMaxDeviceSet = 8;

// util::create_random_array(set_size, 0, n - 1, engine): make_size = size_t(set_size * 1.2) draws of uniform_int_distribution<unsigned>,
// sort + unique (truncated to set_size), repeated until set_size remain, then std::shuffle.  Lane 0 writes out.
__host__ __device__ inline void create_random_array(MtRef& e, uint32_t set_size, uint32_t n, uint32_t* v, int32_t* out) {
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
    if (e.lane == 0)
        for (uint32_t k = 0; k < set_size; ++k) out[k] = (int32_t)v[k];
}

}  // namespace rnd
}  // namespace b200
