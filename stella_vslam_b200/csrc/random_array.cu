// random_array.cu -- the minimal-set sampler of the RANSAC solvers: std::mt19937 and util::create_random_array
// (src/stella_vslam/util/random_array.cc) as libstdc++ evaluates them (random_array.cuh).  The solvers draw their minimal sets here on
// the host, in draw order, and pass them to b200_pnp_ransac, b200_essential_ransac and b200_twoview_ransac; the device sampler draws
// them where the match count is only known on the device (b200_robust_match_based_track).
#include <climits>
#include <cstdint>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "random_array.cuh"
#include "staging.cuh"
#include "track_chain.cuh"

namespace b200 {
namespace rnd {

// One warp per engine: max_num_iter calls of create_random_array(set_size, 0, n[p] - 1) for every problem p with n[p] >= set_size, the
// engine's state in shared memory.  engines == null: default-constructed engines (seed 5489), built here.
__global__ void __launch_bounds__(32) draw_min_sets_kernel(const b200_mt19937_t* __restrict__ engines, const int* __restrict__ n, uint32_t set_size,
                                                           uint32_t max_num_iter, int32_t* __restrict__ out) {
    __shared__ uint32_t x[624];
    const int p = blockIdx.x;
    const int np = n[p];
    if (np < (int)set_size) return;
    MtRef e{x, 624u, threadIdx.x, 32u};
    if (engines) {
        for (int k = threadIdx.x; k < 624; k += 32) x[k] = engines[p].state[k];
        e.index = engines[p].index;
    } else if (threadIdx.x == 0) {
        x[0] = 5489u;
        for (uint32_t i = 1; i < 624; ++i) x[i] = 1812433253u * (x[i - 1] ^ (x[i - 1] >> 30)) + i;
    }
    __syncwarp();
    uint32_t v[scratch_size(kMaxDeviceSet)];
    int32_t* o = out + (size_t)p * max_num_iter * set_size;
    for (uint32_t it = 0; it < max_num_iter; ++it) create_random_array(e, set_size, (uint32_t)np, v, o + (size_t)set_size * it);
}

}  // namespace rnd

namespace chain {
int draw_min_sets(cudaStream_t st, int n_problems, const b200_mt19937_t* d_engines, const int* d_n, uint32_t set_size, uint32_t max_num_iter,
                  int32_t* d_out) {
    if (set_size < 1 || set_size > rnd::kMaxDeviceSet) return B200_ERR_INVALID;
    if (n_problems > 0 && max_num_iter > 0) rnd::draw_min_sets_kernel<<<n_problems, 32, 0, st>>>(d_engines, d_n, set_size, max_num_iter, d_out);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}
}  // namespace chain
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

uint32_t b200_mt19937_next(b200_mt19937_t* e) {
    if (!e) return 0u;
    b200::rnd::MtRef r{e->state, e->index, 0, 1};
    const uint32_t y = b200::rnd::mt_next(r);
    e->index = r.index;
    return y;
}

int b200_draw_min_sets(b200_mt19937_t* e, uint32_t set_size, uint32_t n_matches, uint32_t max_num_iter, int32_t* out) {
    // set_size <= 65535 keeps set_size^2 within the engine's range (the paired shuffle) and the products below in 32 bits
    if (!e || set_size < 1 || set_size > 65535u || n_matches < set_size || (max_num_iter > 0 && !out)) return B200_ERR_INVALID;
    std::vector<uint32_t> v(b200::rnd::scratch_size(set_size));
    b200::rnd::MtRef r{e->state, e->index, 0, 1};
    for (uint32_t it = 0; it < max_num_iter; ++it) b200::rnd::create_random_array(r, set_size, n_matches, v.data(), out + (size_t)set_size * it);
    e->index = r.index;
    return B200_OK;
}

int b200_pnp_draw_min_sets(b200_mt19937_t* e, uint32_t n_matches, uint32_t max_num_iter, int32_t* out) {
    return b200_draw_min_sets(e, 4, n_matches, max_num_iter, out);
}

int b200_draw_min_sets_batch(b200_lba_t h, int n_engines, const b200_mt19937_t* engines, uint32_t set_size, const uint32_t* n_matches,
                             uint32_t max_num_iter, int32_t* out) {
    B200_RANGE("b200:random:draw_min_sets_batch");
    if (!h || n_engines < 0 || set_size < 1 || set_size > b200::rnd::kMaxDeviceSet || max_num_iter > (1u << 24)) return B200_ERR_INVALID;
    if (n_engines == 0 || max_num_iter == 0) return B200_OK;
    if (!n_matches || !out) return B200_ERR_INVALID;
    for (int p = 0; p < n_engines; ++p)
        if (n_matches[p] < set_size || n_matches[p] > (uint32_t)INT32_MAX || (engines && engines[p].index > 624u)) {
            b200::set_error("b200_draw_min_sets_batch: engine %d: n_matches %u below the set size or a bad engine index", p, n_matches[p]);
            return B200_ERR_INVALID;
        }
    const size_t out_bytes = sizeof(int32_t) * set_size * (size_t)max_num_iter * n_engines;
    b200::Layout a;
    const size_t o_eng = a.take<b200_mt19937_t>(engines ? n_engines : 0), o_n = a.take<int>(n_engines);
    const size_t in_bytes = a.end;
    const size_t o_out = a.take(out_bytes);
    cudaStream_t st;
    b200::StagingArena* A;
    int rc = b200::lba::staging(h, a.end, a.end, &st, &A);
    if (rc) return rc;
    if (engines) A->put(o_eng, engines, sizeof(b200_mt19937_t) * n_engines);
    A->put(o_n, n_matches, sizeof(int) * n_engines);
    B200_CUDA(A->upload(in_bytes, st));
    if ((rc = b200::chain::draw_min_sets(st, n_engines, engines ? A->dev<const b200_mt19937_t>(o_eng) : nullptr, A->dev<const int>(o_n), set_size,
                                         max_num_iter, A->dev<int32_t>(o_out))))
        return rc;
    B200_CUDA(A->download(o_out, o_out + out_bytes, st));
    B200_CUDA(cudaStreamSynchronize(st));
    std::memcpy(out, A->host(o_out), out_bytes);
    return B200_OK;
}

}  // extern "C"
