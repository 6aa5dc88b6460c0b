// ransac_host.cuh -- what b200_pnp_ransac, b200_essential_ransac and b200_twoview_ransac share: the minimal-set check and copy,
// and the select kernels' inlier compaction.  Each entry point keeps its own problem checks, device structs and selection rule.
#pragma once

#include <climits>
#include <cstdint>
#include <cstring>

#include "common.cuh"

namespace b200 {

// A problem that runs RANSAC has max_num_iter within int, min_sets when it iterates, and every one of its set_size * max_num_iter
// entries in [0, n).  Reports through set_error under fn's name.
inline bool min_sets_ok(const char* fn, int q, bool runs, uint32_t max_num_iter, const int32_t* min_sets, int set_size, int n) {
    if (!runs) return true;
    if (max_num_iter > (uint32_t)INT_MAX || (max_num_iter > 0 && !min_sets)) {
        set_error("%s: problem %d: bad max_num_iter or null min_sets", fn, q);
        return false;
    }
    for (long long k = 0; k < (long long)set_size * max_num_iter; ++k)
        if (min_sets[k] < 0 || min_sets[k] >= n) {
            set_error("%s: problem %d: min_sets entry %lld = %d outside [0, %d)", fn, q, k, min_sets[k], n);
            return false;
        }
    return true;
}

// Stages problem q's n_hyp minimal sets of set_size entries at entry ms_off of ms, and maps its hypotheses hyp_off.. to q.
inline void stage_min_sets(int q, const int32_t* min_sets, int set_size, int n_hyp, size_t ms_off, int hyp_off, int32_t* ms, int* hyp_problem) {
    if (n_hyp) std::memcpy(ms + ms_off, min_sets, sizeof(int32_t) * set_size * (size_t)n_hyp);
    for (int k = 0; k < n_hyp; ++k) hyp_problem[hyp_off + k] = q;
}

// The indices of the set flags in ascending order; returns their count.
__device__ __forceinline__ int compact_inliers(const uint8_t* flags, int n, int32_t* idx) {
    int m = 0;
    for (int j = 0; j < n; ++j)
        if (flags[j]) idx[m++] = j;
    return m;
}

}  // namespace b200
