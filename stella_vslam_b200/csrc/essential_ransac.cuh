// essential_ransac.cuh -- the device side of find_via_ransac of the five-point essential solver (essential_kernels.cu), shared by
// b200_essential_ransac (problems staged from the host) and b200_robust_match_based_track (problems built on the device from the
// brute-force matches).  Every array is a device array.
#pragma once

#include <cstdint>

#include "common.cuh"

namespace b200 {
namespace ess {

constexpr int kMinSet = 5;
constexpr int kMaxCand = 10;

struct ProblemDev {
    int n;          // matches
    int match_off;  // first row in the concatenated bearings / flags
    int hyp_off;    // first iteration in the concatenated minimal sets
    int n_hyp;      // max_num_iter (0 on the early return)
    int runs;       // 0: find_via_ransac returns before drawing (n < min_set_size); its hypotheses do no work
    int recompute;
};

struct HypDev {
    int count;  // candidates written
    int flags;  // ES_STATUS_* bits
};

struct ScoreDev {
    float cost;
    unsigned num_inliers;
};

struct ResultDev {
    double E[9];
    float best_cost;
    int valid, best_iter, best_candidate, num_inliers, status;
};

struct RansacDev {
    const int* hyp_problem;   // per hypothesis: its problem
    const ProblemDev* probs;  // per problem
    const double *b1, *b2;    // 3 per match row
    const int32_t* min_sets;  // kMinSet per hypothesis
    double* cand;             // scratch: 9 * kMaxCand per hypothesis
    HypDev* hyps;             // scratch: per hypothesis
    ScoreDev* scores;         // scratch: kMaxCand per hypothesis
    int32_t* idx;             // scratch: per match row
    double* mat;              // scratch: 9 per match row
    uint8_t* flags;           // out: inlier flags per match row (written for the problems that run)
    ResultDev* results;       // out: per problem
};

// The hypothesis, score and select launches of find_via_ransac on st over n_hyp hypotheses and n_problems problems.
int enqueue_ransac(cudaStream_t st, int n_problems, int n_hyp, const RansacDev& d);

}  // namespace ess
}  // namespace b200
