// twoview_ransac.cuh -- the device side of find_via_ransac of the homography and fundamental solvers (twoview_kernels.cu), shared by
// b200_twoview_ransac (problems staged from the host) and b200_initialize (one H and one F problem per perspective pair, followed by the
// reconstruction launches of initialize_kernels.cu).  Every array is a device array.
#pragma once

#include <cstdint>

#include "common.cuh"

namespace b200 {
namespace twoview {

constexpr int kMinRows = 8;  // both models return early below 8 matches (H: min_set_size * 2)

struct ProblemDev {
    int model;
    int n;          // matches
    int match_off;  // first match in the concatenated matches / flags
    int n1, kp1_off, n2, kp2_off;
    int set_size;   // 4 (H) or 8 (F)
    int hyp_off;    // first iteration in the concatenated iterations
    int ms_off;     // first entry in the concatenated minimal sets
    int n_hyp;      // max_num_iter (0 on the early return)
    int runs;       // 0: find_via_ransac returns before drawing (n < 8)
    int recompute;
    float sigma;
};

struct NormDev {
    double T1[9];  // transform_1
    double D2[9];  // transform_2.inverse() (H) or transform_2.transpose() (F)
};

struct HypDev {
    double M[9];  // the denormalised estimate
    int ok;       // 0: H's minimal set was degenerate (the iteration is skipped)
    int status;   // ES_STATUS_SVD
};

struct ScoreDev {
    float cost;
    unsigned num_inliers;
};

struct ResultDev {
    double M[9];
    float best_cost;
    int valid, best_iter, num_inliers, status;
};

struct RansacDev {
    const ProblemDev* probs;   // per problem; problems own disjoint keypoint and match ranges
    const float *kp1, *kp2;    // 2 per keypoint
    const int32_t* matches;    // 2 per match
    const int32_t* min_sets;   // set_size per hypothesis
    const int* hyp_problem;    // per hypothesis: its problem
    float *kn1, *kn2;          // scratch: the normalised keypoints
    NormDev* norms;            // scratch: per problem
    HypDev* hyps;              // scratch: per hypothesis
    ScoreDev* scores;          // scratch: per hypothesis
    int32_t* idx;              // scratch: per match
    double* mat;               // scratch: 18 per match
    uint8_t* flags;            // out: inlier flags per match (written for the problems that run)
    ResultDev* results;        // out: per problem
};

// The normalisation, hypothesis, score and select launches of find_via_ransac on st over n_hyp hypotheses and n_problems problems.
int enqueue_ransac(cudaStream_t st, int n_problems, int n_hyp, const RansacDev& d);

}  // namespace twoview
}  // namespace b200
