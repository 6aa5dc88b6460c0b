/* cull_oracle.c -- single-thread C restatement of b200_remove_redundant_keyframes (test infrastructure): local_map_cleaner::
 * remove_redundant_keyframes and count_redundant_observations (module/local_map_cleaner.cc:68-193) with the observation erasure of
 * keyframe::prepare_for_erasing and landmark::erase_observation, on the flat tables of b200_cull_problem_t.  Each rank is counted and,
 * when removed, erased before the next one, as the reference loop does. */
#include <stdlib.h>

#include "../include/b200vslam.h"

/* the live observation of landmark l by rank r */
static int own_obs(const b200_cull_problem_t* P, const unsigned char* erased, int l, int r) {
    for (int j = P->obs_offsets[l]; j < P->obs_offsets[l + 1]; ++j)
        if (P->obs_rank[j] == r && !erased[j]) return j;
    return -1;
}

void cull_oracle(b200_cull_problem_t* P) {
    const int L = P->n_landmarks, total = L ? P->obs_offsets[L] : 0;
    unsigned* num_observations = calloc((size_t)L + 1, sizeof(unsigned)); /* landmark::num_observations_ */
    int* n_left = calloc((size_t)L + 1, sizeof(int));                     /* observations_.size(); 0 = will_be_erased */
    unsigned char* erased = calloc((size_t)total + 1, 1);
    for (int l = 0; l < L; ++l)
        for (int j = P->obs_offsets[l]; j < P->obs_offsets[l + 1]; ++j) {
            num_observations[l] += P->obs_weight[j];
            ++n_left[l];
        }
    const unsigned num_better_obs_thr = 3, window_size_not_to_remove = 2;
    unsigned num_removed = 0;
    for (int r = 0; r < P->n_covisibilities; ++r) {
        b200_cull_keyframe_t* K = &P->covisibilities[r];
        K->n_valid = K->n_redundant = K->skipped = K->removed = 0;
        if (K->is_root) {
            K->skipped = 1;
            continue;
        }
        if (K->id <= P->cur_id && P->cur_id <= K->id + window_size_not_to_remove) {
            K->skipped = 2;
            continue;
        }
        unsigned num_valid_obs = 0, num_redundant_obs = 0;
        for (int idx = 0; idx < K->n_keypoints; ++idx) {
            const int l = K->kp_landmark[idx];
            if (l < 0 || n_left[l] == 0) continue;
            if (K->depth) {
                const float depth = K->depth[idx];
                if (depth < 0.0 || K->depth_thr < depth) continue;
            }
            ++num_valid_obs;
            if (num_observations[l] <= num_better_obs_thr) continue;
            const int scale_level = P->obs_octave[own_obs(P, erased, l, r)];
            unsigned num_better_obs = 0;
            int redundant = 0;
            for (int j = P->obs_offsets[l]; j < P->obs_offsets[l + 1]; ++j) {
                if (erased[j] || P->obs_rank[j] == r) continue;
                if (P->obs_octave[j] <= (long long)scale_level + 1) {
                    ++num_better_obs;
                    if (num_better_obs_thr <= num_better_obs) {
                        redundant = 1;
                        break;
                    }
                }
            }
            if (redundant) ++num_redundant_obs;
        }
        K->n_valid = (int32_t)num_valid_obs;
        K->n_redundant = (int32_t)num_redundant_obs;
        if (P->redundant_obs_ratio_thr <= (float)num_redundant_obs / num_valid_obs) {
            K->removed = 1;
            ++num_removed;
            for (int idx = 0; idx < K->n_keypoints; ++idx) {
                const int l = K->kp_landmark[idx];
                if (l < 0 || n_left[l] == 0) continue;
                const int j = own_obs(P, erased, l, r);
                erased[j] = 1;
                num_observations[l] -= P->obs_weight[j];
                --n_left[l];
            }
        }
    }
    P->n_removed = (int32_t)num_removed;
    P->status = B200_OK;
    free(num_observations);
    free(n_left);
    free(erased);
}
