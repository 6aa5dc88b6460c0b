// Per-keyframe gather shared by the adapters that feed the all-pairs matchers (bow_tree_b200.cc) and the landmark-creation chain
// (create_new_landmarks_b200.cc): the BoW node of every keypoint and the per-keypoint arrays of b200_pairs_problem_t.
#pragma once

#include <cstdint>
#include <vector>

#include "stella_vslam/data/bow_vocabulary.h"
#include "stella_vslam/data/frame_observation.h"
#include "stella_vslam/feature/orb_params.h"

namespace stella_vslam {
namespace b200_gather {

// node id per keypoint (-1: the keypoint is in no node and is never visited)
inline std::vector<int32_t> node_of(const data::bow_feature_vector& fv, size_t n) {
    std::vector<int32_t> node(n, -1);
    for (const auto& kv : fv)
        for (const auto idx : kv.second) node.at(idx) = static_cast<int32_t>(kv.first);
    return node;
}

struct side {
    std::vector<float> angle, scale;
    std::vector<uint8_t> valid, stereo;
    std::vector<double> bearing;
    void fill(const data::frame_observation& obs, const feature::orb_params* prm) {
        const size_t n = obs.undist_keypts_.size();
        angle.resize(n); scale.resize(n); valid.assign(n, 0); stereo.assign(n, 0); bearing.resize(3 * n);
        for (size_t i = 0; i < n; ++i) {
            angle[i] = obs.undist_keypts_[i].angle;
            scale[i] = prm->scale_factors_.at(obs.undist_keypts_[i].octave);
            stereo[i] = !obs.stereo_x_right_.empty() && 0 <= obs.stereo_x_right_.at(i);
            if (i < obs.bearings_.size())
                for (int k = 0; k < 3; ++k) bearing[3 * i + k] = obs.bearings_[i](k);
        }
    }
};

}  // namespace b200_gather
}  // namespace stella_vslam
