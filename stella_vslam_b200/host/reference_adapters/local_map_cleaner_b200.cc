// Keyframe culling on the device: module::local_map_cleaner::remove_redundant_keyframes (module/local_map_cleaner.cc:68-193) as one
// call of b200_remove_redundant_keyframes.  The device counts every rank in order and erases the observations of each removed rank
// before the next one counts; the map itself is changed here, by the reference's own prepare_for_erasing, in rank order.
//
// Call site (USE_B200), mapping_module::mapping_with_new_keyframe (mapping_module.cc:239), in place of
// `local_map_cleaner_->remove_redundant_keyframes(cur_keyfrm_);`:
//       remove_redundant_keyframes_b200(map_db_, bow_db_, cur_keyfrm_, redundant_obs_ratio_thr_, top_n_covisibilities_to_search_);
//   with mapping_module members read from the same YAML node and keys ("redundant_obs_ratio_thr", default 0.9;
//   "top_n_covisibilities_to_search", default 30) as local_map_cleaner's constructor, which keeps its copies private.
// A keyframe pinned by set_not_to_be_erased() is counted as removed, as the reference counts it, but prepare_for_erasing leaves it in
// the map; the device's later ranks assumed it was erased, so the ranks after it are gathered and decided again.
#include "stella_vslam/camera/base.h"
#include "stella_vslam/data/bow_database.h"
#include "stella_vslam/data/graph_node.h"
#include "stella_vslam/data/keyframe.h"
#include "stella_vslam/data/landmark.h"
#include "stella_vslam/data/map_database.h"

#include <memory>
#include <mutex>
#include <stdexcept>
#include <unordered_map>
#include <vector>

#include "b200vslam.h"

namespace stella_vslam {
namespace module {
namespace {

b200_matcher_t cull_matcher() {
    static thread_local b200_matcher_t h = nullptr;
    if (!h && b200_matcher_create(0, &h) != B200_OK) throw std::runtime_error(b200_last_error());
    return h;
}

// The flat tables of the ranks [begin, end) of `covs`, gathered under mtx_database_: get_observations() is called once per landmark.
struct cull_tables {
    std::vector<b200_cull_keyframe_t> covs;
    std::vector<std::vector<int32_t>> kp_landmark;
    std::vector<int32_t> offsets{0}, rank, octave;
    std::vector<uint8_t> weight;

    cull_tables(const std::vector<std::shared_ptr<data::keyframe>>& all, size_t begin, size_t end) {
        std::unordered_map<const data::keyframe*, int32_t> rank_of;
        for (size_t r = begin; r < end; ++r) rank_of[all[r].get()] = static_cast<int32_t>(r - begin);
        std::unordered_map<const data::landmark*, int32_t> row_of;
        std::vector<std::shared_ptr<data::landmark>> rows;
        covs.resize(end - begin);
        kp_landmark.resize(end - begin);
        for (size_t r = begin; r < end; ++r) {
            const auto& kf = all[r];
            const auto landmarks = kf->get_landmarks();
            auto& kl = kp_landmark[r - begin];
            kl.assign(landmarks.size(), -1);
            for (size_t idx = 0; idx < landmarks.size(); ++idx) {
                const auto& lm = landmarks[idx];
                if (!lm || lm->will_be_erased()) continue;
                const auto ins = row_of.emplace(lm.get(), static_cast<int32_t>(rows.size()));
                if (ins.second) rows.push_back(lm);
                kl[idx] = ins.first->second;
            }
            b200_cull_keyframe_t& c = covs[r - begin];
            c = b200_cull_keyframe_t{};
            c.id = kf->id_;
            c.is_root = kf->graph_node_->is_spanning_root() ? 1 : 0;
            c.n_keypoints = static_cast<int32_t>(kl.size());
            c.kp_landmark = kl.data();
            c.depth = kf->depth_is_available() ? kf->frm_obs_.depths_.data() : nullptr;
            c.depth_thr = kf->camera_->depth_thr_;
        }
        for (const auto& lm : rows) {
            for (const auto& obs : lm->get_observations()) {
                const auto ngh = obs.first.lock();
                const auto it = rank_of.find(ngh.get());
                rank.push_back(it == rank_of.end() ? -1 : it->second);
                octave.push_back(ngh->frm_obs_.undist_keypts_.at(obs.second).octave);
                const auto& x_right = ngh->frm_obs_.stereo_x_right_;
                weight.push_back(!x_right.empty() && 0 <= x_right.at(obs.second) ? 2 : 1);  // landmark::add_observation
            }
            offsets.push_back(static_cast<int32_t>(rank.size()));
        }
    }
};

}  // namespace

unsigned int remove_redundant_keyframes_b200(data::map_database* map_db, data::bow_database* bow_db, const std::shared_ptr<data::keyframe>& cur_keyfrm,
                                             double redundant_obs_ratio_thr, unsigned int top_n_covisibilities_to_search) {
    if (redundant_obs_ratio_thr < 0.0 || top_n_covisibilities_to_search <= 0) {
        return 0;
    }
    std::lock_guard<std::mutex> lock(data::map_database::mtx_database_);
    const auto cur_covisibilities = cur_keyfrm->graph_node_->get_top_n_covisibilities(top_n_covisibilities_to_search);
    unsigned int num_removed = 0;
    size_t begin = 0;
    while (begin < cur_covisibilities.size()) {
        cull_tables t(cur_covisibilities, begin, cur_covisibilities.size());
        b200_cull_problem_t p{};
        p.cur_id = cur_keyfrm->id_;
        p.redundant_obs_ratio_thr = redundant_obs_ratio_thr;
        p.n_covisibilities = static_cast<int32_t>(t.covs.size());
        p.covisibilities = t.covs.data();
        p.n_landmarks = static_cast<int32_t>(t.offsets.size() - 1);
        p.obs_offsets = t.offsets.data();
        p.obs_rank = t.rank.data();
        p.obs_octave = t.octave.data();
        p.obs_weight = t.weight.data();
        if (b200_remove_redundant_keyframes(cull_matcher(), 1, &p) != B200_OK) throw std::runtime_error(b200_last_error());
        size_t restart = cur_covisibilities.size();
        for (size_t r = 0; r < t.covs.size(); ++r) {
            if (!t.covs[r].removed) continue;
            ++num_removed;
            const auto& covisibility = cur_covisibilities[begin + r];
            const auto cur_landmarks = covisibility->get_landmarks();
            covisibility->prepare_for_erasing(map_db, bow_db);
            for (const auto& lm : cur_landmarks) {  // local_map_cleaner.cc:101-116
                if (!lm) {
                    continue;
                }
                if (lm->will_be_erased()) {
                    continue;
                }
                if (!lm->has_representative_descriptor()) {
                    lm->compute_descriptor();
                }
                if (!lm->has_valid_prediction_parameters()) {
                    lm->update_mean_normal_and_obs_scale_variance();
                }
            }
            if (!covisibility->will_be_erased()) {  // pinned: the later ranks are decided again on the map as it now is
                restart = begin + r + 1;
                break;
            }
        }
        begin = restart;
    }
    return num_removed;
}

}  // namespace module
}  // namespace stella_vslam
