// optimize::graph_optimizer on the GPU: this translation unit REPLACES src/stella_vslam/optimize/graph_optimizer.cc when USE_B200 is set
// (link-time, like the global bundle adjuster).  It keeps the header, builds the vertices and edges with the reference's own g2o::Sim3
// by the rules of graph_optimizer.cc:43-250, makes one b200_graph_optimize call (steps 4-5 of the reference: LM, 50 iterations,
// terminate action at gain 1e-3) and writes back under mtx_database_ as :261-302 does.
#include "stella_vslam/data/keyframe.h"
#include "stella_vslam/data/graph_node.h"
#include "stella_vslam/data/landmark.h"
#include "stella_vslam/data/map_database.h"
#include "stella_vslam/optimize/graph_optimizer.h"
#include "stella_vslam/util/converter.h"

#include <mutex>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "b200vslam.h"

namespace stella_vslam {
namespace optimize {

namespace {
b200_sim3_t to_b200(const g2o::Sim3& s) {
    b200_sim3_t o;
    const auto& q = s.rotation();
    o.q[0] = q.x(); o.q[1] = q.y(); o.q[2] = q.z(); o.q[3] = q.w();
    for (int k = 0; k < 3; ++k) o.t[k] = s.translation()(k);
    o.s = s.scale();
    return o;
}

b200_lba_t handle() {
    static b200_lba_t h = [] {
        b200_lba_t x = nullptr;
        if (b200_lba_create(0, &x) != B200_OK) throw std::runtime_error(std::string("b200_lba_create: ") + b200_last_error());
        return x;
    }();
    return h;
}
}  // namespace

graph_optimizer::graph_optimizer(const YAML::Node& yaml_node, const bool fix_scale)
    : fix_scale_(fix_scale), min_num_shared_lms_(yaml_node["min_num_shared_lms"].as<unsigned int>(100)) {}

void graph_optimizer::optimize(const std::shared_ptr<data::keyframe>& loop_keyfrm, const std::shared_ptr<data::keyframe>& curr_keyfrm,
                               const module::keyframe_Sim3_pairs_t& non_corrected_Sim3s, const module::keyframe_Sim3_pairs_t& pre_corrected_Sim3s,
                               const std::map<std::shared_ptr<data::keyframe>, std::set<std::shared_ptr<data::keyframe>>>& loop_connections,
                               std::unordered_map<unsigned int, unsigned int>& found_lm_to_ref_keyfrm_id) const {
    const auto all_keyfrms = curr_keyfrm->graph_node_->get_keyframes_from_root();
    // the landmarks of those keyframes, once each (:46-66)
    std::unordered_set<unsigned int> seen_lms;
    std::vector<std::shared_ptr<data::landmark>> all_lms;
    for (const auto& keyfrm : all_keyfrms) {
        for (const auto& lm : keyfrm->get_landmarks()) {
            if (!lm || lm->will_be_erased() || seen_lms.count(lm->id_)) continue;
            seen_lms.insert(lm->id_);
            all_lms.push_back(lm);
        }
    }

    // vertices (:68-106): the pre-corrected Sim3 where there is one, else Sim3(rot_cw, trans_cw, 1)
    std::unordered_map<unsigned int, g2o::Sim3> Sim3s_cw;
    std::unordered_map<unsigned int, int32_t> vidx;
    std::vector<b200_sim3_t> estimate;
    std::vector<uint8_t> fixed;
    for (const auto& keyfrm : all_keyfrms) {
        if (keyfrm->will_be_erased()) continue;
        const auto it = pre_corrected_Sim3s.find(keyfrm);
        const g2o::Sim3 S = it != pre_corrected_Sim3s.end() ? it->second : g2o::Sim3(keyfrm->get_rot_cw(), keyfrm->get_trans_cw(), 1.0);
        Sim3s_cw[keyfrm->id_] = S;
        vidx[keyfrm->id_] = (int32_t)estimate.size();
        estimate.push_back(to_b200(S));
        fixed.push_back((*keyfrm == *loop_keyfrm || *keyfrm == *curr_keyfrm || keyfrm->graph_node_->is_spanning_root()) ? 1 : 0);
    }

    // edges (:108-250), in the reference's insertion order
    std::vector<int32_t> e_v1, e_v2;
    std::vector<b200_sim3_t> e_meas;
    std::set<std::pair<unsigned int, unsigned int>> inserted;
    const auto insert_edge = [&](unsigned int id1, unsigned int id2, const g2o::Sim3& Sim3_21) {
        e_v1.push_back(vidx.at(id1));
        e_v2.push_back(vidx.at(id2));
        e_meas.push_back(to_b200(Sim3_21));
        inserted.insert(std::make_pair(std::min(id1, id2), std::max(id1, id2)));
    };
    for (const auto& loop_connection : loop_connections) {
        const auto& keyfrm = loop_connection.first;
        const auto id1 = keyfrm->id_;
        const g2o::Sim3 Sim3_w1 = Sim3s_cw.at(id1).inverse();
        for (const auto& connected : loop_connection.second) {
            const auto id2 = connected->id_;
            if (!(id1 == curr_keyfrm->id_ && id2 == loop_keyfrm->id_)
                && keyfrm->graph_node_->get_num_shared_landmarks(connected) < min_num_shared_lms_) {
                continue;
            }
            insert_edge(id1, id2, Sim3s_cw.at(id2) * Sim3_w1);
        }
    }
    const auto Sim3_2w_of = [&](const std::shared_ptr<data::keyframe>& kf) -> g2o::Sim3 {
        const auto it = non_corrected_Sim3s.find(kf);
        return it != non_corrected_Sim3s.end() ? it->second : Sim3s_cw.at(kf->id_);
    };
    for (const auto& keyfrm : all_keyfrms) {
        const auto id1 = keyfrm->id_;
        const g2o::Sim3 Sim3_w1 = Sim3_2w_of(keyfrm).inverse();
        const auto parent_node = keyfrm->graph_node_->get_spanning_parent();
        if (parent_node) {
            if (id1 <= parent_node->id_) continue;  // the reference skips the rest of this keyframe
            insert_edge(id1, parent_node->id_, Sim3_2w_of(parent_node) * Sim3_w1);
        }
        const auto loop_edges = keyfrm->graph_node_->get_loop_edges();
        for (const auto& connected : loop_edges) {
            if (id1 <= connected->id_) continue;
            insert_edge(id1, connected->id_, Sim3_2w_of(connected) * Sim3_w1);
        }
        for (const auto& connected : keyfrm->graph_node_->get_covisibilities_over_min_num_shared_lms(min_num_shared_lms_)) {
            if (!connected || !parent_node) continue;
            if (*connected == *parent_node || keyfrm->graph_node_->has_spanning_child(connected)) continue;
            if (loop_edges.count(connected) || connected->will_be_erased()) continue;
            const auto id2 = connected->id_;
            if (id1 <= id2 || inserted.count(std::make_pair(std::min(id1, id2), std::max(id1, id2)))) continue;
            insert_edge(id1, id2, Sim3_2w_of(connected) * Sim3_w1);
        }
    }

    // landmark correction input (:283-300)
    std::vector<double> points;
    std::vector<int32_t> point_ref;
    for (const auto& lm : all_lms) {
        const auto ref_id = found_lm_to_ref_keyfrm_id.count(lm->id_) ? found_lm_to_ref_keyfrm_id.at(lm->id_) : lm->get_ref_keyframe()->id_;
        const Vec3_t pos_w = lm->get_pos_in_world();
        points.insert(points.end(), {pos_w(0), pos_w(1), pos_w(2)});
        point_ref.push_back(vidx.at(ref_id));
    }

    std::vector<b200_sim3_t> estimate_out(estimate.size());
    std::vector<double> pose_cw_out(16 * estimate.size()), points_out(points.size());
    b200_pose_graph_t g{};
    g.n_vertices = (int32_t)estimate.size();
    g.n_edges = (int32_t)e_v1.size();
    g.fix_scale = fix_scale_ ? 1 : 0;
    g.estimate = estimate.data();
    g.fixed = fixed.data();
    g.e_v1 = e_v1.data();
    g.e_v2 = e_v2.data();
    g.e_meas = e_meas.data();
    g.n_points = (int32_t)point_ref.size();
    g.points = points.data();
    g.point_ref = point_ref.data();
    g.estimate_out = estimate_out.data();
    g.pose_cw_out = pose_cw_out.data();
    g.points_out = points_out.empty() ? nullptr : points_out.data();
    if (b200_graph_optimize(handle(), &g, 50, 1e-3, nullptr) != B200_OK) {
        throw std::runtime_error(std::string("b200_graph_optimize: ") + b200_last_error());
    }

    // write-back (:261-302)
    std::lock_guard<std::mutex> lock(data::map_database::mtx_database_);
    for (const auto& keyfrm : all_keyfrms) {
        const auto it = vidx.find(keyfrm->id_);
        if (it == vidx.end()) continue;
        Mat44_t pose_cw;
        for (int r = 0; r < 4; ++r)
            for (int c = 0; c < 4; ++c) pose_cw(r, c) = pose_cw_out[16 * (size_t)it->second + 4 * r + c];
        keyfrm->set_pose_cw(pose_cw);
    }
    for (size_t i = 0; i < all_lms.size(); ++i) {
        const auto& lm = all_lms[i];
        if (lm->will_be_erased()) continue;
        lm->set_pos_in_world(Vec3_t(points_out[3 * i], points_out[3 * i + 1], points_out[3 * i + 2]));
        lm->update_mean_normal_and_obs_scale_variance();
    }
}

}  // namespace optimize
}  // namespace stella_vslam
