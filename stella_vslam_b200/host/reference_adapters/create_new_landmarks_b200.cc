// mapping_module::create_new_landmarks (src/stella_vslam/mapping_module.cc) with the numeric chain on the device: for the current
// keyframe and its top-N covisibilities, match_for_triangulation and two_view_triangulator::triangulate run as ONE call of
// b200_create_new_landmarks; the keypoint rows a neighbour creates landmarks on are closed to the later neighbours on the device.
//
// Call site (mapping_module::mapping_with_new_keyframe, USE_B200): the body of create_new_landmarks becomes
//     create_new_landmarks_b200(map_db_, cur_keyfrm_, num_covisibilities_for_landmark_generation_, use_baseline_dist_thr_ratio_,
//                               baseline_dist_thr_ratio_, baseline_dist_thr_, residual_rad_thr_, bow_db_ && bow_vocab_,
//                               local_map_cleaner_.get(), abort_create_new_landmarks);
// What needs the map stays here: the covisibility walk, the baseline test, E and the epiplane (with the reference's own code), and
// the landmark objects, created in the returned order under mtx_database_ exactly as triangulate_with_two_keyframes does.
// Deviation: the reference polls abort_create_new_landmarks between neighbours (from the second one on); the device chain is not
// interruptible, so the flag is tested once before the call, and the outcome is the reference's outcome without an abort.
#include "stella_vslam/camera/base.h"
#include "stella_vslam/camera/fisheye.h"
#include "stella_vslam/camera/perspective.h"
#include "stella_vslam/camera/radial_division.h"
#include "stella_vslam/data/graph_node.h"
#include "stella_vslam/data/keyframe.h"
#include "stella_vslam/data/landmark.h"
#include "stella_vslam/data/map_database.h"
#include "stella_vslam/module/local_map_cleaner.h"
#include "stella_vslam/solve/essential_solver.h"

#include <atomic>
#include <cstring>
#include <mutex>
#include <stdexcept>

#include "b200vslam.h"
#include "pairs_gather_b200.h"

namespace stella_vslam {
namespace {

b200_matcher_t mapping_matcher() {
    static thread_local b200_matcher_t h = nullptr;
    if (!h && b200_matcher_create(0, &h) != B200_OK) throw std::runtime_error(b200_last_error());
    return h;
}

// one keyframe as b200_tri_keyframe_t; the arrays it points to live in this struct
struct tri_view {
    b200_tri_keyframe_t kf{};
    std::vector<float> x, y;
    std::vector<int32_t> octave;
    std::vector<double> bearing;
    std::vector<uint8_t> no_landmark;
    std::vector<int32_t> node;

    template <class Cam>
    void intrinsics(const camera::base* cam) {
        const auto* c = static_cast<const Cam*>(cam);
        kf.fx = c->fx_; kf.fy = c->fy_; kf.cx = c->cx_; kf.cy = c->cy_; kf.fx_inv = c->fx_inv_; kf.fy_inv = c->fy_inv_;
    }

    void fill(const std::shared_ptr<data::keyframe>& keyfrm, bool bow) {
        const Mat44_t pose_cw = keyfrm->get_pose_cw(), pose_wc = keyfrm->get_pose_wc();
        for (int r = 0; r < 4; ++r)
            for (int c = 0; c < 4; ++c) {
                kf.pose_cw[4 * r + c] = pose_cw(r, c);
                kf.pose_wc[4 * r + c] = pose_wc(r, c);
            }
        const camera::base* cam = keyfrm->camera_;
        switch (cam->model_type_) {
            case camera::model_type_t::Perspective: intrinsics<camera::perspective>(cam); break;
            case camera::model_type_t::Fisheye: intrinsics<camera::fisheye>(cam); break;
            case camera::model_type_t::RadialDivision: intrinsics<camera::radial_division>(cam); break;
            case camera::model_type_t::Equirectangular: break;
        }
        kf.model = cam->model_type_ == camera::model_type_t::Equirectangular ? 1 : 0;
        kf.focal_x_baseline = cam->focal_x_baseline_;
        kf.true_baseline = cam->true_baseline_;
        kf.cols = cam->cols_;
        kf.rows = cam->rows_;
        const feature::orb_params* prm = keyfrm->orb_params_;
        kf.scale_factor = prm->scale_factor_;
        kf.num_levels = static_cast<int32_t>(prm->scale_factors_.size());
        kf.scale_factors = prm->scale_factors_.data();
        kf.level_sigma_sq = prm->level_sigma_sq_.data();
        const auto& obs = keyfrm->frm_obs_;
        const size_t n = obs.undist_keypts_.size();
        x.resize(n); y.resize(n); octave.resize(n); bearing.resize(3 * n); no_landmark.resize(n);
        const auto lms = keyfrm->get_landmarks();
        for (size_t i = 0; i < n; ++i) {
            x[i] = obs.undist_keypts_[i].pt.x;
            y[i] = obs.undist_keypts_[i].pt.y;
            octave[i] = obs.undist_keypts_[i].octave;
            for (int k = 0; k < 3; ++k) bearing[3 * i + k] = obs.bearings_.at(i)(k);
            no_landmark[i] = !lms.at(i);  // robust.cc:44-48, 66-69
        }
        if (bow) node = b200_gather::node_of(keyfrm->bow_feat_vec_, n);
        kf.n_keypoints = static_cast<int32_t>(n);
        kf.x = x.data(); kf.y = y.data(); kf.octave = octave.data(); kf.bearings = bearing.data();
        kf.x_right = obs.stereo_x_right_.empty() ? nullptr : obs.stereo_x_right_.data();
        kf.depth = obs.depths_.empty() ? nullptr : obs.depths_.data();
    }
};

}  // namespace

void create_new_landmarks_b200(data::map_database* map_db, const std::shared_ptr<data::keyframe>& cur_keyfrm, unsigned int num_covisibilities,
                               bool use_baseline_dist_thr_ratio, double baseline_dist_thr_ratio, double baseline_dist_thr, float residual_rad_thr,
                               bool use_bow, module::local_map_cleaner* local_map_cleaner, std::atomic<bool>& abort_create_new_landmarks) {
    const auto cur_covisibilities = cur_keyfrm->graph_node_->get_top_n_covisibilities(num_covisibilities);
    const Vec3_t cur_cam_center = cur_keyfrm->get_trans_wc();
    // the baseline test (mapping_module.cc): keep the neighbours it passes, in covisibility order
    std::vector<std::shared_ptr<data::keyframe>> nghs;
    for (const auto& ngh_keyfrm : cur_covisibilities) {
        const double baseline_dist = (ngh_keyfrm->get_trans_wc() - cur_cam_center).norm();
        if (use_baseline_dist_thr_ratio) {
            const float median_scale_in_ngh = ngh_keyfrm->camera_->model_type_ == camera::model_type_t::Equirectangular
                                                  ? ngh_keyfrm->compute_median_distance()
                                                  : ngh_keyfrm->compute_median_depth(true);
            if (baseline_dist < baseline_dist_thr_ratio * median_scale_in_ngh) continue;
        }
        else if (baseline_dist < baseline_dist_thr) {
            continue;
        }
        nghs.push_back(ngh_keyfrm);
    }
    if (nghs.empty() || abort_create_new_landmarks) return;

    tri_view cur;
    cur.fill(cur_keyfrm, use_bow);
    std::vector<tri_view> views(nghs.size());
    std::vector<b200_new_landmarks_neighbour_t> nb(nghs.size());
    for (size_t r = 0; r < nghs.size(); ++r) {
        const auto& ngh_keyfrm = nghs[r];
        views[r].fill(ngh_keyfrm, use_bow);
        b200_new_landmarks_neighbour_t& N = nb[r];
        N = b200_new_landmarks_neighbour_t{};
        N.keyfrm = &views[r].kf;
        N.desc = ngh_keyfrm->frm_obs_.descriptors_.data;
        N.valid = views[r].no_landmark.data();
        N.node = use_bow ? views[r].node.data() : nullptr;
        const Mat33_t E_ngh_to_cur = solve::essential_solver::create_E_21(ngh_keyfrm->get_rot_cw(), ngh_keyfrm->get_trans_cw(),
                                                                          cur_keyfrm->get_rot_cw(), cur_keyfrm->get_trans_cw());
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) N.E_12[3 * i + j] = E_ngh_to_cur(i, j);
        Vec3_t epiplane_in_keyfrm_2;  // robust.cc:22-27
        const bool valid_epiplane = ngh_keyfrm->camera_->reproject_to_bearing(ngh_keyfrm->get_rot_cw(), ngh_keyfrm->get_trans_cw(), cur_cam_center,
                                                                              epiplane_in_keyfrm_2);
        for (int k = 0; k < 3; ++k) N.epiplane_in_keyfrm_2[k] = epiplane_in_keyfrm_2(k);
        N.valid_epiplane = valid_epiplane ? 1 : 0;
    }
    const size_t n1 = cur.x.size();
    std::vector<int32_t> created_rank(n1), created_idx(2 * n1);
    std::vector<double> created_pos(3 * n1);
    b200_new_landmarks_problem_t P{};
    P.keyfrm = &cur.kf;
    P.desc = cur_keyfrm->frm_obs_.descriptors_.data;
    P.valid = cur.no_landmark.data();
    P.node = use_bow ? cur.node.data() : nullptr;
    P.n_neighbours = static_cast<int32_t>(nb.size());
    P.neighbours = nb.data();
    P.created_rank = created_rank.data();
    P.created_idx = created_idx.data();
    P.created_pos_w = created_pos.data();
    // matchers of create_new_landmarks: lowe_ratio 0.95, no orientation check; triangulator: 1 degree
    if (b200_create_new_landmarks(mapping_matcher(), 1, &P, 0.95f, residual_rad_thr, 1.0f, 0) != B200_OK)
        throw std::runtime_error(b200_last_error());

    // triangulate_with_two_keyframes, in creation order
    std::lock_guard<std::mutex> lock(data::map_database::mtx_database_);
    for (int32_t c = 0; c < P.n_created; ++c) {
        const auto& ngh_keyfrm = nghs.at(created_rank[c]);
        const unsigned int idx_1 = created_idx[2 * c], idx_2 = created_idx[2 * c + 1];
        const Vec3_t pos_w(created_pos[3 * c], created_pos[3 * c + 1], created_pos[3 * c + 2]);
        auto lm = std::make_shared<data::landmark>(map_db->next_landmark_id_++, pos_w, cur_keyfrm);
        lm->connect_to_keyframe(cur_keyfrm, idx_1);
        lm->connect_to_keyframe(ngh_keyfrm, idx_2);
        lm->compute_descriptor();
        lm->update_mean_normal_and_obs_scale_variance();
        map_db->add_landmark(lm);
        local_map_cleaner->add_fresh_landmark(lm);
    }
}

}  // namespace stella_vslam
