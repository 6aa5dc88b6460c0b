// optimize::transform_optimizer on the GPU: this translation unit REPLACES src/stella_vslam/optimize/transform_optimizer.cc when
// USE_B200 is set (link-time, like the graph optimiser).  It keeps the header, gathers the mutual pairs on the host by the rules of
// transform_optimizer.cc:58-94, makes one b200_transform_optimize call (steps 3-7: optimize(5), the outlier test, optimize(num_iter),
// the inlier count), nulls the entries of matched_lms_in_keyfrm_2 the device rejected and writes the Sim3 back through g2o::Sim3.
#include "stella_vslam/camera/base.h"
#include "stella_vslam/camera/perspective.h"
#include "stella_vslam/camera/fisheye.h"
#include "stella_vslam/camera/radial_division.h"
#include "stella_vslam/camera/equirectangular.h"
#include "stella_vslam/data/keyframe.h"
#include "stella_vslam/data/landmark.h"
#include "stella_vslam/feature/orb_params.h"
#include "stella_vslam/optimize/transform_optimizer.h"

#include <stdexcept>
#include <string>
#include <vector>

#include "b200vslam.h"

namespace stella_vslam {
namespace optimize {

namespace {
b200_lba_t handle() {
    static b200_lba_t h = [] {
        b200_lba_t x = nullptr;
        if (b200_lba_create(0, &x) != B200_OK) throw std::runtime_error(std::string("b200_lba_create: ") + b200_last_error());
        return x;
    }();
    return h;
}

// mutual_reproj_edge_wrapper.h: Perspective / Fisheye / RadialDivision use the perspective edges on undistorted keypoints
b200_camera_t to_b200(const camera::base* camera) {
    b200_camera_t cam{};
    switch (camera->model_type_) {
        case camera::model_type_t::Perspective: { const auto c = static_cast<const camera::perspective*>(camera); cam = {0, c->fx_, c->fy_, c->cx_, c->cy_, 0, 0, 0}; break; }
        case camera::model_type_t::Fisheye: { const auto c = static_cast<const camera::fisheye*>(camera); cam = {0, c->fx_, c->fy_, c->cx_, c->cy_, 0, 0, 0}; break; }
        case camera::model_type_t::RadialDivision: { const auto c = static_cast<const camera::radial_division*>(camera); cam = {0, c->fx_, c->fy_, c->cx_, c->cy_, 0, 0, 0}; break; }
        case camera::model_type_t::Equirectangular: { const auto c = static_cast<const camera::equirectangular*>(camera); cam = {1, 0, 0, 0, 0, 0, double(c->cols_), double(c->rows_)}; break; }
    }
    return cam;
}

void pose_of(const std::shared_ptr<data::keyframe>& kf, double* rot, double* trans) {
    const Mat33_t R = kf->get_rot_cw();
    const Vec3_t t = kf->get_trans_cw();
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) rot[3 * r + c] = R(r, c);
        trans[r] = t(r);
    }
}
}  // namespace

transform_optimizer::transform_optimizer(const bool fix_scale, const unsigned int num_iter) : fix_scale_(fix_scale), num_iter_(num_iter) {}

unsigned int transform_optimizer::optimize(const std::shared_ptr<data::keyframe>& keyfrm_1, const std::shared_ptr<data::keyframe>& keyfrm_2,
                                           std::vector<std::shared_ptr<data::landmark>>& matched_lms_in_keyfrm_2, ::g2o::Sim3& g2o_Sim3_12,
                                           const float chi_sq) const {
    // 3. the mutual pairs (:58-94)
    const auto lms_in_keyfrm_1 = keyfrm_1->get_landmarks();
    std::vector<unsigned int> idx1s;
    std::vector<float> obs_1, w1, obs_2, w2;
    std::vector<double> pos_w_2, pos_w_1;
    for (unsigned int idx1 = 0; idx1 < matched_lms_in_keyfrm_2.size(); ++idx1) {
        if (!matched_lms_in_keyfrm_2.at(idx1)) continue;
        const auto& lm_1 = lms_in_keyfrm_1.at(idx1);
        const auto& lm_2 = matched_lms_in_keyfrm_2.at(idx1);
        if (!lm_1 || !lm_2) continue;
        if (lm_1->will_be_erased() || lm_2->will_be_erased()) continue;
        const auto idx2 = lm_2->get_index_in_keyframe(keyfrm_2);
        if (idx2 < 0) continue;
        const auto& kp1 = keyfrm_1->frm_obs_.undist_keypts_.at(idx1);
        const auto& kp2 = keyfrm_2->frm_obs_.undist_keypts_.at(idx2);
        obs_1.push_back(kp1.pt.x);
        obs_1.push_back(kp1.pt.y);
        w1.push_back(keyfrm_1->orb_params_->inv_level_sigma_sq_.at(kp1.octave));
        obs_2.push_back(kp2.pt.x);
        obs_2.push_back(kp2.pt.y);
        w2.push_back(keyfrm_2->orb_params_->inv_level_sigma_sq_.at(kp2.octave));
        const Vec3_t p2 = lm_2->get_pos_in_world(), p1 = lm_1->get_pos_in_world();
        for (int k = 0; k < 3; ++k) {
            pos_w_2.push_back(p2(k));
            pos_w_1.push_back(p1(k));
        }
        idx1s.push_back(idx1);
    }

    b200_transform_problem_t P{};
    P.n_matches = (int32_t)idx1s.size();
    P.fix_scale = fix_scale_ ? 1 : 0;
    const auto& q = g2o_Sim3_12.rotation();
    P.sim3_12.q[0] = q.x(); P.sim3_12.q[1] = q.y(); P.sim3_12.q[2] = q.z(); P.sim3_12.q[3] = q.w();
    for (int k = 0; k < 3; ++k) P.sim3_12.t[k] = g2o_Sim3_12.translation()(k);
    P.sim3_12.s = g2o_Sim3_12.scale();
    pose_of(keyfrm_1, P.rot_1w, P.trans_1w);
    pose_of(keyfrm_2, P.rot_2w, P.trans_2w);
    P.cam_1 = to_b200(keyfrm_1->camera_);
    P.cam_2 = to_b200(keyfrm_2->camera_);
    P.obs_1 = obs_1.data(); P.inv_sigma_sq_1 = w1.data(); P.pos_w_2 = pos_w_2.data();
    P.obs_2 = obs_2.data(); P.inv_sigma_sq_2 = w2.data(); P.pos_w_1 = pos_w_1.data();
    std::vector<uint8_t> keep(idx1s.size() + 1);
    P.keep = keep.data();
    if (b200_transform_optimize(handle(), 1, &P, chi_sq, (int)num_iter_) != B200_OK)
        throw std::runtime_error(std::string("b200_transform_optimize: ") + b200_last_error());

    // the outlier tests' nulls (:115, :146) stand whether or not the second round ran
    for (size_t i = 0; i < idx1s.size(); ++i)
        if (!keep[i]) matched_lms_in_keyfrm_2.at(idx1s[i]) = nullptr;
    if (P.n_matches - P.n_outliers_round1 < 10) return 0;  // :121-123: g2o_Sim3_12 stays as the caller built it

    // 7. the result (:155)
    const auto& o = P.sim3_12_out;
    g2o_Sim3_12.rotation() = ::g2o::Quaternion(o.q[3], o.q[0], o.q[1], o.q[2]);
    for (int k = 0; k < 3; ++k) g2o_Sim3_12.translation()(k) = o.t[k];
    g2o_Sim3_12.scale() = o.s;
    return P.num_inliers;
}

}  // namespace optimize
}  // namespace stella_vslam
