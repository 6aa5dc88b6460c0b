// Drop-in replacement for src/stella_vslam/solve/pnp_solver.cc (same header, same members): link this translation unit instead of the
// original one.  The constructor fills the header's members as the reference does (max_cos_errors_ with util::cos); find_via_ransac
// returns early exactly where the reference does, without touching the engine, and otherwise draws its max_num_iter minimal sets with
// the reference's own util::create_random_array on random_engine_, so the sequence is the reference's whatever the standard library;
// EPnP, the scoring and the selection run on the device (b200_pnp_ransac).  The static compute_pose (also marker_detector::base's)
// calls b200_epnp_compute_pose.
//
// The header keeps no octaves or scale factors, only max_cos_errors_; the per-match scale factor the device needs is kept in a side
// table keyed by `this` (as orb_extractor_b200.cc keeps its handle).  Each thread that calls the solver gets its own b200_lba_t handle.
// Deviations: a hypothesis whose compute_pose writes no pose is rejected (the reference rescores the previous pose, which cannot win,
// or reads uninitialised memory for hypothesis 0); Eigen's vectorised summation order is not reproduced (DESIGN.md section 8).
#include "stella_vslam/solve/pnp_solver.h"
#include "stella_vslam/util/random_array.h"
#include "stella_vslam/util/trigonometric.h"

#include <spdlog/spdlog.h>

#include <cassert>
#include <cmath>
#include <mutex>
#include <stdexcept>
#include <unordered_map>
#include <vector>

#include "b200vslam.h"

namespace stella_vslam {
namespace solve {

namespace {
std::mutex g_mtx;
std::unordered_map<const pnp_solver*, std::vector<float>> g_match_scale;  // scale_factors.at(octaves.at(i)) per match

struct thread_handle {
    b200_lba_t h = nullptr;
    ~thread_handle() {
        if (h) b200_lba_destroy(h);
    }
};

b200_lba_t lba_handle() {
    thread_local thread_handle t;
    if (!t.h && b200_lba_create(0, &t.h) != B200_OK) throw std::runtime_error(b200_last_error());
    return t.h;
}

std::vector<double> flatten(const eigen_alloc_vector<Vec3_t>& v) {
    std::vector<double> out(3 * v.size());
    for (size_t i = 0; i < v.size(); ++i)
        for (int k = 0; k < 3; ++k) out[3 * i + k] = v[i](k);
    return out;
}
}  // namespace

pnp_solver::pnp_solver(const eigen_alloc_vector<Vec3_t>& valid_bearings,
                       const std::vector<int>& octaves,
                       const eigen_alloc_vector<Vec3_t>& valid_points,
                       const std::vector<float>& scale_factors,
                       const unsigned int min_num_inliers,
                       const bool use_fixed_seed,
                       const unsigned int gauss_newton_num_iter)
    : num_matches_(valid_bearings.size()), valid_bearings_(valid_bearings),
      valid_points_(valid_points), min_num_inliers_(min_num_inliers),
      random_engine_(util::create_random_engine(use_fixed_seed)),
      gauss_newton_num_iter_(gauss_newton_num_iter) {
    spdlog::trace("CONSTRUCT: solve::pnp_solver (b200)");
    max_cos_errors_.resize(num_matches_);
    std::vector<float> match_scale(num_matches_);
    constexpr double max_rad_error = 1.0 * M_PI / 180.0;
    for (unsigned int i = 0; i < num_matches_; ++i) {
        match_scale.at(i) = scale_factors.at(octaves.at(i));
        max_cos_errors_.at(i) = util::cos(match_scale.at(i) * max_rad_error);
    }
    assert(num_matches_ == octaves.size());
    assert(num_matches_ == valid_points_.size());
    std::lock_guard<std::mutex> lock(g_mtx);
    g_match_scale[this] = std::move(match_scale);
}

pnp_solver::~pnp_solver() {
    spdlog::trace("DESTRUCT: solve::pnp_solver (b200)");
    std::lock_guard<std::mutex> lock(g_mtx);
    g_match_scale.erase(this);
}

void pnp_solver::find_via_ransac(const unsigned int max_num_iter, const bool recompute) {
    static constexpr unsigned int min_set_size = 4;
    if (num_matches_ < min_set_size || num_matches_ < min_num_inliers_) {
        solution_is_valid_ = false;
        return;
    }
    std::vector<int32_t> min_sets;
    min_sets.reserve(4 * (size_t)max_num_iter);
    for (unsigned int iter = 0; iter < max_num_iter; ++iter)
        for (const auto i : util::create_random_array(min_set_size, 0U, num_matches_ - 1, random_engine_)) min_sets.push_back(static_cast<int32_t>(i));
    std::vector<float> match_scale;
    {
        std::lock_guard<std::mutex> lock(g_mtx);
        match_scale = g_match_scale.at(this);
    }
    // one "level" per match: octave i selects the match's own scale factor
    std::vector<int32_t> octaves(num_matches_);
    for (unsigned int i = 0; i < num_matches_; ++i) octaves[i] = static_cast<int32_t>(i);
    const std::vector<double> bearings = flatten(valid_bearings_), points = flatten(valid_points_);
    std::vector<uint8_t> flags(num_matches_);
    b200_pnp_problem_t P{};
    P.n_matches = static_cast<int32_t>(num_matches_);
    P.bearings = bearings.data();
    P.points = points.data();
    P.octaves = octaves.data();
    P.num_levels = static_cast<int32_t>(num_matches_);
    P.scale_factors = match_scale.data();
    P.min_num_inliers = min_num_inliers_;
    P.gauss_newton_num_iter = gauss_newton_num_iter_;
    P.max_num_iter = max_num_iter;
    P.recompute = recompute ? 1 : 0;
    P.min_sets = min_sets.data();
    P.inlier_flags = flags.data();
    if (b200_pnp_ransac(lba_handle(), 1, &P) != B200_OK) throw std::runtime_error(b200_last_error());
    if (P.status != B200_OK) spdlog::warn("pnp_solver (b200): a Jacobi SVD hit its sweep bound; the solution is unreliable");
    solution_is_valid_ = P.valid != 0;
    is_inlier_match = std::vector<bool>(flags.begin(), flags.end());
    if (solution_is_valid_) {
        for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c) best_rot_cw_(r, c) = P.rot_cw[r * 3 + c];
            best_trans_cw_(r) = P.trans_cw[r];
        }
    }
}

double pnp_solver::compute_pose(const eigen_alloc_vector<Vec3_t>& bearing_vectors,
                                const eigen_alloc_vector<Vec3_t>& pos_ws,
                                Mat33_t& rot_cw, Vec3_t& trans_cw, const unsigned int num_iter) {
    const std::vector<double> bearings = flatten(bearing_vectors), points = flatten(pos_ws);
    b200_epnp_problem_t P{};
    P.n = static_cast<int32_t>(bearing_vectors.size());
    P.bearings = bearings.data();
    P.points = points.data();
    P.num_iter = num_iter;
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) P.rot_cw[r * 3 + c] = rot_cw(r, c);
        P.trans_cw[r] = trans_cw(r);
    }
    if (b200_epnp_compute_pose(lba_handle(), 1, &P) != B200_OK) throw std::runtime_error(b200_last_error());
    if (P.wrote) {
        for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c) rot_cw(r, c) = P.rot_cw[r * 3 + c];
            trans_cw(r) = P.trans_cw[r];
        }
    }
    return P.reproj_error;
}

}  // namespace solve
}  // namespace stella_vslam
