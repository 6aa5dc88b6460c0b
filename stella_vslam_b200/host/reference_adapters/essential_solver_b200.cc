// Replacement body for solve::essential_solver::find_via_ransac (src/stella_vslam/solve/essential_solver.cc:15-102).  Compile this TU
// next to essential_solver.cc with the original definition guarded by #ifndef USE_B200; the constructor, compute_E_21_nonminimal,
// compute_E_21_minimal, decompose, create_E_21 and check_inliers stay in the reference's TU.  match::robust::match_frame_and_keyframe,
// and through it frame_tracker::robust_match_based_track and the relocaliser's robust-matcher option, then run both halves (the
// brute-force match and this RANSAC) on the device with no change of their own; so does equirectangular initialisation.
//
// find_via_ransac returns early exactly where the reference does, without touching the engine; otherwise it draws its max_num_iter
// minimal sets with the reference's own util::create_random_array on random_engine_ (so the sequence is the reference's whatever the
// standard library), then makes one b200_essential_ransac call (five-point solver, scoring, selection and the eight-point recompute on
// the device) and fills solution_is_valid_, best_cost_, best_E_21_ and is_inlier_match_ as the reference leaves them.  Each calling
// thread gets its own b200_lba_t handle.  Only the five-point minimal set is supported: every caller in the reference passes the
// default min_set_size = 5, and any other value throws std::invalid_argument.  Deviations (DESIGN.md section 8): Eigen's vectorised
// summation and blocked triangular-solve order are not reproduced; a RealSchur that does not converge gives no candidates.
#include "stella_vslam/solve/essential_solver.h"
#include "stella_vslam/util/random_array.h"

#include <spdlog/spdlog.h>

#include <stdexcept>
#include <vector>

#include "b200vslam.h"

namespace stella_vslam {
namespace solve {

namespace {
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
}  // namespace

void essential_solver::find_via_ransac(const unsigned int max_num_iter, const bool recompute, const unsigned int min_set_size) {
    if (min_set_size != 5) throw std::invalid_argument("essential_solver (b200): only the five-point minimal set is supported");
    const auto num_matches = static_cast<unsigned int>(matches_12_.size());
    if (num_matches < min_set_size) {
        solution_is_valid_ = false;
        return;
    }

    std::vector<double> b1(3 * (size_t)num_matches), b2(3 * (size_t)num_matches);
    for (unsigned int i = 0; i < num_matches; ++i) {
        const Vec3_t& x1 = bearings_1_.at(matches_12_.at(i).first);
        const Vec3_t& x2 = bearings_2_.at(matches_12_.at(i).second);
        for (int k = 0; k < 3; ++k) {
            b1[3 * i + k] = x1(k);
            b2[3 * i + k] = x2(k);
        }
    }
    std::vector<int32_t> min_sets((size_t)min_set_size * max_num_iter);
    for (unsigned int iter = 0; iter < max_num_iter; ++iter) {
        const auto indices = util::create_random_array(min_set_size, 0U, num_matches - 1, random_engine_);
        for (unsigned int i = 0; i < min_set_size; ++i) min_sets[(size_t)min_set_size * iter + i] = static_cast<int32_t>(indices.at(i));
    }

    std::vector<uint8_t> flags(num_matches);
    b200_essential_problem_t P{};
    P.n_matches = static_cast<int32_t>(num_matches);
    P.bearings_1 = b1.data();
    P.bearings_2 = b2.data();
    P.min_set_size = min_set_size;
    P.max_num_iter = max_num_iter;
    P.recompute = recompute ? 1 : 0;
    P.min_sets = min_sets.data();
    P.inlier_flags = flags.data();
    if (b200_essential_ransac(lba_handle(), 1, &P) != B200_OK) throw std::runtime_error(b200_last_error());
    if (P.status != B200_OK) spdlog::debug("essential_solver (b200): a RealSchur or Jacobi SVD did not converge");

    solution_is_valid_ = P.valid != 0;
    best_cost_ = P.best_cost;
    if (solution_is_valid_)
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) best_E_21_(r, c) = P.E_21[3 * r + c];
    is_inlier_match_ = std::vector<bool>(flags.begin(), flags.end());
}

}  // namespace solve
}  // namespace stella_vslam
