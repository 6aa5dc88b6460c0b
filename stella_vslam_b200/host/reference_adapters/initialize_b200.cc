// Replacement bodies for initialize::perspective::initialize (src/stella_vslam/initialize/perspective.cc:32-81) and
// initialize::bearing_vector::initialize (bearing_vector.cc:26-56).  Compile this TU next to perspective.cc and bearing_vector.cc with
// both original definitions guarded by #ifndef USE_B200; the constructors, reconstruct_with_H / _F / _E, get_camera_matrix and all of
// base.cc stay in the reference's TUs (the reconstruct_* functions are then unused).  module::initializer then runs the whole attempt
// -- RANSAC, the rel_cost_H choice, the decomposition, the triangulation of every hypothesis and find_most_plausible_pose -- in one
// b200_initialize call.
//
// initialize() fills cur_camera_, cur_undist_keypts_, cur_bearings_, ref_cur_matches_ (and cur_cam_matrix_) as the reference does.  Each
// solver's engine is constructed per attempt with util::create_random_engine(use_fixed_seed_) and draws its minimal sets with the
// reference's own util::create_random_array, only when its RANSAC runs (8 matches for H and F, 5 for E).  base's members are left as the
// reference leaves them: rot_ref_to_cur_ / trans_ref_to_cur_ are zeroed once find_most_plausible_pose has run and rejected, set on
// success and untouched when RANSAC or the decomposition failed first; triangulated_pts_ / is_triangulated_ are set on success (points
// that are not triangulated are zeros; the reference leaves them uninitialised).  Each calling thread gets its own b200_lba_t handle.
// Deviations (DESIGN.md section 8): sums run left to right; Jacobi sweeps are bounded and reported at debug level.
#include "stella_vslam/data/frame.h"
#include "stella_vslam/initialize/bearing_vector.h"
#include "stella_vslam/initialize/perspective.h"
#include "stella_vslam/util/random_array.h"

#include <spdlog/spdlog.h>

#include <random>
#include <stdexcept>
#include <vector>

#include "b200vslam.h"
#include "track_params_b200.h"

namespace stella_vslam {
namespace initialize {

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

// num_iters calls of util::create_random_array(set_size, 0, n - 1) on a newly constructed solver engine
std::vector<int32_t> draw(unsigned int set_size, unsigned int n, unsigned int num_iters, bool use_fixed_seed) {
    std::mt19937 engine = util::create_random_engine(use_fixed_seed);
    std::vector<int32_t> sets;
    sets.reserve((size_t)set_size * num_iters);
    for (unsigned int it = 0; it < num_iters; ++it)
        for (const auto i : util::create_random_array(set_size, 0U, n - 1, engine)) sets.push_back(static_cast<int32_t>(i));
    return sets;
}

void put_frame(const std::vector<cv::KeyPoint>& kps, const eigen_alloc_vector<Vec3_t>& bearings, std::vector<float>& undist,
               std::vector<double>& b) {
    undist.resize(2 * kps.size());
    b.resize(3 * bearings.size());
    for (size_t i = 0; i < kps.size(); ++i) {
        undist[2 * i] = kps[i].pt.x;
        undist[2 * i + 1] = kps[i].pt.y;
    }
    for (size_t i = 0; i < bearings.size(); ++i)
        for (int k = 0; k < 3; ++k) b[3 * i + k] = bearings[i](k);
}

// The b200_initialize call of one attempt; the caller copies the outputs into base's members.
struct attempt {
    b200_init_problem_t P{};
    std::vector<float> undist_ref, undist_cur;
    std::vector<double> bearings_ref, bearings_cur, pts;
    std::vector<int32_t> matches, sets_H, sets_F, sets_E;
    std::vector<uint8_t> flags;

    void run(camera::base* ref_cam, const std::vector<cv::KeyPoint>& ref_kps, const eigen_alloc_vector<Vec3_t>& ref_bearings,
             camera::base* cur_cam, const std::vector<cv::KeyPoint>& cur_kps, const eigen_alloc_vector<Vec3_t>& cur_bearings,
             const std::vector<int>& ref_matches_with_cur, unsigned int num_ransac_iters, unsigned int min_num_triangulated,
             unsigned int min_num_valid_pts, float parallax_deg_thr, float reproj_err_thr) {
        fill_camera_intrinsics(ref_cam, P.cam_ref, P.img_bounds_ref);
        fill_camera_intrinsics(cur_cam, P.cam_cur, P.img_bounds_cur);
        put_frame(ref_kps, ref_bearings, undist_ref, bearings_ref);
        put_frame(cur_kps, cur_bearings, undist_cur, bearings_cur);
        matches.assign(ref_matches_with_cur.begin(), ref_matches_with_cur.end());
        if (matches.size() != ref_kps.size()) throw std::invalid_argument("initialize (b200): one match entry per ref keypoint");
        pts.assign(3 * ref_kps.size(), 0.0);
        flags.assign(ref_kps.size(), 0);
        P.n_ref = static_cast<int32_t>(ref_kps.size());
        P.n_cur = static_cast<int32_t>(cur_kps.size());
        P.undist_ref = undist_ref.data();
        P.bearings_ref = bearings_ref.data();
        P.undist_cur = undist_cur.data();
        P.bearings_cur = bearings_cur.data();
        P.ref_matches_with_cur = matches.data();
        P.num_ransac_iters = num_ransac_iters;
        P.min_num_triangulated = min_num_triangulated;
        P.min_num_valid_pts = min_num_valid_pts;
        P.parallax_deg_thr = parallax_deg_thr;
        P.reproj_err_thr = reproj_err_thr;
        P.min_sets_H = sets_H.empty() ? nullptr : sets_H.data();
        P.min_sets_F = sets_F.empty() ? nullptr : sets_F.data();
        P.min_sets_E = sets_E.empty() ? nullptr : sets_E.data();
        P.triangulated_pts = pts.data();
        P.triangulated_flags = flags.data();
        if (b200_initialize(lba_handle(), 1, &P) != B200_OK) throw std::runtime_error(b200_last_error());
        if (P.status != B200_OK) spdlog::debug("initialize (b200): a Jacobi SVD or RealSchur did not converge");
    }
};

unsigned int count_matches(const std::vector<int>& ref_matches_with_cur) {
    unsigned int n = 0;
    for (const int m : ref_matches_with_cur) n += 0 <= m;
    return n;
}
}  // namespace

#define B200_STORE_OUTPUTS(A)                                                                             \
    do {                                                                                                  \
        if ((A).P.n_hypotheses > 0) {                                                                     \
            for (int r = 0; r < 3; ++r) {                                                                 \
                for (int c = 0; c < 3; ++c) rot_ref_to_cur_(r, c) = (A).P.rot_ref_to_cur[3 * r + c];      \
                trans_ref_to_cur_(r) = (A).P.trans_ref_to_cur[r];                                         \
            }                                                                                             \
        }                                                                                                 \
        if ((A).P.succeeded) {                                                                            \
            triangulated_pts_.resize((A).pts.size() / 3);                                                 \
            for (size_t i = 0; i < triangulated_pts_.size(); ++i)                                         \
                triangulated_pts_[i] = Vec3_t((A).pts[3 * i], (A).pts[3 * i + 1], (A).pts[3 * i + 2]);    \
            is_triangulated_.assign((A).flags.begin(), (A).flags.end());                                  \
        }                                                                                                 \
    } while (0)

bool perspective::initialize(const data::frame& cur_frm, const std::vector<int>& ref_matches_with_cur) {
    cur_camera_ = cur_frm.camera_;
    cur_undist_keypts_ = cur_frm.frm_obs_.undist_keypts_;
    cur_bearings_ = cur_frm.frm_obs_.bearings_;
    ref_cur_matches_.clear();
    ref_cur_matches_.reserve(cur_frm.frm_obs_.undist_keypts_.size());
    for (unsigned int ref_idx = 0; ref_idx < ref_matches_with_cur.size(); ++ref_idx) {
        const auto cur_idx = ref_matches_with_cur.at(ref_idx);
        if (0 <= cur_idx) ref_cur_matches_.emplace_back(std::make_pair(ref_idx, cur_idx));
    }
    cur_cam_matrix_ = get_camera_matrix(cur_frm.camera_);

    attempt a;
    const unsigned int n = count_matches(ref_matches_with_cur);
    if (n >= 8) {  // homography_solver / fundamental_solver return before drawing below 8 matches
        a.sets_H = draw(4, n, num_ransac_iters_, use_fixed_seed_);
        a.sets_F = draw(8, n, num_ransac_iters_, use_fixed_seed_);
    }
    a.run(ref_camera_, ref_undist_keypts_, ref_bearings_, cur_camera_, cur_undist_keypts_, cur_bearings_, ref_matches_with_cur, num_ransac_iters_,
          min_num_triangulated_, min_num_valid_pts_, parallax_deg_thr_, reproj_err_thr_);
    B200_STORE_OUTPUTS(a);
    if (a.P.succeeded) spdlog::info("initialization succeeded with {}", a.P.model == B200_INIT_MODEL_H ? "H" : "F");
    return a.P.succeeded != 0;
}

bool bearing_vector::initialize(const data::frame& cur_frm, const std::vector<int>& ref_matches_with_cur) {
    cur_camera_ = cur_frm.camera_;
    cur_undist_keypts_ = cur_frm.frm_obs_.undist_keypts_;
    cur_bearings_ = cur_frm.frm_obs_.bearings_;
    ref_cur_matches_.clear();
    ref_cur_matches_.reserve(cur_frm.frm_obs_.undist_keypts_.size());
    for (unsigned int ref_idx = 0; ref_idx < ref_matches_with_cur.size(); ++ref_idx) {
        const auto cur_idx = ref_matches_with_cur.at(ref_idx);
        if (0 <= cur_idx) ref_cur_matches_.emplace_back(std::make_pair(ref_idx, cur_idx));
    }

    attempt a;
    const unsigned int n = count_matches(ref_matches_with_cur);
    if (n >= 5) a.sets_E = draw(5, n, num_ransac_iters_, use_fixed_seed_);  // essential_solver returns before drawing below 5
    a.run(ref_camera_, ref_undist_keypts_, ref_bearings_, cur_camera_, cur_undist_keypts_, cur_bearings_, ref_matches_with_cur, num_ransac_iters_,
          min_num_triangulated_, min_num_valid_pts_, parallax_deg_thr_, reproj_err_thr_);
    B200_STORE_OUTPUTS(a);
    if (a.P.succeeded) spdlog::info("initialization succeeded with E");
    return a.P.succeeded != 0;
}

#undef B200_STORE_OUTPUTS

}  // namespace initialize
}  // namespace stella_vslam
