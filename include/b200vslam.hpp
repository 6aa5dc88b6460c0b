// b200vslam.hpp -- C++ host-side mirror of the reference's class surfaces on top of the C ABI (b200vslam.h).
//
// Header-only, no OpenCV/Eigen/g2o dependency: images are raw 8-bit buffers, keypoints are b200_keypoint_t.  The names,
// constructor arguments and error behaviour follow the reference so that the thin adapters in
// stella_vslam_b200/host/reference_adapters/ (which DO include the reference's headers) are one-liners:
//   b200::feature::orb_params      <->  stella_vslam::feature::orb_params      (feature/orb_params.h:11-54)
//   b200::feature::orb_extractor   <->  stella_vslam::feature::orb_extractor   (feature/orb_extractor.h:46-122)
//   b200::match::robust            <->  stella_vslam::match::robust            (match/robust.h, match/base.h:81-91)
//   b200::match::projection / fuse / area / bow_tree / stereo  <->  match/projection.h, fuse.h, area.h, bow_tree.h, stereo.h
//   b200::optimize::local_bundle_adjuster <-> stella_vslam::optimize::local_bundle_adjuster (optimize/local_bundle_adjuster.h:15-24)
//   b200::optimize::pose_optimizer        <-> stella_vslam::optimize::pose_optimizer        (optimize/pose_optimizer.h:24-40)
//   b200::optimize::transform_optimizer   <-> stella_vslam::optimize::transform_optimizer   (optimize/transform_optimizer.h:17-48)
//   b200::util::stereo_rectifier          <-> stella_vslam::util::stereo_rectifier          (util/stereo_rectifier.h:14-46)
//   b200::solve::pnp_solver               <-> stella_vslam::solve::pnp_solver               (solve/pnp_solver.h:13-142)
//   b200::solve::essential_solver         <-> stella_vslam::solve::essential_solver         (solve/essential_solver.h)
//   b200::initialize::perspective / bearing_vector <-> stella_vslam::initialize::perspective / bearing_vector (initialize/*.h)
//   b200::module::depth_landmarks         <-> the depth branches of module::keyframe_inserter and module::initializer
//   b200::module::local_map_cleaner       <-> stella_vslam::module::local_map_cleaner::remove_redundant_keyframes (module/local_map_cleaner.h)
#pragma once

#include <cmath>
#include <cstdint>
#include <random>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "b200vslam.h"

namespace b200 {

inline void check(int rc, const char* what) {
    if (rc != B200_OK) throw std::runtime_error(std::string(what) + ": " + b200_last_error());
}

namespace feature {

enum class descriptor_type { ORB, HASH_SIFT };  // feature/orb_extractor.h:17-44

struct orb_params {  // feature/orb_params.cc:12-71 (float recurrences, not pow)
    std::string name_;
    float scale_factor_ = 1.2f;
    float log_scale_factor_;
    unsigned int num_levels_ = 8, ini_fast_thr_ = 20, min_fast_thr_ = 7;
    std::vector<float> scale_factors_, inv_scale_factors_, level_sigma_sq_, inv_level_sigma_sq_;

    explicit orb_params(const std::string& name = "default ORB feature extraction setting", float scale_factor = 1.2f,
                        unsigned int num_levels = 8, unsigned int ini_fast_thr = 20, unsigned int min_fast_thr = 7)
        : name_(name), scale_factor_(scale_factor), log_scale_factor_(std::log(scale_factor)), num_levels_(num_levels),
          ini_fast_thr_(ini_fast_thr), min_fast_thr_(min_fast_thr) {
        scale_factors_.assign(num_levels, 1.0f);
        inv_scale_factors_.assign(num_levels, 1.0f);
        level_sigma_sq_.assign(num_levels, 1.0f);
        inv_level_sigma_sq_.assign(num_levels, 1.0f);
        float s = 1.0f;
        for (unsigned int l = 1; l < num_levels; ++l) {
            scale_factors_[l] = scale_factor * scale_factors_[l - 1];
            inv_scale_factors_[l] = (1.0f / scale_factor) * inv_scale_factors_[l - 1];
            s = scale_factor * s;
            level_sigma_sq_[l] = s * s;
            inv_level_sigma_sq_[l] = 1.0f / (s * s);
        }
    }
};

class orb_extractor {
public:
    // orb_extractor(const orb_params*, unsigned min_area, descriptor_type, mask_rects) -- orb_extractor.h:51-54
    orb_extractor(const orb_params* params, unsigned int min_area, descriptor_type desc_type = descriptor_type::ORB,
                  const std::vector<std::vector<float>>& mask_rects = {}, int device = 0, int max_batch = 1)
        : orb_params_(params), mask_rects_(mask_rects) {
        if (desc_type == descriptor_type::HASH_SIFT) throw std::runtime_error("cuda_efficient_features is not available");  // orb_extractor.cc:121
        b200_orb_params_t p;
        b200_orb_default_params(&p);
        p.scale_factor = params->scale_factor_;
        p.num_levels = (int32_t)params->num_levels_;
        p.ini_fast_thr = (int32_t)params->ini_fast_thr_;
        p.min_fast_thr = (int32_t)params->min_fast_thr_;
        p.min_area = min_area;
        for (const auto& r : mask_rects) flat_rects_.insert(flat_rects_.end(), r.begin(), r.begin() + 4);
        p.n_mask_rects = (int32_t)mask_rects.size();
        p.mask_rects = flat_rects_.empty() ? nullptr : flat_rects_.data();
        p.device = device;
        p.max_batch = max_batch;
        check(b200_orb_create(&p, &h_), "b200_orb_create");
    }
    ~orb_extractor() { b200_orb_destroy(h_); }
    orb_extractor(const orb_extractor&) = delete;
    orb_extractor& operator=(const orb_extractor&) = delete;

    // extract(in_image, in_image_mask, keypts, out_descriptors) -- orb_extractor.h:60-61.  One CV_8UC1 frame in host memory;
    // descriptors come back as N x 32 bytes (cv::Mat(N, 32, CV_8U) layout).  Empty image -> silent return (orb_extractor.cc:30-32).
    void extract(const uint8_t* image, int width, int height, size_t pitch, const uint8_t* mask, size_t mask_pitch,
                 std::vector<b200_keypoint_t>& keypts, std::vector<uint8_t>& descriptors) {
        extract_batch(image, width, height, pitch, pitch * (size_t)height, 1, mask, mask_pitch, keypts, descriptors, counts_);
        keypts.resize(counts_.empty() ? 0 : counts_[0]);
        descriptors.resize(keypts.size() * 32);
    }
    // `batch` same-sized frames; frame f's results start at f * cap (cap = max_keypoints(width, height)).
    void extract_batch(const uint8_t* images, int width, int height, size_t pitch, size_t frame_stride, int batch, const uint8_t* mask,
                       size_t mask_pitch, std::vector<b200_keypoint_t>& keypts, std::vector<uint8_t>& descriptors, std::vector<int32_t>& counts) {
        keypts.clear();
        descriptors.clear();
        counts.assign(batch > 0 ? batch : 0, 0);
        if (!images || width == 0 || height == 0 || batch == 0) return;
        const int cap = max_keypoints(width, height);
        keypts.resize((size_t)cap * batch);
        descriptors.resize((size_t)cap * batch * 32);
        check(b200_orb_extract(h_, images, width, height, pitch, frame_stride, batch, mask, mask_pitch, keypts.data(), descriptors.data(), cap,
                               counts.data()),
              "b200_orb_extract");
    }
    int max_keypoints(int width, int height) const { return b200_orb_max_keypoints(h_, width, height); }
    // image_pyramid_ (orb_extractor.h:71): level >= 1 of the last extract, tightly packed
    std::vector<uint8_t> pyramid_level(int frame, int level, int* w = nullptr, int* hgt = nullptr) const {
        int lw = 0, lh = 0;
        check(b200_orb_level_info(h_, level, &lw, &lh, nullptr, nullptr), "b200_orb_level_info");
        std::vector<uint8_t> out((size_t)lw * lh);
        check(b200_orb_pyramid_level_host(h_, frame, level, out.data(), (size_t)lw), "b200_orb_pyramid_level_host");
        if (w) *w = lw;
        if (hgt) *hgt = lh;
        return out;
    }
    // system::create_RGBD_frame after the extraction (system.cc:467-530), b200_rgbd_depths: the first n_frames frames of the last
    // extract; frame f's results start at f * cap (cap = max_keypoints(width, height)), counts[f] = its keypoints.  depth_type:
    // B200_DEPTH_16UC1 or B200_DEPTH_32FC1 (cv::Mat::type()); the maps are host buffers of the extracted frames' size.
    struct rgbd_frames {
        int cap = 0;
        std::vector<b200_keypoint_t> undist_keypts;
        std::vector<double> bearings;
        std::vector<float> depths, x_right;
        std::vector<int32_t> counts;
    };
    rgbd_frames rgbd_depths(const b200_camera_intrinsics_t& cam, double focal_x_baseline, double depthmap_factor, int depth_type,
                            const void* depth_maps, int width, int height, size_t pitch, size_t frame_stride, int n_frames) const {
        rgbd_frames r;
        r.cap = max_keypoints(width, height);
        check(r.cap < 0 ? r.cap : B200_OK, "b200_orb_max_keypoints");
        const size_t m = (size_t)r.cap * (n_frames > 0 ? n_frames : 0);
        r.undist_keypts.resize(m);
        r.bearings.resize(3 * m);
        r.depths.resize(m);
        r.x_right.resize(m);
        r.counts.assign(n_frames > 0 ? n_frames : 0, 0);
        check(b200_rgbd_depths(h_, n_frames, &cam, focal_x_baseline, depthmap_factor, depth_type, depth_maps, width, height, pitch, frame_stride, r.cap,
                               r.undist_keypts.data(), r.bearings.data(), r.depths.data(), r.x_right.data(), r.counts.data()),
              "b200_rgbd_depths");
        return r;
    }
    b200_orb_t handle() const { return h_; }

    const orb_params* orb_params_;                  // orb_extractor.h:64
    std::vector<std::vector<float>> mask_rects_;    // orb_extractor.h:68

private:
    b200_orb_t h_ = nullptr;
    std::vector<float> flat_rects_;
    std::vector<int32_t> counts_;
};

}  // namespace feature

namespace match {

constexpr unsigned int HAMMING_DIST_THR_LOW = 50, HAMMING_DIST_THR_HIGH = 100, MAX_HAMMING_DIST = 256;  // match/base.h:15-17

class base {  // match/base.h:81-91
public:
    base(float lowe_ratio, bool check_orientation) : lowe_ratio_(lowe_ratio), check_orientation_(check_orientation) {}
    virtual ~base() = default;

protected:
    const float lowe_ratio_;
    const bool check_orientation_;
};

class robust final : public base {
public:
    robust(float lowe_ratio, bool check_orientation, int device = 0) : base(lowe_ratio, check_orientation) {
        check(b200_matcher_create(device, &h_), "b200_matcher_create");
    }
    ~robust() override { b200_matcher_destroy(h_); }
    // brute_force_match (match/robust.cc:232-328): frame keypoints (descriptors 32 B each, angles with a byte stride) against the
    // keyframe's; keyfrm_has_landmark[i] != 0 <=> lms_2[i] && !will_be_erased().  Returns (idx_1, idx_2) sorted by idx_1.
    unsigned int brute_force_match(const uint8_t* frm_desc, const void* frm_angles, size_t frm_angle_stride, int n1, const uint8_t* keyfrm_desc,
                                   const void* keyfrm_angles, size_t keyfrm_angle_stride, const uint8_t* keyfrm_has_landmark, int n2,
                                   std::vector<std::pair<int, int>>& matches) const {
        matches.clear();
        if (n1 <= 0 || n2 <= 0) return 0;
        std::vector<int32_t> pairs((size_t)2 * n1);
        const int32_t off = 0;
        int32_t n = 0;
        check(b200_match_bruteforce(h_, 1, frm_desc, frm_angles, frm_angle_stride, &off, &n1, keyfrm_desc, keyfrm_angles, keyfrm_angle_stride,
                                    keyfrm_has_landmark, &off, &n2, lowe_ratio_, check_orientation_ ? 1 : 0, pairs.data(), n1, &n),
              "b200_match_bruteforce");
        matches.reserve(n);
        for (int i = 0; i < n; ++i) matches.emplace_back(pairs[2 * i], pairs[2 * i + 1]);
        return (unsigned int)n;
    }

    // match_for_triangulation (match/robust.cc:14-146): the problem carries bearings, E_12, the epipole and the "has no landmark"
    // masks; returns matched_idx_pairs sorted by idx_1.
    unsigned int match_for_triangulation(b200_pairs_problem_t& problem, std::vector<std::pair<unsigned int, unsigned int>>& matched_idx_pairs) const {
        return run_pairs(h_, problem, B200_PAIRS_TRIANGULATION, lowe_ratio_, check_orientation_, matched_idx_pairs);
    }
    b200_matcher_t handle() const { return h_; }

    static unsigned int run_pairs(b200_matcher_t h, b200_pairs_problem_t& problem, int variant, float lowe_ratio, bool check_orientation,
                                  std::vector<std::pair<unsigned int, unsigned int>>& out) {
        std::vector<int32_t> match((size_t)(problem.n1 > 0 ? problem.n1 : 1), -1);
        problem.match_out = match.data();
        check(b200_match_pairs(h, 1, &problem, variant, lowe_ratio, check_orientation ? 1 : 0, 0), "b200_match_pairs");
        out.clear();
        for (int i = 0; i < problem.n1; ++i)
            if (match[i] >= 0) out.emplace_back((unsigned int)i, (unsigned int)match[i]);
        problem.match_out = nullptr;
        return (unsigned int)problem.n_matches;
    }

private:
    b200_matcher_t h_ = nullptr;
};

// One matcher handle (stream + staging) shared by the guided / all-pairs / stereo mirrors below.
class device_matcher {
public:
    explicit device_matcher(int device = 0) { check(b200_matcher_create(device, &h_), "b200_matcher_create"); }
    ~device_matcher() { b200_matcher_destroy(h_); }
    device_matcher(const device_matcher&) = delete;
    device_matcher& operator=(const device_matcher&) = delete;
    b200_matcher_t get() const { return h_; }

private:
    b200_matcher_t h_ = nullptr;
};

// match::projection (match/projection.h:24-67).  The adapter fills one b200_guided_problem_t per call (landmarks in the reference's
// order, reprojected; see reference_adapters/projection_b200.cc); match_out / n_matches come back in the struct.
class projection final : public base {
public:
    explicit projection(float lowe_ratio = 0.6f, bool check_orientation = true, int device = 0) : base(lowe_ratio, check_orientation), m_(device) {}
    unsigned int match_frame_and_landmarks(b200_guided_problem_t& p) const { return run(p, B200_GUIDED_LANDMARKS, HAMMING_DIST_THR_HIGH, false); }
    unsigned int match_current_and_last_frames(b200_guided_problem_t& p) const {
        return run(p, B200_GUIDED_LAST_FRAME, HAMMING_DIST_THR_HIGH, check_orientation_);
    }
    unsigned int match_frame_and_keyframe(b200_guided_problem_t& p, unsigned int hamm_dist_thr) const {
        return run(p, B200_GUIDED_LAST_FRAME, hamm_dist_thr, check_orientation_);
    }
    unsigned int match_by_Sim3_transform(b200_guided_problem_t& p) const { return run(p, B200_GUIDED_LAST_FRAME, HAMMING_DIST_THR_LOW, false); }
    // match_keyframes_mutually: p12 = landmarks of keyframe 1 searched in keyframe 2, p21 the other direction; mutual[i] = idx_2 or -1
    unsigned int match_keyframes_mutually(b200_guided_problem_t& p12, b200_guided_problem_t& p21, std::vector<int32_t>& mutual) const {
        b200_guided_problem_t both[2] = {p12, p21};
        check(b200_match_guided(m_.get(), 2, both, B200_GUIDED_INDEPENDENT, HAMMING_DIST_THR_HIGH, lowe_ratio_, 0, 0), "b200_match_guided");
        mutual.assign((size_t)(p12.n_queries > 0 ? p12.n_queries : 1), -1);
        int32_t n = 0;
        check(b200_match_cross_check(p12.match_out, p12.n_queries, p21.match_out, p21.n_queries, mutual.data(), &n), "b200_match_cross_check");
        mutual.resize((size_t)p12.n_queries);
        return (unsigned int)n;
    }

private:
    unsigned int run(b200_guided_problem_t& p, int mode, unsigned int thr, bool orientation) const {
        check(b200_match_guided(m_.get(), 1, &p, mode, thr, lowe_ratio_, orientation ? 1 : 0, 0), "b200_match_guided");
        return (unsigned int)p.n_matches;
    }
    device_matcher m_;
};

class fuse final : public base {  // match/fuse.h, fuse.cc:12-154
public:
    explicit fuse(float lowe_ratio = 0.6f, bool check_orientation = true, int device = 0) : base(lowe_ratio, check_orientation), m_(device) {}
    unsigned int detect_duplication(b200_guided_problem_t& p) const {
        check(b200_match_guided(m_.get(), 1, &p, B200_GUIDED_FUSE, HAMMING_DIST_THR_LOW, lowe_ratio_, 0, 0), "b200_match_guided");
        return (unsigned int)p.n_matches;
    }

private:
    device_matcher m_;
};

class area final : public base {  // match/area.h, area.cc:8-98
public:
    explicit area(float lowe_ratio = 0.9f, bool check_orientation = true, int device = 0) : base(lowe_ratio, check_orientation), m_(device) {}
    unsigned int match_in_consistent_area(b200_guided_problem_t& p) const {
        check(b200_match_guided(m_.get(), 1, &p, B200_GUIDED_AREA, HAMMING_DIST_THR_LOW, lowe_ratio_, check_orientation_ ? 1 : 0, 0), "b200_match_guided");
        return (unsigned int)p.n_matches;
    }

private:
    device_matcher m_;
};

class bow_tree final : public base {  // match/bow_tree.h, bow_tree.cc:11-366 (node1 / node2 = BoW node of every keypoint)
public:
    explicit bow_tree(float lowe_ratio = 0.6f, bool check_orientation = true, int device = 0) : base(lowe_ratio, check_orientation), m_(device) {}
    unsigned int match_for_triangulation(b200_pairs_problem_t& p, std::vector<std::pair<unsigned int, unsigned int>>& matched_idx_pairs) const {
        return robust::run_pairs(m_.get(), p, B200_PAIRS_TRIANGULATION, lowe_ratio_, check_orientation_, matched_idx_pairs);
    }
    // match_frame_and_keyframe / match_keyframes: (row, candidate) pairs; the adapter maps them to matched_lms_in_frm / _in_keyfrm_1
    unsigned int match_frame_and_keyframe(b200_pairs_problem_t& p, std::vector<std::pair<unsigned int, unsigned int>>& pairs) const {
        return robust::run_pairs(m_.get(), p, B200_PAIRS_BOW, lowe_ratio_, check_orientation_, pairs);
    }
    unsigned int match_keyframes(b200_pairs_problem_t& p, std::vector<std::pair<unsigned int, unsigned int>>& pairs) const {
        return robust::run_pairs(m_.get(), p, B200_PAIRS_BOW, lowe_ratio_, check_orientation_, pairs);
    }

private:
    device_matcher m_;
};

// match::stereo (match/stereo.h:17-101): built from the two extractors whose pyramids stay on the device (system.cc:443)
class stereo {
public:
    stereo(const feature::orb_extractor& left, const feature::orb_extractor& right, const std::vector<b200_keypoint_t>& keypts_left,
           const std::vector<b200_keypoint_t>& keypts_right, const std::vector<uint8_t>& descs_left, const std::vector<uint8_t>& descs_right,
           float focal_x_baseline, float true_baseline, int frame_left = 0, int frame_right = 0, int device = 0)
        : left_(left), right_(right), kl_(keypts_left), kr_(keypts_right), dl_(descs_left), dr_(descs_right), fxb_(focal_x_baseline),
          baseline_(true_baseline), fl_(frame_left), fr_(frame_right), m_(device) {}
    void compute(std::vector<float>& stereo_x_right, std::vector<float>& depths) const {
        stereo_x_right.assign(kl_.size(), -1.0f);
        depths.assign(kl_.size(), -1.0f);
        int32_t n = 0;
        check(b200_stereo_compute(m_.get(), left_.handle(), fl_, right_.handle(), fr_, kl_.data(), dl_.data(), (int)kl_.size(), kr_.data(), dr_.data(),
                                  (int)kr_.size(), fxb_, baseline_, stereo_x_right.data(), depths.data(), &n),
              "b200_stereo_compute");
    }

private:
    const feature::orb_extractor &left_, &right_;
    const std::vector<b200_keypoint_t>&kl_, &kr_;
    const std::vector<uint8_t>&dl_, &dr_;
    float fxb_, baseline_;
    int fl_, fr_;
    device_matcher m_;
};

}  // namespace match

namespace module {

// The depth-seeded landmarks of stereo / RGB-D keyframes (b200_depth_landmarks): keyframe_inserter::create_new_keyframe's depth branch
// (mode B200_DEPTH_LM_KEYFRAME, module/keyframe_inserter.cc:160-212) and initializer::create_map_for_stereo's landmark loop
// (B200_DEPTH_LM_INITIAL, module/initializer.cc:363-387) for many frames in one call.
class depth_landmarks {
public:
    struct result {
        std::vector<int32_t> idx;  // keypoint of each created landmark, in creation order
        std::vector<double> pos_w, mean_normal;
        std::vector<float> min_valid_dist, max_valid_dist;
        int32_t status = B200_OK;
    };
    explicit depth_landmarks(int device = 0) : m_(device) {}
    // Problems with their inputs filled (the output pointers are set here).  Throws on the first rejected problem unless
    // throw_on_error is false; then result::status tells which ones ran.
    std::vector<result> create(std::vector<b200_depth_landmarks_problem_t> problems, bool throw_on_error = true) {
        std::vector<result> out(problems.size());
        for (size_t k = 0; k < problems.size(); ++k) {
            auto& p = problems[k];
            const size_t n = p.n_keypoints > 0 ? (size_t)p.n_keypoints : 0;
            auto& r = out[k];
            r.idx.resize(n);
            r.pos_w.resize(3 * n);
            r.mean_normal.resize(3 * n);
            r.min_valid_dist.resize(n);
            r.max_valid_dist.resize(n);
            p.created_idx = r.idx.data();
            p.pos_w = r.pos_w.data();
            p.mean_normal = r.mean_normal.data();
            p.min_valid_dist = r.min_valid_dist.data();
            p.max_valid_dist = r.max_valid_dist.data();
        }
        const int rc = b200_depth_landmarks(m_.get(), (int)problems.size(), problems.data());
        if (throw_on_error) check(rc, "b200_depth_landmarks");
        for (size_t k = 0; k < problems.size(); ++k) {
            const size_t c = (size_t)problems[k].n_created;
            auto& r = out[k];
            r.status = problems[k].status;
            r.idx.resize(c);
            r.pos_w.resize(3 * c);
            r.mean_normal.resize(3 * c);
            r.min_valid_dist.resize(c);
            r.max_valid_dist.resize(c);
        }
        return out;
    }

private:
    match::device_matcher m_;
};

// module::local_map_cleaner's keyframe culling (module/local_map_cleaner.cc:68-193) on gathered tables (b200_remove_redundant_keyframes),
// for many maps in one call.  The caller gathers each problem from get_top_n_covisibilities(top_n_covisibilities_to_search()), applies
// prepare_for_erasing to the removed ranks in rank order, and calls again for the ranks after a removed keyframe it could not erase.
class local_map_cleaner {
public:
    explicit local_map_cleaner(double redundant_obs_ratio_thr = 0.9, unsigned int top_n_covisibilities_to_search = 30, int device = 0)
        : redundant_obs_ratio_thr_(redundant_obs_ratio_thr), top_n_covisibilities_to_search_(top_n_covisibilities_to_search), m_(device) {}
    unsigned int top_n_covisibilities_to_search() const { return top_n_covisibilities_to_search_; }
    // Sets each problem's threshold, runs them and returns each n_removed; the per-rank results are in the problems' covisibilities.
    // The reference's early return (a negative threshold or top_n of 0) returns zeros without a call.
    std::vector<unsigned int> remove_redundant_keyframes(std::vector<b200_cull_problem_t>& problems) const {
        std::vector<unsigned int> n_removed(problems.size(), 0);
        if (redundant_obs_ratio_thr_ < 0.0 || top_n_covisibilities_to_search_ == 0 || problems.empty()) return n_removed;
        for (auto& p : problems) p.redundant_obs_ratio_thr = redundant_obs_ratio_thr_;
        check(b200_remove_redundant_keyframes(m_.get(), (int)problems.size(), problems.data()), "b200_remove_redundant_keyframes");
        for (size_t k = 0; k < problems.size(); ++k) n_removed[k] = (unsigned int)problems[k].n_removed;
        return n_removed;
    }

private:
    double redundant_obs_ratio_thr_;
    unsigned int top_n_covisibilities_to_search_;
    match::device_matcher m_;
};

}  // namespace module

namespace optimize {

class local_bundle_adjuster {  // optimize/local_bundle_adjuster_g2o.h:16-46 with Mapping.backend: "b200"
public:
    explicit local_bundle_adjuster(unsigned int num_first_iter = 5, unsigned int num_second_iter = 10, int device = 0)
        : num_first_iter_(num_first_iter), num_second_iter_(num_second_iter) {
        check(b200_lba_create(device, &h_), "b200_lba_create");
    }
    ~local_bundle_adjuster() { b200_lba_destroy(h_); }
    local_bundle_adjuster(const local_bundle_adjuster&) = delete;
    // steps 5-7 of local_bundle_adjuster_g2o::optimize on the flattened window; returns false when the abort flag was already set
    // (local_bundle_adjuster_g2o.cc:308-310), in which case nothing is written.
    bool optimize(const b200_lba_problem_t& problem, volatile uint8_t* force_stop_flag, std::vector<double>& pose_cw_out,
                  std::vector<double>& points_out, std::vector<uint8_t>& outlier_out, b200_lba_stats_t* stats = nullptr) const {
        pose_cw_out.resize((size_t)16 * problem.n_poses);
        points_out.resize((size_t)3 * problem.n_points);
        outlier_out.resize((size_t)problem.n_edges);
        const int rc = b200_lba_solve(h_, &problem, (int)num_first_iter_, (int)num_second_iter_, force_stop_flag, pose_cw_out.data(),
                                      points_out.data(), outlier_out.data(), stats);
        if (rc == B200_ERR_ABORTED) return false;
        check(rc, "b200_lba_solve");
        return true;
    }

    // many windows per launch sequence (b200_lba_solve_batch); ok[w] = false for windows whose flag was already set
    void optimize_batch(const std::vector<b200_lba_problem_t>& problems, const std::vector<volatile uint8_t*>& force_stop_flags,
                        std::vector<std::vector<double>>& pose_cw_out, std::vector<std::vector<double>>& points_out,
                        std::vector<std::vector<uint8_t>>& outlier_out, std::vector<bool>& ok) const {
        const size_t n = problems.size();
        pose_cw_out.resize(n); points_out.resize(n); outlier_out.resize(n);
        std::vector<double*> pp(n), qq(n);
        std::vector<uint8_t*> oo(n);
        std::vector<int32_t> status(n, 0);
        for (size_t w = 0; w < n; ++w) {
            pose_cw_out[w].resize((size_t)16 * problems[w].n_poses);
            points_out[w].resize((size_t)3 * problems[w].n_points);
            outlier_out[w].resize((size_t)(problems[w].n_edges > 0 ? problems[w].n_edges : 1));
            pp[w] = pose_cw_out[w].data(); qq[w] = points_out[w].data(); oo[w] = outlier_out[w].data();
        }
        const int rc = b200_lba_solve_batch(h_, (int)n, problems.data(), (int)num_first_iter_, (int)num_second_iter_,
                                            force_stop_flags.empty() ? nullptr : force_stop_flags.data(), pp.data(), qq.data(), oo.data(), nullptr, status.data());
        ok.assign(n, true);
        for (size_t w = 0; w < n; ++w)
            if (status[w] == B200_ERR_ABORTED) ok[w] = false;
            else if (status[w] != B200_OK) check(status[w], "b200_lba_solve_batch");
        if (rc != B200_OK && rc != B200_ERR_ABORTED) check(rc, "b200_lba_solve_batch");
    }

private:
    const unsigned int num_first_iter_, num_second_iter_;
    b200_lba_t h_ = nullptr;
};

class global_bundle_adjuster {  // optimize/global_bundle_adjuster.h:18-62
public:
    explicit global_bundle_adjuster(unsigned int num_iter = 10, bool use_huber_kernel = true, int device = 0)
        : num_iter_(num_iter), use_huber_kernel_(use_huber_kernel) {
        check(b200_lba_create(device, &h_), "b200_lba_create");
    }
    ~global_bundle_adjuster() { b200_lba_destroy(h_); }
    global_bundle_adjuster(const global_bundle_adjuster&) = delete;
    // one LM round over the flattened map (problem.e_robust carries use_huber_kernel per edge); false = aborted by the caller's flag
    bool optimize(const b200_lba_problem_t& problem, volatile uint8_t* force_stop_flag, std::vector<double>& pose_cw_out, std::vector<double>& points_out,
                  double gain_threshold = 1e-3) const {
        pose_cw_out.resize((size_t)16 * problem.n_poses);
        points_out.resize((size_t)3 * problem.n_points);
        const int rc = b200_global_ba_solve(h_, &problem, (int)num_iter_, gain_threshold, force_stop_flag, pose_cw_out.data(), points_out.data(), nullptr);
        if (rc == B200_ERR_ABORTED) return false;
        check(rc, "b200_global_ba_solve");
        return true;
    }
    const unsigned int num_iter_;
    const bool use_huber_kernel_;

private:
    b200_lba_t h_ = nullptr;
};

class pose_optimizer {  // optimize/pose_optimizer.h:24-40 with Tracking.backend: "b200" (pose_optimizer_g2o.h:30-37 defaults)
public:
    explicit pose_optimizer(unsigned int num_trials_robust = 2, unsigned int num_trials = 2, unsigned int num_each_iter = 10, int device = 0)
        : num_trials_robust_(num_trials_robust), num_trials_(num_trials), num_each_iter_(num_each_iter) {
        check(b200_lba_create(device, &h_), "b200_lba_create");
    }
    ~pose_optimizer() { b200_lba_destroy(h_); }
    pose_optimizer(const pose_optimizer&) = delete;
    // one flattened frame (one free pose, fixed landmarks, one edge per observation); returns num_init_obs - num_bad_obs
    unsigned int optimize(const b200_lba_problem_t& frame, double (&optimized_pose)[16], std::vector<bool>& outlier_flags) const {
        std::vector<uint8_t> flags((size_t)(frame.n_edges > 0 ? frame.n_edges : 1));
        uint32_t n_valid = 0;
        check(b200_pose_optimize(h_, 1, &frame, (int)num_trials_robust_, (int)num_trials_, (int)num_each_iter_, optimized_pose, flags.data(), &n_valid),
              "b200_pose_optimize");
        outlier_flags.assign((size_t)frame.n_edges, false);
        for (int e = 0; e < frame.n_edges; ++e) outlier_flags[e] = flags[e] != 0;
        return n_valid;
    }
    b200_lba_t handle() const { return h_; }

private:
    const unsigned int num_trials_robust_, num_trials_, num_each_iter_;
    b200_lba_t h_ = nullptr;
};

class graph_optimizer {  // optimize/graph_optimizer.h:20-45: steps 4-5 on a graph built as graph_optimizer.cc:43-250 builds it
public:
    explicit graph_optimizer(bool fix_scale, unsigned int min_num_shared_lms = 100, int device = 0)
        : fix_scale_(fix_scale), min_num_shared_lms_(min_num_shared_lms) {
        check(b200_lba_create(device, &h_), "b200_lba_create");
    }
    ~graph_optimizer() { b200_lba_destroy(h_); }
    graph_optimizer(const graph_optimizer&) = delete;
    // estimate / fixed per vertex, e_v1 / e_v2 / e_meas per edge, landmarks (points, point_ref) to correct; fills the outputs
    void optimize(const std::vector<b200_sim3_t>& estimate, const std::vector<uint8_t>& fixed, const std::vector<int32_t>& e_v1,
                  const std::vector<int32_t>& e_v2, const std::vector<b200_sim3_t>& e_meas, const std::vector<double>& points,
                  const std::vector<int32_t>& point_ref, std::vector<b200_sim3_t>& estimate_out, std::vector<double>& pose_cw_out,
                  std::vector<double>& points_out, b200_pgo_stats_t* stats = nullptr, int max_iter = 50, double gain_threshold = 1e-3) const {
        estimate_out.resize(estimate.size());
        pose_cw_out.resize(16 * estimate.size());
        points_out.resize(points.size());
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
        check(b200_graph_optimize(h_, &g, max_iter, gain_threshold, stats), "b200_graph_optimize");
    }
    const bool fix_scale_;
    const unsigned int min_num_shared_lms_;

private:
    b200_lba_t h_ = nullptr;
};

class transform_optimizer {  // optimize/transform_optimizer.h:17-48: optimize() on pairs gathered as transform_optimizer.cc:58-94 does
public:
    explicit transform_optimizer(bool fix_scale, unsigned int num_iter = 10, int device = 0) : fix_scale_(fix_scale), num_iter_(num_iter) {
        check(b200_lba_create(device, &h_), "b200_lba_create");
    }
    ~transform_optimizer() { b200_lba_destroy(h_); }
    transform_optimizer(const transform_optimizer&) = delete;
    // problems: inputs filled by the caller (n_matches, sim3_12, poses, cameras, the pair arrays, keep); fix_scale is set here.
    // Writes the outputs of every problem; returns nothing (each problem's num_inliers is optimize()'s return value).
    void optimize_batch(std::vector<b200_transform_problem_t>& problems, float chi_sq = 10.0f) const {
        for (auto& p : problems) p.fix_scale = fix_scale_ ? 1 : 0;
        check(b200_transform_optimize(h_, (int)problems.size(), problems.data(), chi_sq, (int)num_iter_), "b200_transform_optimize");
    }
    unsigned int optimize(b200_transform_problem_t& problem, float chi_sq = 10.0f) const {
        problem.fix_scale = fix_scale_ ? 1 : 0;
        check(b200_transform_optimize(h_, 1, &problem, chi_sq, (int)num_iter_), "b200_transform_optimize");
        return problem.num_inliers;
    }
    b200_lba_t handle() const { return h_; }

private:
    const bool fix_scale_;
    const unsigned int num_iter_;
    b200_lba_t h_ = nullptr;
};

}  // namespace optimize

namespace tracking {
// tracking_module::search_local_landmarks + pose_optimizer::optimize for a batch of frames that stay on the GPU (b200_track_local_map)
class local_map_tracker {
public:
    local_map_tracker(const feature::orb_extractor& extractor, const b200_track_params_t& params, int device = 0)
        : ex_(extractor), prm_(params), m_(device), opt_(params.num_trials_robust, params.num_trials, params.num_each_iter, device) {}
    void track(std::vector<b200_track_frame_t>& frames) {
        check(b200_track_local_map(ex_.handle(), m_.get(), opt_.handle(), &prm_, (int)frames.size(), frames.data()), "b200_track_local_map");
    }

private:
    const feature::orb_extractor& ex_;
    b200_track_params_t prm_;
    match::device_matcher m_;
    optimize::pose_optimizer opt_;
};

// module::frame_tracker::motion_based_track (module/frame_tracker.h, frame_tracker.cc:20-59), bow_match_based_track (:61-95) and
// robust_match_based_track (:97-131) for a batch of frames that stay on the GPU (b200_motion_based_track, b200_bow_match_based_track,
// b200_robust_match_based_track).  params.margin = margin_last_frame_projection; true_baseline = camera::base::true_baseline_.
class frame_tracker {
public:
    frame_tracker(const feature::orb_extractor& extractor, const b200_track_params_t& params, double true_baseline, unsigned int num_matches_thr = 10,
                  int device = 0)
        : ex_(extractor), prm_(params), prm_bow_(params), true_baseline_(true_baseline), num_matches_thr_(num_matches_thr), m_(device),
          opt_(params.num_trials_robust, params.num_trials, params.num_each_iter, device) {
        prm_bow_.lowe_ratio = 0.7f;  // match::bow_tree bow_matcher(0.7, true) (frame_tracker.cc:62)
    }
    void motion_based_track(std::vector<b200_motion_track_frame_t>& frames) {
        check(b200_motion_based_track(ex_.handle(), m_.get(), opt_.handle(), &prm_, true_baseline_, num_matches_thr_, (int)frames.size(), frames.data()),
              "b200_motion_based_track");
    }
    float stage_ms(int stage) const {
        float ms = 0.f;
        check(b200_motion_track_stage_ms(m_.get(), stage, &ms), "b200_motion_track_stage_ms");
        return ms;
    }
    // robust_match_based_track (frame_tracker.cc:97-131) with match::robust(params.lowe_ratio = 0.8, true) (b200_robust_match_based_track).
    // frames[f].engine: the solver's engine; nullptr = default-constructed (use_fixed_seed), else one from solve::create_random_engine.
    void robust_match_based_track(std::vector<b200_robust_track_frame_t>& frames) {
        check(b200_robust_match_based_track(ex_.handle(), m_.get(), opt_.handle(), &prm_, num_matches_thr_, (int)frames.size(), frames.data()),
              "b200_robust_match_based_track");
    }
    float robust_stage_ms(int stage) const {
        float ms = 0.f;
        check(b200_robust_track_stage_ms(m_.get(), stage, &ms), "b200_robust_track_stage_ms");
        return ms;
    }
    // bow_match_based_track (frame_tracker.cc:61-95) with match::bow_tree(0.7, true) (b200_bow_match_based_track); params.max_candidates
    // bounds the gated candidates of one keyframe keypoint (0 = 64).  frames[f].kp_node / kf_node: the BoW node of every keypoint, -1 = none.
    void bow_match_based_track(std::vector<b200_bow_track_frame_t>& frames) {
        check(b200_bow_match_based_track(ex_.handle(), m_.get(), opt_.handle(), &prm_bow_, num_matches_thr_, (int)frames.size(), frames.data()),
              "b200_bow_match_based_track");
    }
    float bow_stage_ms(int stage) const {
        float ms = 0.f;
        check(b200_bow_track_stage_ms(m_.get(), stage, &ms), "b200_bow_track_stage_ms");
        return ms;
    }

private:
    const feature::orb_extractor& ex_;
    b200_track_params_t prm_, prm_bow_;
    double true_baseline_;
    unsigned int num_matches_thr_;
    match::device_matcher m_;
    optimize::pose_optimizer opt_;
};
}  // namespace tracking

namespace mapping {
// module::two_view_triangulator (module/two_view_triangulator.h): triangulate(matches) over (idx_1, idx_2) pairs (b200_triangulate_pairs)
class two_view_triangulator {
public:
    two_view_triangulator(const b200_tri_keyframe_t& keyfrm_1, const b200_tri_keyframe_t& keyfrm_2, float rays_parallax_deg_thr = 1.0f,
                          int device = 0)
        : k1_(keyfrm_1), k2_(keyfrm_2), deg_(rays_parallax_deg_thr), m_(device) {}
    // pos_w: 3 per match, ok: 1 per match; returns the number accepted
    int triangulate(const std::vector<std::pair<int32_t, int32_t>>& matches, std::vector<double>& pos_w, std::vector<uint8_t>& ok) {
        std::vector<int32_t> flat(2 * matches.size());
        for (size_t k = 0; k < matches.size(); ++k) {
            flat[2 * k] = matches[k].first;
            flat[2 * k + 1] = matches[k].second;
        }
        pos_w.assign(3 * matches.size(), 0.0);
        ok.assign(matches.size(), 0);
        b200_triangulate_problem_t P{};
        P.keyfrm_1 = &k1_;
        P.keyfrm_2 = &k2_;
        P.rays_parallax_deg_thr = deg_;
        P.n_matches = static_cast<int32_t>(matches.size());
        P.matches = flat.data();
        P.pos_w = pos_w.data();
        P.ok = ok.data();
        check(b200_triangulate_pairs(m_.get(), 1, &P), "b200_triangulate_pairs");
        return P.n_ok;
    }

private:
    b200_tri_keyframe_t k1_, k2_;
    float deg_;
    match::device_matcher m_;
};

// mapping_module::create_new_landmarks after the baseline test, for a batch of current keyframes (b200_create_new_landmarks); the
// problems' created_* / per-neighbour outputs are filled in place.  Defaults: the mapping module's matchers (lowe_ratio 0.95,
// residual 0.2 degrees) and triangulator (1 degree).
class new_landmark_creator {
public:
    explicit new_landmark_creator(int device = 0, float lowe_ratio = 0.95f, float residual_rad_thr = 0.2f * 3.14159265358979f / 180.0f,
                                  float rays_parallax_deg_thr = 1.0f)
        : m_(device), lowe_(lowe_ratio), residual_(residual_rad_thr), deg_(rays_parallax_deg_thr) {}
    void create(std::vector<b200_new_landmarks_problem_t>& problems, int max_candidates = 0) {
        check(b200_create_new_landmarks(m_.get(), static_cast<int>(problems.size()), problems.data(), lowe_, residual_, deg_, max_candidates),
              "b200_create_new_landmarks");
    }

private:
    match::device_matcher m_;
    float lowe_, residual_, deg_;
};
}  // namespace mapping

namespace util {
// util::stereo_rectifier (util/stereo_rectifier.h): both eyes' maps are built at construction (b200_rectifier_create); rectify() is
// cv::remap(INTER_LINEAR) of one pair of 8-bit frames in host memory, rectify_device() of a batch already on the device.
class stereo_rectifier {
public:
    explicit stereo_rectifier(const b200_rectifier_params_t& params) : cols_(params.cols), rows_(params.rows) {
        check(b200_rectifier_create(&params, &h_), "b200_rectifier_create");
    }
    ~stereo_rectifier() { b200_rectifier_destroy(h_); }
    stereo_rectifier(const stereo_rectifier&) = delete;
    stereo_rectifier& operator=(const stereo_rectifier&) = delete;

    // rectify(in_img_l, in_img_r, out_img_l, out_img_r) -- stereo_rectifier.h:25-26; all four frames cols x rows x channels
    void rectify(int channels, const uint8_t* in_l, size_t in_l_pitch, const uint8_t* in_r, size_t in_r_pitch, uint8_t* out_l, size_t out_l_pitch,
                 uint8_t* out_r, size_t out_r_pitch) const {
        check(b200_stereo_rectify(h_, channels, in_l, in_l_pitch, in_r, in_r_pitch, out_l, out_l_pitch, out_r, out_r_pitch), "b200_stereo_rectify");
    }
    void rectify_device(int channels, const void* d_l, const void* d_r, size_t src_pitch, size_t src_frame_stride, void* d_out_l, void* d_out_r,
                        size_t out_pitch, size_t out_frame_stride, int batch) const {
        check(b200_stereo_rectify_device(h_, channels, d_l, d_r, src_pitch, src_frame_stride, d_out_l, d_out_r, out_pitch, out_frame_stride, batch),
              "b200_stereo_rectify_device");
    }
    void set_stream(void* stream, bool use_own = false) { check(b200_rectifier_set_stream(h_, stream, use_own ? 1 : 0), "b200_rectifier_set_stream"); }
    // undist_map_{x,y}_{l,r}_ (stereo_rectifier.h:38-45): eye 0 left, 1 right; rows x cols floats each
    void maps(int eye, std::vector<float>& map_x, std::vector<float>& map_y) const {
        map_x.resize((size_t)cols_ * rows_);
        map_y.resize((size_t)cols_ * rows_);
        check(b200_rectifier_maps(h_, eye, map_x.data(), map_y.data()), "b200_rectifier_maps");
    }
    b200_rectifier_t handle() const { return h_; }

private:
    b200_rectifier_t h_ = nullptr;
    int cols_, rows_;
};
}  // namespace util
}  // namespace b200

namespace b200 {
namespace solve {

// util::create_random_engine: a default-constructed engine, or one seeded by std::seed_seq over ten std::random_device words
inline void create_random_engine(b200_mt19937_t& engine, bool use_fixed_seed) {
    if (use_fixed_seed) {
        check(b200_mt19937_seed(&engine, nullptr, 0), "b200_mt19937_seed");
        return;
    }
    std::random_device rd;
    uint32_t words[10];
    for (auto& w : words) w = rd();
    check(b200_mt19937_seed(&engine, words, 10), "b200_mt19937_seed");
}

// util::create_random_array(set_size, 0, n - 1, engine), max_num_iter times from one engine (b200_draw_min_sets), max_num_iter x set_size
inline std::vector<int32_t> draw_min_sets(b200_mt19937_t& engine, uint32_t set_size, uint32_t n_matches, uint32_t max_num_iter) {
    std::vector<int32_t> out((size_t)set_size * max_num_iter);
    check(b200_draw_min_sets(&engine, set_size, n_matches, max_num_iter, out.data()), "b200_draw_min_sets");
    return out;
}

// PnP's minimal sets of 4
inline std::vector<int32_t> draw_min_sets(b200_mt19937_t& engine, uint32_t n_matches, uint32_t max_num_iter) {
    return draw_min_sets(engine, 4, n_matches, max_num_iter);
}

// find_via_ransac for many problems in one call (b200_pnp_ransac); the problems' out fields are filled
inline void pnp_ransac_batch(b200_lba_t h, std::vector<b200_pnp_problem_t>& problems) {
    check(b200_pnp_ransac(h, (int)problems.size(), problems.data()), "b200_pnp_ransac");
}

// solve::pnp_solver (solve/pnp_solver.h:13-142).  bearings / points: n x 3 row-major; rotations row-major 3 x 3.  The engine is the
// solver's member: find_via_ransac continues its state across calls.  The solver owns a b200_lba_t handle unless one is given.
class pnp_solver {
public:
    pnp_solver(const std::vector<double>& valid_bearings, const std::vector<int>& octaves, const std::vector<double>& valid_points,
               const std::vector<float>& scale_factors, unsigned int min_num_inliers = 10, bool use_fixed_seed = false,
               unsigned int gauss_newton_num_iter = 10, b200_lba_t handle = nullptr)
        : num_matches_((unsigned int)octaves.size()), bearings_(valid_bearings), points_(valid_points), octaves_(octaves.begin(), octaves.end()),
          scale_factors_(scale_factors), min_num_inliers_(min_num_inliers), gauss_newton_num_iter_(gauss_newton_num_iter), h_(handle) {
        if (bearings_.size() != 3 * (size_t)num_matches_ || points_.size() != 3 * (size_t)num_matches_)
            throw std::invalid_argument("pnp_solver: bearings, octaves and points must have one entry per match");
        for (int32_t o : octaves_)
            if (o < 0 || (size_t)o >= scale_factors_.size()) throw std::out_of_range("pnp_solver: octave outside the scale factors");
        create_random_engine(engine_, use_fixed_seed);
        if (!h_) {
            check(b200_lba_create(0, &h_), "b200_lba_create");
            own_ = true;
        }
    }
    ~pnp_solver() {
        if (own_) b200_lba_destroy(h_);
    }
    pnp_solver(const pnp_solver&) = delete;
    pnp_solver& operator=(const pnp_solver&) = delete;

    void find_via_ransac(unsigned int max_num_iter, bool recompute = true) {
        if (num_matches_ < 4 || num_matches_ < min_num_inliers_) {  // before any draw (pnp_solver.cc:48-52)
            solution_is_valid_ = false;
            return;
        }
        const std::vector<int32_t> sets = draw_min_sets(engine_, num_matches_, max_num_iter);
        std::vector<uint8_t> flags(num_matches_);
        b200_pnp_problem_t P{};
        P.n_matches = (int32_t)num_matches_;
        P.bearings = bearings_.data();
        P.points = points_.data();
        P.octaves = octaves_.data();
        P.num_levels = (int32_t)scale_factors_.size();
        P.scale_factors = scale_factors_.data();
        P.min_num_inliers = min_num_inliers_;
        P.gauss_newton_num_iter = gauss_newton_num_iter_;
        P.max_num_iter = max_num_iter;
        P.recompute = recompute ? 1 : 0;
        P.min_sets = sets.data();
        P.inlier_flags = flags.data();
        check(b200_pnp_ransac(h_, 1, &P), "b200_pnp_ransac");
        status_ = P.status;
        solution_is_valid_ = P.valid != 0;
        if (solution_is_valid_) {
            for (int k = 0; k < 9; ++k) best_rot_cw_[k] = P.rot_cw[k];
            for (int k = 0; k < 3; ++k) best_trans_cw_[k] = P.trans_cw[k];
        }
        is_inlier_match_.assign(flags.begin(), flags.end());
    }
    bool solution_is_valid() const { return solution_is_valid_; }
    const double* get_best_rotation() const { return best_rot_cw_; }
    const double* get_best_translation() const { return best_trans_cw_; }
    void get_best_cam_pose(double (&pose_cw)[16]) const {
        for (int r = 0; r < 4; ++r)
            for (int c = 0; c < 4; ++c) pose_cw[r * 4 + c] = r < 3 ? (c < 3 ? best_rot_cw_[r * 3 + c] : best_trans_cw_[r]) : (c == 3 ? 1.0 : 0.0);
    }
    std::vector<bool> get_inlier_flags() const { return is_inlier_match_; }
    int status() const { return status_; }  // B200_ERR_INVALID when a Jacobi SVD of the last call hit its sweep bound

    // compute_pose (pnp_solver.h:95-97): rot_cw / trans_cw are written only when a candidate reaches reproj_error < DBL_MAX
    static double compute_pose(b200_lba_t h, const std::vector<double>& bearing_vectors, const std::vector<double>& pos_ws, double (&rot_cw)[9],
                               double (&trans_cw)[3], unsigned int num_iter = 5) {
        b200_epnp_problem_t P{};
        P.n = (int32_t)(bearing_vectors.size() / 3);
        P.bearings = bearing_vectors.data();
        P.points = pos_ws.data();
        P.num_iter = num_iter;
        for (int k = 0; k < 9; ++k) P.rot_cw[k] = rot_cw[k];
        for (int k = 0; k < 3; ++k) P.trans_cw[k] = trans_cw[k];
        check(b200_epnp_compute_pose(h, 1, &P), "b200_epnp_compute_pose");
        check(P.status, "b200_epnp_compute_pose: Jacobi SVD");
        for (int k = 0; k < 9; ++k) rot_cw[k] = P.rot_cw[k];
        for (int k = 0; k < 3; ++k) trans_cw[k] = P.trans_cw[k];
        return P.reproj_error;
    }

private:
    unsigned int num_matches_;
    std::vector<double> bearings_, points_;
    std::vector<int32_t> octaves_;
    std::vector<float> scale_factors_;
    unsigned int min_num_inliers_, gauss_newton_num_iter_;
    b200_mt19937_t engine_;
    b200_lba_t h_ = nullptr;
    bool own_ = false;
    bool solution_is_valid_ = false;
    int status_ = B200_OK;
    double best_rot_cw_[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, best_trans_cw_[3] = {0, 0, 0};
    std::vector<bool> is_inlier_match_;
};

// essential_solver::find_via_ransac for many problems in one call (b200_essential_ransac); the problems' out fields are filled
inline void essential_ransac_batch(b200_lba_t h, std::vector<b200_essential_problem_t>& problems) {
    check(b200_essential_ransac(h, (int)problems.size(), problems.data()), "b200_essential_ransac");
}

// solve::essential_solver (solve/essential_solver.h).  bearings: n x 3 row-major; matches_12: (first, second) index pairs; E_21
// row-major.  The engine is the solver's member: find_via_ransac continues its state across calls.  The solver owns a b200_lba_t
// handle unless one is given.  Only the five-point minimal set (min_set_size = 5, every caller's value) is supported.
class essential_solver {
public:
    essential_solver(const std::vector<double>& bearings_1, const std::vector<double>& bearings_2,
                     const std::vector<std::pair<int, int>>& matches_12, bool use_fixed_seed = false, b200_lba_t handle = nullptr)
        : num_matches_((unsigned int)matches_12.size()), h_(handle) {
        b1_.reserve(3 * matches_12.size());
        b2_.reserve(3 * matches_12.size());
        for (const auto& m : matches_12) {
            if (m.first < 0 || 3 * (size_t)m.first + 3 > bearings_1.size() || m.second < 0 || 3 * (size_t)m.second + 3 > bearings_2.size())
                throw std::out_of_range("essential_solver: match index outside the bearings");
            b1_.insert(b1_.end(), bearings_1.begin() + 3 * m.first, bearings_1.begin() + 3 * m.first + 3);
            b2_.insert(b2_.end(), bearings_2.begin() + 3 * m.second, bearings_2.begin() + 3 * m.second + 3);
        }
        create_random_engine(engine_, use_fixed_seed);
    }
    ~essential_solver() {
        if (own_) b200_lba_destroy(h_);
    }
    essential_solver(const essential_solver&) = delete;
    essential_solver& operator=(const essential_solver&) = delete;

    void find_via_ransac(unsigned int max_num_iter, bool recompute = true, unsigned int min_set_size = 5) {
        if (min_set_size != 5) throw std::invalid_argument("essential_solver: only the five-point minimal set is supported");
        if (num_matches_ < min_set_size) {  // before any draw (essential_solver.cc:23-26)
            solution_is_valid_ = false;
            return;
        }
        if (!h_) {
            check(b200_lba_create(0, &h_), "b200_lba_create");
            own_ = true;
        }
        const std::vector<int32_t> sets = draw_min_sets(engine_, 5, num_matches_, max_num_iter);
        std::vector<uint8_t> flags(num_matches_);
        b200_essential_problem_t P{};
        P.n_matches = (int32_t)num_matches_;
        P.bearings_1 = b1_.data();
        P.bearings_2 = b2_.data();
        P.min_set_size = 5;
        P.max_num_iter = max_num_iter;
        P.recompute = recompute ? 1 : 0;
        P.min_sets = sets.data();
        P.inlier_flags = flags.data();
        check(b200_essential_ransac(h_, 1, &P), "b200_essential_ransac");
        status_ = P.status;
        solution_is_valid_ = P.valid != 0;
        best_cost_ = P.best_cost;
        if (solution_is_valid_)
            for (int k = 0; k < 9; ++k) best_E_21_[k] = P.E_21[k];
        is_inlier_match_.assign(flags.begin(), flags.end());
    }
    bool solution_is_valid() const { return solution_is_valid_; }
    float get_best_cost() const { return best_cost_; }
    const double* get_best_E_21() const { return best_E_21_; }
    std::vector<bool> get_inlier_matches() const { return is_inlier_match_; }
    int status() const { return status_; }  // B200_ERR_INVALID when a RealSchur or a Jacobi SVD of the last call did not converge

private:
    unsigned int num_matches_;
    std::vector<double> b1_, b2_;
    b200_mt19937_t engine_;
    b200_lba_t h_ = nullptr;
    bool own_ = false;
    bool solution_is_valid_ = false;
    int status_ = B200_OK;
    float best_cost_ = 0.0f;
    double best_E_21_[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    std::vector<bool> is_inlier_match_;
};

}  // namespace solve
}  // namespace b200

namespace b200 {
namespace initialize {

// One frame as the initialisers read it: the camera (b200_camera_intrinsics_t model codes), its image bounds (min_x, max_x, min_y,
// max_y), every undistorted keypoint (n x 2) and bearing (n x 3).
struct frame {
    b200_camera_intrinsics_t camera{};
    float img_bounds[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    std::vector<float> undist_keypts;
    std::vector<double> bearings;
};

// initialize() for many frame pairs in one call (b200_initialize); the problems' out fields are filled
inline void initialize_batch(b200_lba_t h, std::vector<b200_init_problem_t>& problems) {
    check(b200_initialize(h, (int)problems.size(), problems.data()), "b200_initialize");
}

// initialize::base (initialize/base.h) with initialize() of perspective (models 0, 2, 3) or bearing_vector (model 1).  Each attempt
// constructs its solvers' engines afresh (util::create_random_engine) and draws only for a RANSAC that runs; a Jacobi SVD or RealSchur
// that hits its bound does not throw (the reference returns normally): status() then reports B200_ERR_INVALID.  R and t are left as
// the reference leaves base's members: zeroed once find_most_plausible_pose has run and rejected, untouched when RANSAC or the
// decomposition failed first.  The initialiser owns a b200_lba_t handle unless one is given.
class base {
public:
    base(const frame& ref_frm, bool bearing, unsigned int num_ransac_iters, unsigned int min_num_triangulated, unsigned int min_num_valid_pts,
         float parallax_deg_thr, float reproj_err_thr, bool use_fixed_seed, b200_lba_t handle)
        : ref_(ref_frm), bearing_(bearing), num_ransac_iters_(num_ransac_iters), min_num_triangulated_(min_num_triangulated),
          min_num_valid_pts_(min_num_valid_pts), parallax_deg_thr_(parallax_deg_thr), reproj_err_thr_(reproj_err_thr),
          use_fixed_seed_(use_fixed_seed), h_(handle) {
        if ((ref_.camera.model == 1) != bearing_)
            throw std::invalid_argument(bearing_ ? "bearing_vector: needs an equirectangular camera" : "perspective: cannot get a camera matrix");
        if (ref_.undist_keypts.size() / 2 != ref_.bearings.size() / 3) throw std::invalid_argument("initialize: one bearing per keypoint");
    }
    virtual ~base() {
        if (own_) b200_lba_destroy(h_);
    }
    base(const base&) = delete;
    base& operator=(const base&) = delete;

    bool initialize(const frame& cur_frm, const std::vector<int>& ref_matches_with_cur) {
        const size_t n_ref = ref_.undist_keypts.size() / 2;
        if (ref_matches_with_cur.size() != n_ref) throw std::invalid_argument("initialize: one match entry per ref keypoint");
        if (!h_) {
            check(b200_lba_create(0, &h_), "b200_lba_create");
            own_ = true;
        }
        uint32_t n = 0;
        for (int m : ref_matches_with_cur) n += m >= 0;
        std::vector<int32_t> sets_H, sets_F, sets_E;
        b200_mt19937_t engine;
        if (bearing_) {
            if (n >= 5) {
                solve::create_random_engine(engine, use_fixed_seed_);
                sets_E = solve::draw_min_sets(engine, 5, n, num_ransac_iters_);
            }
        } else if (n >= 8) {
            solve::create_random_engine(engine, use_fixed_seed_);
            sets_H = solve::draw_min_sets(engine, 4, n, num_ransac_iters_);
            solve::create_random_engine(engine, use_fixed_seed_);
            sets_F = solve::draw_min_sets(engine, 8, n, num_ransac_iters_);
        }
        const std::vector<int32_t> matches(ref_matches_with_cur.begin(), ref_matches_with_cur.end());
        std::vector<double> pts(3 * n_ref);
        std::vector<uint8_t> flags(n_ref);
        b200_init_problem_t P{};
        P.cam_ref = ref_.camera;
        P.cam_cur = cur_frm.camera;
        for (int k = 0; k < 4; ++k) {
            P.img_bounds_ref[k] = ref_.img_bounds[k];
            P.img_bounds_cur[k] = cur_frm.img_bounds[k];
        }
        P.n_ref = (int32_t)n_ref;
        P.n_cur = (int32_t)(cur_frm.undist_keypts.size() / 2);
        P.undist_ref = ref_.undist_keypts.data();
        P.bearings_ref = ref_.bearings.data();
        P.undist_cur = cur_frm.undist_keypts.data();
        P.bearings_cur = cur_frm.bearings.data();
        P.ref_matches_with_cur = matches.data();
        P.num_ransac_iters = num_ransac_iters_;
        P.min_num_triangulated = min_num_triangulated_;
        P.min_num_valid_pts = min_num_valid_pts_;
        P.parallax_deg_thr = parallax_deg_thr_;
        P.reproj_err_thr = reproj_err_thr_;
        P.min_sets_H = sets_H.empty() ? nullptr : sets_H.data();
        P.min_sets_F = sets_F.empty() ? nullptr : sets_F.data();
        P.min_sets_E = sets_E.empty() ? nullptr : sets_E.data();
        P.triangulated_pts = pts.data();
        P.triangulated_flags = flags.data();
        check(b200_initialize(h_, 1, &P), "b200_initialize");
        status_ = P.status;
        stage_ = P.stage;
        model_ = P.model;
        if (P.n_hypotheses > 0) {
            for (int k = 0; k < 9; ++k) rot_ref_to_cur_[k] = P.rot_ref_to_cur[k];
            for (int k = 0; k < 3; ++k) trans_ref_to_cur_[k] = P.trans_ref_to_cur[k];
        }
        if (P.succeeded) {
            triangulated_pts_ = pts;
            is_triangulated_.assign(flags.begin(), flags.end());
        }
        return P.succeeded != 0;
    }

    const double* get_rotation_ref_to_cur() const { return rot_ref_to_cur_; }  // row-major
    const double* get_translation_ref_to_cur() const { return trans_ref_to_cur_; }
    const std::vector<double>& get_triangulated_pts() const { return triangulated_pts_; }  // n_ref x 3
    std::vector<bool> get_triangulated_flags() const { return is_triangulated_; }
    int status() const { return status_; }
    int stage() const { return stage_; }  // B200_INIT_STAGE_* of the last attempt
    int model() const { return model_; }  // B200_INIT_MODEL_*

private:
    frame ref_;
    bool bearing_;
    unsigned int num_ransac_iters_, min_num_triangulated_, min_num_valid_pts_;
    float parallax_deg_thr_, reproj_err_thr_;
    bool use_fixed_seed_;
    b200_lba_t h_ = nullptr;
    bool own_ = false;
    int status_ = B200_OK, stage_ = B200_INIT_STAGE_NO_MODEL, model_ = B200_INIT_MODEL_NONE;
    double rot_ref_to_cur_[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};  // base.h: Mat33_t::Identity(), Vec3_t::Zero()
    double trans_ref_to_cur_[3] = {0, 0, 0};
    std::vector<double> triangulated_pts_;
    std::vector<bool> is_triangulated_;
};

// initialize::perspective (initialize/perspective.h): H and F RANSAC and the reconstruction with the model rel_cost_H picks
class perspective final : public base {
public:
    explicit perspective(const frame& ref_frm, unsigned int num_ransac_iters = 100, unsigned int min_num_triangulated = 50,
                         unsigned int min_num_valid_pts = 50, float parallax_deg_thr = 1.0f, float reproj_err_thr = 4.0f, bool use_fixed_seed = false,
                         b200_lba_t handle = nullptr)
        : base(ref_frm, false, num_ransac_iters, min_num_triangulated, min_num_valid_pts, parallax_deg_thr, reproj_err_thr, use_fixed_seed, handle) {}
};

// initialize::bearing_vector (initialize/bearing_vector.h): E RANSAC and its reconstruction (equirectangular cameras)
class bearing_vector final : public base {
public:
    explicit bearing_vector(const frame& ref_frm, unsigned int num_ransac_iters = 100, unsigned int min_num_triangulated = 50,
                            unsigned int min_num_valid_pts = 50, float parallax_deg_thr = 1.0f, float reproj_err_thr = 4.0f,
                            bool use_fixed_seed = false, b200_lba_t handle = nullptr)
        : base(ref_frm, true, num_ransac_iters, min_num_triangulated, min_num_valid_pts, parallax_deg_thr, reproj_err_thr, use_fixed_seed, handle) {}
};

}  // namespace initialize
}  // namespace b200
