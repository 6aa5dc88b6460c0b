// Drives the C++ mirror of BoW-match tracking (include/b200vslam.hpp: tracking::frame_tracker::bow_match_based_track) on frames
// written by tests/test_cpp_bow_track_api.py, and prints the results as hex words so that the driver can compare them with the Python
// mirror bit for bit.
//   bow_track_api_test track <file>   file: int32 n, w, h; n gray frames (u8); camera: int32 model, monocular, 7 doubles
//                                     (fx fy cx cy fxb cols rows); uint32 num_matches_thr; then per frame: int32 frame, n_kp_in, stereo, n_kf;
//                                     last_pose_cw (16 doubles); kp_node (i32 x n_kp_in); kp_x_right (f32 x n_kp_in, when stereo);
//                                     desc (32 u8 x n_kf); angle (f32 x n_kf); node (i32 x n_kf); valid (u8 x n_kf); pos_w (3 doubles x n_kf)
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iterator>
#include <vector>

#include "b200vslam.hpp"

namespace {

struct reader {
    std::vector<char> buf;
    size_t pos = 0;
    explicit reader(const char* path) {
        std::ifstream f(path, std::ios::binary);
        buf.assign(std::istreambuf_iterator<char>(f), {});
    }
    template <class T>
    T get() {
        T v;
        std::memcpy(&v, buf.data() + pos, sizeof(T));
        pos += sizeof(T);
        return v;
    }
    template <class T>
    std::vector<T> arr(size_t n) {
        std::vector<T> v(n);
        if (n) std::memcpy(v.data(), buf.data() + pos, sizeof(T) * n);
        pos += sizeof(T) * n;
        return v;
    }
};

template <class T>
void hex(const char* name, const T* p, size_t n) {
    std::printf("%s", name);
    const unsigned char* b = reinterpret_cast<const unsigned char*>(p);
    for (size_t i = 0; i < n * sizeof(T); ++i) std::printf("%s%02x", i % sizeof(T) ? "" : " ", b[i]);
    std::printf("\n");
}

struct frame_data {
    std::vector<double> last, pos;
    std::vector<float> xr, angle;
    std::vector<uint8_t> desc, valid;
    std::vector<int32_t> kp_node, node, kp_landmark;
};

}  // namespace

int main(int argc, char** argv) {
    if (argc < 3 || std::strcmp(argv[1], "track")) {
        std::fprintf(stderr, "usage: %s track <file>\n", argv[0]);
        return 2;
    }
    reader r(argv[2]);
    const int n = r.get<int32_t>(), w = r.get<int32_t>(), h = r.get<int32_t>();
    const auto gray = r.arr<uint8_t>((size_t)n * w * h);
    b200_track_params_t prm{};
    prm.cam.model = r.get<int32_t>();
    prm.monocular = r.get<int32_t>();
    prm.cam.fx = r.get<double>();
    prm.cam.fy = r.get<double>();
    prm.cam.cx = r.get<double>();
    prm.cam.cy = r.get<double>();
    prm.focal_x_baseline = r.get<double>();
    prm.cam.cols = r.get<double>();
    prm.cam.rows = r.get<double>();
    const uint32_t thr = r.get<uint32_t>();
    b200::feature::orb_params op;
    b200::feature::orb_extractor ex(&op, 800, b200::feature::descriptor_type::ORB, {}, 0, n);
    std::vector<b200_keypoint_t> kps;
    std::vector<uint8_t> desc;
    std::vector<int32_t> counts;
    ex.extract_batch(gray.data(), w, h, w, (size_t)w * h, n, nullptr, 0, kps, desc, counts);
    prm.num_levels = op.num_levels_;
    prm.log_scale_factor = op.log_scale_factor_;
    prm.scale_factors = op.scale_factors_.data();
    prm.inv_level_sigma_sq = op.inv_level_sigma_sq_.data();
    prm.lowe_ratio = 0.8f;  // the mirror sets bow_tree's 0.7 itself
    prm.num_trials_robust = 2;
    prm.num_trials = 2;
    prm.num_each_iter = 10;
    std::vector<frame_data> data(n);
    std::vector<b200_bow_track_frame_t> frames(n);
    const int kp_cap = b200_orb_max_keypoints(ex.handle(), w, h);
    for (int f = 0; f < n; ++f) {
        b200_bow_track_frame_t& F = frames[f];
        frame_data& D = data[f];
        F = b200_bow_track_frame_t{};
        F.frame = r.get<int32_t>();
        F.n_keypoints_in = r.get<int32_t>();
        const int stereo = r.get<int32_t>();
        F.n_kf_keypoints = r.get<int32_t>();
        const size_t nk = (size_t)F.n_keypoints_in, nkf = (size_t)F.n_kf_keypoints;
        D.last = r.arr<double>(16);
        D.kp_node = r.arr<int32_t>(nk);
        if (stereo) D.xr = r.arr<float>(nk);
        D.desc = r.arr<uint8_t>(32 * nkf);
        D.angle = r.arr<float>(nkf);
        D.node = r.arr<int32_t>(nkf);
        D.valid = r.arr<uint8_t>(nkf);
        D.pos = r.arr<double>(3 * nkf);
        D.kp_landmark.assign((size_t)kp_cap, -1);
        F.last_pose_cw = D.last.data();
        F.kp_node = D.kp_node.data();
        F.kp_x_right = stereo ? D.xr.data() : nullptr;
        F.kf_desc = D.desc.data();
        F.kf_angle = D.angle.data();
        F.kf_node = D.node.data();
        F.kf_valid = D.valid.data();
        F.kf_pos_w = D.pos.data();
        F.kp_cap = kp_cap;
        F.kp_landmark_out = D.kp_landmark.data();
    }
    b200::tracking::frame_tracker tracker(ex, prm, 0.0, thr);
    tracker.bow_match_based_track(frames);
    for (int f = 0; f < n; ++f) {
        const b200_bow_track_frame_t& F = frames[f];
        std::printf("frame %d %d %d %u %d\n", F.n_keypoints, F.n_matches, F.applied, F.n_valid, F.tracked);
        hex("kp", data[f].kp_landmark.data(), (size_t)F.n_keypoints);
        hex("pose", F.pose_cw_out, 16);
    }
    std::printf("chain_ms_positive %d\n", tracker.bow_stage_ms(6) > 0.f ? 1 : 0);
    return 0;
}
