// Drives the C++ mirror of keyframe culling (include/b200vslam.hpp: b200::module::local_map_cleaner) on problems written by
// tests/test_cpp_cull_api.py and prints the results, so that the driver can compare them with the Python mirror.
//   cull_api_test <file> <redundant_obs_ratio_thr> <top_n>
//   file: int32 n_problems; per problem: uint32 cur_id, int32 n_covisibilities, then per covisibility uint32 id, int32 is_root,
//         int32 n_keypoints, int32 has_depth, double depth_thr, int32 kp_landmark x n, float depth x n when has_depth; then int32
//         n_landmarks, int32 obs_offsets x (n_landmarks + 1), int32 obs_rank x total, int32 obs_octave x total, uint8 obs_weight x total
//   output: "problem <k> <n_removed>", then one line "rank <r> <skipped> <n_valid> <n_redundant> <removed>" per covisibility
#include <cstdio>
#include <cstdlib>
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

struct owned {  // the arrays one problem points into
    std::vector<b200_cull_keyframe_t> covs;
    std::vector<std::vector<int32_t>> kp_landmark;
    std::vector<std::vector<float>> depth;
    std::vector<int32_t> offsets, rank, octave;
    std::vector<uint8_t> weight;
};

}  // namespace

int main(int argc, char** argv) {
    if (argc < 4) {
        std::fprintf(stderr, "usage: %s <file> <redundant_obs_ratio_thr> <top_n>\n", argv[0]);
        return 2;
    }
    reader r(argv[1]);
    const int n = r.get<int32_t>();
    std::vector<owned> own(n);
    std::vector<b200_cull_problem_t> problems(n);
    for (int k = 0; k < n; ++k) {
        owned& o = own[k];
        b200_cull_problem_t& p = problems[k];
        p = b200_cull_problem_t{};
        p.cur_id = r.get<uint32_t>();
        const int n_cov = r.get<int32_t>();
        o.covs.assign(n_cov, b200_cull_keyframe_t{});
        o.kp_landmark.resize(n_cov);
        o.depth.resize(n_cov);
        for (int c = 0; c < n_cov; ++c) {
            b200_cull_keyframe_t& kf = o.covs[c];
            kf.id = r.get<uint32_t>();
            kf.is_root = r.get<int32_t>();
            kf.n_keypoints = r.get<int32_t>();
            const int has_depth = r.get<int32_t>();
            kf.depth_thr = r.get<double>();
            o.kp_landmark[c] = r.arr<int32_t>(kf.n_keypoints);
            kf.kp_landmark = o.kp_landmark[c].data();
            if (has_depth) {
                o.depth[c] = r.arr<float>(kf.n_keypoints);
                kf.depth = o.depth[c].data();
            }
        }
        p.n_covisibilities = n_cov;
        p.covisibilities = o.covs.data();
        p.n_landmarks = r.get<int32_t>();
        o.offsets = r.arr<int32_t>(p.n_landmarks + 1);
        const size_t total = (size_t)o.offsets[p.n_landmarks];
        o.rank = r.arr<int32_t>(total);
        o.octave = r.arr<int32_t>(total);
        o.weight = r.arr<uint8_t>(total);
        p.obs_offsets = o.offsets.data();
        p.obs_rank = o.rank.data();
        p.obs_octave = o.octave.data();
        p.obs_weight = o.weight.data();
    }
    b200::module::local_map_cleaner cleaner(std::atof(argv[2]), (unsigned int)std::atoi(argv[3]));
    const auto n_removed = cleaner.remove_redundant_keyframes(problems);
    for (int k = 0; k < n; ++k) {
        std::printf("problem %d %u\n", k, n_removed[k]);
        for (int c = 0; c < problems[k].n_covisibilities; ++c) {
            const b200_cull_keyframe_t& kf = problems[k].covisibilities[c];
            std::printf("rank %d %d %d %d %d\n", c, kf.skipped, kf.n_valid, kf.n_redundant, kf.removed);
        }
    }
    return 0;
}
