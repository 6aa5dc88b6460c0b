// Drives the C++ mirror of the RGB-D frame step and the depth-seeded landmarks (include/b200vslam.hpp) on problems written by
// tests/test_cpp_rgbd_api.py, and prints the results as hex words so that the driver can compare them with the Python mirror bit for bit.
//   rgbd_api_test rgbd <file>       file: int32 n, w, h; n gray frames (u8); n depth maps (u16); camera: int32 model, 13 doubles
//                                   (fx fy cx cy k1 k2 p1 p2 k3 cols rows k4 distortion); double focal_x_baseline, depthmap_factor
//   rgbd_api_test landmarks <file>  file: int32 mode, n; x, y, depth (f32 x n); octave (i32 x n); has_landmark (u8 x n);
//                                   pose_wc (16 doubles); fx_inv fy_inv cx cy depth_thr (doubles); 8 scale factors, inv_last (floats)
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

}  // namespace

int main(int argc, char** argv) {
    if (argc < 3) {
        std::fprintf(stderr, "usage: %s rgbd|landmarks <file>\n", argv[0]);
        return 2;
    }
    reader r(argv[2]);
    if (!std::strcmp(argv[1], "rgbd")) {
        const int n = r.get<int32_t>(), w = r.get<int32_t>(), h = r.get<int32_t>();
        const auto gray = r.arr<uint8_t>((size_t)n * w * h);
        const auto depth = r.arr<uint16_t>((size_t)n * w * h);
        b200_camera_intrinsics_t cam{};
        cam.model = r.get<int32_t>();
        double* f = &cam.fx;  // fx fy cx cy k1 k2 p1 p2 k3 cols rows k4 distortion are consecutive doubles
        for (int k = 0; k < 13; ++k) f[k] = r.get<double>();
        const double fxb = r.get<double>(), factor = r.get<double>();
        b200::feature::orb_params prm;
        b200::feature::orb_extractor ex(&prm, 800, b200::feature::descriptor_type::ORB, {}, 0, n);
        std::vector<b200_keypoint_t> kps;
        std::vector<uint8_t> desc;
        std::vector<int32_t> counts;
        ex.extract_batch(gray.data(), w, h, w, (size_t)w * h, n, nullptr, 0, kps, desc, counts);
        const auto res = ex.rgbd_depths(cam, fxb, factor, B200_DEPTH_16UC1, depth.data(), w, h, 2 * (size_t)w, 2 * (size_t)w * h, n);
        for (int fr = 0; fr < n; ++fr) {
            const size_t o = (size_t)fr * res.cap, c = (size_t)res.counts[fr];
            std::printf("frame %d %d\n", fr, res.counts[fr]);
            hex("undist", reinterpret_cast<const uint32_t*>(res.undist_keypts.data() + o), 6 * c);  // six 4-byte fields per keypoint
            hex("bearings", res.bearings.data() + 3 * o, 3 * c);
            hex("depths", res.depths.data() + o, c);
            hex("x_right", res.x_right.data() + o, c);
        }
        return 0;
    }
    if (!std::strcmp(argv[1], "landmarks")) {
        b200_depth_landmarks_problem_t p{};
        p.mode = r.get<int32_t>();
        const int n = r.get<int32_t>();
        const auto x = r.arr<float>(n), y = r.arr<float>(n), depth = r.arr<float>(n);
        const auto octave = r.arr<int32_t>(n);
        const auto has_lm = r.arr<uint8_t>(n);
        for (int k = 0; k < 16; ++k) p.pose_wc[k] = r.get<double>();
        p.fx_inv = r.get<double>();
        p.fy_inv = r.get<double>();
        p.cx = r.get<double>();
        p.cy = r.get<double>();
        p.depth_thr = r.get<double>();
        const auto sf = r.arr<float>(8);
        p.inv_scale_factor_last = r.get<float>();
        p.n_keypoints = n;
        p.x = x.data();
        p.y = y.data();
        p.depth = depth.data();
        p.octave = octave.data();
        p.has_landmark = has_lm.data();
        p.num_levels = 8;
        p.scale_factors = sf.data();
        b200::module::depth_landmarks creator;
        const auto res = creator.create({p, p})[1];  // the same problem twice in one call: the second equals the first
        std::printf("created %zu\n", res.idx.size());
        hex("idx", res.idx.data(), res.idx.size());
        hex("pos_w", res.pos_w.data(), res.pos_w.size());
        hex("mean_normal", res.mean_normal.data(), res.mean_normal.size());
        hex("min_valid_dist", res.min_valid_dist.data(), res.min_valid_dist.size());
        hex("max_valid_dist", res.max_valid_dist.data(), res.max_valid_dist.size());
        return 0;
    }
    return 2;
}
