// Drives b200::optimize::graph_optimizer (include/b200vslam.hpp) for tests/test_cpp_pgo_api.py, which compares the output with the
// Python mirror.
//   pgo_api_test FILE   FILE: int32 n_vertices, n_edges, n_points, fix_scale; n_vertices x 8 estimates (double); n_vertices fixed
//                       (uint8); n_edges e_v1, n_edges e_v2 (int32); n_edges x 8 measurements; n_points x 3 points; n_points point_ref
// Prints the estimates, the poses and the points, every double with 17 significant digits, then "iterations N".
#include <cstdio>
#include <vector>

#include "b200vslam.hpp"

template <class T> static void rd(std::FILE* f, std::vector<T>& v, size_t n) {
    v.resize(n);
    if (n && std::fread(v.data(), sizeof(T), n, f) != n) throw std::runtime_error("short file");
}

int main(int argc, char** argv) {
    if (argc != 2) return 2;
    std::FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 2;
    int32_t hdr[4];
    if (std::fread(hdr, sizeof(int32_t), 4, f) != 4) return 2;
    std::vector<b200_sim3_t> est, meas, est_out;
    std::vector<uint8_t> fixed;
    std::vector<int32_t> e1, e2, pref;
    std::vector<double> pts, pose_out, pts_out;
    rd(f, est, hdr[0]);
    rd(f, fixed, hdr[0]);
    rd(f, e1, hdr[1]);
    rd(f, e2, hdr[1]);
    rd(f, meas, hdr[1]);
    rd(f, pts, 3 * (size_t)hdr[2]);
    rd(f, pref, hdr[2]);
    std::fclose(f);
    b200::optimize::graph_optimizer opt(hdr[3] != 0);
    b200_pgo_stats_t st{};
    opt.optimize(est, fixed, e1, e2, meas, pts, pref, est_out, pose_out, pts_out, &st);
    for (const auto& s : est_out) {
        for (double q : s.q) std::printf("%.17g ", q);
        for (double t : s.t) std::printf("%.17g ", t);
        std::printf("%.17g\n", s.s);
    }
    for (double v : pose_out) std::printf("%.17g\n", v);
    for (double v : pts_out) std::printf("%.17g\n", v);
    std::printf("iterations %d\n", st.iterations);
    return 0;
}
