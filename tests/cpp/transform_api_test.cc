// Drives b200::optimize::transform_optimizer (include/b200vslam.hpp) for tests/test_cpp_transform_api.py, which compares the output
// with the Python mirror.
//   transform_api_test FILE   FILE: int32 n, fix_scale; 8 doubles sim3_12; 9 + 3 + 9 + 3 doubles rot_1w, trans_1w, rot_2w, trans_2w;
//                             2 x (int32 model, 7 doubles fx fy cx cy fxb cols rows); n x 2 float obs_1; n float inv_sigma_sq_1;
//                             n x 3 double pos_w_2; n x 2 float obs_2; n float inv_sigma_sq_2; n x 3 double pos_w_1
// Prints the refined Sim3 (8 doubles, 17 significant digits), the keep flags, then "inliers N".
#include <cstdio>
#include <vector>

#include "b200vslam.hpp"

template <class T> static void rd(std::FILE* f, T* v, size_t n) {
    if (n && std::fread(v, sizeof(T), n, f) != n) throw std::runtime_error("short file");
}

int main(int argc, char** argv) {
    if (argc != 2) return 2;
    std::FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 2;
    int32_t hdr[2];
    rd(f, hdr, 2);
    const size_t n = (size_t)hdr[0];
    b200_transform_problem_t p{};
    p.n_matches = hdr[0];
    rd(f, p.sim3_12.q, 4);
    rd(f, p.sim3_12.t, 3);
    rd(f, &p.sim3_12.s, 1);
    rd(f, p.rot_1w, 9);
    rd(f, p.trans_1w, 3);
    rd(f, p.rot_2w, 9);
    rd(f, p.trans_2w, 3);
    for (b200_camera_t* c : {&p.cam_1, &p.cam_2}) {
        rd(f, &c->model, 1);
        double v[7];
        rd(f, v, 7);
        c->fx = v[0]; c->fy = v[1]; c->cx = v[2]; c->cy = v[3]; c->fxb = v[4]; c->cols = v[5]; c->rows = v[6];
    }
    std::vector<float> obs_1(2 * n), w1(n), obs_2(2 * n), w2(n);
    std::vector<double> pw2(3 * n), pw1(3 * n);
    std::vector<uint8_t> keep(n + 1);
    rd(f, obs_1.data(), 2 * n);
    rd(f, w1.data(), n);
    rd(f, pw2.data(), 3 * n);
    rd(f, obs_2.data(), 2 * n);
    rd(f, w2.data(), n);
    rd(f, pw1.data(), 3 * n);
    std::fclose(f);
    p.obs_1 = obs_1.data(); p.inv_sigma_sq_1 = w1.data(); p.pos_w_2 = pw2.data();
    p.obs_2 = obs_2.data(); p.inv_sigma_sq_2 = w2.data(); p.pos_w_1 = pw1.data();
    p.keep = keep.data();
    b200::optimize::transform_optimizer opt(hdr[1] != 0);
    const unsigned int inliers = opt.optimize(p);
    for (double q : p.sim3_12_out.q) std::printf("%.17g ", q);
    for (double t : p.sim3_12_out.t) std::printf("%.17g ", t);
    std::printf("%.17g\n", p.sim3_12_out.s);
    for (size_t i = 0; i < n; ++i) std::printf("%d\n", keep[i]);
    std::printf("inliers %u\n", inliers);
    return 0;
}
