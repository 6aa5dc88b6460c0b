// Drives b200::initialize::{perspective, bearing_vector} (include/b200vslam.hpp) for tests/test_cpp_initialize_api.py, which compares
// the output with the Python mirror.
//   initialize_api_test FILE   the initialiser of the camera's model (use_fixed_seed, default parameters) built on the ref frame in
//                              FILE, one initialize() with the current frame; every double printed with 17 significant digits
// FILE (both frames share the camera): 14 doubles (model fx fy cx cy k1 k2 p1 p2 k3 cols rows k4 distortion), 4 floats (image bounds),
// int32 n_ref, int32 n_cur, n_ref x 2 floats, n_ref x 3 doubles, n_cur x 2 floats, n_cur x 3 doubles, n_ref int32 ref_matches_with_cur.
#include <cstdio>
#include <memory>
#include <string>
#include <vector>

#include "b200vslam.hpp"

template <typename T>
static bool read(FILE* f, std::vector<T>& v, size_t n) {
    v.resize(n);
    return std::fread(v.data(), sizeof(T), n, f) == n;
}

int main(int argc, char** argv) {
    if (argc != 2) return 2;
    FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 3;
    std::vector<double> cam;
    std::vector<float> bounds;
    std::vector<int32_t> counts, matches;
    b200::initialize::frame ref, cur;
    if (!read(f, cam, 14) || !read(f, bounds, 4) || !read(f, counts, 2)) return 4;
    b200_camera_intrinsics_t c{};
    c.model = (int32_t)cam[0];
    c.fx = cam[1], c.fy = cam[2], c.cx = cam[3], c.cy = cam[4], c.k1 = cam[5], c.k2 = cam[6], c.p1 = cam[7], c.p2 = cam[8], c.k3 = cam[9];
    c.cols = cam[10], c.rows = cam[11], c.k4 = cam[12], c.distortion = cam[13];
    for (auto* fr : {&ref, &cur}) {
        fr->camera = c;
        for (int k = 0; k < 4; ++k) fr->img_bounds[k] = bounds[k];
    }
    if (!read(f, ref.undist_keypts, 2 * (size_t)counts[0]) || !read(f, ref.bearings, 3 * (size_t)counts[0]) ||
        !read(f, cur.undist_keypts, 2 * (size_t)counts[1]) || !read(f, cur.bearings, 3 * (size_t)counts[1]) || !read(f, matches, (size_t)counts[0]))
        return 5;
    std::fclose(f);
    std::unique_ptr<b200::initialize::base> ini;
    if (c.model == 1)
        ini.reset(new b200::initialize::bearing_vector(ref, 100, 50, 50, 1.0f, 4.0f, true));
    else
        ini.reset(new b200::initialize::perspective(ref, 100, 50, 50, 1.0f, 4.0f, true));
    const bool ok = ini->initialize(cur, std::vector<int>(matches.begin(), matches.end()));
    std::printf("succeeded %d status %d stage %d model %d\nR", ok ? 1 : 0, ini->status(), ini->stage(), ini->model());
    for (int k = 0; k < 9; ++k) std::printf(" %.17g", ini->get_rotation_ref_to_cur()[k]);
    std::printf("\nt");
    for (int k = 0; k < 3; ++k) std::printf(" %.17g", ini->get_translation_ref_to_cur()[k]);
    std::printf("\npts");
    for (double v : ini->get_triangulated_pts()) std::printf(" %.17g", v);
    std::printf("\nflags ");
    for (bool v : ini->get_triangulated_flags()) std::putchar(v ? '1' : '0');
    std::printf("\n");
    return 0;
}
