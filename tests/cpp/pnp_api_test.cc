// Drives b200::solve (include/b200vslam.hpp) for tests/test_cpp_pnp_api.py, which compares the output with the Python mirror.
//   pnp_api_test sampler N ITERS [SEED_WORDS...]   the minimal sets of one engine, one set per line (host only, no GPU)
//   pnp_api_test ransac FILE                        pnp_solver(use_fixed_seed) on the problem in FILE: find_via_ransac(30, true), then
//                                                   find_via_ransac(30, false) on the continued engine, then compute_pose on the first
//                                                   min(n, 50) matches; every double printed with 17 significant digits
// FILE: int32 n, int32 num_levels, n x 3 bearings, n x 3 points (double), n octaves (int32), num_levels scale factors (float).
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "b200vslam.hpp"

static void print_result(const b200::solve::pnp_solver& s) {
    std::printf("valid %d\n", s.solution_is_valid() ? 1 : 0);
    std::printf("pose");
    for (int k = 0; k < 9; ++k) std::printf(" %.17g", s.get_best_rotation()[k]);
    for (int k = 0; k < 3; ++k) std::printf(" %.17g", s.get_best_translation()[k]);
    std::printf("\nflags ");
    for (bool f : s.get_inlier_flags()) std::putchar(f ? '1' : '0');
    std::printf("\n");
}

int main(int argc, char** argv) {
    if (argc >= 4 && std::string(argv[1]) == "sampler") {
        std::vector<uint32_t> words;
        for (int i = 4; i < argc; ++i) words.push_back((uint32_t)std::strtoul(argv[i], nullptr, 10));
        b200_mt19937_t e;
        b200::check(b200_mt19937_seed(&e, words.empty() ? nullptr : words.data(), (int)words.size()), "b200_mt19937_seed");
        const std::vector<int32_t> sets = b200::solve::draw_min_sets(e, (uint32_t)std::atoi(argv[2]), (uint32_t)std::atoi(argv[3]));
        for (size_t i = 0; i < sets.size(); i += 4) std::printf("%d %d %d %d\n", sets[i], sets[i + 1], sets[i + 2], sets[i + 3]);
        return 0;
    }
    if (argc != 3 || std::string(argv[1]) != "ransac") return 2;
    FILE* f = std::fopen(argv[2], "rb");
    if (!f) return 3;
    int32_t hdr[2];
    if (std::fread(hdr, 4, 2, f) != 2) return 4;
    const int n = hdr[0], levels = hdr[1];
    std::vector<double> bearings(3 * (size_t)n), points(3 * (size_t)n);
    std::vector<int32_t> oct(n);
    std::vector<float> sf(levels);
    if (std::fread(bearings.data(), 8, bearings.size(), f) != bearings.size() || std::fread(points.data(), 8, points.size(), f) != points.size()
        || std::fread(oct.data(), 4, oct.size(), f) != oct.size() || std::fread(sf.data(), 4, sf.size(), f) != sf.size())
        return 5;
    std::fclose(f);
    const std::vector<int> octaves(oct.begin(), oct.end());
    b200::solve::pnp_solver s(bearings, octaves, points, sf, 10, true);
    s.find_via_ransac(30, true);
    print_result(s);
    s.find_via_ransac(30, false);
    print_result(s);
    b200_lba_t h = nullptr;
    b200::check(b200_lba_create(0, &h), "b200_lba_create");
    const size_t m = (size_t)(n < 50 ? n : 50);
    const std::vector<double> b(bearings.begin(), bearings.begin() + 3 * m), p(points.begin(), points.begin() + 3 * m);
    double R[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, t[3] = {0, 0, 0};
    const double err = b200::solve::pnp_solver::compute_pose(h, b, p, R, t, 10);
    std::printf("compute_pose %.17g", err);
    for (double v : R) std::printf(" %.17g", v);
    for (double v : t) std::printf(" %.17g", v);
    std::printf("\n");
    b200_lba_destroy(h);
    return 0;
}
