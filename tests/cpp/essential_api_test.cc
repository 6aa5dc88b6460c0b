// Drives b200::solve::essential_solver (include/b200vslam.hpp) for tests/test_cpp_essential_api.py, which compares the output with the
// Python mirror.
//   essential_api_test sampler SET_SIZE N ITERS [SEED_WORDS...]   the minimal sets of one engine, one set per line (host only, no GPU)
//   essential_api_test ransac FILE                                 essential_solver(use_fixed_seed) on the problem in FILE:
//                                                                  find_via_ransac(200, true), then find_via_ransac(200, false) on the
//                                                                  continued engine; every double printed with 17 significant digits
// FILE: int32 n1, int32 n2, int32 m, n1 x 3 bearings_1, n2 x 3 bearings_2 (double), m x 2 matches (int32).
#include <cstdio>
#include <cstdlib>
#include <string>
#include <utility>
#include <vector>

#include "b200vslam.hpp"

static void print_result(const b200::solve::essential_solver& s) {
    std::printf("valid %d status %d\ncost %.9g\nE", s.solution_is_valid() ? 1 : 0, s.status(), (double)s.get_best_cost());
    for (int k = 0; k < 9; ++k) std::printf(" %.17g", s.get_best_E_21()[k]);
    std::printf("\nflags ");
    for (bool f : s.get_inlier_matches()) std::putchar(f ? '1' : '0');
    std::printf("\n");
}

int main(int argc, char** argv) {
    if (argc >= 5 && std::string(argv[1]) == "sampler") {
        std::vector<uint32_t> words;
        for (int i = 5; i < argc; ++i) words.push_back((uint32_t)std::strtoul(argv[i], nullptr, 10));
        b200_mt19937_t e;
        b200::check(b200_mt19937_seed(&e, words.empty() ? nullptr : words.data(), (int)words.size()), "b200_mt19937_seed");
        const uint32_t k = (uint32_t)std::atoi(argv[2]);
        const std::vector<int32_t> sets = b200::solve::draw_min_sets(e, k, (uint32_t)std::atoi(argv[3]), (uint32_t)std::atoi(argv[4]));
        for (size_t i = 0; i < sets.size(); ++i) std::printf("%d%c", sets[i], (i + 1) % k ? ' ' : '\n');
        return 0;
    }
    if (argc != 3 || std::string(argv[1]) != "ransac") return 2;
    FILE* f = std::fopen(argv[2], "rb");
    if (!f) return 3;
    int32_t hdr[3];
    if (std::fread(hdr, 4, 3, f) != 3) return 4;
    std::vector<double> b1(3 * (size_t)hdr[0]), b2(3 * (size_t)hdr[1]);
    std::vector<int32_t> m(2 * (size_t)hdr[2]);
    if (std::fread(b1.data(), 8, b1.size(), f) != b1.size() || std::fread(b2.data(), 8, b2.size(), f) != b2.size()
        || std::fread(m.data(), 4, m.size(), f) != m.size())
        return 5;
    std::fclose(f);
    std::vector<std::pair<int, int>> matches;
    for (int i = 0; i < hdr[2]; ++i) matches.emplace_back(m[2 * i], m[2 * i + 1]);
    b200::solve::essential_solver s(b1, b2, matches, true);
    s.find_via_ransac(200, true);
    print_result(s);
    s.find_via_ransac(200, false);
    print_result(s);
    return 0;
}
