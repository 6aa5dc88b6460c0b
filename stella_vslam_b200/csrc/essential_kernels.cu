// essential_kernels.cu -- solve::essential_solver (src/stella_vslam/solve/essential_solver.cc) on the device: find_via_ransac with the
// five-point minimal set for many problems in one launch sequence on the b200_lba_t handle's stream.  The minimal sets are drawn on the
// host (random_array.cu), or on the device in the robust-match tracking chain (match_kernels.cu).
//
// find_via_ransac is split in three launches (enqueue_ransac, essential_ransac.cuh), which read each problem's match count and whether it
// runs from device memory:
//   essential_hypothesis_kernel  one thread per (problem, iteration): compute_E_21_minimal on the minimal set (essential_core.h),
//                                up to ten candidates written to scratch in eigenvalue order;
//   essential_score_kernel       one thread per (problem, iteration, candidate slot): check_inliers, the float cost accumulated over
//                                the matches in ascending order (a tree sum could change which candidate wins);
//   essential_select_kernel      one thread per problem: the first-wins selection in (iteration, candidate) order
//                                (num_inliers > min_set_size and best_cost > cost), the winner's inlier flags and, with recompute and
//                                at least 8 inliers, compute_E_21_nonminimal over the inliers and check_inliers again.
// The arithmetic is fp64 with explicit round-to-nearest intrinsics; tests/essential_oracle.c compiles the same essential_core.h as C.
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "epnp.cuh"
#include "essential_ransac.cuh"
#include "ransac_host.cuh"
#include "staging.cuh"
#include "util_trig.cuh"

namespace b200 {
namespace ess {

using pnp::apply_householder_left;
using pnp::svd_core;
using tri::da;
using tri::dd;
using tri::dm;
using tri::ds;

#include "essential_core.cuh"

__global__ void __launch_bounds__(32) essential_hypothesis_kernel(int n_hyp_total, const int* __restrict__ hyp_problem,
                                                                   const ProblemDev* __restrict__ probs, const double* __restrict__ b1,
                                                                   const double* __restrict__ b2, const int32_t* __restrict__ min_sets,
                                                                   double* __restrict__ cand, HypDev* __restrict__ hyps) {
    const int h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= n_hyp_total) return;
    const ProblemDev P = probs[hyp_problem[h]];
    HypDev out;
    out.flags = 0;
    out.count = 0;
    if (P.runs)
        out.count = es_minimal(b1 + 3 * (size_t)P.match_off, b2 + 3 * (size_t)P.match_off, min_sets + kMinSet * (size_t)h,
                               cand + 9 * kMaxCand * (size_t)h, &out.flags);
    hyps[h] = out;
}

__global__ void __launch_bounds__(64) essential_score_kernel(long long n_slots, const int* __restrict__ hyp_problem,
                                                              const ProblemDev* __restrict__ probs, const double* __restrict__ b1,
                                                              const double* __restrict__ b2, const double* __restrict__ cand,
                                                              const HypDev* __restrict__ hyps, ScoreDev* __restrict__ scores) {
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_slots) return;
    const long long h = s / kMaxCand;
    if ((int)(s - h * kMaxCand) >= hyps[h].count) return;
    const ProblemDev P = probs[hyp_problem[h]];
    ScoreDev out;
    out.num_inliers = es_check_inliers(b1 + 3 * (size_t)P.match_off, b2 + 3 * (size_t)P.match_off, P.n, cand + 9 * (size_t)s,
                                       es_cos_angle_thr(), nullptr, &out.cost);
    scores[s] = out;
}

__global__ void __launch_bounds__(64) essential_select_kernel(int n_problems, const ProblemDev* __restrict__ probs,
                                                              const double* __restrict__ b1, const double* __restrict__ b2,
                                                              const double* __restrict__ cand, const HypDev* __restrict__ hyps,
                                                              const ScoreDev* __restrict__ scores, int32_t* __restrict__ idx_scratch,
                                                              double* __restrict__ mat_scratch, uint8_t* __restrict__ flags,
                                                              ResultDev* __restrict__ results) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n_problems) return;
    const ProblemDev P = probs[q];
    ResultDev r;
    r.valid = 0;
    r.best_iter = -1;
    r.best_candidate = -1;
    r.num_inliers = 0;
    r.best_cost = 0.0f;  // the member's initial value, kept on the early return
    r.status = 0;
    if (!P.runs) {
        results[q] = r;
        return;
    }
    r.best_cost = FLT_MAX;
    for (int it = 0; it < P.n_hyp; ++it) {
        const HypDev H = hyps[P.hyp_off + it];
        r.status |= H.flags & (ES_STATUS_SCHUR | ES_STATUS_SVD);
        for (int k = 0; k < H.count; ++k) {
            const ScoreDev S = scores[(size_t)(P.hyp_off + it) * kMaxCand + k];
            if (S.num_inliers > (unsigned)kMinSet && r.best_cost > S.cost) {
                r.best_cost = S.cost;
                r.best_iter = it;
                r.best_candidate = k;
                r.num_inliers = (int)S.num_inliers;
            }
        }
    }
    r.valid = r.best_cost < FLT_MAX;
    const double* pb1 = b1 + 3 * (size_t)P.match_off;
    const double* pb2 = b2 + 3 * (size_t)P.match_off;
    uint8_t* fl = flags + P.match_off;
    if (!r.valid) {
        for (int j = 0; j < P.n; ++j) fl[j] = 0;
        results[q] = r;
        return;
    }
    const double* W = cand + 9 * ((size_t)(P.hyp_off + r.best_iter) * kMaxCand + r.best_candidate);
    for (int k = 0; k < 9; ++k) r.E[k] = W[k];
    const float thr = es_cos_angle_thr();
    float cost;
    es_check_inliers(pb1, pb2, P.n, r.E, thr, fl, &cost);
    if (P.recompute && r.num_inliers >= 8) {
        int32_t* idx = idx_scratch + P.match_off;
        const int m = compact_inliers(fl, P.n, idx);
        r.status |= es_nonminimal(pb1, pb2, idx, m, mat_scratch + 9 * (size_t)P.match_off, r.E);
        es_check_inliers(pb1, pb2, P.n, r.E, thr, fl, &r.best_cost);
    }
    results[q] = r;
}

int enqueue_ransac(cudaStream_t st, int n_problems, int n_hyp, const RansacDev& d) {
    if (n_hyp > 0) {
        // 32-thread blocks: one problem of 1 000 iterations spreads over 32 SMs rather than 8 (the tracker's fallback is one problem)
        essential_hypothesis_kernel<<<b200::ceil_div(n_hyp, 32), 32, 0, st>>>(n_hyp, d.hyp_problem, d.probs, d.b1, d.b2, d.min_sets, d.cand, d.hyps);
        B200_CUDA(cudaGetLastError());
        const long long slots = (long long)n_hyp * kMaxCand;
        essential_score_kernel<<<(unsigned)((slots + 63) / 64), 64, 0, st>>>(slots, d.hyp_problem, d.probs, d.b1, d.b2, d.cand, d.hyps, d.scores);
        B200_CUDA(cudaGetLastError());
    }
    essential_select_kernel<<<b200::ceil_div(n_problems, 64), 64, 0, st>>>(n_problems, d.probs, d.b1, d.b2, d.cand, d.hyps, d.scores, d.idx, d.mat,
                                                                          d.flags, d.results);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

}  // namespace ess
}  // namespace b200

extern "C" {

int b200_essential_ransac(b200_lba_t h, int n_problems, b200_essential_problem_t* problems) {
    B200_RANGE("b200:essential:ransac");
    using namespace b200::ess;
    if (!h || n_problems < 0) return B200_ERR_INVALID;
    if (n_problems == 0) return B200_OK;
    if (!problems) return B200_ERR_INVALID;
    std::vector<ProblemDev> pd(n_problems);
    long long total = 0, total_hyp = 0;
    for (int q = 0; q < n_problems; ++q) {
        const b200_essential_problem_t& P = problems[q];
        const int n = P.n_matches;
        if (P.min_set_size != (uint32_t)kMinSet) {
            b200::set_error("b200_essential_ransac: problem %d: min_set_size %u (only the five-point minimal set is supported)", q, P.min_set_size);
            return B200_ERR_INVALID;
        }
        if (n < 0 || (n > 0 && (!P.bearings_1 || !P.bearings_2 || !P.inlier_flags))) {
            b200::set_error("b200_essential_ransac: problem %d: negative count or null buffer", q);
            return B200_ERR_INVALID;
        }
        const bool runs = n >= kMinSet;
        if (!b200::min_sets_ok("b200_essential_ransac", q, runs, P.max_num_iter, P.min_sets, kMinSet, n)) return B200_ERR_INVALID;
        const int n_hyp = runs ? (int)P.max_num_iter : 0;
        pd[q] = ProblemDev{n, (int)total, (int)total_hyp, n_hyp, runs, P.recompute != 0};
        total += n;
        total_hyp += n_hyp;
        if (total > INT_MAX / 16 || total_hyp > INT_MAX / 16) {
            b200::set_error("b200_essential_ransac: too many matches or iterations in one call");
            return B200_ERR_INVALID;
        }
    }
    const size_t T = (size_t)std::max(total, 1LL), NH = (size_t)std::max(total_hyp, 1LL);
    b200::Layout a;
    const size_t o_probs = a.take(sizeof(ProblemDev) * n_problems), o_b1 = a.take(24 * T), o_b2 = a.take(24 * T);
    const size_t o_ms = a.take(4 * kMinSet * NH), o_hp = a.take(4 * NH);
    const size_t in_bytes = a.end;
    const size_t o_res = a.take(sizeof(ResultDev) * n_problems), o_fl = a.take(T);
    const size_t out_end = a.end;
    const size_t o_cand = a.take(8 * 9 * kMaxCand * NH), o_hyp = a.take(sizeof(HypDev) * NH), o_sc = a.take(sizeof(ScoreDev) * kMaxCand * NH);
    const size_t o_idx = a.take(4 * T), o_mat = a.take(72 * T);
    cudaStream_t st;
    b200::StagingArena* A;
    int rc = b200::lba::staging(h, a.end, out_end, &st, &A);
    if (rc) return rc;
    unsigned char *db = A->d, *hb = A->h;
    std::memcpy(hb + o_probs, pd.data(), sizeof(ProblemDev) * n_problems);
    for (int q = 0; q < n_problems; ++q) {
        const b200_essential_problem_t& P = problems[q];
        const size_t off = (size_t)pd[q].match_off, n = (size_t)P.n_matches;
        if (n) {
            std::memcpy(hb + o_b1 + 24 * off, P.bearings_1, 24 * n);
            std::memcpy(hb + o_b2 + 24 * off, P.bearings_2, 24 * n);
        }
        b200::stage_min_sets(q, P.min_sets, kMinSet, pd[q].n_hyp, kMinSet * (size_t)pd[q].hyp_off, pd[q].hyp_off, (int32_t*)(hb + o_ms),
                             (int*)(hb + o_hp));
    }
    B200_CUDA(A->upload(in_bytes, st));
    const RansacDev dev{(const int*)(db + o_hp), (const ProblemDev*)(db + o_probs), (const double*)(db + o_b1), (const double*)(db + o_b2),
                        (const int32_t*)(db + o_ms), (double*)(db + o_cand), (HypDev*)(db + o_hyp), (ScoreDev*)(db + o_sc), (int32_t*)(db + o_idx),
                        (double*)(db + o_mat), db + o_fl, (ResultDev*)(db + o_res)};
    if ((rc = enqueue_ransac(st, n_problems, (int)total_hyp, dev))) return rc;
    B200_CUDA(A->download(o_res, out_end, st));
    B200_CUDA(cudaStreamSynchronize(st));
    const ResultDev* res = reinterpret_cast<const ResultDev*>(hb + o_res);
    for (int q = 0; q < n_problems; ++q) {
        b200_essential_problem_t& P = problems[q];
        const ResultDev& r = res[q];
        P.status = r.status ? B200_ERR_INVALID : B200_OK;
        P.valid = r.valid;
        P.best_iter = r.best_iter;
        P.best_candidate = r.best_candidate;
        P.num_inliers = r.num_inliers;
        P.best_cost = r.best_cost;
        if (r.valid) std::memcpy(P.E_21, r.E, sizeof r.E);
        if (pd[q].runs) std::memcpy(P.inlier_flags, hb + o_fl + pd[q].match_off, (size_t)P.n_matches);
    }
    return B200_OK;
}

}  // extern "C"
