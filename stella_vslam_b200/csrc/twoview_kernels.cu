// twoview_kernels.cu -- solve::homography_solver and solve::fundamental_solver (src/stella_vslam/solve/homography_solver.cc,
// fundamental_solver.cc) on the device: find_via_ransac for many problems of either model in one launch sequence on the b200_lba_t
// handle's stream.
//
// find_via_ransac is split in four launches (enqueue_ransac, twoview_ransac.cuh):
//   twoview_normalize_kernel   one CTA per (problem, frame): solve::normalize.  Thread 0 forms the float centroid and L1 deviation in
//                              keypoint order (the sums are sequential in the reference) and the transform; every thread then
//                              scales its keypoints;
//   twoview_hypothesis_kernel  one thread per (problem, iteration): compute_H_21 / compute_F_21 on the minimal set (the wide 8 x 9
//                              JacobiSVD path), H's rank() test, the denormalisation;
//   twoview_score_kernel       one warp per (problem, iteration): check_inliers.  The lanes form the per-match terms of 32 matches at
//                              a time; lane 0 adds them to the float cost in match order (a tree sum could change which iteration
//                              wins);
//   twoview_select_kernel      one thread per problem: the first-wins selection (num_inliers > min_set_size and best_cost > cost), the
//                              winner's inlier flags and, with recompute, compute_H_21 / compute_F_21 over the inliers (tall or
//                              square path) and check_inliers again.
// The arithmetic is csrc/twoview_core.h; tests/twoview_oracle.c compiles the same header as C.
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "epnp.cuh"
#include "ransac_host.cuh"
#include "staging.cuh"
#include "twoview_ransac.cuh"
#include "util_trig.cuh"  // util_cos, which essential_core.h (included below for its SVD pieces) calls in es_cos_angle_thr

namespace b200 {
namespace twoview {

using pnp::apply_householder_left;
using pnp::svd_core;
using tri::da;
using tri::dd;
using tri::dm;
using tri::ds;

__device__ __forceinline__ float tv_fa(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float tv_fs(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float tv_fm(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float tv_fd(float a, float b) { return __fdiv_rn(a, b); }

#include "essential_core.cuh"
#include "twoview_core.h"

__global__ void __launch_bounds__(128) twoview_normalize_kernel(const ProblemDev* __restrict__ probs, const float* __restrict__ kp1,
                                                                 const float* __restrict__ kp2, float* __restrict__ kn1,
                                                                 float* __restrict__ kn2, NormDev* __restrict__ norms) {
    const int q = blockIdx.x >> 1, side = blockIdx.x & 1;
    const ProblemDev P = probs[q];
    if (!P.runs) return;
    const int n = side ? P.n2 : P.n1;
    const float* pts = (side ? kp2 : kp1) + 2 * (size_t)(side ? P.kp2_off : P.kp1_off);
    float* out = (side ? kn2 : kn1) + 2 * (size_t)(side ? P.kp2_off : P.kp1_off);
    __shared__ float mean[2], l1[2];
    if (threadIdx.x == 0) {
        double T[9];
        tv_normalize_stats(n, pts, mean, l1, T);
        if (side == 0)
            for (int k = 0; k < 9; ++k) norms[q].T1[k] = T[k];
        else
            tv_left_factor(P.model, T, norms[q].D2);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) tv_normalize_point(pts + 2 * (size_t)i, mean, l1, out + 2 * (size_t)i);
}

__global__ void __launch_bounds__(32) twoview_hypothesis_kernel(int n_hyp_total, const int* __restrict__ hyp_problem,
                                                                 const ProblemDev* __restrict__ probs, const NormDev* __restrict__ norms,
                                                                 const float* __restrict__ kn1, const float* __restrict__ kn2,
                                                                 const int32_t* __restrict__ matches, const int32_t* __restrict__ min_sets,
                                                                 HypDev* __restrict__ hyps) {
    const int h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= n_hyp_total) return;
    const int q = hyp_problem[h];
    const ProblemDev P = probs[q];
    const NormDev& N = norms[q];
    double S[72], Mn[9];
    HypDev out;
    out.status = 0;
    out.ok = tv_estimate(P.model, kn1 + 2 * (size_t)P.kp1_off, kn2 + 2 * (size_t)P.kp2_off, matches + 2 * (size_t)P.match_off,
                         min_sets + P.ms_off + (size_t)P.set_size * (h - P.hyp_off), P.set_size, S, Mn, &out.status);
    if (out.ok) tv_denormalise(N.D2, Mn, N.T1, out.M);
    hyps[h] = out;
}

__global__ void __launch_bounds__(128) twoview_score_kernel(int n_hyp_total, const int* __restrict__ hyp_problem,
                                                             const ProblemDev* __restrict__ probs, const float* __restrict__ kp1,
                                                             const float* __restrict__ kp2, const int32_t* __restrict__ matches,
                                                             const HypDev* __restrict__ hyps, ScoreDev* __restrict__ scores) {
    const int h = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (h >= n_hyp_total || !hyps[h].ok) return;  // warp-uniform
    const ProblemDev P = probs[hyp_problem[h]];
    double M[9], Mi[9];
    for (int k = 0; k < 9; ++k) M[k] = hyps[h].M[k];
    if (P.model == TV_MODEL_H) tv_inverse33(M, Mi);
    const float thr = tv_thr(P.sigma);
    const float* k1 = kp1 + 2 * (size_t)P.kp1_off;
    const float* k2 = kp2 + 2 * (size_t)P.kp2_off;
    const int32_t* mt = matches + 2 * (size_t)P.match_off;
    float cost = 0.0f;
    unsigned num = 0;
    for (int base = 0; base < P.n; base += 32) {
        const int j = base + lane;
        int in = 0;
        double t = 0.0;
        if (j < P.n) t = tv_term(P.model, M, Mi, k1 + 2 * (size_t)mt[2 * (size_t)j], k2 + 2 * (size_t)mt[2 * (size_t)j + 1], thr, &in);
        num += __popc(__ballot_sync(0xffffffffu, in));
        const int cnt = min(32, P.n - base);
        for (int k = 0; k < cnt; ++k) {
            const double tk = __shfl_sync(0xffffffffu, t, k);
            const int ik = __shfl_sync(0xffffffffu, in, k);
            if (lane == 0) cost = tv_accumulate(P.model, cost, tk, ik);
        }
    }
    if (lane == 0) scores[h] = ScoreDev{cost, num};
}

__global__ void __launch_bounds__(64) twoview_select_kernel(int n_problems, const ProblemDev* __restrict__ probs,
                                                             const NormDev* __restrict__ norms, const float* __restrict__ kp1,
                                                             const float* __restrict__ kp2, const float* __restrict__ kn1,
                                                             const float* __restrict__ kn2, const int32_t* __restrict__ matches,
                                                             const HypDev* __restrict__ hyps, const ScoreDev* __restrict__ scores,
                                                             int32_t* __restrict__ idx_scratch, double* __restrict__ mat_scratch,
                                                             uint8_t* __restrict__ flags, ResultDev* __restrict__ results) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n_problems) return;
    const ProblemDev P = probs[q];
    ResultDev r;
    r.valid = 0;
    r.best_iter = -1;
    r.num_inliers = 0;
    r.best_cost = 0.0f;  // the member's initial value, kept on the early return
    r.status = 0;
    if (!P.runs) {
        results[q] = r;
        return;
    }
    r.best_cost = FLT_MAX;
    const unsigned min_set = (unsigned)P.set_size;
    for (int it = 0; it < P.n_hyp; ++it) {
        const HypDev& H = hyps[P.hyp_off + it];
        r.status |= H.status;
        if (!H.ok) continue;
        const ScoreDev S = scores[P.hyp_off + it];
        if (S.num_inliers > min_set && r.best_cost > S.cost) {
            r.best_cost = S.cost;
            r.best_iter = it;
            r.num_inliers = (int)S.num_inliers;
        }
    }
    r.valid = r.best_cost < FLT_MAX;
    uint8_t* fl = flags + P.match_off;
    if (!r.valid) {
        for (int j = 0; j < P.n; ++j) fl[j] = 0;
        results[q] = r;
        return;
    }
    const float* k1 = kp1 + 2 * (size_t)P.kp1_off;
    const float* k2 = kp2 + 2 * (size_t)P.kp2_off;
    const int32_t* mt = matches + 2 * (size_t)P.match_off;
    for (int k = 0; k < 9; ++k) r.M[k] = hyps[P.hyp_off + r.best_iter].M[k];
    float cost;
    tv_check_inliers(P.model, k1, k2, mt, P.n, r.M, P.sigma, fl, &cost);
    if (P.recompute) {
        int32_t* idx = idx_scratch + P.match_off;
        const int m = compact_inliers(fl, P.n, idx);
        double Mn[9];
        if (tv_estimate(P.model, kn1 + 2 * (size_t)P.kp1_off, kn2 + 2 * (size_t)P.kp2_off, mt, idx, m, mat_scratch + 18 * (size_t)P.match_off,
                        Mn, &r.status)) {
            const NormDev& N = norms[q];
            tv_denormalise(N.D2, Mn, N.T1, r.M);
            tv_check_inliers(P.model, k1, k2, mt, P.n, r.M, P.sigma, fl, &r.best_cost);
        }
    }
    results[q] = r;
}

int enqueue_ransac(cudaStream_t st, int n_problems, int n_hyp, const RansacDev& d) {
    twoview_normalize_kernel<<<2 * n_problems, 128, 0, st>>>(d.probs, d.kp1, d.kp2, d.kn1, d.kn2, d.norms);
    B200_CUDA(cudaGetLastError());
    if (n_hyp > 0) {
        // 32-thread blocks: one attempt's 100 iterations spread over 4 SMs rather than 1
        twoview_hypothesis_kernel<<<b200::ceil_div(n_hyp, 32), 32, 0, st>>>(n_hyp, d.hyp_problem, d.probs, d.norms, d.kn1, d.kn2, d.matches,
                                                                            d.min_sets, d.hyps);
        B200_CUDA(cudaGetLastError());
        twoview_score_kernel<<<b200::ceil_div(n_hyp, 4), 128, 0, st>>>(n_hyp, d.hyp_problem, d.probs, d.kp1, d.kp2, d.matches, d.hyps, d.scores);
        B200_CUDA(cudaGetLastError());
    }
    twoview_select_kernel<<<b200::ceil_div(n_problems, 64), 64, 0, st>>>(n_problems, d.probs, d.norms, d.kp1, d.kp2, d.kn1, d.kn2, d.matches,
                                                                        d.hyps, d.scores, d.idx, d.mat, d.flags, d.results);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

}  // namespace twoview
}  // namespace b200

extern "C" {

int b200_twoview_ransac(b200_lba_t h, int n_problems, b200_twoview_problem_t* problems) {
    B200_RANGE("b200:twoview:ransac");
    using namespace b200::twoview;
    if (!h || n_problems < 0) return B200_ERR_INVALID;
    if (n_problems == 0) return B200_OK;
    if (!problems) return B200_ERR_INVALID;
    std::vector<ProblemDev> pd(n_problems);
    long long total = 0, total_k1 = 0, total_k2 = 0, total_hyp = 0, total_ms = 0;
    for (int q = 0; q < n_problems; ++q) {
        const b200_twoview_problem_t& P = problems[q];
        const int n = P.n_matches, n1 = P.n_keypts_1, n2 = P.n_keypts_2;
        if (P.model != B200_TWOVIEW_H && P.model != B200_TWOVIEW_F) {
            b200::set_error("b200_twoview_ransac: problem %d: model %d is neither B200_TWOVIEW_H nor B200_TWOVIEW_F", q, P.model);
            return B200_ERR_INVALID;
        }
        if (n < 0 || n1 < 0 || n2 < 0 || (n > 0 && (!P.matches_12 || !P.inlier_flags)) || (n1 > 0 && !P.keypts_1) || (n2 > 0 && !P.keypts_2)) {
            b200::set_error("b200_twoview_ransac: problem %d: negative count or null buffer", q);
            return B200_ERR_INVALID;
        }
        for (int j = 0; j < n; ++j)
            if (P.matches_12[2 * j] < 0 || P.matches_12[2 * j] >= n1 || P.matches_12[2 * j + 1] < 0 || P.matches_12[2 * j + 1] >= n2) {
                b200::set_error("b200_twoview_ransac: problem %d: match %d = (%d, %d) outside the keypoints (%d, %d)", q, j, P.matches_12[2 * j],
                                P.matches_12[2 * j + 1], n1, n2);
                return B200_ERR_INVALID;
            }
        const int set_size = P.model == B200_TWOVIEW_H ? 4 : 8;
        const bool runs = n >= kMinRows;
        if (!b200::min_sets_ok("b200_twoview_ransac", q, runs, P.max_num_iter, P.min_sets, set_size, n)) return B200_ERR_INVALID;
        const int n_hyp = runs ? (int)P.max_num_iter : 0;
        pd[q] = ProblemDev{P.model, n, (int)total, n1, (int)total_k1, n2, (int)total_k2, set_size, (int)total_hyp, (int)total_ms, n_hyp,
                           runs, P.recompute != 0, P.sigma};
        total += n;
        total_k1 += n1;
        total_k2 += n2;
        total_hyp += n_hyp;
        total_ms += (long long)set_size * n_hyp;
        if (total > INT_MAX / 32 || total_k1 > INT_MAX / 16 || total_k2 > INT_MAX / 16 || total_hyp > INT_MAX / 64 || total_ms > INT_MAX / 8) {
            b200::set_error("b200_twoview_ransac: too many keypoints, matches or iterations in one call");
            return B200_ERR_INVALID;
        }
    }
    const size_t T = (size_t)std::max(total, 1LL), K1 = (size_t)std::max(total_k1, 1LL), K2 = (size_t)std::max(total_k2, 1LL);
    const size_t NH = (size_t)std::max(total_hyp, 1LL), NMS = (size_t)std::max(total_ms, 1LL);
    b200::Layout a;
    const size_t o_probs = a.take(sizeof(ProblemDev) * n_problems), o_k1 = a.take(8 * K1), o_k2 = a.take(8 * K2), o_mt = a.take(8 * T);
    const size_t o_ms = a.take(4 * NMS), o_hp = a.take(4 * NH);
    const size_t in_bytes = a.end;
    const size_t o_res = a.take(sizeof(ResultDev) * n_problems), o_fl = a.take(T);
    const size_t out_end = a.end;
    const size_t o_n1 = a.take(8 * K1), o_n2 = a.take(8 * K2), o_norm = a.take(sizeof(NormDev) * n_problems);
    const size_t o_hyp = a.take(sizeof(HypDev) * NH), o_sc = a.take(sizeof(ScoreDev) * NH);
    const size_t o_idx = a.take(4 * T), o_mat = a.take(8 * 18 * T);
    cudaStream_t st;
    b200::StagingArena* A;
    int rc = b200::lba::staging(h, a.end, out_end, &st, &A);
    if (rc) return rc;
    unsigned char *db = A->d, *hb = A->h;
    std::memcpy(hb + o_probs, pd.data(), sizeof(ProblemDev) * n_problems);
    for (int q = 0; q < n_problems; ++q) {
        const b200_twoview_problem_t& P = problems[q];
        const ProblemDev& D = pd[q];
        if (D.n1) std::memcpy(hb + o_k1 + 8 * (size_t)D.kp1_off, P.keypts_1, 8 * (size_t)D.n1);
        if (D.n2) std::memcpy(hb + o_k2 + 8 * (size_t)D.kp2_off, P.keypts_2, 8 * (size_t)D.n2);
        if (D.n) std::memcpy(hb + o_mt + 8 * (size_t)D.match_off, P.matches_12, 8 * (size_t)D.n);
        b200::stage_min_sets(q, P.min_sets, D.set_size, D.n_hyp, (size_t)D.ms_off, D.hyp_off, (int32_t*)(hb + o_ms), (int*)(hb + o_hp));
    }
    B200_CUDA(A->upload(in_bytes, st));
    const RansacDev dev{(const ProblemDev*)(db + o_probs), (const float*)(db + o_k1), (const float*)(db + o_k2), (const int32_t*)(db + o_mt),
                        (const int32_t*)(db + o_ms), (const int*)(db + o_hp), (float*)(db + o_n1), (float*)(db + o_n2), (NormDev*)(db + o_norm),
                        (HypDev*)(db + o_hyp), (ScoreDev*)(db + o_sc), (int32_t*)(db + o_idx), (double*)(db + o_mat), db + o_fl,
                        (ResultDev*)(db + o_res)};
    if ((rc = enqueue_ransac(st, n_problems, (int)total_hyp, dev))) return rc;
    B200_CUDA(A->download(o_res, out_end, st));
    B200_CUDA(cudaStreamSynchronize(st));
    const ResultDev* res = reinterpret_cast<const ResultDev*>(hb + o_res);
    for (int q = 0; q < n_problems; ++q) {
        b200_twoview_problem_t& P = problems[q];
        const ResultDev& r = res[q];
        P.status = r.status ? B200_ERR_INVALID : B200_OK;
        P.valid = r.valid;
        P.best_iter = r.best_iter;
        P.num_inliers = r.num_inliers;
        P.best_cost = r.best_cost;
        if (r.valid) std::memcpy(P.M_21, r.M, sizeof r.M);
        if (pd[q].runs) std::memcpy(P.inlier_flags, hb + o_fl + pd[q].match_off, (size_t)P.n_matches);
    }
    return B200_OK;
}

}  // extern "C"
