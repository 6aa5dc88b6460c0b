// pnp_kernels.cu -- solve::pnp_solver (src/stella_vslam/solve/pnp_solver.cc) on the device: find_via_ransac for many problems in one
// launch sequence, and the static compute_pose.  The minimal sets are drawn on the host (random_array.cu).
//
// find_via_ransac is split in two launches:
//   pnp_hypothesis_kernel  one thread per (problem, hypothesis): EPnP on the minimal set (epnp.cuh), then check_inliers' cost summed
//                          over the matches in ascending index order (a tree sum could change which hypothesis wins);
//   pnp_select_kernel      one thread per problem: the first-wins selection in hypothesis order (num_inliers > min_num_inliers and
//                          min_cost > cost), the winner's inlier flags, and with recompute EPnP over all its inliers.
// Hypotheses are independent once their minimal sets are drawn, and problems are independent (each reference solver owns its engine).
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "epnp.cuh"
#include "ransac_host.cuh"
#include "staging.cuh"
#include "util_trig.cuh"

namespace b200 {
namespace pnp {

struct ProblemDev {
    int n;             // matches
    int match_off;     // first row in the concatenated bearings / points / max_cos / flags
    int hyp_off;       // first hypothesis in the concatenated minimal sets
    int n_hyp;         // max_num_iter (0 when find_via_ransac returns before drawing)
    int runs;          // 0: find_via_ransac returns before drawing (n < 4 or n < min_num_inliers)
    unsigned min_num_inliers, gn_iter;
    int recompute;
};

struct HypDev {
    double R[9], t[3];
    double cost;
    unsigned num_inliers;
    int wrote;         // compute_pose wrote a pose
    int unconverged;
};

struct ResultDev {
    double R[9], t[3];
    double min_cost;
    int valid, best_iter, num_inliers, unconverged;
};

// max_cos_errors_: util::cos(float(scale_factors[octave] * 1 deg in rad)), stored as float
__global__ void pnp_max_cos_kernel(int total, const float* __restrict__ scale, float* __restrict__ max_cos) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    max_cos[i] = util_cos(__double2float_rn(dm((double)scale[i], 1.0 * M_PI / 180.0)));
}

// check_inliers: the cost is summed in ascending match order; flags (may be null) receive the per-match decision
__device__ __forceinline__ unsigned check_inliers(const double* b, const double* p, const float* max_cos, int n, const double* R,
                                                  const double* t, uint8_t* flags, double& cost) {
    unsigned num = 0;
    double c = 0.0;
    for (int j = 0; j < n; ++j) {
        const double ca = cos_angle(R, t, p + 3 * (size_t)j, b + 3 * (size_t)j);
        const float mc = max_cos[j];
        const bool in = (double)mc < ca;
        if (in) {
            c = da(c, ds(1.0, ca));
            ++num;
        } else {
            c = da(c, (double)__fsub_rn(1.0f, mc));  // `1 - max_cos_errors_.at(i)` is float arithmetic
        }
        if (flags) flags[j] = in;
    }
    cost = c;
    return num;
}

__global__ void __launch_bounds__(128) pnp_hypothesis_kernel(int n_hyp_total, const int* __restrict__ hyp_problem,
                                                             const ProblemDev* __restrict__ probs, const double* __restrict__ bearings,
                                                             const double* __restrict__ points, const float* __restrict__ max_cos,
                                                             const int32_t* __restrict__ min_sets, HypDev* __restrict__ hyps) {
    const int h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= n_hyp_total) return;
    const ProblemDev P = probs[hyp_problem[h]];
    const double* b = bearings + 3 * (size_t)P.match_off;
    const double* p = points + 3 * (size_t)P.match_off;
    HypDev out;
    bool wrote;
    int status;
    const Pts s{b, p, min_sets + 4 * (size_t)h, 4};
    compute_pose(s, P.gn_iter, out.R, out.t, wrote, status);
    out.wrote = wrote;
    out.unconverged = status != 0;
    out.cost = 0.0;
    out.num_inliers = 0;
    if (wrote) out.num_inliers = check_inliers(b, p, max_cos + P.match_off, P.n, out.R, out.t, nullptr, out.cost);
    hyps[h] = out;
}

__global__ void __launch_bounds__(64) pnp_select_kernel(int n_problems, const ProblemDev* __restrict__ probs, const double* __restrict__ bearings,
                                                        const double* __restrict__ points, const float* __restrict__ max_cos,
                                                        const HypDev* __restrict__ hyps, int32_t* __restrict__ idx_scratch,
                                                        uint8_t* __restrict__ flags, ResultDev* __restrict__ results) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n_problems) return;
    const ProblemDev P = probs[q];
    ResultDev r;
    r.valid = 0;
    r.best_iter = -1;
    r.num_inliers = 0;
    r.min_cost = DBL_MAX;
    r.unconverged = 0;
    if (!P.runs) {  // returned before drawing
        results[q] = r;
        return;
    }
    const double* b = bearings + 3 * (size_t)P.match_off;
    const double* p = points + 3 * (size_t)P.match_off;
    for (int it = 0; it < P.n_hyp; ++it) {
        const HypDev& H = hyps[P.hyp_off + it];
        r.unconverged |= H.unconverged;
        // a hypothesis without a pose would score the previous hypothesis' pose again: an equal cost never wins (DESIGN.md 8)
        if (H.wrote && H.num_inliers > P.min_num_inliers && r.min_cost > H.cost) {
            r.min_cost = H.cost;
            r.best_iter = it;
            r.num_inliers = (int)H.num_inliers;
        }
    }
    r.valid = r.min_cost < DBL_MAX;
    uint8_t* fl = flags + P.match_off;
    if (!r.valid) {
        for (int j = 0; j < P.n; ++j) fl[j] = 0;
        results[q] = r;
        return;
    }
    const HypDev& B = hyps[P.hyp_off + r.best_iter];
    for (int k = 0; k < 9; ++k) r.R[k] = B.R[k];
    for (int k = 0; k < 3; ++k) r.t[k] = B.t[k];
    double cost;
    check_inliers(b, p, max_cos + P.match_off, P.n, r.R, r.t, fl, cost);
    if (P.recompute) {
        int32_t* idx = idx_scratch + P.match_off;
        const int m = compact_inliers(fl, P.n, idx);
        bool wrote;
        int status;
        compute_pose(Pts{b, p, idx, m}, P.gn_iter, r.R, r.t, wrote, status);
        r.unconverged |= status != 0;
    }
    results[q] = r;
}

struct EpnpDev {
    double R[9], t[3];
    double err;
    int n, off, wrote, unconverged;
    unsigned num_iter;
};

__global__ void __launch_bounds__(64) epnp_kernel(int n_problems, const double* __restrict__ bearings, const double* __restrict__ points,
                                                  EpnpDev* __restrict__ probs) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n_problems) return;
    EpnpDev E = probs[q];
    bool wrote;
    int status;
    E.err = compute_pose(Pts{bearings + 3 * (size_t)E.off, points + 3 * (size_t)E.off, nullptr, E.n}, E.num_iter, E.R, E.t, wrote, status);
    E.wrote = wrote;
    E.unconverged = status != 0;
    probs[q] = E;
}

}  // namespace pnp
}  // namespace b200

extern "C" {

int b200_pnp_ransac(b200_lba_t h, int n_problems, b200_pnp_problem_t* problems) {
    B200_RANGE("b200:pnp:ransac");
    using namespace b200::pnp;
    if (!h || n_problems < 0) return B200_ERR_INVALID;
    if (n_problems == 0) return B200_OK;
    if (!problems) return B200_ERR_INVALID;
    std::vector<ProblemDev> pd(n_problems);
    long long total = 0, total_hyp = 0;
    for (int q = 0; q < n_problems; ++q) {
        const b200_pnp_problem_t& P = problems[q];
        const int n = P.n_matches;
        if (n < 0 || (n > 0 && (!P.bearings || !P.points || !P.octaves || !P.scale_factors || !P.inlier_flags || P.num_levels <= 0))) {
            b200::set_error("b200_pnp_ransac: problem %d: negative count or null buffer", q);
            return B200_ERR_INVALID;
        }
        for (int j = 0; j < n; ++j)
            if (P.octaves[j] < 0 || P.octaves[j] >= P.num_levels) {
                b200::set_error("b200_pnp_ransac: problem %d match %d: octave %d outside [0, %d)", q, j, P.octaves[j], P.num_levels);
                return B200_ERR_INVALID;
            }
        const bool runs = !((unsigned)n < 4u || (unsigned)n < P.min_num_inliers);
        if (!b200::min_sets_ok("b200_pnp_ransac", q, runs, P.max_num_iter, P.min_sets, 4, n)) return B200_ERR_INVALID;
        const int n_hyp = runs ? (int)P.max_num_iter : 0;
        pd[q] = ProblemDev{n, (int)total, (int)total_hyp, n_hyp, runs, P.min_num_inliers, P.gauss_newton_num_iter, P.recompute != 0};
        total += n;
        total_hyp += n_hyp;
        if (total > INT_MAX / 4 || total_hyp > INT_MAX / 4) {
            b200::set_error("b200_pnp_ransac: too many matches or hypotheses in one call");
            return B200_ERR_INVALID;
        }
    }
    const size_t T = (size_t)std::max(total, 1LL), NH = (size_t)std::max(total_hyp, 1LL);
    b200::Layout a;
    const size_t o_probs = a.take(sizeof(ProblemDev) * n_problems), o_b = a.take(24 * T), o_p = a.take(24 * T), o_sf = a.take(4 * T);
    const size_t o_ms = a.take(16 * NH), o_hp = a.take(4 * NH);
    const size_t in_bytes = a.end;
    const size_t o_res = a.take(sizeof(ResultDev) * n_problems), o_fl = a.take(T);
    const size_t out_end = a.end;
    const size_t o_mc = a.take(4 * T), o_hyp = a.take(sizeof(HypDev) * NH), o_idx = a.take(4 * T);
    cudaStream_t st;
    b200::StagingArena* A;
    int rc = b200::lba::staging(h, a.end, out_end, &st, &A);
    if (rc) return rc;
    unsigned char *db = A->d, *hb = A->h;
    std::memcpy(hb + o_probs, pd.data(), sizeof(ProblemDev) * n_problems);
    for (int q = 0; q < n_problems; ++q) {
        const b200_pnp_problem_t& P = problems[q];
        const size_t off = (size_t)pd[q].match_off, n = (size_t)P.n_matches;
        if (n) {
            std::memcpy(hb + o_b + 24 * off, P.bearings, 24 * n);
            std::memcpy(hb + o_p + 24 * off, P.points, 24 * n);
            float* sf = reinterpret_cast<float*>(hb + o_sf) + off;
            for (size_t j = 0; j < n; ++j) sf[j] = P.scale_factors[P.octaves[j]];
        }
        b200::stage_min_sets(q, P.min_sets, 4, pd[q].n_hyp, 4 * (size_t)pd[q].hyp_off, pd[q].hyp_off, (int32_t*)(hb + o_ms), (int*)(hb + o_hp));
    }
    B200_CUDA(A->upload(in_bytes, st));
    const double* d_b = (const double*)(db + o_b);
    const double* d_p = (const double*)(db + o_p);
    const float* d_mc = (const float*)(db + o_mc);
    if (total > 0) {
        pnp_max_cos_kernel<<<b200::ceil_div((int)total, 256), 256, 0, st>>>((int)total, (const float*)(db + o_sf), (float*)(db + o_mc));
        B200_CUDA(cudaGetLastError());
    }
    if (total_hyp > 0) {
        pnp_hypothesis_kernel<<<b200::ceil_div((int)total_hyp, 128), 128, 0, st>>>((int)total_hyp, (const int*)(db + o_hp),
                                                                                   (const ProblemDev*)(db + o_probs), d_b, d_p, d_mc,
                                                                                   (const int32_t*)(db + o_ms), (HypDev*)(db + o_hyp));
        B200_CUDA(cudaGetLastError());
    }
    pnp_select_kernel<<<b200::ceil_div(n_problems, 64), 64, 0, st>>>(n_problems, (const ProblemDev*)(db + o_probs), d_b, d_p, d_mc,
                                                                      (const HypDev*)(db + o_hyp), (int32_t*)(db + o_idx), db + o_fl,
                                                                      (ResultDev*)(db + o_res));
    B200_CUDA(cudaGetLastError());
    B200_CUDA(A->download(o_res, out_end, st));
    B200_CUDA(cudaStreamSynchronize(st));
    const ResultDev* res = reinterpret_cast<const ResultDev*>(hb + o_res);
    for (int q = 0; q < n_problems; ++q) {
        b200_pnp_problem_t& P = problems[q];
        const ResultDev& r = res[q];
        P.status = r.unconverged ? B200_ERR_INVALID : B200_OK;
        P.valid = r.valid;
        P.best_iter = r.best_iter;
        P.num_inliers = r.num_inliers;
        P.min_cost = r.min_cost;
        if (r.valid) {
            std::memcpy(P.rot_cw, r.R, sizeof r.R);
            std::memcpy(P.trans_cw, r.t, sizeof r.t);
        }
        if (pd[q].runs) std::memcpy(P.inlier_flags, hb + o_fl + pd[q].match_off, (size_t)P.n_matches);
    }
    return B200_OK;
}

int b200_epnp_compute_pose(b200_lba_t h, int n_problems, b200_epnp_problem_t* problems) {
    B200_RANGE("b200:pnp:compute_pose");
    using namespace b200::pnp;
    if (!h || n_problems < 0) return B200_ERR_INVALID;
    if (n_problems == 0) return B200_OK;
    if (!problems) return B200_ERR_INVALID;
    long long total = 0;
    for (int q = 0; q < n_problems; ++q) {
        const b200_epnp_problem_t& P = problems[q];
        if (P.n < 1 || !P.bearings || !P.points) {
            b200::set_error("b200_epnp_compute_pose: problem %d: fewer than one point or null buffer", q);
            return B200_ERR_INVALID;
        }
        total += P.n;
        if (total > INT_MAX / 4) return B200_ERR_INVALID;
    }
    b200::Layout a;
    const size_t o_probs = a.take(sizeof(EpnpDev) * n_problems), o_b = a.take(24 * (size_t)total), o_p = a.take(24 * (size_t)total);
    const size_t bytes = a.end;
    cudaStream_t st;
    b200::StagingArena* A;
    int rc = b200::lba::staging(h, bytes, bytes, &st, &A);
    if (rc) return rc;
    unsigned char *db = A->d, *hb = A->h;
    EpnpDev* E = reinterpret_cast<EpnpDev*>(hb + o_probs);
    size_t off = 0;
    for (int q = 0; q < n_problems; ++q) {
        const b200_epnp_problem_t& P = problems[q];
        std::memcpy(E[q].R, P.rot_cw, sizeof E[q].R);
        std::memcpy(E[q].t, P.trans_cw, sizeof E[q].t);
        E[q].n = P.n;
        E[q].off = (int)off;
        E[q].num_iter = P.num_iter;
        std::memcpy(hb + o_b + 24 * off, P.bearings, 24 * (size_t)P.n);
        std::memcpy(hb + o_p + 24 * off, P.points, 24 * (size_t)P.n);
        off += (size_t)P.n;
    }
    B200_CUDA(A->upload(bytes, st));
    epnp_kernel<<<b200::ceil_div(n_problems, 64), 64, 0, st>>>(n_problems, (const double*)(db + o_b), (const double*)(db + o_p), (EpnpDev*)(db + o_probs));
    B200_CUDA(cudaGetLastError());
    B200_CUDA(A->download(o_probs, o_probs + sizeof(EpnpDev) * n_problems, st));
    B200_CUDA(cudaStreamSynchronize(st));
    for (int q = 0; q < n_problems; ++q) {
        b200_epnp_problem_t& P = problems[q];
        P.reproj_error = E[q].err;
        P.wrote = E[q].wrote;
        P.status = E[q].unconverged ? B200_ERR_INVALID : B200_OK;
        if (E[q].wrote) {
            std::memcpy(P.rot_cw, E[q].R, sizeof E[q].R);
            std::memcpy(P.trans_cw, E[q].t, sizeof E[q].t);
        }
    }
    return B200_OK;
}

}  // extern "C"
