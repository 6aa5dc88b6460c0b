// transform_kernels.cu -- optimize::transform_optimizer (the Sim3 refinement of a loop candidate) on sm_90a, fp64.
//
// Reference path (relative to the reference checkout):
//   transform_optimizer::optimize                src/stella_vslam/optimize/transform_optimizer.cc:20-158
//   forward / backward reprojection edges        optimize/internal/sim3/forward_reproj_edge.h, backward_reproj_edge.h
//   edge wrapper (information, Huber delta)      optimize/internal/sim3/mutual_reproj_edge_wrapper.h
//   transform_vertex::oplusImpl                  optimize/internal/sim3/transform_vertex.h
// and upstream g2o (tag 20230223_git, not vendored): g2o::Sim3 (sim3.cuh), BaseFixedSizedEdge's numeric Jacobian (central difference,
// delta 1e-9, errors restored afterwards), RobustKernelHuber, OptimizationAlgorithmLevenberg (tau 1e-5, rho rule, at most 10 trials)
// and SparseOptimizer::optimize, here without a terminate action: every round runs all its iterations unless an LM step fails.
//
// One CTA per problem runs steps 3-7 of the reference in one launch: the LM loops of both rounds with their decisions on the device,
// the outlier test, the early return and the inlier count.  Each thread takes a strided subset of the pairs and sums the 7x7 normal
// equations (28 upper entries), b and the robust chi2 of both edges of each; the CTA combines them in a fixed order (cta_sum) and
// thread 0 solves the damped system.  The 14 perturbed states Sim3(+-delta e_d) * estimate and their inverses are the same for every
// edge, so they are formed once per linearisation in shared memory (g2o forms them per edge: the values are identical).
//
// Which errors the outlier tests read: edge->chi2() returns the error g2o computed last.  SparseOptimizer::optimize does not
// recompute the errors after its last iteration, so that is the error at the last trial state of the round, accepted or rejected
// (EXT? g2o's optimization_algorithm_levenberg.cpp / sparse_optimizer.cpp).  The kernel keeps that state (s_trial) for the tests.
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "lm_common.cuh"
#include "sim3.cuh"
#include "staging.cuh"

namespace b200 {

namespace tfo {

using sim3::Sim3;
constexpr int kThreads = 256;
constexpr double kDelta = 1e-9;                     // BaseFixedSizedEdge::linearizeOplus
constexpr double kPi = 3.14159265358979323846;      // M_PI

static_assert(sizeof(Sim3) == sizeof(b200_sim3_t), "Sim3 layout");

struct Cam {
    int model;
    double fx, fy, cx, cy, cols, rows;
};
struct Prob {
    int n, off, fix_scale;
    Sim3 init;
    double R1[9], t1[3], R2[9], t2[3];
    Cam c1, c2;
};
struct Pair {
    double pw2[3], pw1[3];  // points of edge_12 (lm_2) and edge_21 (lm_1)
    float o1[2], o2[2];     // observations of edge_12 (keyfrm_1) and edge_21 (keyfrm_2)
    float w1, w2;           // inv_level_sigma_sq
};
struct Out {
    Sim3 s;
    unsigned num_inliers;
    int n_outliers1, iterations[2], trials[2];
    double chi2[2], lambda_init[2];
};

// rot * pos_w + trans (the product is evaluated first, in mat3_vec's order)
__device__ __forceinline__ void rigid(const double* R, const double* t, const double* p, double* out) {
    sim3::mat3_vec(R, p, out);
    out[0] += t[0];
    out[1] += t[1];
    out[2] += t[2];
}

// cam_project of the perspective and equirectangular edges (forward_reproj_edge.h, backward_reproj_edge.h)
__device__ __forceinline__ void project(const Cam& c, const double* p, double* u) {
    if (c.model == 1) {
        const double theta = atan2(p[0], p[2]);
        const double phi = -asin(p[1] / sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]));  // EXT? Eigen's norm() summation order
        u[0] = c.cols * (0.5 + theta / (2 * kPi));
        u[1] = c.rows * (0.5 - phi / kPi);
    } else {
        u[0] = c.fx * p[0] / p[2] + c.cx;
        u[1] = c.fy * p[1] / p[2] + c.cy;
    }
}

// computeError: e = obs - cam_project(S.map(pc)); returns chi2() = e . (Omega e) with Omega = w I
__device__ __forceinline__ double edge_chi2(const Sim3& S, const double* pc, const Cam& c, const float* obs, double w, double* e) {
    double p[3], u[2];
    sim3::map(S, pc, p);
    project(c, p, u);
    e[0] = (double)obs[0] - u[0];
    e[1] = (double)obs[1] - u[1];
    return e[0] * (w * e[0]) + e[1] * (w * e[1]);
}

// (A + lambda I) x = b for a 7x7 SPD A given as its 28 upper entries (row-major) by a dense Cholesky; false on a non-positive pivot
__device__ __forceinline__ bool damped_solve7(const double* Hu, const double* b, double lambda, double* x) {
    double A[49];
    int k = 0;
    for (int a = 0; a < 7; ++a)
        for (int c = a; c < 7; ++c) {
            A[a * 7 + c] = Hu[k];
            A[c * 7 + a] = Hu[k];
            ++k;
        }
    for (int a = 0; a < 7; ++a) {
        A[a * 8] += lambda;
        x[a] = b[a];
    }
    for (int j = 0; j < 7; ++j) {
        double d = A[j * 7 + j];
        for (int kk = 0; kk < j; ++kk) d -= A[j * 7 + kk] * A[j * 7 + kk];
        if (!(d > 0) || !isfinite(d)) return false;
        d = sqrt(d);
        A[j * 7 + j] = d;
        for (int i = j + 1; i < 7; ++i) {
            double sv = A[i * 7 + j];
            for (int kk = 0; kk < j; ++kk) sv -= A[i * 7 + kk] * A[j * 7 + kk];
            A[i * 7 + j] = sv / d;
        }
    }
    for (int i = 0; i < 7; ++i) {
        double sv = x[i];
        for (int kk = 0; kk < i; ++kk) sv -= A[i * 7 + kk] * x[kk];
        x[i] = sv / A[i * 8];
    }
    for (int i = 6; i >= 0; --i) {
        double sv = x[i];
        for (int kk = i + 1; kk < 7; ++kk) sv -= A[kk * 7 + i] * x[kk];
        x[i] = sv / A[i * 8];
    }
    return true;
}

constexpr int kAcc = 36;  // 28 upper entries of H, 7 of b, the robust chi2

__global__ void __launch_bounds__(kThreads) transform_optimize_kernel(const Prob* __restrict__ probs, const Pair* __restrict__ pairs_all,
                                                                      unsigned char* __restrict__ keep_all, Out* __restrict__ outs, double delta,
                                                                      double chi_sq, int num_iter) {
    __shared__ double scratch[(kThreads / 32) * kAcc];
    __shared__ double red[kAcc];
    __shared__ Sim3 s_cur, s_cur_inv, s_trial, s_trial_inv, s_pert[14], s_pert_inv[14];
    __shared__ double x[7], s_lambda, s_ni, s_cur_chi;
    __shared__ int s_go_inner, s_go_outer, s_qmax, s_it, s_ok, s_ok2, s_trials, s_bad, s_good;
    __shared__ Prob pb;
    const int tid = threadIdx.x;
    if (tid == 0) pb = probs[blockIdx.x];
    __syncthreads();
    const int n = pb.n, fix_scale = pb.fix_scale;
    const Pair* __restrict__ pairs = pairs_all + pb.off;
    unsigned char* __restrict__ keep = keep_all + pb.off;
    Out* out = outs + blockIdx.x;
    for (int i = tid; i < n; i += kThreads) keep[i] = 1;
    if (tid == 0) {
        s_cur = pb.init;
        s_trial = pb.init;
        s_bad = 0;
        s_good = 0;
        for (int r = 0; r < 2; ++r) {
            out->iterations[r] = 0;
            out->trials[r] = 0;
            out->chi2[r] = 0.0;
            out->lambda_init[r] = 0.0;
        }
        out->n_outliers1 = 0;
        out->num_inliers = 0;
        out->s = pb.init;
    }
    __syncthreads();

    // chi2 of both edges of pair i at the state S (S_inv = S.inverse() for the backward edge)
    auto pair_chi2 = [&](const Pair& pr, const Sim3& S, const Sim3& S_inv, double* c12, double* c21) {
        double p2[3], p1[3], e[2];
        rigid(pb.R2, pb.t2, pr.pw2, p2);
        rigid(pb.R1, pb.t1, pr.pw1, p1);
        *c12 = edge_chi2(S, p2, pb.c1, pr.o1, (double)pr.w1, e);
        *c21 = edge_chi2(S_inv, p1, pb.c2, pr.o2, (double)pr.w2, e);
    };
    // robust chi2 and (optionally) the normal equations of this thread's active pairs at the state S
    auto accumulate = [&](const Sim3& S, const Sim3& S_inv, bool linearize, double (&acc)[kAcc]) {
#pragma unroll
        for (int i = 0; i < kAcc; ++i) acc[i] = 0.0;
        for (int i = tid; i < n; i += kThreads) {
            if (!keep[i]) continue;
            const Pair pr = pairs[i];
            double pc[2][3];
            rigid(pb.R2, pb.t2, pr.pw2, pc[0]);
            rigid(pb.R1, pb.t1, pr.pw1, pc[1]);
            for (int side = 0; side < 2; ++side) {  // edge_12 then edge_21
                const Cam& c = side ? pb.c2 : pb.c1;
                const float* obs = side ? pr.o2 : pr.o1;
                const double w = (double)(side ? pr.w2 : pr.w1);
                double e[2];
                const double chi = edge_chi2(side ? S_inv : S, pc[side], c, obs, w, e);
                acc[35] += huber_cost(chi, delta);
                if (!linearize) continue;
                double J[2][7];
                for (int d = 0; d < 7; ++d) {
                    double ep[2], em[2];
                    edge_chi2(side ? s_pert_inv[2 * d] : s_pert[2 * d], pc[side], c, obs, w, ep);
                    edge_chi2(side ? s_pert_inv[2 * d + 1] : s_pert[2 * d + 1], pc[side], c, obs, w, em);
                    J[0][d] = (1 / (2 * kDelta)) * (ep[0] - em[0]);
                    J[1][d] = (1 / (2 * kDelta)) * (ep[1] - em[1]);
                }
                const double ww = w * huber_weight(chi, delta);
                int k = 0;
#pragma unroll
                for (int a = 0; a < 7; ++a)
#pragma unroll
                    for (int b = a; b < 7; ++b) acc[k++] += ww * (J[0][a] * J[0][b] + J[1][a] * J[1][b]);
#pragma unroll
                for (int a = 0; a < 7; ++a) acc[28 + a] += -ww * (J[0][a] * e[0] + J[1][a] * e[1]);
            }
        }
    };
    // SparseOptimizer::optimize(iters) with OptimizationAlgorithmLevenberg over the active pairs
    auto lm_round = [&](int r, int iters) {
        if (tid == 0) {
            s_it = 0;
            s_ok = 1;
            s_trials = 0;
            s_go_outer = iters > 0 && n > 0;  // no edge, no active vertex: g2o's optimize() returns without iterating
        }
        __syncthreads();
        while (s_go_outer) {
            if (tid < 14) {  // the perturbed states of linearizeOplus: Sim3(+-delta e_d) * estimate
                double u[7] = {0, 0, 0, 0, 0, 0, 0};
                u[tid >> 1] = (tid & 1) ? -kDelta : kDelta;
                s_pert[tid] = sim3::oplus(s_cur, u, fix_scale != 0);
                s_pert_inv[tid] = sim3::inverse(s_pert[tid]);
            } else if (tid == 14) {
                s_cur_inv = sim3::inverse(s_cur);
            }
            __syncthreads();
            double acc[kAcc];
            accumulate(s_cur, s_cur_inv, true, acc);
            cta_sum<kThreads>(acc, red, scratch);
            if (tid == 0) {
                s_cur_chi = red[35];
                if (s_it == 0) {  // computeLambdaInit
                    double mx = 0.0;
                    int k = 0;
                    for (int a = 0; a < 7; ++a) {
                        mx = fmax(mx, fabs(red[k]));
                        k += 7 - a;
                    }
                    s_lambda = 1e-5 * mx;
                    s_ni = 2.0;
                    out->lambda_init[r] = s_lambda;
                }
                s_qmax = 0;
                s_go_inner = 1;
            }
            __syncthreads();
            while (s_go_inner) {
                if (tid == 0) {
                    const bool ok2 = damped_solve7(red, red + 28, s_lambda, x);
                    s_trial = ok2 ? sim3::oplus(s_cur, x, fix_scale != 0) : s_cur;
                    s_trial_inv = sim3::inverse(s_trial);
                    s_ok2 = ok2;
                }
                __syncthreads();
                double tacc[kAcc];
                accumulate(s_trial, s_trial_inv, false, tacc);
                double chi1[1] = {tacc[35]};
                cta_sum<kThreads>(chi1, red + 35, scratch);  // red[0..34] (H, b of the current state) stay valid for the next trial
                if (tid == 0) {
                    const bool ok2 = s_ok2 != 0;
                    s_trials++;
                    const double temp_chi = ok2 ? red[35] : DBL_MAX;
                    double rho = s_cur_chi - temp_chi;
                    double scale = 0.0;  // computeScale
                    if (ok2)
                        for (int i = 0; i < 7; ++i) scale += x[i] * (s_lambda * x[i] + red[28 + i]);
                    scale = ok2 ? scale + 1e-3 : 1;
                    rho /= scale;
                    bool broke = false;
                    if (rho > 0 && isfinite(temp_chi) && ok2) {
                        double alpha = 1. - pow(2 * rho - 1, 3.0);
                        alpha = fmin(alpha, 2. / 3.);
                        s_lambda *= fmax(1. / 3., alpha);
                        s_ni = 2.0;
                        s_cur_chi = temp_chi;
                        s_cur = s_trial;
                    } else {
                        s_lambda *= s_ni;
                        s_ni *= 2.0;
                        if (!isfinite(s_lambda)) broke = true;
                    }
                    if (!broke) s_qmax++;
                    const bool again = !broke && rho < 0 && s_qmax < 10;
                    s_go_inner = again ? 1 : 0;
                    if (!again) {
                        if (s_qmax == 10 || rho == 0 || !isfinite(s_lambda)) s_ok = 0;  // SolverResult::Terminate
                        s_it++;
                        s_go_outer = (s_it < iters && s_ok) ? 1 : 0;
                    }
                }
                __syncthreads();
            }
        }
        if (tid == 0) {
            out->iterations[r] = s_it;
            out->trials[r] = s_trials;
            out->chi2[r] = s_it > 0 ? s_cur_chi : 0.0;
        }
        __syncthreads();
    };

    lm_round(0, 5);  // :98-99
    // :104-119 round-1 outlier test at the errors computed last; outliers go to level 1
    int bad = 0;
    for (int i = tid; i < n; i += kThreads) {
        double c12, c21;
        pair_chi2(pairs[i], s_trial, s_trial_inv, &c12, &c21);
        if (c12 < chi_sq && c21 < chi_sq) continue;
        keep[i] = 0;
        ++bad;
    }
    atomicAdd(&s_bad, bad);
    __syncthreads();
    if (tid == 0) out->n_outliers1 = s_bad;
    if (n - s_bad < 10) return;  // :121-123: the caller's Sim3 stays as it was, the round-1 nulls stand
    lm_round(1, num_iter);       // :127-128
    // :132-151 inlier count of the surviving pairs
    int good = 0;
    for (int i = tid; i < n; i += kThreads) {
        if (!keep[i]) continue;
        double c12, c21;
        pair_chi2(pairs[i], s_trial, s_trial_inv, &c12, &c21);
        if (chi_sq < c12 || chi_sq < c21) {
            keep[i] = 0;
            continue;
        }
        ++good;
    }
    atomicAdd(&s_good, good);
    __syncthreads();
    if (tid == 0) {
        out->num_inliers = (unsigned)s_good;
        out->s = s_cur;  // :155
    }
}

static bool finite_n(const double* v, int n) {
    for (int i = 0; i < n; ++i)
        if (!std::isfinite(v[i])) return false;
    return true;
}
static bool cam_ok(const b200_camera_t& c) {
    const double v[6] = {c.fx, c.fy, c.cx, c.cy, c.cols, c.rows};
    return (c.model == 0 || c.model == 1) && finite_n(v, 6);
}
static bool obs_ok(const float* obs, const float* w, int n) {
    for (int i = 0; i < n; ++i)
        if (!std::isfinite(obs[2 * i]) || !std::isfinite(obs[2 * i + 1]) || !std::isfinite(w[i]) || !(w[i] > 0.f)) return false;
    return true;
}

static int validate(int n_problems, const b200_transform_problem_t* problems) {
    for (int p = 0; p < n_problems; ++p) {
        const b200_transform_problem_t& P = problems[p];
        const int n = P.n_matches;
        if (n < 0 || (n > 0 && (!P.obs_1 || !P.inv_sigma_sq_1 || !P.pos_w_2 || !P.obs_2 || !P.inv_sigma_sq_2 || !P.pos_w_1 || !P.keep))) {
            set_error("b200_transform_optimize: problem %d has a negative count or a null array", p);
            return B200_ERR_INVALID;
        }
        if (!sim3::well_formed(P.sim3_12.q, P.sim3_12.t, P.sim3_12.s) || !finite_n(P.rot_1w, 9) || !finite_n(P.trans_1w, 3)
            || !finite_n(P.rot_2w, 9) || !finite_n(P.trans_2w, 3)) {
            set_error("b200_transform_optimize: problem %d has a non-finite pose, a scale <= 0 or a quaternion far from unit norm", p);
            return B200_ERR_INVALID;
        }
        if (!cam_ok(P.cam_1) || !cam_ok(P.cam_2)) {
            set_error("b200_transform_optimize: problem %d has a camera model other than 0 / 1 or a non-finite intrinsic", p);
            return B200_ERR_INVALID;
        }
        if (n > 0 && (!obs_ok(P.obs_1, P.inv_sigma_sq_1, n) || !obs_ok(P.obs_2, P.inv_sigma_sq_2, n) || !finite_n(P.pos_w_1, 3 * n)
                      || !finite_n(P.pos_w_2, 3 * n))) {
            set_error("b200_transform_optimize: problem %d has a non-finite observation or point, or an inv_sigma_sq <= 0", p);
            return B200_ERR_INVALID;
        }
    }
    return B200_OK;
}

static Cam to_cam(const b200_camera_t& c) { return Cam{c.model, c.fx, c.fy, c.cx, c.cy, c.cols, c.rows}; }

}  // namespace tfo
}  // namespace b200

extern "C" {

int b200_transform_optimize(b200_lba_t h, int n_problems, b200_transform_problem_t* problems, float chi_sq, int num_iter) {
    B200_RANGE("b200:lba:transform_optimize");
    using namespace b200::tfo;
    if (!h || n_problems < 0 || (n_problems > 0 && !problems) || !(chi_sq > 0.f) || !std::isfinite(chi_sq) || num_iter < 0) {
        b200::set_error("b200_transform_optimize: null or out-of-range argument");
        return B200_ERR_INVALID;
    }
    int rc = validate(n_problems, problems);
    if (rc) return rc;
    if (n_problems == 0) return B200_OK;
    size_t total = 0;
    for (int p = 0; p < n_problems; ++p) total += (size_t)problems[p].n_matches;
    b200::Layout L;
    const size_t o_probs = L.take<Prob>(n_problems), o_pairs = L.take<Pair>(total);
    const size_t in_bytes = L.end;
    const size_t o_out = L.take<Out>(n_problems), o_keep = L.take(total);
    cudaStream_t st;
    b200::StagingArena* A;
    if ((rc = b200::lba::staging(h, L.end, L.end, &st, &A))) return rc;
    unsigned char *d = A->d, *hs = A->h;
    Prob* hp = reinterpret_cast<Prob*>(hs + o_probs);
    Pair* hq = reinterpret_cast<Pair*>(hs + o_pairs);
    size_t off = 0;
    for (int p = 0; p < n_problems; ++p) {
        const b200_transform_problem_t& P = problems[p];
        Prob pb{};
        pb.n = P.n_matches;
        pb.off = (int)off;
        pb.fix_scale = P.fix_scale ? 1 : 0;
        std::memcpy(&pb.init, &P.sim3_12, sizeof(Sim3));
        std::memcpy(pb.R1, P.rot_1w, sizeof(pb.R1));
        std::memcpy(pb.t1, P.trans_1w, sizeof(pb.t1));
        std::memcpy(pb.R2, P.rot_2w, sizeof(pb.R2));
        std::memcpy(pb.t2, P.trans_2w, sizeof(pb.t2));
        pb.c1 = to_cam(P.cam_1);
        pb.c2 = to_cam(P.cam_2);
        hp[p] = pb;
        for (int i = 0; i < P.n_matches; ++i) {
            Pair& q = hq[off + i];
            for (int k = 0; k < 3; ++k) {
                q.pw2[k] = P.pos_w_2[3 * i + k];
                q.pw1[k] = P.pos_w_1[3 * i + k];
            }
            q.o1[0] = P.obs_1[2 * i]; q.o1[1] = P.obs_1[2 * i + 1];
            q.o2[0] = P.obs_2[2 * i]; q.o2[1] = P.obs_2[2 * i + 1];
            q.w1 = P.inv_sigma_sq_1[i];
            q.w2 = P.inv_sigma_sq_2[i];
        }
        off += (size_t)P.n_matches;
    }
    const float sqrt_chi_sq = std::sqrt(chi_sq);  // transform_optimizer.cc:23: the Huber delta is computed in float
    B200_CUDA(A->upload(in_bytes, st));
    transform_optimize_kernel<<<n_problems, kThreads, 0, st>>>((const Prob*)(d + o_probs), (const Pair*)(d + o_pairs), d + o_keep, (Out*)(d + o_out),
                                                              (double)sqrt_chi_sq, (double)chi_sq, num_iter);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(A->download(o_out, L.end, st));
    B200_CUDA(cudaStreamSynchronize(st));
    const Out* ho = reinterpret_cast<const Out*>(hs + o_out);
    off = 0;
    for (int p = 0; p < n_problems; ++p) {
        b200_transform_problem_t& P = problems[p];
        const Out& o = ho[p];
        std::memcpy(&P.sim3_12_out, &o.s, sizeof(Sim3));
        if (P.n_matches > 0) std::memcpy(P.keep, hs + o_keep + off, (size_t)P.n_matches);
        P.num_inliers = o.num_inliers;
        P.n_outliers_round1 = o.n_outliers1;
        for (int r = 0; r < 2; ++r) {
            P.iterations[r] = o.iterations[r];
            P.trials[r] = o.trials[r];
            P.chi2[r] = o.chi2[r];
            P.lambda_init[r] = o.lambda_init[r];
        }
        off += (size_t)P.n_matches;
    }
    return B200_OK;
}

}  // extern "C"
