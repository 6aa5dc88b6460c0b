// initialize_kernels.cu -- initialize::perspective::initialize and initialize::bearing_vector::initialize
// (src/stella_vslam/initialize/perspective.cc, bearing_vector.cc, base.cc) for many frame pairs in one launch sequence on the
// b200_lba_t handle's stream:
//   the RANSAC launches of b200_twoview_ransac (one H and one F problem per perspective pair) and of b200_essential_ransac (one E
//   problem per bearing-vector pair), recompute = false;
//   init_choose_kernel       one CTA per pair: the rel_cost_H rule and the decomposition of the winner (thread 0), the chosen
//                            solver's inlier flags copied by the whole CTA;
//   init_triangulate_kernel  one CTA per (pair, hypothesis): base::triangulate, the threads striding over the matches; the counts by
//                            block reductions, the 50th-smallest parallax cosine by a radix select on the float bits;
//   init_select_kernel       one CTA per pair: find_most_plausible_pose's rules (thread 0), then the winner's points and flags
//                            scattered to their ref keypoints.
// The arithmetic is csrc/initialize_core.h; tests/initialize_oracle.c compiles the same header as C.  This file is compiled with
// -fmad=false for reproject_to_image (camera_model.cuh).
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>

#include "camera_model.cuh"
#include "common.cuh"
#include "epnp.cuh"
#include "essential_ransac.cuh"
#include "ransac_host.cuh"
#include "staging.cuh"
#include "track_chain.cuh"
#include "twoview_ransac.cuh"
#include "util_trig.cuh"

namespace b200 {
namespace init {

using pnp::apply_householder_left;  // es_svd_n9 (essential_core.h) calls both unqualified
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

struct InitCam {
    orb::CamModel cam;
    float bounds[4];  // min_x, max_x, min_y, max_y
};
typedef InitCam in_cam_t;

__device__ __forceinline__ int in_reproject(const InitCam* c, const double* Rt, const double* p, double* q) {
    float x_right;
    return orb::reproject_to_image(c->cam, 0.0, c->bounds[0], c->bounds[1], c->bounds[2], c->bounds[3], Rt, p[0], p[1], p[2], q[0], q[1],
                                   x_right);
}

#define IN_FSQRT(x) __fsqrt_rn(x)
#include "initialize_core.h"

static_assert(IN_MODEL_H == B200_INIT_MODEL_H && IN_MODEL_F == B200_INIT_MODEL_F && IN_MODEL_E == B200_INIT_MODEL_E, "model codes");
static_assert(IN_STAGE_DECOMPOSE == B200_INIT_STAGE_DECOMPOSE && IN_STAGE_SUCCEEDED == B200_INIT_STAGE_SUCCEEDED &&
                  IN_STAGE_MIN_TRIANGULATED == B200_INIT_STAGE_MIN_TRIANGULATED,
              "stage codes");

constexpr int kMaxHyp = 8;
constexpr int kThreads = 128;

struct InitDev {
    InitCam cam[2];  // ref, cur
    double K[2][9];  // eigen_cam_matrix_ of each view (perspective path)
    int bearing;     // 0: perspective (H and F), 1: bearing_vector (E)
    int n_ref, ref_off, n_cur, cur_off;  // keypoints in the concatenated undistorted keypoints / bearings
    int n, match_off;                    // ref_cur_matches_ in the concatenated matches / flags
    int solver;      // perspective: the H problem among the two-view problems (F is solver + 1); bearing vector: the essential problem
    unsigned min_num_triangulated, min_num_valid_pts;
    float thr_sq;    // reproj_err_thr * reproj_err_thr
    double cos_thr;  // cos(parallax_deg_thr / 180 pi)
};

struct HypPoses {
    double Rt[kMaxHyp][12];  // rotation row-major, then translation
};

struct ResultDev {
    int status, model, stage, n_hyp, best;
    float cost[3];  // H, F, E
    int valid[3], num_inliers[3];
    int32_t nums_valid[kMaxHyp], num_triangulated[kMaxHyp];
    float parallax_cos[kMaxHyp];
    double R[9], t[3];
};

__global__ void __launch_bounds__(64) init_choose_kernel(const InitDev* __restrict__ probs, const twoview::ProblemDev* __restrict__ tv_probs,
                                                         const twoview::ResultDev* __restrict__ tv_res, const uint8_t* __restrict__ tv_flags,
                                                         const ess::ProblemDev* __restrict__ es_probs, const ess::ResultDev* __restrict__ es_res,
                                                         const uint8_t* __restrict__ es_flags, HypPoses* __restrict__ poses,
                                                         uint8_t* __restrict__ inlier, ResultDev* __restrict__ results) {
    const int q = blockIdx.x;
    const InitDev& P = probs[q];
    __shared__ const uint8_t* s_flags;
    if (threadIdx.x == 0) {
        ResultDev r;
        memset(&r, 0, sizeof r);
        r.model = IN_MODEL_NONE;
        r.stage = IN_STAGE_NO_MODEL;
        const uint8_t* fl = nullptr;
        const double* M = nullptr;
        if (!P.bearing) {
            const twoview::ResultDev &H = tv_res[P.solver], &F = tv_res[P.solver + 1];
            r.cost[0] = H.best_cost, r.valid[0] = H.valid, r.num_inliers[0] = H.num_inliers;
            r.cost[1] = F.best_cost, r.valid[1] = F.valid, r.num_inliers[1] = F.num_inliers;
            r.status |= H.status | F.status;
            if (in_choose_H(H.best_cost, F.best_cost, H.valid)) {
                r.model = IN_MODEL_H, M = H.M, fl = tv_flags + tv_probs[P.solver].match_off;
            } else if (F.valid) {
                r.model = IN_MODEL_F, M = F.M, fl = tv_flags + tv_probs[P.solver + 1].match_off;
            }
        } else {
            const ess::ResultDev& E = es_res[P.solver];
            r.cost[2] = E.best_cost, r.valid[2] = E.valid, r.num_inliers[2] = E.num_inliers;
            r.status |= E.status;
            if (E.valid) r.model = IN_MODEL_E, M = E.E, fl = es_flags + es_probs[P.solver].match_off;
        }
        double R[kMaxHyp * 9], t[kMaxHyp * 3];
        if (r.model == IN_MODEL_H) {
            double nrm[kMaxHyp * 3];
            if (in_decompose_H(M, P.K[0], P.K[1], R, t, nrm, &r.status))
                r.n_hyp = 8;
            else
                r.stage = IN_STAGE_DECOMPOSE;
        } else if (r.model != IN_MODEL_NONE) {
            double E[9];
            if (r.model == IN_MODEL_F) {
                in_essential_of_F(M, P.K[0], P.K[1], E);
                M = E;
            }
            in_decompose_E(M, R, t, &r.status);
            r.n_hyp = 4;
        }
        for (int h = 0; h < r.n_hyp; ++h) {
            for (int k = 0; k < 9; ++k) poses[q].Rt[h][k] = R[9 * h + k];
            for (int k = 0; k < 3; ++k) poses[q].Rt[h][9 + k] = t[3 * h + k];
        }
        results[q] = r;
        s_flags = fl;
    }
    __syncthreads();
    const uint8_t* fl = s_flags;
    if (fl)
        for (int j = threadIdx.x; j < P.n; j += blockDim.x) inlier[P.match_off + j] = fl[j];
}

__device__ __forceinline__ unsigned float_key(float f) {  // ascending keys in ascending float order
    const unsigned b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_float(unsigned k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k); }

__device__ __forceinline__ unsigned block_sum(unsigned v, unsigned* red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    unsigned s = 0;
    for (int w = 0; w < kThreads / 32; ++w) s += red[w];
    __syncthreads();
    return s;
}

// Per match row (8 rows of n per pair): state IN_TRI_*, its parallax cosine and, when triangulated, its point.
__global__ void __launch_bounds__(kThreads) init_triangulate_kernel(const InitDev* __restrict__ probs, const float* __restrict__ undist,
                                                                    const double* __restrict__ bearings, const int32_t* __restrict__ matches,
                                                                    const uint8_t* __restrict__ inlier, const HypPoses* __restrict__ poses,
                                                                    uint8_t* __restrict__ state, float* __restrict__ cosp, double* __restrict__ pts,
                                                                    ResultDev* __restrict__ results) {
    const int q = blockIdx.x, hyp = blockIdx.y;
    if (hyp >= results[q].n_hyp) return;  // block-uniform
    const InitDev& P = probs[q];
    double Rt[12], ctr[3];
    for (int k = 0; k < 12; ++k) Rt[k] = poses[q].Rt[hyp][k];
    in_neg_rt_t(Rt, Rt + 9, ctr);
    const InitCam cam_ref = P.cam[0], cam_cur = P.cam[1];
    const size_t row = (size_t)kMaxHyp * P.match_off + (size_t)hyp * P.n;
    const int32_t* mt = matches + 2 * (size_t)P.match_off;
    unsigned n_valid = 0, n_tri = 0;
    for (int j = threadIdx.x; j < P.n; j += blockDim.x) {
        int s = IN_TRI_REJECTED;
        if (inlier[P.match_off + j]) {
            const int kr = P.ref_off + mt[2 * j], kc = P.cur_off + mt[2 * j + 1];
            double p[3];
            float c;
            s = in_match(&cam_ref, &cam_cur, Rt, ctr, !P.bearing, P.thr_sq, bearings + 3 * (size_t)kr, bearings + 3 * (size_t)kc,
                         undist + 2 * (size_t)kr, undist + 2 * (size_t)kc, p, &c);
            if (s != IN_TRI_REJECTED) {
                cosp[row + j] = c;
                ++n_valid;
            }
            if (s == IN_TRI_TRIANGULATED) {
                for (int k = 0; k < 3; ++k) pts[3 * (row + j) + k] = p[k];
                ++n_tri;
            }
        }
        state[row + j] = (uint8_t)s;
    }
    __shared__ unsigned red[kThreads / 32];
    n_valid = block_sum(n_valid, red);
    n_tri = block_sum(n_tri, red);
    float parallax = 1.0f;
    if (n_valid > 0) {
        // the element at index min(50, n_valid - 1) of the ascending cosines: a radix select, 8 bits per pass from the top
        __shared__ unsigned hist[256], s_prefix, s_k;
        if (threadIdx.x == 0) {
            s_prefix = 0;
            s_k = min(50u, n_valid - 1);
        }
        unsigned mask = 0;
        for (int shift = 24; shift >= 0; shift -= 8) {
            for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
            __syncthreads();
            const unsigned prefix = s_prefix;
            for (int j = threadIdx.x; j < P.n; j += blockDim.x)
                if (state[row + j] != IN_TRI_REJECTED) {
                    const unsigned key = float_key(cosp[row + j]);
                    if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
                }
            __syncthreads();
            if (threadIdx.x == 0) {
                unsigned k = s_k, b = 0;
                while (hist[b] <= k) k -= hist[b++];
                s_k = k;
                s_prefix = prefix | (b << shift);
            }
            mask |= 255u << shift;
            __syncthreads();
        }
        parallax = key_float(s_prefix);
    }
    if (threadIdx.x == 0) {
        results[q].nums_valid[hyp] = (int32_t)n_valid;
        results[q].num_triangulated[hyp] = (int32_t)n_tri;
        results[q].parallax_cos[hyp] = parallax;
    }
}

__global__ void __launch_bounds__(kThreads) init_select_kernel(const InitDev* __restrict__ probs, const int32_t* __restrict__ matches,
                                                               const HypPoses* __restrict__ poses, const uint8_t* __restrict__ state,
                                                               const double* __restrict__ pts, ResultDev* __restrict__ results,
                                                               double* __restrict__ pts_out, uint8_t* __restrict__ tri_out) {
    const int q = blockIdx.x;
    const InitDev& P = probs[q];
    __shared__ int s_ok, s_best;
    if (threadIdx.x == 0) {
        ResultDev& r = results[q];
        s_ok = 0;
        if (r.n_hyp > 0) {
            int best;
            r.stage = in_select(r.n_hyp, r.nums_valid, r.num_triangulated, r.parallax_cos, P.min_num_valid_pts, P.min_num_triangulated, P.cos_thr,
                                &best);
            r.best = best;
            s_ok = r.stage == IN_STAGE_SUCCEEDED;
            s_best = best;
            for (int k = 0; k < 9; ++k) r.R[k] = s_ok ? poses[q].Rt[best][k] : 0.0;
            for (int k = 0; k < 3; ++k) r.t[k] = s_ok ? poses[q].Rt[best][9 + k] : 0.0;
        }
    }
    __syncthreads();
    if (!s_ok) return;
    for (int i = threadIdx.x; i < P.n_ref; i += blockDim.x) {
        tri_out[P.ref_off + i] = 0;
        for (int k = 0; k < 3; ++k) pts_out[3 * (size_t)(P.ref_off + i) + k] = 0.0;
    }
    __syncthreads();
    const size_t row = (size_t)kMaxHyp * P.match_off + (size_t)s_best * P.n;
    const int32_t* mt = matches + 2 * (size_t)P.match_off;
    for (int j = threadIdx.x; j < P.n; j += blockDim.x)
        if (state[row + j] == IN_TRI_TRIANGULATED) {
            const size_t r = (size_t)(P.ref_off + mt[2 * j]);
            tri_out[r] = 1;
            for (int k = 0; k < 3; ++k) pts_out[3 * r + k] = pts[3 * (row + j) + k];
        }
}

static bool check_problem(int q, const b200_init_problem_t& P) {
    if (!b200::chain::camera_valid(P.cam_ref) || !b200::chain::camera_valid(P.cam_cur)) {
        b200::set_error("b200_initialize: problem %d: camera model outside 0-3 or non-finite intrinsics", q);
        return false;
    }
    if ((P.cam_ref.model == 1) != (P.cam_cur.model == 1)) {
        b200::set_error("b200_initialize: problem %d: equirectangular on one view only", q);
        return false;
    }
    if (P.n_ref < 0 || P.n_cur < 0 || P.num_ransac_iters > (uint32_t)INT_MAX) {
        b200::set_error("b200_initialize: problem %d: negative keypoint count or num_ransac_iters above INT_MAX", q);
        return false;
    }
    if ((P.n_ref > 0 && (!P.undist_ref || !P.bearings_ref || !P.ref_matches_with_cur || !P.triangulated_pts || !P.triangulated_flags)) ||
        (P.n_cur > 0 && (!P.undist_cur || !P.bearings_cur))) {
        b200::set_error("b200_initialize: problem %d: null buffer", q);
        return false;
    }
    for (int i = 0; i < P.n_ref; ++i)
        if (P.ref_matches_with_cur[i] >= P.n_cur) {
            b200::set_error("b200_initialize: problem %d: ref keypoint %d matched to %d, outside the %d current keypoints", q, i,
                            P.ref_matches_with_cur[i], P.n_cur);
            return false;
        }
    return true;
}

}  // namespace init
}  // namespace b200

extern "C" {

int b200_initialize(b200_lba_t h, int n_problems, b200_init_problem_t* problems) {
    B200_RANGE("b200:initialize");
    using namespace b200::init;
    namespace tv = b200::twoview;
    namespace es = b200::ess;
    if (!h || n_problems < 0) return B200_ERR_INVALID;
    if (n_problems == 0) return B200_OK;
    if (!problems) return B200_ERR_INVALID;
    const int iters_bound = INT_MAX / 64;
    std::vector<InitDev> pd(n_problems);
    std::vector<tv::ProblemDev> tvd;
    std::vector<es::ProblemDev> esd;
    long long tot_kp = 0, tot_m = 0, tv_kp = 0, tv_m = 0, tv_hyp = 0, tv_ms = 0, es_m = 0, es_hyp = 0;
    for (int q = 0; q < n_problems; ++q) {
        const b200_init_problem_t& P = problems[q];
        if (!check_problem(q, P)) return B200_ERR_INVALID;
        int n = 0;
        for (int i = 0; i < P.n_ref; ++i) n += P.ref_matches_with_cur[i] >= 0;
        InitDev& D = pd[q];
        memset(&D, 0, sizeof D);
        const b200_camera_intrinsics_t* cams[2] = {&P.cam_ref, &P.cam_cur};
        const float* bounds[2] = {P.img_bounds_ref, P.img_bounds_cur};
        for (int v = 0; v < 2; ++v) {
            D.cam[v].cam = b200::orb::cam_model(*cams[v]);
            for (int k = 0; k < 4; ++k) D.cam[v].bounds[k] = bounds[v][k];
            const double K[9] = {cams[v]->fx, 0.0, cams[v]->cx, 0.0, cams[v]->fy, cams[v]->cy, 0.0, 0.0, 1.0};
            for (int k = 0; k < 9; ++k) D.K[v][k] = K[k];
        }
        D.bearing = P.cam_ref.model == 1;
        D.n_ref = P.n_ref, D.ref_off = (int)tot_kp, D.n_cur = P.n_cur, D.cur_off = (int)(tot_kp + P.n_ref);
        D.n = n, D.match_off = (int)tot_m;
        D.min_num_triangulated = P.min_num_triangulated, D.min_num_valid_pts = P.min_num_valid_pts;
        D.thr_sq = P.reproj_err_thr * P.reproj_err_thr;
        D.cos_thr = std::cos((double)P.parallax_deg_thr / 180.0 * M_PI);
        const int iters = (int)P.num_ransac_iters;
        if (!D.bearing) {
            D.solver = (int)tvd.size();
            const bool runs = n >= tv::kMinRows;
            if (!b200::min_sets_ok("b200_initialize", q, runs, P.num_ransac_iters, P.min_sets_H, 4, n) ||
                !b200::min_sets_ok("b200_initialize", q, runs, P.num_ransac_iters, P.min_sets_F, 8, n))
                return B200_ERR_INVALID;
            for (int model = 0; model < 2; ++model) {
                const int set_size = model == TV_MODEL_H ? 4 : 8, n_hyp = runs ? iters : 0;
                tvd.push_back(tv::ProblemDev{model, n, (int)tv_m, P.n_ref, (int)tv_kp, P.n_cur, (int)tv_kp + P.n_ref, set_size, (int)tv_hyp,
                                             (int)tv_ms, n_hyp, runs, 0, 1.0f});
                tv_kp += P.n_ref + P.n_cur;
                tv_m += n;
                tv_hyp += n_hyp;
                tv_ms += (long long)set_size * n_hyp;
            }
        } else {
            D.solver = (int)esd.size();
            const bool runs = n >= es::kMinSet;
            if (!b200::min_sets_ok("b200_initialize", q, runs, P.num_ransac_iters, P.min_sets_E, es::kMinSet, n)) return B200_ERR_INVALID;
            const int n_hyp = runs ? iters : 0;
            esd.push_back(es::ProblemDev{n, (int)es_m, (int)es_hyp, n_hyp, runs, 0});
            es_m += n;
            es_hyp += n_hyp;
        }
        tot_kp += P.n_ref + P.n_cur;
        tot_m += n;
        if (tot_kp > INT_MAX / 32 || tot_m > INT_MAX / 256 || tv_kp > INT_MAX / 16 || tv_hyp > iters_bound || tv_ms > INT_MAX / 8 ||
            es_hyp > iters_bound) {
            b200::set_error("b200_initialize: too many keypoints, matches or iterations in one call");
            return B200_ERR_INVALID;
        }
    }
    const int n_tv = (int)tvd.size(), n_es = (int)esd.size();
    auto sz = [](long long v) { return (size_t)std::max(v, 1LL); };
    b200::Layout a;
    const size_t o_probs = a.take(sizeof(InitDev) * n_problems), o_kp = a.take(8 * sz(tot_kp)), o_br = a.take(24 * sz(tot_kp));
    const size_t o_mt = a.take(8 * sz(tot_m));
    const size_t o_tvp = a.take(sizeof(tv::ProblemDev) * sz(n_tv)), o_tvk = a.take(8 * sz(tv_kp)), o_tvm = a.take(8 * sz(tv_m));
    const size_t o_tvms = a.take(4 * sz(tv_ms)), o_tvhp = a.take(4 * sz(tv_hyp));
    const size_t o_esp = a.take(sizeof(es::ProblemDev) * sz(n_es)), o_esb1 = a.take(24 * sz(es_m)), o_esb2 = a.take(24 * sz(es_m));
    const size_t o_esms = a.take(4 * es::kMinSet * sz(es_hyp)), o_eshp = a.take(4 * sz(es_hyp));
    const size_t in_bytes = a.end;
    const size_t o_res = a.take(sizeof(ResultDev) * n_problems), o_pts = a.take(24 * sz(tot_kp)), o_tri = a.take(sz(tot_kp));
    const size_t o_inl = a.take(sz(tot_m));
    const size_t out_end = a.end;
    const size_t o_tvkn = a.take(8 * sz(tv_kp)), o_tvnorm = a.take(sizeof(tv::NormDev) * sz(n_tv));
    const size_t o_tvhyp = a.take(sizeof(tv::HypDev) * sz(tv_hyp)), o_tvsc = a.take(sizeof(tv::ScoreDev) * sz(tv_hyp));
    const size_t o_tvidx = a.take(4 * sz(tv_m)), o_tvmat = a.take(8 * 18 * sz(tv_m)), o_tvfl = a.take(sz(tv_m));
    const size_t o_tvres = a.take(sizeof(tv::ResultDev) * sz(n_tv));
    const size_t o_escand = a.take(8 * 9 * es::kMaxCand * sz(es_hyp)), o_eshyp = a.take(sizeof(es::HypDev) * sz(es_hyp));
    const size_t o_essc = a.take(sizeof(es::ScoreDev) * es::kMaxCand * sz(es_hyp)), o_esidx = a.take(4 * sz(es_m));
    const size_t o_esmat = a.take(72 * sz(es_m)), o_esfl = a.take(sz(es_m)), o_esres = a.take(sizeof(es::ResultDev) * sz(n_es));
    const size_t o_poses = a.take(sizeof(HypPoses) * n_problems), o_state = a.take(kMaxHyp * sz(tot_m));
    const size_t o_cosp = a.take(4 * kMaxHyp * sz(tot_m)), o_hpts = a.take(24 * kMaxHyp * sz(tot_m));
    cudaStream_t st;
    b200::StagingArena* A;
    int rc = b200::lba::staging(h, a.end, out_end, &st, &A);
    if (rc) return rc;
    unsigned char *db = A->d, *hb = A->h;
    std::memcpy(hb + o_probs, pd.data(), sizeof(InitDev) * n_problems);
    if (n_tv) std::memcpy(hb + o_tvp, tvd.data(), sizeof(tv::ProblemDev) * n_tv);
    if (n_es) std::memcpy(hb + o_esp, esd.data(), sizeof(es::ProblemDev) * n_es);
    for (int q = 0; q < n_problems; ++q) {
        const b200_init_problem_t& P = problems[q];
        const InitDev& D = pd[q];
        A->put(o_kp + 8 * (size_t)D.ref_off, P.undist_ref, 8 * (size_t)P.n_ref);
        A->put(o_kp + 8 * (size_t)D.cur_off, P.undist_cur, 8 * (size_t)P.n_cur);
        A->put(o_br + 24 * (size_t)D.ref_off, P.bearings_ref, 24 * (size_t)P.n_ref);
        A->put(o_br + 24 * (size_t)D.cur_off, P.bearings_cur, 24 * (size_t)P.n_cur);
        int32_t* mt = (int32_t*)(hb + o_mt) + 2 * (size_t)D.match_off;
        int m = 0;
        for (int i = 0; i < P.n_ref; ++i)
            if (P.ref_matches_with_cur[i] >= 0) {
                mt[2 * m] = i;
                mt[2 * m + 1] = P.ref_matches_with_cur[i];
                ++m;
            }
        if (!D.bearing) {
            const int32_t* sets[2] = {P.min_sets_H, P.min_sets_F};
            for (int k = 0; k < 2; ++k) {
                const tv::ProblemDev& T = tvd[D.solver + k];
                A->put(o_tvk + 8 * (size_t)T.kp1_off, P.undist_ref, 8 * (size_t)P.n_ref);
                A->put(o_tvk + 8 * (size_t)T.kp2_off, P.undist_cur, 8 * (size_t)P.n_cur);
                A->put(o_tvm + 8 * (size_t)T.match_off, mt, 8 * (size_t)D.n);
                b200::stage_min_sets(D.solver + k, sets[k], T.set_size, T.n_hyp, (size_t)T.ms_off, T.hyp_off, (int32_t*)(hb + o_tvms),
                                     (int*)(hb + o_tvhp));
            }
        } else {
            const es::ProblemDev& E = esd[D.solver];
            double* b1 = (double*)(hb + o_esb1) + 3 * (size_t)E.match_off;
            double* b2 = (double*)(hb + o_esb2) + 3 * (size_t)E.match_off;
            for (int j = 0; j < D.n; ++j) {
                std::memcpy(b1 + 3 * (size_t)j, P.bearings_ref + 3 * (size_t)mt[2 * j], 24);
                std::memcpy(b2 + 3 * (size_t)j, P.bearings_cur + 3 * (size_t)mt[2 * j + 1], 24);
            }
            b200::stage_min_sets(D.solver, P.min_sets_E, es::kMinSet, E.n_hyp, es::kMinSet * (size_t)E.hyp_off, E.hyp_off, (int32_t*)(hb + o_esms),
                                 (int*)(hb + o_eshp));
        }
    }
    B200_CUDA(A->upload(in_bytes, st));
    if (n_tv) {
        const tv::RansacDev dev{(const tv::ProblemDev*)(db + o_tvp), (const float*)(db + o_tvk), (const float*)(db + o_tvk),
                                (const int32_t*)(db + o_tvm), (const int32_t*)(db + o_tvms), (const int*)(db + o_tvhp), (float*)(db + o_tvkn),
                                (float*)(db + o_tvkn), (tv::NormDev*)(db + o_tvnorm), (tv::HypDev*)(db + o_tvhyp), (tv::ScoreDev*)(db + o_tvsc),
                                (int32_t*)(db + o_tvidx), (double*)(db + o_tvmat), db + o_tvfl, (tv::ResultDev*)(db + o_tvres)};
        if ((rc = tv::enqueue_ransac(st, n_tv, (int)tv_hyp, dev))) return rc;
    }
    if (n_es) {
        const es::RansacDev dev{(const int*)(db + o_eshp), (const es::ProblemDev*)(db + o_esp), (const double*)(db + o_esb1),
                                (const double*)(db + o_esb2), (const int32_t*)(db + o_esms), (double*)(db + o_escand), (es::HypDev*)(db + o_eshyp),
                                (es::ScoreDev*)(db + o_essc), (int32_t*)(db + o_esidx), (double*)(db + o_esmat), db + o_esfl,
                                (es::ResultDev*)(db + o_esres)};
        if ((rc = es::enqueue_ransac(st, n_es, (int)es_hyp, dev))) return rc;
    }
    const InitDev* d_probs = (const InitDev*)(db + o_probs);
    ResultDev* d_res = (ResultDev*)(db + o_res);
    init_choose_kernel<<<n_problems, 64, 0, st>>>(d_probs, (const tv::ProblemDev*)(db + o_tvp), (const tv::ResultDev*)(db + o_tvres), db + o_tvfl,
                                                  (const es::ProblemDev*)(db + o_esp), (const es::ResultDev*)(db + o_esres), db + o_esfl,
                                                  (HypPoses*)(db + o_poses), db + o_inl, d_res);
    B200_CUDA(cudaGetLastError());
    init_triangulate_kernel<<<dim3(n_problems, kMaxHyp), kThreads, 0, st>>>(d_probs, (const float*)(db + o_kp), (const double*)(db + o_br),
                                                                           (const int32_t*)(db + o_mt), db + o_inl, (const HypPoses*)(db + o_poses),
                                                                           db + o_state, (float*)(db + o_cosp), (double*)(db + o_hpts), d_res);
    B200_CUDA(cudaGetLastError());
    init_select_kernel<<<n_problems, kThreads, 0, st>>>(d_probs, (const int32_t*)(db + o_mt), (const HypPoses*)(db + o_poses), db + o_state,
                                                        (const double*)(db + o_hpts), d_res, (double*)(db + o_pts), db + o_tri);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(A->download(o_res, out_end, st));
    B200_CUDA(cudaStreamSynchronize(st));
    const ResultDev* res = reinterpret_cast<const ResultDev*>(hb + o_res);
    for (int q = 0; q < n_problems; ++q) {
        b200_init_problem_t& P = problems[q];
        const InitDev& D = pd[q];
        const ResultDev& r = res[q];
        P.status = r.status ? B200_ERR_INVALID : B200_OK;
        P.succeeded = r.stage == IN_STAGE_SUCCEEDED;
        P.model = r.model;
        P.stage = r.stage;
        P.n_matches = D.n;
        P.cost_H = r.cost[0], P.cost_F = r.cost[1], P.cost_E = r.cost[2];
        P.valid_H = r.valid[0], P.valid_F = r.valid[1], P.valid_E = r.valid[2];
        P.num_inliers_H = r.num_inliers[0], P.num_inliers_F = r.num_inliers[1], P.num_inliers_E = r.num_inliers[2];
        P.n_hypotheses = r.n_hyp;
        for (int k = 0; k < kMaxHyp; ++k) {
            const bool ran = k < r.n_hyp;
            P.nums_valid[k] = ran ? r.nums_valid[k] : 0;
            P.num_triangulated[k] = ran ? r.num_triangulated[k] : 0;
            P.parallax_cos[k] = ran ? r.parallax_cos[k] : 0.0f;
        }
        if (r.n_hyp > 0) {
            std::memcpy(P.rot_ref_to_cur, r.R, sizeof r.R);
            std::memcpy(P.trans_ref_to_cur, r.t, sizeof r.t);
        }
        if (P.succeeded) {
            std::memcpy(P.triangulated_pts, hb + o_pts + 24 * (size_t)D.ref_off, 24 * (size_t)P.n_ref);
            std::memcpy(P.triangulated_flags, hb + o_tri + D.ref_off, (size_t)P.n_ref);
        }
        if (P.inlier_flags && r.model != IN_MODEL_NONE) std::memcpy(P.inlier_flags, hb + o_inl + D.match_off, (size_t)D.n);
    }
    return B200_OK;
}

}  // extern "C"
