// lba_kernels.cu -- optimize::local_bundle_adjuster on sm_90a (fp64).
//
// Reference path (paths relative to the reference checkout):
//   local_bundle_adjuster_g2o::optimize steps 5-7     src/stella_vslam/optimize/local_bundle_adjuster_g2o.cc:306-375
//   mono/stereo perspective reprojection edges         optimize/internal/se3/perspective_reproj_edge.h:67-120, 175-239
//   equirectangular reprojection edge                  optimize/internal/se3/equirectangular_reproj_edge.h:64-134
//   edge wrapper (information, Huber delta, mono test) optimize/internal/se3/reproj_edge_wrapper.h:57-268
//   shot_vertex / landmark_vertex oplus                optimize/internal/se3/shot_vertex.h:55-58, internal/landmark_vertex.h:50-53
//   terminate_action (gain threshold 1e-3)             optimize/terminate_action.cc:36-76
// and g2o's published algorithm (tag 20230223_git, not vendored): BaseBinaryEdge::constructQuadraticForm with
// RobustKernelHuber, BlockSolver_6_3 (Schur complement over the landmarks), OptimizationAlgorithmLevenberg.
//
// Layout: edges are sorted by landmark (CSR, built on the device), so every landmark-side quantity (Hll, bl, Dinv,
// back-substitution) is a contiguous, atomics-free reduction; pose-side blocks are built by one CTA per free keyframe; the Schur
// complement is a block-sparse  Hschur(i,j) = Hpp(i,j) - sum_l Hpl(i,l) Dinv(l) Hpl(j,l)^T  evaluated from device-built lists of
// the edge pairs that share a landmark, one list per block (i, j >= i), cut into chunks whose 6x6 partials are small GEMMs on the
// fp64 tensor cores (DMMA).  Many windows are solved per launch sequence (b200_lba_solve_batch).  Everything is deterministic
// (fixed reduction orders, no floating-point atomics).
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <new>
#include <sched.h>

#include <chrono>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

#include "common.cuh"
#include "lm_common.cuh"
#include "quat.cuh"
#include "staging.cuh"
#include "track_chain.cuh"

namespace b200 {
namespace lba {

constexpr double kPi = 3.14159265358979323846;

struct Cam {
    int model;
    double fx, fy, cx, cy, fxb, cols, rows;
};

// per-edge static data (sorted by landmark)
struct EdgeS {
    int pose;        // keyframe index
    int pcol;        // free-pose column or -1
    int point;       // landmark index
    int lcol;        // free-landmark column or -1
    float ox, oy, oxr;
    float inv_sigma_sq;
    float delta;
    unsigned char cam, robust, can_outlier, pad;
};


// ---------------------------------------------------------------------------------------------------------------
// geometry
// ---------------------------------------------------------------------------------------------------------------
using b200::quat_normalize;  // quat.cuh
using b200::quat_to_rot;
using b200::rot_to_quat;

// Residual of one edge at pose Rt = [R(9) t(3)], landmark p.  dim = 2 (mono / equirect) or 3 (stereo).
__device__ __forceinline__ void edge_residual(const EdgeS& e, const Cam& c, const double* Rt, const double* p, double* err, double* pc) {
    pc[0] = Rt[0] * p[0] + Rt[1] * p[1] + Rt[2] * p[2] + Rt[9];
    pc[1] = Rt[3] * p[0] + Rt[4] * p[1] + Rt[5] * p[2] + Rt[10];
    pc[2] = Rt[6] * p[0] + Rt[7] * p[1] + Rt[8] * p[2] + Rt[11];
    if (c.model == 1) {  // equirectangular_reproj_edge.h:130-134
        const double theta = atan2(pc[0], pc[2]);
        const double phi = -asin(pc[1] / sqrt(pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2]));
        err[0] = (double)e.ox - c.cols * (0.5 + theta / (2 * kPi));
        err[1] = (double)e.oy - c.rows * (0.5 - phi / kPi);
        err[2] = 0.0;
    } else {  // perspective_reproj_edge.h:118-120, 236-239
        const double rx = c.fx * pc[0] / pc[2] + c.cx;
        err[0] = (double)e.ox - rx;
        err[1] = (double)e.oy - (c.fy * pc[1] / pc[2] + c.cy);
        err[2] = (e.oxr < 0.f) ? 0.0 : (double)e.oxr - (rx - c.fxb / pc[2]);
    }
}

// linearizeOplus: Ji (3 rows x 3, landmark) and Jj (3 rows x 6, pose, rotation first); unused rows are zero.
__device__ __forceinline__ void edge_jacobians(const EdgeS& e, const Cam& c, const double* Rt, const double* pc, double* Ji, double* Jj) {
    const double x = pc[0], y = pc[1], z = pc[2];
#pragma unroll
    for (int i = 0; i < 9; ++i) Ji[i] = 0.0;
#pragma unroll
    for (int i = 0; i < 18; ++i) Jj[i] = 0.0;
    if (c.model == 1) {  // equirectangular_reproj_edge.h:71-128
        const double L = sqrt(x * x + y * y + z * z);
        const double dx[9] = {0, z, -y, 1, 0, 0, Rt[0], Rt[1], Rt[2]};
        const double dy[9] = {-z, 0, x, 0, 1, 0, Rt[3], Rt[4], Rt[5]};
        const double dz[9] = {y, -x, 0, 0, 0, 1, Rt[6], Rt[7], Rt[8]};
        const double k0 = -(c.cols / (2 * kPi)) * (1.0 / (x * x + z * z));
        const double k1 = -(c.rows / kPi) * (1.0 / (L * sqrt(x * x + z * z)));
#pragma unroll
        for (int j = 0; j < 9; ++j) {
            const double dL = (1.0 / L) * (x * dx[j] + y * dy[j] + z * dz[j]);
            const double j0 = k0 * (z * dx[j] - x * dz[j]);
            const double j1 = k1 * (L * dy[j] - y * dL);
            if (j < 6) {
                Jj[j] = j0;
                Jj[6 + j] = j1;
            } else {
                Ji[j - 6] = j0;
                Ji[3 + j - 6] = j1;
            }
        }
        return;
    }
    const double fx = c.fx, fy = c.fy, z_sq = z * z;
#pragma unroll
    for (int j = 0; j < 3; ++j) {  // perspective_reproj_edge.h:89-95
        Ji[j] = -fx * Rt[j] / z + fx * x * Rt[6 + j] / z_sq;
        Ji[3 + j] = -fy * Rt[3 + j] / z + fy * y * Rt[6 + j] / z_sq;
    }
    Jj[0] = x * y / z_sq * fx; Jj[1] = -(1.0 + (x * x / z_sq)) * fx; Jj[2] = y / z * fx;
    Jj[3] = -1.0 / z * fx;     Jj[4] = 0.0;                            Jj[5] = x / z_sq * fx;
    Jj[6] = (1.0 + y * y / z_sq) * fy; Jj[7] = -x * y / z_sq * fy; Jj[8] = -x / z * fy;
    Jj[9] = 0.0;                       Jj[10] = -1.0 / z * fy;     Jj[11] = y / z_sq * fy;
    if (e.oxr >= 0.f) {  // perspective_reproj_edge.h:203-205, 221-226
        const double fxb = c.fxb;
#pragma unroll
        for (int j = 0; j < 3; ++j) Ji[6 + j] = Ji[j] - fxb * Rt[6 + j] / z_sq;
        Jj[12] = Jj[0] - fxb * y / z_sq; Jj[13] = Jj[1] + fxb * x / z_sq; Jj[14] = Jj[2];
        Jj[15] = Jj[3];                  Jj[16] = 0.0;                    Jj[17] = Jj[5] - fxb / z_sq;
    }
}

using b200::huber_cost;  // lm_common.cuh
using b200::huber_weight;

__device__ __forceinline__ double block_sum(double v, double* sh) {  // deterministic tree reduction, blockDim.x power of two <= 1024
    const int tid = threadIdx.x;
    sh[tid] = v;
    __syncthreads();
    for (int s = blockDim.x >> 1; s > 0; s >>= 1) {
        if (tid < s) sh[tid] += sh[tid + s];
        __syncthreads();
    }
    const double r = sh[0];
    __syncthreads();
    return r;
}


// Factored Hpl record.  All three edge models factor their Jacobians through the camera-frame point pc = R P + t:
//     Jj = Jpi [-[pc]x | I]  (rotation columns first),   Ji = Jpi R,
// so with A = ww Jpi^T Ji (3x3; rows 3..5 of Hpl)  the 6x3 block is  Hpl = ww Jj^T Ji = [ [pc]x A ; A ].
// A record holds A (row-major, 9 doubles) and pc (3): 96 bytes = three whole 32-byte sectors, read and written as pairs of 128-bit
// accesses (Hopper has no 256-bit access).  The Schur kernel, which runs at the L2 bandwidth, gathers 40 % fewer bytes than with the
// 18 entries padded to 160 bytes.  An edge that contributes no Hpl (inactive, fixed landmark or fixed keyframe) has an all-zero record.
constexpr int kHplStride = 12;
__device__ __forceinline__ void ld256(const double* p, double& a, double& b, double& c, double& d) {
    const double2 lo = reinterpret_cast<const double2*>(p)[0], hi = reinterpret_cast<const double2*>(p)[1];
    a = lo.x, b = lo.y, c = hi.x, d = hi.y;
}
__device__ __forceinline__ void st256(double* p, double a, double b, double c, double d) {
    reinterpret_cast<double2*>(p)[0] = make_double2(a, b);
    reinterpret_cast<double2*>(p)[1] = make_double2(c, d);
}
// out = {A (9), pc (3)}
__device__ __forceinline__ void load_hpl_record(const double* __restrict__ p, double* out) {
#pragma unroll
    for (int i = 0; i < 3; ++i) ld256(p + 4 * i, out[4 * i], out[4 * i + 1], out[4 * i + 2], out[4 * i + 3]);
}
// the 6x3 block (row-major) from a record: rows 0..2 = [pc]x A, rows 3..5 = A
__device__ __forceinline__ void expand_hpl(const double* r, double* h) {
    const double* A = r;
    const double x = r[9], y = r[10], z = r[11];
#pragma unroll
    for (int b = 0; b < 3; ++b) {
        h[b] = y * A[6 + b] - z * A[3 + b];
        h[3 + b] = z * A[b] - x * A[6 + b];
        h[6 + b] = x * A[3 + b] - y * A[b];
        h[9 + b] = A[b];
        h[12 + b] = A[3 + b];
        h[15 + b] = A[6 + b];
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Batched windows.  b200_lba_solve_batch solves n independent local-BA windows in LOCKSTEP: every kernel below takes the
// array of per-window descriptors and uses blockIdx.y (or a cluster index) as the window, so one launch sequence serves the
// whole batch.  Each window owns a Levenberg-Marquardt control block on the device; the numeric kernels read lambda, the
// index of the current state and the "go" flags from it and skip windows that are not in the phase the kernel implements
// (a window whose trial was rejected skips the next build, a window that has finished its round skips everything).  The LM
// bookkeeping itself (g2o's OptimizationAlgorithmLevenberg::solve / SparseOptimizer::optimize / terminate_action) runs in
// the LAST CTA of the producing kernel of that window, so the host never takes part in a decision: it enqueues repetitions of
// {build; trial} and looks at the control blocks every few repetitions only to know when to stop enqueueing.
// ---------------------------------------------------------------------------------------------------------------
struct LmCtl {
    double lambda, ni, current_chi, last_chi, rho;
    double lambda_init, chi2[2], lambda_final[2];
    int cur, it, iterations, qmax, ok, stop_flag, round, skip_round2;
    double gain_thr;  // terminate_action::setGainThreshold (1e-3 for local / global BA; the initializer passes its own)
    int outer_go;    // the window still iterates in this round
    int need_build;  // the next repetition starts with buildSystem (0 after a rejected trial: H and b are unchanged)
    int iters_done[2];
    int trials;      // LM trials run so far (statistics)
    int pad;
    const volatile int* abort_word;  // mapped host word mirroring the caller's force_stop flag (NULL: no flag)
};
__device__ __forceinline__ bool lm_aborted(const LmCtl* c) { return c->stop_flag || (c->abort_word && *c->abort_word); }

// Everything a kernel needs to know about one window (device pointers into the solver's arena).
struct WinDev {
    int K, L, E, Kf, Lf, n, ld, n_cams;
    int lbc;  // CTAs of the landmark pass = max(1, ceil(L / 16)) = number of chi2 / diagonal / scale partials
    int pad0;
    // inputs as the caller gave them (original edge order)
    const int* e_pose;
    const int* e_point;
    const unsigned char* e_cam;
    const unsigned char* e_robust;
    const unsigned char* e_can_outlier;
    const float* e_obs;
    const float* e_isig;
    const float* e_delta;
    const int* pose_col;  // K: free-pose column or -1
    const int* pt_col;    // L: free-landmark column or -1
    const Cam* cams;
    // plan (built on the device)
    int* pt_cnt;      // L   (zeroed; histogram, then placement cursor)
    int* pt_start;    // L+1
    int* order;       // E: sorted slot -> original edge index
    EdgeS* edges;     // E, sorted by landmark (original order inside a landmark)
    int* epcol;       // E: free-pose column of the sorted edge (compact copy for the scans)
    int* pose_cnt;    // Kf (zeroed)
    int* pose_start;  // Kf+1
    int* pose_edges;  // sorted-edge ids grouped by free pose, ascending (= landmark order)
    int4* rowrec;     // aligned with pose_edges: {edge a, its landmark (-1: the landmark is fixed), first edge of that landmark, its edge count}
    // pair-list form of the Schur complement: the (edge a, edge c) pairs that share a landmark, grouped by the upper block
    // (i <= j) of the reduced system they fall into, in landmark order, cut into chunks of kSchurChunk pairs
    unsigned long long* lm_mask;  // L x mask_words: bit p set <=> the (free) landmark has an edge of free keyframe column p
    int mask_words, n_blocks;
    int* blk_cnt;          // n_blocks: pairs per block
    int* blk_pair_start;   // n_blocks + 1
    int* blk_chunk_start;  // n_blocks + 1
    int4* pairs;           // {a, c, free-landmark column, 0}
    struct SchurBlock* blocks;
    struct SchurChunk* chunks;
    double* chunk_part;    // 42 doubles per chunk
    int* blk_done;         // (zeroed) chunks of the block that have published their partial
    unsigned char* level;   // E (zeroed): 0 active, 1 outlier
    unsigned char* robust;  // E: Huber on/off in the current round
    // state (current / trial double buffers; LmCtl::cur says which one is current)
    double* q[2];
    double* t[2];
    double* Rt[2];
    double* pts[2];
    double* chi[2];
    double *Hpl, *Hll, *bl, *Dinv, *Hpp, *bp, *M, *xp;
    double *r_chi, *r_diag, *r_scale, *r_result;
    double *gP, *gD, *ginvd;  // reduced systems too large for the on-chip panel (global BA): panel (kNB x mp), diagonal block, 1 / L[j][j]
    int* fail;       // (zeroed) the linear solve of the current trial failed
    int* tickets;    // (zeroed) 2 "last CTA" tickets
    int* bad_input;  // (zeroed) 1 + index of the first edge with an invalid vertex / camera reference
    LmCtl* ctl;
    // export block (contiguous per window): qf[4K] tf[3K] pf[3L] out[E]
    double *qf, *tf, *pf;
    unsigned char* out;
};

// ---------------------------------------------------------------------------------------------------------------
// Plan: the host only copies the caller's arrays; sorting the edges by landmark and listing them by keyframe happens here.
// ---------------------------------------------------------------------------------------------------------------
// P1: validate + histogram of edges per landmark
__global__ void __launch_bounds__(256) plan_count_kernel(const WinDev* __restrict__ wins) {
    const WinDev& W = wins[blockIdx.y];
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= W.E) return;
    const int p = W.e_point[e], k = W.e_pose[e];
    if (p < 0 || p >= W.L || k < 0 || k >= W.K || (int)W.e_cam[e] >= W.n_cams) {
        atomicMax(W.bad_input, e + 1);
        return;
    }
    atomicAdd(&W.pt_cnt[p], 1);
}
// P2: exclusive scan of the histogram (one CTA per window); the histogram becomes the placement cursor (zero)
__global__ void __launch_bounds__(1024) plan_scan_kernel(const WinDev* __restrict__ wins) {
    const WinDev& W = wins[blockIdx.x];
    if (*W.bad_input) return;
    __shared__ int warp_sums[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int carry = 0;
    for (int base = 0; base < W.L; base += 1024) {
        const int i = base + tid;
        const int v = i < W.L ? W.pt_cnt[i] : 0;
        int x = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int y = __shfl_up_sync(0xFFFFFFFFu, x, d);
            if (lane >= d) x += y;
        }
        if (lane == 31) warp_sums[warp] = x;
        __syncthreads();
        if (warp == 0) {
            int s = warp_sums[lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int y = __shfl_up_sync(0xFFFFFFFFu, s, d);
                if (lane >= d) s += y;
            }
            warp_sums[lane] = s;
        }
        __syncthreads();
        const int excl = carry + (warp ? warp_sums[warp - 1] : 0) + x - v;
        if (i < W.L) {
            W.pt_start[i] = excl;
            W.pt_cnt[i] = 0;
        }
        carry += warp_sums[31];
        __syncthreads();
    }
    if (tid == 0) W.pt_start[W.L] = carry;
}
// P3: place every edge somewhere inside its landmark's segment
__global__ void __launch_bounds__(256) plan_place_kernel(const WinDev* __restrict__ wins) {
    const WinDev& W = wins[blockIdx.y];
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= W.E || *W.bad_input) return;
    const int p = W.e_point[e];
    W.order[W.pt_start[p] + atomicAdd(&W.pt_cnt[p], 1)] = e;
}
// P4: one thread per landmark puts its (few) edges back into the caller's order -- the placement above is not deterministic,
//     the sorted segment is -- and writes the edge records; histogram of edges per free keyframe
__global__ void __launch_bounds__(128) plan_sort_kernel(const WinDev* __restrict__ wins) {
    const WinDev& W = wins[blockIdx.y];
    const int l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= W.L || *W.bad_input) return;
    const int a = W.pt_start[l], b = W.pt_start[l + 1];
    int* __restrict__ ord = W.order;
    for (int i = a + 1; i < b; ++i) {
        const int v = ord[i];
        int j = i - 1;
        while (j >= a && ord[j] > v) {
            ord[j + 1] = ord[j];
            --j;
        }
        ord[j + 1] = v;
    }
    const int lc = W.pt_col[l];
    // this thread owns the landmark's mask row: bit j of it says free keyframe column j observes the landmark
    unsigned long long* __restrict__ mask = W.lm_mask + (size_t)l * W.mask_words;
    for (int w2 = 0; w2 < W.mask_words; ++w2) mask[w2] = 0ull;
    for (int s = a; s < b; ++s) {
        const int e = ord[s];
        EdgeS d;
        d.pose = W.e_pose[e];
        d.pcol = W.pose_col[d.pose];
        d.point = l;
        d.lcol = lc;
        d.ox = W.e_obs[3 * (size_t)e];
        d.oy = W.e_obs[3 * (size_t)e + 1];
        d.oxr = W.e_obs[3 * (size_t)e + 2];
        d.inv_sigma_sq = W.e_isig[e];
        d.delta = W.e_delta[e];
        d.cam = W.e_cam[e];
        d.robust = W.e_robust[e];
        d.can_outlier = W.e_can_outlier[e];
        d.pad = 0;
        W.edges[s] = d;
        W.epcol[s] = d.pcol;
        W.robust[s] = d.robust;
        if (d.pcol >= 0) {
            atomicAdd(&W.pose_cnt[d.pcol], 1);
            if (lc >= 0) mask[d.pcol >> 6] |= 1ull << (d.pcol & 63);
        }
    }
}
// P5: one CTA per free keyframe lists its edges in ascending sorted-edge order (= landmark order) by an ordered compaction
//     over the window's edges
constexpr int kListThreads = 256;
__global__ void __launch_bounds__(kListThreads) plan_pose_lists_kernel(const WinDev* __restrict__ wins) {
    const WinDev& W = wins[blockIdx.y];
    const int i = blockIdx.x;
    if (i >= W.Kf || *W.bad_input) return;
    __shared__ int s_start;
    __shared__ int warp_cnt[kListThreads / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (warp == 0) {
        int s = 0;
        for (int j = lane; j < i; j += 32) s += W.pose_cnt[j];
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) s += __shfl_down_sync(0xFFFFFFFFu, s, d);
        if (lane == 0) {
            s_start = s;
            W.pose_start[i] = s;
            if (i == W.Kf - 1) W.pose_start[W.Kf] = s + W.pose_cnt[i];
        }
    }
    __syncthreads();
    int run = s_start;
    for (int base = 0; base < W.E; base += kListThreads) {
        const int s = base + tid;
        const bool mine = s < W.E && W.epcol[s] == i;
        const unsigned bal = __ballot_sync(0xFFFFFFFFu, mine);
        if (lane == 0) warp_cnt[warp] = __popc(bal);
        __syncthreads();
        int off = 0, tot = 0;
#pragma unroll
        for (int w2 = 0; w2 < kListThreads / 32; ++w2) {
            const int c = warp_cnt[w2];
            if (w2 < warp) off += c;
            tot += c;
        }
        if (mine) {
            const int slot = run + off + __popc(bal & ((1u << lane) - 1u));
            W.pose_edges[slot] = s;
            const EdgeS* ed = W.edges + s;
            const int l = ed->point, c_lo = W.pt_start[l];
            W.rowrec[slot] = make_int4(s, ed->lcol >= 0 ? l : -1, c_lo, W.pt_start[l + 1] - c_lo);
        }
        run += tot;
        __syncthreads();
    }
}

// P6-P8: the pair list of the Schur complement.  Block b = (i, j >= i) of the reduced system collects the landmarks seen by both
//     keyframes; one warp per block walks keyframe i's edge list (landmark order) and tests bit j of each landmark's mask, so the
//     pairs of a block come out in landmark order without any sort: count, scan over the blocks, emit.
constexpr int kSchurChunk = 64;
struct SchurBlock {
    int i, j, chunk_start, chunk_end;
};
struct SchurChunk {
    int start, end, diag, block;
};
__device__ __forceinline__ void block_to_ij(int b, int Kf, int& i, int& j) {  // b = i * Kf - i (i - 1) / 2 + (j - i)
    const double t = 2.0 * Kf + 1.0;
    i = (int)((t - sqrt(t * t - 8.0 * b)) * 0.5);
    i = max(0, min(i, Kf - 1));
    while (i > 0 && i * Kf - i * (i - 1) / 2 > b) --i;
    while (i + 1 < Kf && (i + 1) * Kf - (i + 1) * i / 2 <= b) ++i;
    j = i + (b - (i * Kf - i * (i - 1) / 2));
}
template <bool EMIT>
__global__ void __launch_bounds__(128) plan_pairs_kernel(const WinDev* __restrict__ wins) {
    const WinDev& W = wins[blockIdx.y];
    const int lane = threadIdx.x & 31, b = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (b >= W.n_blocks || *W.bad_input) return;
    int i, j;
    block_to_ij(b, W.Kf, i, j);
    const int a_lo = W.pose_start[i], a_hi = W.pose_start[i + 1], mw = W.mask_words;
    int run = EMIT ? W.blk_pair_start[b] : 0;
    for (int base = a_lo; base < a_hi; base += 32) {
        const int pos = base + lane;
        bool hit = false;
        int4 rec = make_int4(0, -1, 0, 0);
        if (pos < a_hi) {
            rec = W.rowrec[pos];
            if (rec.y >= 0) hit = (W.lm_mask[(size_t)rec.y * mw + (j >> 6)] >> (j & 63)) & 1ull;
        }
        const unsigned bal = __ballot_sync(0xFFFFFFFFu, hit);
        if (EMIT && hit) {
            int c = rec.z;
            for (int q = 0; q < rec.w; ++q)
                if (W.epcol[rec.z + q] == j) {
                    c = rec.z + q;
                    break;
                }
            W.pairs[run + __popc(bal & ((1u << lane) - 1u))] = make_int4(rec.x, c, W.pt_col[rec.y], 0);
        }
        run += __popc(bal);
    }
    if (!EMIT) {
        if (lane == 0) W.blk_cnt[b] = run;
        return;
    }
    const int ps = W.blk_pair_start[b], total = W.blk_pair_start[b + 1] - ps, cs = W.blk_chunk_start[b];
    for (int ch = lane; ch * kSchurChunk < total; ch += 32)
        W.chunks[cs + ch] = SchurChunk{ps + ch * kSchurChunk, ps + min(total, (ch + 1) * kSchurChunk), i == j ? 1 : 0, b};
    if (lane == 0) W.blocks[b] = SchurBlock{i, j, cs, W.blk_chunk_start[b + 1]};
}
// exclusive scans of the pairs and of the chunks per block (one CTA per window)
__global__ void __launch_bounds__(1024) plan_pair_scan_kernel(const WinDev* __restrict__ wins) {
    const WinDev& W = wins[blockIdx.x];
    if (*W.bad_input) return;
    __shared__ int ws_p[32], ws_c[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nb = W.n_blocks;
    int carry_p = 0, carry_c = 0;
    for (int base = 0; base < nb; base += 1024) {
        const int b = base + tid;
        const int vp = b < nb ? W.blk_cnt[b] : 0, vc = ceil_div(vp, kSchurChunk);
        int xp = vp, xc = vc;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int yp = __shfl_up_sync(0xFFFFFFFFu, xp, d), yc = __shfl_up_sync(0xFFFFFFFFu, xc, d);
            if (lane >= d) {
                xp += yp;
                xc += yc;
            }
        }
        if (lane == 31) {
            ws_p[warp] = xp;
            ws_c[warp] = xc;
        }
        __syncthreads();
        if (warp == 0) {
            int sp = ws_p[lane], sc = ws_c[lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int yp = __shfl_up_sync(0xFFFFFFFFu, sp, d), yc = __shfl_up_sync(0xFFFFFFFFu, sc, d);
                if (lane >= d) {
                    sp += yp;
                    sc += yc;
                }
            }
            ws_p[lane] = sp;
            ws_c[lane] = sc;
        }
        __syncthreads();
        if (b < nb) {
            W.blk_pair_start[b] = carry_p + (warp ? ws_p[warp - 1] : 0) + xp - vp;
            W.blk_chunk_start[b] = carry_c + (warp ? ws_c[warp - 1] : 0) + xc - vc;
        }
        carry_p += ws_p[31];
        carry_c += ws_c[31];
        __syncthreads();
    }
    if (tid == 0) {
        W.blk_pair_start[nb] = carry_p;
        W.blk_chunk_start[nb] = carry_c;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// LM control.  Sums of the per-CTA partials are taken by thread 0 in index order (staged through shared memory), exactly
// like a host loop over the read-back array would.
// ---------------------------------------------------------------------------------------------------------------
__device__ double ordered_sum(const double* __restrict__ p, int n, double* stage) {
    double s = 0.0;
    for (int base = 0; base < n; base += 1024) {
        const int m = min(1024, n - base);
        __syncthreads();
        for (int i = threadIdx.x; i < m; i += blockDim.x) stage[i] = __ldcg(p + base + i);  // L2: the partials come from other CTAs of this launch
        __syncthreads();
        if (threadIdx.x == 0)
            for (int i = 0; i < m; ++i) s += stage[i];
    }
    return s;  // valid in thread 0
}

// Dinv = (Hll + lambda I)^-1 for every free landmark of the window (symmetric 3x3, cofactor inverse like Eigen's fixed-size
// path), by all threads of the control CTA right after lambda has been decided.
__device__ void compute_dinv(const WinDev& W, double lambda) {
    const int Lf = W.Lf;
    const double* __restrict__ Hll = W.Hll;
    double* __restrict__ Dinv = W.Dinv;
    for (int lc = threadIdx.x; lc < Lf; lc += blockDim.x) {
        const double A0 = __ldcg(Hll + lc) + lambda, A1 = __ldcg(Hll + (size_t)Lf + lc), A2 = __ldcg(Hll + (size_t)2 * Lf + lc);
        const double A4 = __ldcg(Hll + (size_t)3 * Lf + lc) + lambda, A5 = __ldcg(Hll + (size_t)4 * Lf + lc), A8 = __ldcg(Hll + (size_t)5 * Lf + lc) + lambda;
        const double c0 = A4 * A8 - A5 * A5, c1 = A5 * A2 - A1 * A8, c2 = A1 * A5 - A4 * A2;
        const double det = A0 * c0 + A1 * c1 + A2 * c2;
        if (det == 0.0 || !isfinite(det)) {
            *W.fail = 1;
            continue;
        }
        const double id = 1.0 / det;
        Dinv[lc] = c0 * id;
        Dinv[(size_t)Lf + lc] = c1 * id;
        Dinv[(size_t)2 * Lf + lc] = c2 * id;
        Dinv[(size_t)3 * Lf + lc] = (A0 * A8 - A2 * A2) * id;
        Dinv[(size_t)4 * Lf + lc] = (A1 * A2 - A0 * A5) * id;
        Dinv[(size_t)5 * Lf + lc] = (A0 * A4 - A1 * A1) * id;
    }
}

// start of SparseOptimizer::optimize(iterations): terminate_action at iteration -1 resets the stop flag (terminate_action.cc:46-51).
// One thread per window.
__global__ void lm_round_begin_kernel(const WinDev* __restrict__ wins, int n_windows, int iterations, int round, double gain_thr) {
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= n_windows) return;
    LmCtl* c = wins[w].ctl;
    c->round = round;
    c->iterations = iterations;
    c->gain_thr = gain_thr;
    c->iters_done[round] = 0;
    c->need_build = 1;
    if (*wins[w].bad_input) {
        c->skip_round2 = 1;
        c->outer_go = 0;
        return;
    }
    // local_bundle_adjuster_g2o.cc:317-321: the second round is skipped only when the CALLER's flag exists and is set (the gain stop
    // of the first round sets it through terminate_action); without a caller flag the stop lands in g2o's own auxiliary flag, which
    // iteration -1 of the next optimize() resets
    if (round == 1 && c->abort_word && lm_aborted(c)) {
        c->skip_round2 = 1;
        c->outer_go = 0;
        return;
    }
    c->stop_flag = 0;
    c->it = 0;
    c->ok = 1;
    c->outer_go = (iterations > 0 && !(c->abort_word && *c->abort_word)) ? 1 : 0;
}

// after computeActiveErrors + buildSystem: at the first iteration of a round take the robust chi2 and computeLambdaInit
// (tau * max |H_jj| over all free vertices, tau = 1e-5); arm the trial loop.  Run by the last CTA of the keyframe-side kernel.
__device__ void lm_after_build(const WinDev& W, double* stage) {
    LmCtl* c = W.ctl;
    const bool first = c->it == 0;
    double chi = 0.0;
    if (first) chi = ordered_sum(W.r_chi, W.lbc, stage);
    if (threadIdx.x == 0) {
        if (first) {
            c->current_chi = chi;
            double mx = 0.0;
            for (int i = 0; i < W.lbc; ++i) mx = fmax(mx, __ldcg(W.r_diag + i));
            for (int p = 0; p < W.Kf; ++p)
                for (int a = 0; a < 6; ++a) mx = fmax(mx, fabs(__ldcg(W.Hpp + 36 * (size_t)p + a * 7)));
            c->lambda = 1e-5 * mx;
            c->ni = 2.0;
            if (c->round == 0) c->lambda_init = c->lambda;
        }
        c->qmax = 0;
        c->rho = 0.0;
        c->need_build = 0;
        *W.fail = 0;
    }
    __syncthreads();
    compute_dinv(W, c->lambda);
}

// after one trial (solve, back-substitution, chi2 at the trial state): the accept / reject rule of
// OptimizationAlgorithmLevenberg::solve, and when the trial loop ends the end-of-iteration bookkeeping of
// SparseOptimizer::optimize + terminate_action (terminate_action.cc:52-73).  Run by the last CTA of the trial's chi2 pass.
__device__ void lm_after_trial(const WinDev& W, double* stage) {
    LmCtl* c = W.ctl;
    const double* r_result = W.r_result;
    const bool ok2 = __ldcg(r_result) != 0.0;
    const double chi_sum = ordered_sum(W.r_chi, W.lbc, stage);
    const double scale_sum = ordered_sum(W.r_scale, W.lbc, stage);
    __shared__ int s_again;
    if (threadIdx.x == 0) {
        c->trials += 1;
        const double temp_chi = ok2 ? chi_sum : 1.7976931348623157e308;
        double rho = c->current_chi - temp_chi;
        double scale = ok2 ? __ldcg(r_result + 1) + scale_sum : 0.0;  // computeScale
        scale += 1e-3;
        rho /= scale;
        bool broke = false;
        if (rho > 0 && isfinite(temp_chi) && ok2) {
            double alpha = 1. - pow(2 * rho - 1, 3.0);
            alpha = fmin(alpha, 2. / 3.);
            c->lambda *= fmax(1. / 3., alpha);
            c->ni = 2.0;
            c->current_chi = temp_chi;
            c->cur ^= 1;  // discardTop: keep the trial state
        } else {
            c->lambda *= c->ni;
            c->ni *= 2.0;  // pop: the current state is untouched
            if (!isfinite(c->lambda)) broke = true;
        }
        if (!broke) c->qmax++;
        c->rho = rho;
        const bool again = !broke && rho < 0 && c->qmax < 10 && !lm_aborted(c);
        s_again = again ? 1 : 0;
        *W.fail = 0;  // re-armed for the next trial
        if (!again) {
            if (c->qmax == 10 || rho == 0 || !isfinite(c->lambda)) c->ok = 0;  // SolverResult::Terminate
            const double chi_now = c->current_chi;
            if (c->it == 0) {
                c->last_chi = chi_now;
            } else {
                const double gain = (c->last_chi - chi_now) / chi_now;
                c->last_chi = chi_now;
                if (gain >= 0 && gain < c->gain_thr) c->stop_flag = 1;
            }
            c->chi2[c->round] = chi_now;
            c->lambda_final[c->round] = c->lambda;
            c->it++;
            c->iters_done[c->round] = c->it;
            c->need_build = 1;
            c->outer_go = (c->it < c->iterations && !lm_aborted(c) && c->ok) ? 1 : 0;
        }
    }
    __syncthreads();
    if (s_again) compute_dinv(W, c->lambda);  // the next trial of this iteration: same H and b, new damping
}

// "last CTA" election among the `n_ctas` CTAs that work on one window: after every one of them has published its results,
// exactly one (the last to arrive) sees true and may consume them; it re-arms the ticket for the next launch.
__device__ __forceinline__ bool last_cta_arrives(int* ticket, int n_ctas, int* smem_flag) {
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const int t = atomicAdd(ticket, 1);
        *smem_flag = (t == n_ctas - 1);
        if (*smem_flag) *ticket = 0;
    }
    __syncthreads();
    const bool last = *smem_flag != 0;
    if (last) __threadfence();
    return last;
}

// end of a round: a round that ran no iteration still reports the chi2 of its (re-evaluated) state.  One CTA per window.
__global__ void __launch_bounds__(256) lm_round_end_kernel(const WinDev* __restrict__ wins, int round) {
    __shared__ double stage[1024];
    const WinDev& W = wins[blockIdx.x];
    LmCtl* c = W.ctl;
    if (*W.bad_input || (round == 1 && c->skip_round2)) return;
    const double chi = ordered_sum(W.r_chi, W.lbc, stage);
    if (threadIdx.x) return;
    if (c->iters_done[round] == 0) c->chi2[round] = chi;
}

// ---------------------------------------------------------------------------------------------------------------
// K1: landmark pass.  Eight lanes share a landmark and split its edges; sixteen landmarks per 128-thread CTA.
//   kBuild : computeActiveErrors + the landmark side of buildSystem at the CURRENT state -- per edge the residual, chi2, Huber
//            weight, the factored Hpl record (96 bytes: A and pc) and the landmark's Hll (6 unique) / bl (3), reduced over the
//            landmark's contiguous edge range in a fixed order; chi2 and max |diag| partials per CTA
//   kTrial : chi2 of the TRIAL state (inactive edges carry the chi2 of their last activation over); the last CTA of the window
//            runs the accept / reject bookkeeping
//   kRoundEnd: chi2 of the current state after a round (terminate_action's computeActiveErrors)
// ---------------------------------------------------------------------------------------------------------------
enum { kBuild = 0, kTrial = 1, kRoundEnd = 2 };
constexpr int kLmThreads = 128;

template <int MODE>
__global__ void __launch_bounds__(kLmThreads, 4) landmark_kernel(const WinDev* __restrict__ wins) {
    __shared__ double sh[kLmThreads];
    const WinDev& W = wins[blockIdx.y];
    if ((int)blockIdx.x >= W.lbc) return;
    const LmCtl* ctl = W.ctl;
    if (MODE == kBuild && !(ctl->outer_go && ctl->need_build)) return;
    if (MODE == kTrial && !ctl->outer_go) return;
    if (MODE == kRoundEnd && (*W.bad_input || (ctl->round == 1 && ctl->skip_round2))) return;
    const int sidx = (ctl->cur ^ (MODE == kTrial ? 1 : 0)) & 1;
    const double* __restrict__ Rt = W.Rt[sidx];
    const double* __restrict__ pts = W.pts[sidx];
    double* __restrict__ chi = W.chi[sidx];
    const double* __restrict__ chi_carry = W.chi[sidx ^ 1];
    const int sub = threadIdx.x & 7;
    const int l = blockIdx.x * 16 + (threadIdx.x >> 3);
    const bool valid = l < W.L;
    const int a0 = valid ? W.pt_start[l] : 0, b0 = valid ? W.pt_start[l + 1] : 0;
    const int lc = valid ? W.pt_col[l] : -1;
    double cost = 0.0;
    double h[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    double P[3] = {0, 0, 0};
    if (valid) {
        P[0] = pts[3 * (size_t)l];
        P[1] = pts[3 * (size_t)l + 1];
        P[2] = pts[3 * (size_t)l + 2];
    }
    for (int e = a0 + sub; e < b0; e += 8) {
        const EdgeS ed = W.edges[e];
        double* __restrict__ rec = W.Hpl + (size_t)e * kHplStride;
        if (W.level[e] == 0) {
            const Cam c = W.cams[ed.cam];
            double err[3], pc[3];
            const double* T = Rt + 12 * (size_t)ed.pose;
            edge_residual(ed, c, T, P, err, pc);
            const double w = (double)ed.inv_sigma_sq;
            const double e2 = w * (err[0] * err[0] + err[1] * err[1] + err[2] * err[2]);
            chi[e] = e2;
            const bool rob = W.robust[e] != 0;
            cost += rob ? huber_cost(e2, (double)ed.delta) : e2;
            if (MODE == kBuild) {
                double Ji[9], Jj[18];
                edge_jacobians(ed, c, T, pc, Ji, Jj);
                const double ww = w * (rob ? huber_weight(e2, (double)ed.delta) : 1.0);
                const bool lfree = lc >= 0, pfree = ed.pcol >= 0;
                if (lfree) {  // Hll (upper 6) and bl
                    h[0] += ww * (Ji[0] * Ji[0] + Ji[3] * Ji[3] + Ji[6] * Ji[6]);
                    h[1] += ww * (Ji[0] * Ji[1] + Ji[3] * Ji[4] + Ji[6] * Ji[7]);
                    h[2] += ww * (Ji[0] * Ji[2] + Ji[3] * Ji[5] + Ji[6] * Ji[8]);
                    h[3] += ww * (Ji[1] * Ji[1] + Ji[4] * Ji[4] + Ji[7] * Ji[7]);
                    h[4] += ww * (Ji[1] * Ji[2] + Ji[4] * Ji[5] + Ji[7] * Ji[8]);
                    h[5] += ww * (Ji[2] * Ji[2] + Ji[5] * Ji[5] + Ji[8] * Ji[8]);
                    h[6] += -ww * (Ji[0] * err[0] + Ji[3] * err[1] + Ji[6] * err[2]);
                    h[7] += -ww * (Ji[1] * err[0] + Ji[4] * err[1] + Ji[7] * err[2]);
                    h[8] += -ww * (Ji[2] * err[0] + Ji[5] * err[1] + Ji[8] * err[2]);
                }
                // factored Hpl record {A = ww Jpi^T Ji, pc}; the translation columns of Jj are Jpi
                const bool both = lfree && pfree;
                double hr[12];
#pragma unroll
                for (int a = 0; a < 3; ++a)
#pragma unroll
                    for (int b = 0; b < 3; ++b) {
                        const double s = ww * (Jj[3 + a] * Ji[b] + Jj[9 + a] * Ji[3 + b] + Jj[15 + a] * Ji[6 + b]);
                        hr[a * 3 + b] = both ? s : 0.0;
                    }
#pragma unroll
                for (int i = 0; i < 3; ++i) hr[9 + i] = both ? pc[i] : 0.0;
#pragma unroll
                for (int i = 0; i < 3; ++i) st256(rec + 4 * i, hr[4 * i], hr[4 * i + 1], hr[4 * i + 2], hr[4 * i + 3]);
            }
        } else if (MODE == kBuild) {
#pragma unroll
            for (int i = 0; i < 3; ++i) st256(rec + 4 * i, 0.0, 0.0, 0.0, 0.0);
        } else if (MODE == kTrial) {
            chi[e] = chi_carry[e];  // inactive edges keep the chi2 of their last activation across the current/trial swap
        }
    }
    if (MODE == kBuild) {
        // fixed-order reduction over the 8 lanes of the landmark
#pragma unroll
        for (int i = 0; i < 9; ++i)
#pragma unroll
            for (int s = 4; s > 0; s >>= 1) h[i] += __shfl_down_sync(0xFFFFFFFFu, h[i], s, 8);
        double mx = 0.0;
        if (valid && sub == 0 && lc >= 0) {
            const int Lf = W.Lf;
#pragma unroll
            for (int i = 0; i < 6; ++i) W.Hll[(size_t)i * Lf + lc] = h[i];
#pragma unroll
            for (int i = 0; i < 3; ++i) W.bl[(size_t)i * Lf + lc] = h[6 + i];
            mx = fmax(fabs(h[0]), fmax(fabs(h[3]), fabs(h[5])));
        }
        // max is order independent
        sh[threadIdx.x] = mx;
        __syncthreads();
        for (int s = blockDim.x >> 1; s > 0; s >>= 1) {
            if (threadIdx.x < s) sh[threadIdx.x] = fmax(sh[threadIdx.x], sh[threadIdx.x + s]);
            __syncthreads();
        }
        if (threadIdx.x == 0) W.r_diag[blockIdx.x] = sh[0];
        __syncthreads();
    }
    const double s = block_sum(cost, sh);
    if (threadIdx.x == 0) W.r_chi[blockIdx.x] = s;
    if (MODE == kTrial) {  // the last CTA of the window runs the accept / reject bookkeeping on the complete partial sums
        __shared__ int last_flag;
        __shared__ double stage[1024];
        if (!last_cta_arrives(W.tickets + 1, W.lbc, &last_flag)) return;
        lm_after_trial(W, stage);
    }
}

// K2: keyframe-side blocks, one CTA per free keyframe.  Its edges (in landmark order) are cut into one contiguous range per
//     warp; a warp reduces its range to 21 unique Hpp entries + 6 bp entries and the warp partials are added in index order.
//     The last CTA of the window then runs the after-build LM bookkeeping and inverts the damped landmark blocks.
constexpr int kRowThreads = 256;
__global__ void __launch_bounds__(kRowThreads) pose_rows_kernel(const WinDev* __restrict__ wins) {
    const WinDev& W = wins[blockIdx.y];
    const LmCtl* ctl = W.ctl;
    if (!(ctl->outer_go && ctl->need_build)) return;
    const int n_rows = max(W.Kf, 1);
    if ((int)blockIdx.x >= n_rows) return;
    __shared__ double part[kRowThreads / 32][27];
    __shared__ int last_flag;
    __shared__ double stage[1024];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if ((int)blockIdx.x < W.Kf) {
        const int i = blockIdx.x;
        const double* __restrict__ Rt = W.Rt[ctl->cur & 1];
        const double* __restrict__ pts = W.pts[ctl->cur & 1];
        const int a = W.pose_start[i], b = W.pose_start[i + 1];
        const int per = round_up(ceil_div(max(b - a, 1), kRowThreads / 32), 32);
        const int lo = a + warp * per, hi = min(b, lo + per);
        double acc[27];
#pragma unroll
        for (int x = 0; x < 27; ++x) acc[x] = 0.0;
        for (int k = lo + lane; k < hi; k += 32) {
            const int e = W.pose_edges[k];
            if (W.level[e]) continue;
            const EdgeS ed = W.edges[e];
            const Cam c = W.cams[ed.cam];
            double err[3], pc[3], Ji[9], Jj[18];
            const double* T = Rt + 12 * (size_t)ed.pose;
            edge_residual(ed, c, T, pts + 3 * (size_t)ed.point, err, pc);
            edge_jacobians(ed, c, T, pc, Ji, Jj);
            const double w = (double)ed.inv_sigma_sq;
            const double e2 = w * (err[0] * err[0] + err[1] * err[1] + err[2] * err[2]);
            const double ww = w * (W.robust[e] ? huber_weight(e2, (double)ed.delta) : 1.0);
            int t = 0;
#pragma unroll
            for (int x = 0; x < 6; ++x)
#pragma unroll
                for (int y = x; y < 6; ++y) acc[t++] += ww * (Jj[x] * Jj[y] + Jj[6 + x] * Jj[6 + y] + Jj[12 + x] * Jj[12 + y]);
#pragma unroll
            for (int x = 0; x < 6; ++x) acc[21 + x] += -ww * (Jj[x] * err[0] + Jj[6 + x] * err[1] + Jj[12 + x] * err[2]);
        }
#pragma unroll
        for (int x = 0; x < 27; ++x)
#pragma unroll
            for (int s = 16; s > 0; s >>= 1) acc[x] += __shfl_down_sync(0xFFFFFFFFu, acc[x], s);
        if (lane == 0)
#pragma unroll
            for (int x = 0; x < 27; ++x) part[warp][x] = acc[x];
        __syncthreads();
        if (tid < 27) {
            double r = 0.0;
#pragma unroll
            for (int w2 = 0; w2 < kRowThreads / 32; ++w2) r += part[w2][tid];
            if (tid < 21) {
                int x = 0, rem = tid;
                while (rem >= 6 - x) {
                    rem -= 6 - x;
                    ++x;
                }
                const int y = x + rem;
                W.Hpp[(size_t)i * 36 + x * 6 + y] = r;
                W.Hpp[(size_t)i * 36 + y * 6 + x] = r;
            } else {
                W.bp[(size_t)i * 6 + (tid - 21)] = r;
            }
        }
    }
    if (!last_cta_arrives(W.tickets, n_rows, &last_flag)) return;
    lm_after_build(W, stage);
}

// one fp64 tensor-core instruction (DMMA): D (8x8) += A (8x4) B (4x8); every lane holds one element of A, one of B and two of D
__device__ __forceinline__ void dmma_m8n8k4(double& c0, double& c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

// K5: Schur complement from the pair lists.  One warp (schur_mma_kernel) reduces one chunk of <= kSchurChunk pairs of one block:
//        partial = sum T(a) Hpl(c)^T,  T(a) = Hpl(a) Dinv(l)   (+ for diagonal blocks  sum T(a) bl(l));
//     the warp that publishes a block's last chunk adds the chunk partials in index order (deterministic) into
//     M = [Hpp + lambda I - sum ; (bp - sum)^T].  Blocks without any pair are filled by the warps past the chunks.
__device__ __forceinline__ void schur_finish_block(const WinDev& W, const SchurBlock sb, double lambda, int lane) {
    const double* __restrict__ partials = W.chunk_part;
    double* __restrict__ M = W.M;
    const int n = W.n, ld = W.ld;
    for (int el = lane; el < 42; el += 32) {
        if (el >= 36 && sb.i != sb.j) continue;
        double sacc = 0.0;
        for (int c = sb.chunk_start; c < sb.chunk_end; ++c) sacc += __ldcg(partials + (size_t)c * 42 + el);
        if (el < 36) {
            const int r = el / 6, c = el - r * 6;
            double val = -sacc;
            if (sb.i == sb.j) val += W.Hpp[(size_t)sb.i * 36 + el] + (r == c ? lambda : 0.0);
            M[(size_t)(6 * sb.j + c) * ld + 6 * sb.i + r] = val;  // lower triangle (j >= i)
            if (sb.i == sb.j) M[(size_t)(6 * sb.i + r) * ld + 6 * sb.j + c] = val;
        } else {
            const int r = el - 36;
            M[(size_t)n * ld + 6 * sb.i + r] = W.bp[(size_t)sb.i * 6 + r] - sacc;  // rhs row
        }
    }
}

// K6: dense Cholesky of the reduced system (<= 6*Kf unknowns), solve, then the keyframe updates
//     (shot_vertex::oplusImpl: T <- exp(dx) * T) into the trial state.  One CTA.
__device__ void se3_oplus(const double* q, const double* t, const double* upd, double* qo, double* to) {
    const double* om = upd;
    const double* up = upd + 3;
    const double theta = sqrt(om[0] * om[0] + om[1] * om[1] + om[2] * om[2]);
    const double O[9] = {0, -om[2], om[1], om[2], 0, -om[0], -om[1], om[0], 0};
    double O2[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) O2[i * 3 + j] = O[i * 3] * O[j] + O[i * 3 + 1] * O[3 + j] + O[i * 3 + 2] * O[6 + j];
    double a, b, c, d;
    if (theta < 0.00001) {  // g2o SE3Quat::exp small-angle branch
        a = 1.0; b = 0.5; c = 0.5; d = 1.0 / 6.0;
    } else {
        a = sin(theta) / theta;
        b = (1 - cos(theta)) / (theta * theta);
        c = b;
        d = (theta - sin(theta)) / (theta * theta * theta);
    }
    double R[9], V[9];
    for (int i = 0; i < 9; ++i) {
        const double I = (i % 4 == 0) ? 1.0 : 0.0;
        R[i] = I + a * O[i] + b * O2[i];
        V[i] = I + c * O[i] + d * O2[i];
    }
    double dq[4], dt[3];
    rot_to_quat(R, dq);
    quat_normalize(dq);
    for (int i = 0; i < 3; ++i) dt[i] = V[i * 3] * up[0] + V[i * 3 + 1] * up[1] + V[i * 3 + 2] * up[2];
    // (dq, dt) * (q, t): rotate t by dq (Eigen: v + w*uv + qv x uv, uv = 2 qv x v)
    double uv[3] = {dq[1] * t[2] - dq[2] * t[1], dq[2] * t[0] - dq[0] * t[2], dq[0] * t[1] - dq[1] * t[0]};
    uv[0] += uv[0]; uv[1] += uv[1]; uv[2] += uv[2];
    to[0] = dt[0] + t[0] + dq[3] * uv[0] + (dq[1] * uv[2] - dq[2] * uv[1]);
    to[1] = dt[1] + t[1] + dq[3] * uv[1] + (dq[2] * uv[0] - dq[0] * uv[2]);
    to[2] = dt[2] + t[2] + dq[3] * uv[2] + (dq[0] * uv[1] - dq[1] * uv[0]);
    double nq[4];
    nq[3] = dq[3] * q[3] - dq[0] * q[0] - dq[1] * q[1] - dq[2] * q[2];
    nq[0] = dq[3] * q[0] + dq[0] * q[3] + dq[1] * q[2] - dq[2] * q[1];
    nq[1] = dq[3] * q[1] + dq[1] * q[3] + dq[2] * q[0] - dq[0] * q[2];
    nq[2] = dq[3] * q[2] + dq[2] * q[3] + dq[0] * q[1] - dq[1] * q[0];
    quat_normalize(nq);
    qo[0] = nq[0]; qo[1] = nq[1]; qo[2] = nq[2]; qo[3] = nq[3];
}

constexpr int kCholThreads = 512;
constexpr int kNB = 24;       // panel width: four 6x6 keyframe blocks
constexpr int kCholCluster = 8;  // CTAs (SMs) that share one factorisation

__device__ __forceinline__ unsigned cluster_ctarank() {
    unsigned r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ unsigned cluster_nctarank() {
    unsigned r;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
    return r;
}
// all threads of all CTAs of the cluster; release/acquire at cluster scope orders the global-memory updates of the trailing matrix
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// Blocked right-looking Cholesky of the augmented matrix M = [Hs ; bs^T] ((n+1) x ld, row-major, lower triangle): the
// right-hand side rides along as row n, so after the factorisation M[n][0..n) = L^-1 bs and only the backward solve
// remains.  Per panel of kNB columns: (1) one warp factors the diagonal block in registers (lane i owns row i, columns
// are exchanged by shuffle); (2) every row below is solved against it, column oriented, with the reciprocal diagonal;
// the solved panel is kept TRANSPOSED in shared memory; (3) rank-kNB trailing update with 4x4 register tiles whose
// operands are two 32-byte vector loads per panel column.
// The kernel runs as ONE thread-block cluster: every CTA repeats the cheap steps (1) and (2) on its own SM (so no panel
// exchange is needed), the tiles of step (3) -- 60 % of the flops -- are dealt round-robin to the CTAs of the cluster, and a
// cluster barrier (release/acquire) separates the panels.  CTA 0 writes the factor back and does the backward solve.
__global__ void __launch_bounds__(kCholThreads) chol_solve_kernel(const WinDev* __restrict__ wins) {
    const unsigned crank = cluster_ctarank(), csize = cluster_nctarank();
    const WinDev& W = wins[blockIdx.x / csize];  // one cluster per window
    const LmCtl* __restrict__ ctl = W.ctl;
    if (!ctl->outer_go) return;  // (uniform over the cluster: nobody waits at a cluster barrier)
    const int n = W.n, ld = W.ld, K = W.K;
    double* __restrict__ M = W.M;
    const double* __restrict__ bp = W.bp;
    double* __restrict__ xp = W.xp;
    const int* __restrict__ pose_col = W.pose_col;
    double* __restrict__ result = W.r_result;
    int* __restrict__ fail = W.fail;
    extern __shared__ __align__(32) double dyn[];
    const double lambda = ctl->lambda;
    const int cur_idx = ctl->cur & 1;
    const double* __restrict__ q_cur = W.q[cur_idx];
    const double* __restrict__ t_cur = W.t[cur_idx];
    double* __restrict__ q_new = W.q[cur_idx ^ 1];
    double* __restrict__ t_new = W.t[cur_idx ^ 1];
    double* __restrict__ Rt_new = W.Rt[cur_idx ^ 1];
    double* D = dyn;                     // kNB x (kNB+1) diagonal block (lower, padded with the identity)
    double* Pn = dyn + kNB * (kNB + 1);  // kNB x mp panel, transposed (k-major); the 600 doubles in front keep it 32-byte aligned
    const int mp = (n + 1 + 3) & ~3;
    __shared__ double xs[1024];
    __shared__ double invd_all[1024];    // 1 / L[j][j]
    __shared__ double sh[kCholThreads];
    __shared__ int bad;
    const int tid = threadIdx.x, nt = blockDim.x;
    const bool lead = crank == 0;
    if (tid == 0) bad = *fail;
    __syncthreads();
    long long t_diag = 0, t_panel = 0, t_trail = 0, t_back = 0, t0 = clock64(), t1;
#define PHASE(acc) do { t1 = clock64(); acc += t1 - t0; t0 = t1; } while (0)
    for (int kb = 0; kb < n && !bad; kb += kNB) {
        const int nb = min(kNB, n - kb);
        if (tid < 32) {
            // (1) diagonal block, warp 0.  A short last block is padded with the identity so everything is fully unrolled.
            double r[kNB];
#pragma unroll
            for (int k = 0; k < kNB; ++k) r[k] = (tid < nb && k <= tid) ? M[(size_t)(kb + tid) * ld + kb + k] : ((k == tid) ? 1.0 : 0.0);
            int b = 0;
#pragma unroll
            for (int j = 0; j < kNB; ++j) {
                const double djj = __shfl_sync(0xFFFFFFFFu, r[j], j);
                b |= (!(djj > 0.0) || !isfinite(djj)) ? 1 : 0;
                const double inv = rsqrt(djj), dd = djj * inv;  // one reciprocal square root instead of sqrt + divide
                if (tid == 0) invd_all[kb + j] = inv;  // (entries past n are never read)
                r[j] = (tid == j) ? dd : ((tid > j) ? r[j] * inv : r[j]);
                const double mine = (tid > j) ? r[j] : 0.0;
#pragma unroll
                for (int k = j + 1; k < kNB; ++k) {
                    const double lkj = __shfl_sync(0xFFFFFFFFu, r[j], k);
                    r[k] = fma(-((tid >= k) ? mine : 0.0), lkj, r[k]);
                }
            }
            if (tid < kNB) {
#pragma unroll
                for (int k = 0; k < kNB; ++k) {
                    D[tid * (kNB + 1) + k] = r[k];
                }
            }
            if (tid == 0 && b) bad = 1;
        }
        __syncthreads();
        PHASE(t_diag);
        if (bad) break;
        // (2) panel solve: every row below the block (including the rhs row n)
        const int r0 = kb + nb, m = n + 1 - r0;
        for (int t = tid; t < m; t += nt) {
            double* row = M + (size_t)(r0 + t) * ld + kb;
            double x[kNB];
#pragma unroll
            for (int j = 0; j < kNB; ++j) x[j] = (j < nb) ? row[j] : 0.0;
#pragma unroll
            for (int j = 0; j < kNB; ++j) {
                x[j] *= invd_all[kb + j];
#pragma unroll
                for (int k = j + 1; k < kNB; ++k) x[k] = fma(-x[j], D[k * (kNB + 1) + j], x[k]);
            }
#pragma unroll
            for (int j = 0; j < kNB; ++j) {
                Pn[(size_t)j * mp + t] = x[j];
            }
        }
        for (int idx = tid; idx < kNB * 4; idx += nt) {  // zero the <= 3 padding rows read by the last 4-row tile
            const int j = idx >> 2, t = m + (idx & 3);
            if (t < mp) Pn[(size_t)j * mp + t] = 0.0;
        }
        __syncthreads();
        PHASE(t_panel);
        // (3) trailing update with 4x4 register tiles over the lower triangle (rhs row included, rhs column excluded)
        const int tm = (m + 3) >> 2;
        const int n_tiles = tm * (tm + 1) / 2;
        for (int tile = tid * csize + crank; tile < n_tiles; tile += nt * csize) {
            int tr = (int)((sqrt(8.0 * tile + 1.0) - 1.0) * 0.5);
            while ((tr + 1) * (tr + 2) / 2 <= tile) ++tr;
            while (tr * (tr + 1) / 2 > tile) --tr;
            const int tc = tile - tr * (tr + 1) / 2;
            double acc[16];
#pragma unroll
            for (int a = 0; a < 16; ++a) acc[a] = 0.0;
            const int rb = tr * 4, cb = tc * 4;
#pragma unroll 4
            for (int k = 0; k < kNB; ++k) {
                const double2* pa = reinterpret_cast<const double2*>(Pn + (size_t)k * mp + rb);
                const double2* pb = reinterpret_cast<const double2*>(Pn + (size_t)k * mp + cb);
                const double2 a0 = pa[0], a1 = pa[1], b0 = pb[0], b1 = pb[1];
                const double a[4] = {a0.x, a0.y, a1.x, a1.y}, b[4] = {b0.x, b0.y, b1.x, b1.y};
#pragma unroll
                for (int u = 0; u < 4; ++u)
#pragma unroll
                    for (int w = 0; w < 4; ++w) acc[u * 4 + w] = fma(a[u], b[w], acc[u * 4 + w]);
            }
#pragma unroll
            for (int u = 0; u < 4; ++u)
#pragma unroll
                for (int w = 0; w < 4; ++w) {
                    const int r = rb + u, c = cb + w;
                    if (r < m && c <= r && r0 + c < n) M[(size_t)(r0 + r) * ld + r0 + c] -= acc[u * 4 + w];
                }
        }
        __syncthreads();
        if (csize > 1) cluster_sync_all();  // every CTA's share of the trailing matrix is visible before the next panel is read
        // The factor of this panel is written back only now: the other CTAs were still reading these columns of M (their own copy
        // of steps 1-2) until the barrier; the next panel touches columns >= kb + nb only.
        if (lead) {
            for (int idx = tid; idx < nb * nb; idx += nt) {
                const int i = idx / nb, j = idx - i * nb;
                if (j <= i) M[(size_t)(kb + i) * ld + kb + j] = D[i * (kNB + 1) + j];
            }
            for (int idx = tid; idx < m * nb; idx += nt) {
                const int t = idx / nb, j = idx - t * nb;
                M[(size_t)(r0 + t) * ld + kb + j] = Pn[(size_t)j * mp + t];
            }
        }
        __syncthreads();
        PHASE(t_trail);
    }
    if (!lead) return;  // the backward solve and the keyframe updates are one CTA's work
    if (bad) {
        if (tid == 0) {
            *fail = 1;
            result[0] = 0.0;
        }
    } else {
        // backward solve L^T x = y, y = M[n][0..n)
        for (int i = tid; i < n; i += nt) xs[i] = M[(size_t)n * ld + i];
        __syncthreads();
        for (int kb = ((n - 1) / kNB) * kNB; kb >= 0; kb -= kNB) {
            const int nb = min(kNB, n - kb);
            for (int idx = tid; idx < kNB * kNB; idx += nt) {
                const int i = idx / kNB, j = idx - i * kNB;
                D[i * (kNB + 1) + j] = (i < nb && j <= i) ? M[(size_t)(kb + i) * ld + kb + j] : 0.0;
            }
            __syncthreads();
            if (tid < 32) {  // diagonal block: lane k owns y[k]; x[j] is broadcast by shuffle
                double y = (tid < nb) ? xs[kb + tid] : 0.0;
#pragma unroll
                for (int j = kNB - 1; j >= 0; --j) {
                    const double xj = __shfl_sync(0xFFFFFFFFu, y, j) * ((j < nb) ? invd_all[kb + j] : 0.0);
                    if (tid == j) y = xj;
                    else if (tid < j) y = fma(-D[j * (kNB + 1) + tid], xj, y);
                }
                if (tid < nb) xs[kb + tid] = y;
            }
            __syncthreads();
            for (int i = tid; i < kb; i += nt) {
                double sacc = xs[i];
                for (int k = 0; k < nb; ++k) sacc = fma(-M[(size_t)(kb + k) * ld + i], xs[kb + k], sacc);
                xs[i] = sacc;
            }
            __syncthreads();
        }
        double sc = 0.0;  // pose part of computeScale: sum x (lambda x + b)
        for (int i = tid; i < n; i += nt) {
            xp[i] = xs[i];
            sc += xs[i] * (lambda * xs[i] + bp[i]);
        }
        const double tot = block_sum(sc, sh);
        PHASE(t_back);
        if (tid == 0) {
            result[0] = 1.0;
            result[1] = tot;
            result[2] = (double)t_diag;
            result[3] = (double)t_panel;
            result[4] = (double)t_trail;
            result[5] = (double)t_back;
        }
    }
#undef PHASE
    __syncthreads();
    // trial keyframe states (fixed keyframes and failed solves keep the current state)
    for (int k = tid; k < K; k += nt) {
        double qn[4], tn[3];
        const int pc = pose_col[k];
        if (pc >= 0 && !bad) {
            se3_oplus(q_cur + 4 * k, t_cur + 3 * k, xs + 6 * pc, qn, tn);
        } else {
            for (int i = 0; i < 4; ++i) qn[i] = q_cur[4 * k + i];
            for (int i = 0; i < 3; ++i) tn[i] = t_cur[3 * k + i];
        }
        for (int i = 0; i < 4; ++i) q_new[4 * k + i] = qn[i];
        for (int i = 0; i < 3; ++i) t_new[3 * k + i] = tn[i];
        double R[9];
        quat_to_rot(qn, R);
        for (int i = 0; i < 9; ++i) Rt_new[12 * k + i] = R[i];
        for (int i = 0; i < 3; ++i) Rt_new[12 * k + 9 + i] = tn[i];
    }
}

// K5 (pair-list chunks, one warp per chunk): a chunk's block partial is formed as a small GEMM on the fp64 tensor cores:
//        S (6 x 6 | rhs) = [T_1 ... T_P] (6 x 3P) . [H_1 | b_1 ... H_P | b_P]^T (3P x 7),   T_p = Hpl(a_p) Dinv(l_p),  H_p = Hpl(c_p)
//     Phase 1 (lane = pair, 32 pairs per pass): load the two 96-byte records and Dinv, expand the records to Hpl, form T, park T and
//     H (and bl for diagonal blocks) in the warp's shared-memory operand tiles, r-major with a row stride of 100 doubles (conflict-free
//     fragment loads).
//     Phase 2: 24 x mma.sync.m8n8k4.f64 (DMMA) per pass, two LDS + one DMMA per lane and step; the 8 x 8 accumulator tile lives in two
//     registers per lane for the whole chunk, so no per-lane accumulators have to be reduced across the warp.  Summation order is
//     fixed => deterministic.
constexpr int kSmmaKS = 100;                               // row stride of the operand tiles (K = 96 per pass, +4: bank spread)
constexpr int kSmmaWarpDoubles = (6 + 7) * kSmmaKS;        // A: 6 rows, B: 7 rows (6 columns of H + the rhs column)
__global__ void __launch_bounds__(128) schur_mma_kernel(const WinDev* __restrict__ wins) {
    extern __shared__ __align__(16) double smma[];
    const WinDev& W = wins[blockIdx.y];
    const LmCtl* ctl = W.ctl;
    if (!ctl->outer_go) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wid = blockIdx.x * 4 + warp;
    const int n_blocks = W.n_blocks, n_chunks = W.blk_chunk_start[n_blocks];
    if (wid >= n_chunks) {
        const int e = wid - n_chunks;
        if (e < n_blocks) {
            const SchurBlock sb = W.blocks[e];
            if (sb.chunk_start == sb.chunk_end) schur_finish_block(W, sb, ctl->lambda, lane);  // no pair: just Hpp + lambda I, or zero
        }
        return;
    }
    double* As = smma + (size_t)warp * kSmmaWarpDoubles;
    double* Bs = As + 6 * kSmmaKS;
    const SchurChunk ch = W.chunks[wid];
    const int Lf = W.Lf;
    const double* __restrict__ Hpl = W.Hpl;
    const double* __restrict__ Dinv = W.Dinv;
    const int g = lane >> 2, t4 = lane & 3;
    const double* a_row = As + min(g, 5) * kSmmaKS + t4;  // rows 6, 7 of the tile are don't-care copies
    const double* b_row = Bs + min(g, 6) * kSmmaKS + t4;
    double c0 = 0.0, c1 = 0.0;
    for (int base = ch.start; base < ch.end; base += 32) {
        const int k = base + lane;
        const int np = min(32, ch.end - base);
        {
            double t[18], hc[18], b3[3];
            if (k < ch.end) {
                const int4 pr = W.pairs[k];
                double ra[12], rc[12], ha[18];
                load_hpl_record(Hpl + (size_t)pr.x * kHplStride, ra);
                load_hpl_record(Hpl + (size_t)pr.y * kHplStride, rc);
                expand_hpl(ra, ha);
                expand_hpl(rc, hc);
                const int lc = pr.z;
                const double D0 = Dinv[lc], D1 = Dinv[(size_t)Lf + lc], D2 = Dinv[(size_t)2 * Lf + lc];
                const double D4 = Dinv[(size_t)3 * Lf + lc], D5 = Dinv[(size_t)4 * Lf + lc], D8 = Dinv[(size_t)5 * Lf + lc];
#pragma unroll
                for (int r = 0; r < 6; ++r) {
                    t[r * 3] = ha[r * 3] * D0 + ha[r * 3 + 1] * D1 + ha[r * 3 + 2] * D2;
                    t[r * 3 + 1] = ha[r * 3] * D1 + ha[r * 3 + 1] * D4 + ha[r * 3 + 2] * D5;
                    t[r * 3 + 2] = ha[r * 3] * D2 + ha[r * 3 + 1] * D5 + ha[r * 3 + 2] * D8;
                }
                b3[0] = b3[1] = b3[2] = 0.0;
                if (ch.diag) {
                    b3[0] = W.bl[lc];
                    b3[1] = W.bl[(size_t)Lf + lc];
                    b3[2] = W.bl[(size_t)2 * Lf + lc];
                }
            } else {
#pragma unroll
                for (int i = 0; i < 18; ++i) t[i] = hc[i] = 0.0;
                b3[0] = b3[1] = b3[2] = 0.0;
            }
            double* ap = As + 3 * lane;
            double* bp2 = Bs + 3 * lane;
#pragma unroll
            for (int r = 0; r < 6; ++r)
#pragma unroll
                for (int kk = 0; kk < 3; ++kk) {
                    ap[r * kSmmaKS + kk] = t[r * 3 + kk];
                    bp2[r * kSmmaKS + kk] = hc[r * 3 + kk];
                }
#pragma unroll
            for (int kk = 0; kk < 3; ++kk) bp2[6 * kSmmaKS + kk] = b3[kk];
        }
        __syncwarp();
        const int steps = (3 * np + 3) >> 2;  // (columns past 3 np inside the last step are zeros written by the idle lanes)
#pragma unroll 4
        for (int s2 = 0; s2 < steps; ++s2) dmma_m8n8k4(c0, c1, a_row[4 * s2], b_row[4 * s2]);
        __syncwarp();
    }
    // accumulator tile -> chunk partial: lane (g, t4) holds S[g][2 t4], S[g][2 t4 + 1]; column 6 is the rhs part
    double* part = W.chunk_part + (size_t)wid * 42;
    if (g < 6) {
        if (t4 < 3) {
            part[g * 6 + 2 * t4] = c0;
            part[g * 6 + 2 * t4 + 1] = c1;
        } else {
            part[36 + g] = c0;
        }
    }
    __threadfence();
    __syncwarp();
    const SchurBlock sb = W.blocks[ch.block];
    int arrived = 0;
    if (lane == 0) arrived = atomicAdd(&W.blk_done[ch.block], 1);
    arrived = __shfl_sync(0xFFFFFFFFu, arrived, 0);
    if (arrived != sb.chunk_end - sb.chunk_start - 1) return;
    __threadfence();
    schur_finish_block(W, sb, ctl->lambda, lane);
    if (lane == 0) W.blk_done[ch.block] = 0;  // re-armed for the next trial
}

// ---- reduced systems beyond the on-chip panel (n > kCholOnChipMax: global bundle adjustment, global_bundle_adjuster.cc:42-45) ----
// The same blocked right-looking factorisation, one panel = two launches over the whole chip instead of one cluster:
//   gchol_panel_kernel : every CTA factors the (tiny) diagonal block itself, solves its 256 rows of the panel, writes them
//                        transposed into the window's global panel buffer gP (L2 resident: kNB x n doubles)
//   gchol_trail_kernel : rank-kNB update of the trailing matrix with 4x4 register tiles read from gP, and the write-back of the
//                        panel's factor into M (columns the update does not touch)
// and gchol_finish_kernel (one CTA): backward solve in global memory, computeScale's pose part, trial keyframe states.
constexpr int kCholOnChipMax = 1000;
constexpr int kCholGlobalMax = 24000;  // (n + 1)^2 doubles = 4.6 GB of the H100's 80 GB
constexpr int kGcholThreads = 256;
__global__ void __launch_bounds__(kGcholThreads) gchol_panel_kernel(const WinDev* __restrict__ wins, int kb) {
    const WinDev& W = wins[blockIdx.y];
    const LmCtl* __restrict__ ctl = W.ctl;
    const int n = W.n, ld = W.ld;
    if (!ctl->outer_go || kb >= n || *W.fail) return;
    const int nb = min(kNB, n - kb), r0 = kb + nb, m = n + 1 - r0, mp = (n + 1 + 3) & ~3;
    if ((int)blockIdx.x * kGcholThreads >= m + 4) return;
    double* __restrict__ M = W.M;
    __shared__ double D[kNB * (kNB + 1)];
    __shared__ double invd[kNB];
    __shared__ int bad;
    const int tid = threadIdx.x;
    if (tid == 0) bad = 0;
    __syncthreads();
    if (tid < 32) {
        double r[kNB];
#pragma unroll
        for (int k = 0; k < kNB; ++k) r[k] = (tid < nb && k <= tid) ? M[(size_t)(kb + tid) * ld + kb + k] : ((k == tid) ? 1.0 : 0.0);
        int b = 0;
#pragma unroll
        for (int j = 0; j < kNB; ++j) {
            const double djj = __shfl_sync(0xFFFFFFFFu, r[j], j);
            b |= (!(djj > 0.0) || !isfinite(djj)) ? 1 : 0;
            const double inv = rsqrt(djj), dd = djj * inv;
            if (tid == 0) invd[j] = inv;
            r[j] = (tid == j) ? dd : ((tid > j) ? r[j] * inv : r[j]);
            const double mine = (tid > j) ? r[j] : 0.0;
#pragma unroll
            for (int k = j + 1; k < kNB; ++k) {
                const double lkj = __shfl_sync(0xFFFFFFFFu, r[j], k);
                r[k] = fma(-((tid >= k) ? mine : 0.0), lkj, r[k]);
            }
        }
        if (tid < kNB) {
#pragma unroll
            for (int k = 0; k < kNB; ++k) D[tid * (kNB + 1) + k] = r[k];
        }
        if (tid == 0 && b) bad = 1;
    }
    __syncthreads();
    if (bad) {  // (every CTA reaches the same verdict from the same numbers; the flag stops the remaining panels)
        if (blockIdx.x == 0 && tid == 0) {
            *W.fail = 1;
            W.r_result[0] = 0.0;
        }
        return;
    }
    if (blockIdx.x == 0) {
        for (int idx = tid; idx < kNB * (kNB + 1); idx += kGcholThreads) W.gD[idx] = D[idx];
        if (tid < kNB && kb + tid < n) W.ginvd[kb + tid] = invd[tid];
    }
    const int t = blockIdx.x * kGcholThreads + tid;
    if (t < m) {
        const double* row = M + (size_t)(r0 + t) * ld + kb;
        double x[kNB];
#pragma unroll
        for (int j = 0; j < kNB; ++j) x[j] = (j < nb) ? row[j] : 0.0;
#pragma unroll
        for (int j = 0; j < kNB; ++j) {
            x[j] *= invd[j];
#pragma unroll
            for (int k = j + 1; k < kNB; ++k) x[k] = fma(-x[j], D[k * (kNB + 1) + j], x[k]);
        }
#pragma unroll
        for (int j = 0; j < kNB; ++j) W.gP[(size_t)j * mp + t] = x[j];
    } else if (t < min(mp, m + 4)) {  // the <= 3 padding rows read by the last 4-row tile
#pragma unroll
        for (int j = 0; j < kNB; ++j) W.gP[(size_t)j * mp + t] = 0.0;
    }
}

__global__ void __launch_bounds__(kGcholThreads) gchol_trail_kernel(const WinDev* __restrict__ wins, int kb) {
    const WinDev& W = wins[blockIdx.y];
    const LmCtl* __restrict__ ctl = W.ctl;
    const int n = W.n, ld = W.ld;
    if (!ctl->outer_go || kb >= n || *W.fail) return;
    const int nb = min(kNB, n - kb), r0 = kb + nb, m = n + 1 - r0, mp = (n + 1 + 3) & ~3;
    double* __restrict__ M = W.M;
    const double* __restrict__ Pn = W.gP;
    const long long gid = (long long)blockIdx.x * kGcholThreads + threadIdx.x;
    const int tm = (m + 3) >> 2;
    const long long n_tiles = (long long)tm * (tm + 1) / 2;
    if (gid < n_tiles) {
        int tr = (int)((sqrt(8.0 * (double)gid + 1.0) - 1.0) * 0.5);
        while ((long long)(tr + 1) * (tr + 2) / 2 <= gid) ++tr;
        while ((long long)tr * (tr + 1) / 2 > gid) --tr;
        const int tc = (int)(gid - (long long)tr * (tr + 1) / 2);
        double acc[16];
#pragma unroll
        for (int a = 0; a < 16; ++a) acc[a] = 0.0;
        const int rb = tr * 4, cb = tc * 4;
#pragma unroll 4
        for (int k = 0; k < kNB; ++k) {
            const double2* pa = reinterpret_cast<const double2*>(Pn + (size_t)k * mp + rb);
            const double2* pb = reinterpret_cast<const double2*>(Pn + (size_t)k * mp + cb);
            const double2 a0 = pa[0], a1 = pa[1], b0 = pb[0], b1 = pb[1];
            const double a[4] = {a0.x, a0.y, a1.x, a1.y}, b[4] = {b0.x, b0.y, b1.x, b1.y};
#pragma unroll
            for (int u = 0; u < 4; ++u)
#pragma unroll
                for (int w2 = 0; w2 < 4; ++w2) acc[u * 4 + w2] = fma(a[u], b[w2], acc[u * 4 + w2]);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
            for (int w2 = 0; w2 < 4; ++w2) {
                const int r = rb + u, c = cb + w2;
                if (r < m && c <= r && r0 + c < n) M[(size_t)(r0 + r) * ld + r0 + c] -= acc[u * 4 + w2];
            }
    }
    // factor of this panel -> M (columns kb .. kb + nb, which the update above neither reads nor writes)
    const long long wb = (long long)m * nb + (long long)nb * nb;
    for (long long idx = gid; idx < wb; idx += (long long)gridDim.x * kGcholThreads) {
        if (idx < (long long)nb * nb) {
            const int i = (int)(idx / nb), j = (int)(idx - (long long)i * nb);
            if (j <= i) M[(size_t)(kb + i) * ld + kb + j] = W.gD[i * (kNB + 1) + j];
        } else {
            const long long id2 = idx - (long long)nb * nb;
            const int t = (int)(id2 / nb), j = (int)(id2 - (long long)t * nb);
            M[(size_t)(r0 + t) * ld + kb + j] = Pn[(size_t)j * mp + t];
        }
    }
}

constexpr int kGfinThreads = 1024;
__global__ void __launch_bounds__(kGfinThreads) gchol_finish_kernel(const WinDev* __restrict__ wins) {
    const WinDev& W = wins[blockIdx.x];
    const LmCtl* __restrict__ ctl = W.ctl;
    if (!ctl->outer_go) return;
    const int n = W.n, ld = W.ld, K = W.K;
    const double* __restrict__ M = W.M;
    double* __restrict__ xs = W.xp;  // the solution is built in place in global memory (one CTA; __syncthreads orders it)
    const double* __restrict__ invd = W.ginvd;
    __shared__ double D[kNB * (kNB + 1)];
    __shared__ double sh[kGfinThreads];
    const int tid = threadIdx.x, nt = blockDim.x;
    const int bad = *W.fail;
    const double lambda = ctl->lambda;
    if (!bad) {
        for (int i = tid; i < n; i += nt) xs[i] = M[(size_t)n * ld + i];
        __syncthreads();
        for (int kb = ((n - 1) / kNB) * kNB; kb >= 0; kb -= kNB) {
            const int nb = min(kNB, n - kb);
            for (int idx = tid; idx < kNB * kNB; idx += nt) {
                const int i = idx / kNB, j = idx - i * kNB;
                D[i * (kNB + 1) + j] = (i < nb && j <= i) ? M[(size_t)(kb + i) * ld + kb + j] : 0.0;
            }
            __syncthreads();
            if (tid < 32) {
                double y = (tid < nb) ? xs[kb + tid] : 0.0;
#pragma unroll
                for (int j = kNB - 1; j >= 0; --j) {
                    const double xj = __shfl_sync(0xFFFFFFFFu, y, j) * ((j < nb) ? invd[kb + j] : 0.0);
                    if (tid == j) y = xj;
                    else if (tid < j) y = fma(-D[j * (kNB + 1) + tid], xj, y);
                }
                if (tid < nb) xs[kb + tid] = y;
            }
            __syncthreads();
            for (int i = tid; i < kb; i += nt) {
                double sacc = xs[i];
                for (int k = 0; k < nb; ++k) sacc = fma(-M[(size_t)(kb + k) * ld + i], xs[kb + k], sacc);
                xs[i] = sacc;
            }
            __syncthreads();
        }
        double sc = 0.0;
        for (int i = tid; i < n; i += nt) sc += xs[i] * (lambda * xs[i] + W.bp[i]);
        const double tot = block_sum(sc, sh);
        if (tid == 0) {
            W.r_result[0] = 1.0;
            W.r_result[1] = tot;
        }
    }
    __syncthreads();
    const int cur_idx = ctl->cur & 1;
    const double* __restrict__ q_cur = W.q[cur_idx];
    const double* __restrict__ t_cur = W.t[cur_idx];
    double* __restrict__ q_new = W.q[cur_idx ^ 1];
    double* __restrict__ t_new = W.t[cur_idx ^ 1];
    double* __restrict__ Rt_new = W.Rt[cur_idx ^ 1];
    for (int k = tid; k < K; k += nt) {
        double qn[4], tn[3];
        const int pc = W.pose_col[k];
        if (pc >= 0 && !bad) {
            se3_oplus(q_cur + 4 * k, t_cur + 3 * k, xs + 6 * pc, qn, tn);
        } else {
            for (int i = 0; i < 4; ++i) qn[i] = q_cur[4 * k + i];
            for (int i = 0; i < 3; ++i) tn[i] = t_cur[3 * k + i];
        }
        for (int i = 0; i < 4; ++i) q_new[4 * k + i] = qn[i];
        for (int i = 0; i < 3; ++i) t_new[3 * k + i] = tn[i];
        double R[9];
        quat_to_rot(qn, R);
        for (int i = 0; i < 9; ++i) Rt_new[12 * k + i] = R[i];
        for (int i = 0; i < 3; ++i) Rt_new[12 * k + 9 + i] = tn[i];
    }
}

// K7: back-substitution x_l = Dinv (bl - sum_e Hpl(e)^T x_p), trial landmark, scale partials.  Eight lanes share a landmark
//     (they split its edges), sixteen landmarks per 128-thread CTA.  Hpl^T x_p is formed from the factored record without expanding it.
__global__ void __launch_bounds__(128) backsub_kernel(const WinDev* __restrict__ wins) {
    __shared__ double sh[128];
    const WinDev& W = wins[blockIdx.y];
    const LmCtl* __restrict__ ctl = W.ctl;
    if ((int)blockIdx.x >= W.lbc || !ctl->outer_go) return;
    struct { int L, Lf; const int* pt_start; const EdgeS* edges; } v = {W.L, W.Lf, W.pt_start, W.edges};
    const double* __restrict__ Dinv = W.Dinv;
    const double* __restrict__ bl = W.bl;
    const double* __restrict__ Hpl = W.Hpl;
    const double* __restrict__ xp = W.xp;
    double* __restrict__ scale_partials = W.r_scale;
    const int* __restrict__ fail = W.fail;
    const double lambda = ctl->lambda;
    const double* __restrict__ pts_cur = W.pts[ctl->cur & 1];
    double* __restrict__ pts_new = W.pts[(ctl->cur & 1) ^ 1];
    const int sub = threadIdx.x & 7;
    const int l = blockIdx.x * 16 + (threadIdx.x >> 3);
    double sc = 0.0;
    const bool valid = l < v.L;
    const int a0 = valid ? v.pt_start[l] : 0, b0 = valid ? v.pt_start[l + 1] : 0;
    const int lc = valid ? W.pt_col[l] : -1;
    const bool solve = lc >= 0 && !*fail;
    double c0 = 0.0, c1 = 0.0, c2 = 0.0;
    if (solve) {
        for (int e = a0 + sub; e < b0; e += 8) {
            const int pcol = v.edges[e].pcol;
            if (pcol < 0) continue;
            double r[12];
            load_hpl_record(Hpl + (size_t)e * kHplStride, r);
            // Hpl^T [w; v] = A^T (v - [pc]x w) = A^T (v + w x pc)
            const double* x = xp + 6 * pcol;
            const double w0 = x[0], w1 = x[1], w2 = x[2];
            const double u[3] = {x[3] + (w1 * r[11] - w2 * r[10]), x[4] + (w2 * r[9] - w0 * r[11]), x[5] + (w0 * r[10] - w1 * r[9])};
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                c0 -= r[k * 3] * u[k];
                c1 -= r[k * 3 + 1] * u[k];
                c2 -= r[k * 3 + 2] * u[k];
            }
        }
    }
    // fixed-order reduction over the 8 lanes of the landmark
#pragma unroll
    for (int s = 4; s > 0; s >>= 1) {
        c0 += __shfl_down_sync(0xFFFFFFFFu, c0, s, 8);
        c1 += __shfl_down_sync(0xFFFFFFFFu, c1, s, 8);
        c2 += __shfl_down_sync(0xFFFFFFFFu, c2, s, 8);
    }
    double pn0 = 0.0, pn1 = 0.0, pn2 = 0.0;  // the landmark's trial position (lane 0 of its eight lanes)
    if (valid && sub == 0) {
        double p0 = pts_cur[3 * (size_t)l], p1 = pts_cur[3 * (size_t)l + 1], p2 = pts_cur[3 * (size_t)l + 2];
        if (solve) {
            const double bb0 = bl[lc], bb1 = bl[(size_t)v.Lf + lc], bb2 = bl[(size_t)2 * v.Lf + lc];
            c0 += bb0; c1 += bb1; c2 += bb2;
            const double D0 = Dinv[lc], D1 = Dinv[(size_t)v.Lf + lc], D2 = Dinv[(size_t)2 * v.Lf + lc];
            const double D4 = Dinv[(size_t)3 * v.Lf + lc], D5 = Dinv[(size_t)4 * v.Lf + lc], D8 = Dinv[(size_t)5 * v.Lf + lc];
            const double x0 = D0 * c0 + D1 * c1 + D2 * c2, x1 = D1 * c0 + D4 * c1 + D5 * c2, x2 = D2 * c0 + D5 * c1 + D8 * c2;
            sc = x0 * (lambda * x0 + bb0) + x1 * (lambda * x1 + bb1) + x2 * (lambda * x2 + bb2);
            p0 += x0; p1 += x1; p2 += x2;  // landmark_vertex::oplusImpl
        }
        pts_new[3 * (size_t)l] = p0; pts_new[3 * (size_t)l + 1] = p1; pts_new[3 * (size_t)l + 2] = p2;
        pn0 = p0; pn1 = p1; pn2 = p2;
    }
    const double tot = block_sum(sc, sh);
    if (threadIdx.x == 0) scale_partials[blockIdx.x] = tot;
    // ---- computeActiveErrors at the TRIAL state (round 2a: a separate launch, landmark_kernel<kTrial>): the eight lanes of the landmark
    //      take its new position from lane 0 and walk its edges once more against the trial keyframe states the Cholesky kernel wrote
    {
        const int base = threadIdx.x & ~7 & 31;
        pn0 = __shfl_sync(0xFFFFFFFFu, pn0, base);
        pn1 = __shfl_sync(0xFFFFFFFFu, pn1, base);
        pn2 = __shfl_sync(0xFFFFFFFFu, pn2, base);
        const int tidx = (ctl->cur & 1) ^ 1;
        const double* __restrict__ Rt = W.Rt[tidx];
        double* __restrict__ chi = W.chi[tidx];
        const double* __restrict__ chi_carry = W.chi[tidx ^ 1];
        const double P[3] = {pn0, pn1, pn2};
        double cost = 0.0;
        for (int e = a0 + sub; e < b0; e += 8) {
            if (W.level[e] == 0) {
                const EdgeS ed = v.edges[e];
                const Cam c = W.cams[ed.cam];
                double err[3], pc[3];
                edge_residual(ed, c, Rt + 12 * (size_t)ed.pose, P, err, pc);
                const double w = (double)ed.inv_sigma_sq;
                const double e2 = w * (err[0] * err[0] + err[1] * err[1] + err[2] * err[2]);
                chi[e] = e2;
                cost += W.robust[e] ? huber_cost(e2, (double)ed.delta) : e2;
            } else {
                chi[e] = chi_carry[e];  // inactive edges keep the chi2 of their last activation across the current/trial swap
            }
        }
        __syncthreads();  // (sh is reused)
        const double cs = block_sum(cost, sh);
        if (threadIdx.x == 0) W.r_chi[blockIdx.x] = cs;
        // the last CTA of the window runs the accept / reject bookkeeping on the complete partial sums
        __shared__ int last_flag;
        __shared__ double stage[1024];
        if (!last_cta_arrives(W.tickets + 1, W.lbc, &last_flag)) return;
        lm_after_trial(W, stage);
    }
}

// K8: outlier test (local_bundle_adjuster_g2o.cc:323-344, 357-375): chi2 of the last activation vs the chi-square
//     threshold, or non-positive depth at the current estimate.  mode 0: mark level + drop the kernel; mode 1: report.
__global__ void __launch_bounds__(128) outlier_kernel(const WinDev* __restrict__ wins, int mode) {
    const WinDev& W = wins[blockIdx.y];
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= W.E || *W.bad_input) return;
    const LmCtl* __restrict__ ctl = W.ctl;
    if (mode == 0 && ctl->skip_round2) return;  // local_bundle_adjuster_g2o.cc:317-321: no second round after an abort
    const double* __restrict__ Rt = W.Rt[ctl->cur & 1];
    const double* __restrict__ pts = W.pts[ctl->cur & 1];
    const double* __restrict__ chi = W.chi[ctl->cur & 1];
    const EdgeS ed = W.edges[e];
    unsigned char o = 0;
    if (ed.can_outlier) {
        const double thr = (ed.oxr < 0.f) ? (double)5.99146f : (double)7.81473f;
        bool depth_ok = true;
        if (W.cams[ed.cam].model != 1) {  // reproj_edge_wrapper.h:233-268 (equirectangular: always true)
            const double* T = Rt + 12 * (size_t)ed.pose;
            const double* P = pts + 3 * (size_t)ed.point;
            depth_ok = 0.0 < T[6] * P[0] + T[7] * P[1] + T[8] * P[2] + T[11];
        }
        o = (thr < chi[e] || !depth_ok) ? 1 : 0;
    }
    if (mode == 0) {
        if (ed.can_outlier) {
            if (o) W.level[e] = 1;
            W.robust[e] = 0;
        }
    } else {
        W.out[W.order[e]] = o;  // reported in the caller's edge order
    }
}

// copy the final (current) keyframe and landmark states into the window's export block
__global__ void __launch_bounds__(256) lm_export_kernel(const WinDev* __restrict__ wins) {
    const WinDev& W = wins[blockIdx.y];
    const int cur = W.ctl->cur & 1;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 4 * W.K) W.qf[i] = W.q[cur][i];
    if (i < 3 * W.K) W.tf[i] = W.t[cur][i];
    if (i < 3 * W.L) W.pf[i] = W.pts[cur][i];
}

// ---------------------------------------------------------------------------------------------------------------
// optimize::pose_optimizer (SURVEY §8f N1): motion-only BA of one frame, the step between the two per-frame matcher calls.
//   pose_optimizer_g2o::optimize            src/stella_vslam/optimize/pose_optimizer_g2o.cc:38-175
//   mono / stereo_perspective_pose_opt_edge optimize/internal/se3/perspective_pose_opt_edge.h  (= pose block of the reprojection edges)
//   equirectangular_pose_opt_edge           optimize/internal/se3/equirectangular_pose_opt_edge.h
// Six unknowns: the whole protocol -- (num_trials_robust + num_trials) calls of optimize(num_each_iter) with LM, the terminate
// action and the outlier re-classification in between -- runs inside ONE kernel launch, one CTA per frame, no host round trip.
// Sums over edges are per-thread strided partials combined in a fixed order (deterministic).
// ---------------------------------------------------------------------------------------------------------------
struct PoseEdge {
    double pw[3];
    float ox, oy, oxr, inv_sigma_sq, delta;
    int pad;
};
struct PoseProb {
    int n;
    int edge_off;  // into the flat edge / flag arrays
    Cam cam;
    double q[4], t[3];
};
constexpr int kPoseThreads = 256;

__device__ __forceinline__ void pose_rt(const double* q, const double* t, double* Rt) {
    quat_to_rot(q, Rt);
    Rt[9] = t[0];
    Rt[10] = t[1];
    Rt[11] = t[2];
}
__global__ void __launch_bounds__(kPoseThreads) pose_optimize_kernel(const PoseProb* __restrict__ probs, const PoseEdge* __restrict__ edges_all,
                                                                     unsigned char* __restrict__ level_all, unsigned char* __restrict__ flags_all,
                                                                     int trials_robust, int trials, int each_iter, double* __restrict__ pose_out,
                                                                     unsigned* __restrict__ n_valid_out) {
    __shared__ double scratch[(kPoseThreads / 32) * 28];
    __shared__ double red[28];
    __shared__ double Rt[12], Rt_trial[12], q_cur[4], t_cur[3], q_trial[4], t_trial[3], x[6];
    __shared__ double s_lambda, s_ni, s_cur_chi, s_last_chi, s_rho;
    __shared__ int s_ok2, s_go_inner, s_go_outer, s_accept, s_it, s_qmax, s_ok, s_stop, s_bad;
    const PoseProb pb = probs[blockIdx.x];
    const PoseEdge* __restrict__ edges = edges_all + pb.edge_off;
    unsigned char* __restrict__ level = level_all + pb.edge_off;
    unsigned char* __restrict__ flags = flags_all + pb.edge_off;
    const int tid = threadIdx.x, n = pb.n;
    const Cam cam = pb.cam;
    if (tid < 4) q_cur[tid] = pb.q[tid];
    if (tid < 3) t_cur[tid] = pb.t[tid];
    for (int e = tid; e < n; e += kPoseThreads) {
        level[e] = 0;
        flags[e] = 0;
    }
    __syncthreads();
    if (n < 5) {  // pose_optimizer_g2o.cc:116-118
        if (tid == 0) n_valid_out[blockIdx.x] = 0;
        if (tid < 16) {
            double Rm[9];
            quat_to_rot(pb.q, Rm);
            const int r = tid >> 2, c = tid & 3;
            pose_out[16 * (size_t)blockIdx.x + tid] = r == 3 ? (c == 3 ? 1.0 : 0.0) : (c == 3 ? pb.t[r] : Rm[r * 3 + c]);
        }
        return;
    }
    bool robust_on = trials_robust != 0;  // :123-127
    // residual / chi2 / (optionally) the normal equations of this thread's edges at pose T
    auto accumulate = [&](const double* T, bool linearize, double (&acc)[28]) {
#pragma unroll
        for (int i = 0; i < 28; ++i) acc[i] = 0.0;
        for (int e = tid; e < n; e += kPoseThreads) {
            if (level[e]) continue;
            const PoseEdge pe = edges[e];
            EdgeS ed;
            ed.ox = pe.ox; ed.oy = pe.oy; ed.oxr = pe.oxr;
            double err[3], pc[3];
            edge_residual(ed, cam, T, pe.pw, err, pc);
            const double w = (double)pe.inv_sigma_sq;
            const double e2 = w * (err[0] * err[0] + err[1] * err[1] + err[2] * err[2]);
            acc[27] += robust_on ? huber_cost(e2, (double)pe.delta) : e2;
            if (linearize) {
                double Ji[9], Jj[18];
                edge_jacobians(ed, cam, T, pc, Ji, Jj);
                const double ww = w * (robust_on ? huber_weight(e2, (double)pe.delta) : 1.0);
                int k = 0;
#pragma unroll
                for (int a = 0; a < 6; ++a)
#pragma unroll
                    for (int b = a; b < 6; ++b) acc[k++] += ww * (Jj[a] * Jj[b] + Jj[6 + a] * Jj[6 + b] + Jj[12 + a] * Jj[12 + b]);
#pragma unroll
                for (int a = 0; a < 6; ++a) acc[21 + a] += -ww * (Jj[a] * err[0] + Jj[6 + a] * err[1] + Jj[12 + a] * err[2]);
            }
        }
    };
    int bad_total = 0;
    for (int trial = 0; trial < trials_robust + trials; ++trial) {
        // ---- SparseOptimizer::optimize(each_iter) with OptimizationAlgorithmLevenberg + terminate_action
        if (tid == 0) {
            s_it = 0;
            s_ok = 1;
            s_stop = 0;
            s_go_outer = each_iter > 0;
        }
        __syncthreads();
        while (s_go_outer) {
            if (tid == 0) pose_rt(q_cur, t_cur, Rt);
            __syncthreads();
            double acc[28];
            accumulate(Rt, true, acc);
            cta_sum<kPoseThreads>(acc, red, scratch);
            if (tid == 0) {
                if (s_it == 0) {  // computeLambdaInit
                    s_cur_chi = red[27];
                    double mx = 0.0;
                    int k = 0;
                    for (int a = 0; a < 6; ++a) {
                        mx = fmax(mx, fabs(red[k]));
                        k += 6 - a;
                    }
                    s_lambda = 1e-5 * mx;
                    s_ni = 2.0;
                }
                s_qmax = 0;
                s_rho = 0.0;
                s_go_inner = 1;
            }
            __syncthreads();
            while (s_go_inner) {
                if (tid == 0) {  // (H + lambda I) x = b, dense Cholesky like the reduced system of the local BA
                    double A[36], b[6];
                    int k = 0;
                    for (int a = 0; a < 6; ++a)
                        for (int c = a; c < 6; ++c) {
                            A[a * 6 + c] = red[k];
                            A[c * 6 + a] = red[k];
                            ++k;
                        }
                    for (int a = 0; a < 6; ++a) {
                        A[a * 7] += s_lambda;
                        b[a] = red[21 + a];
                    }
                    int ok2 = 1;
                    for (int j = 0; j < 6 && ok2; ++j) {
                        double d = A[j * 6 + j];
                        for (int kk = 0; kk < j; ++kk) d -= A[j * 6 + kk] * A[j * 6 + kk];
                        if (!(d > 0) || !isfinite(d)) {
                            ok2 = 0;
                            break;
                        }
                        d = sqrt(d);
                        A[j * 6 + j] = d;
                        for (int i = j + 1; i < 6; ++i) {
                            double sv = A[i * 6 + j];
                            for (int kk = 0; kk < j; ++kk) sv -= A[i * 6 + kk] * A[j * 6 + kk];
                            A[i * 6 + j] = sv / d;
                        }
                    }
                    if (ok2) {
                        for (int i = 0; i < 6; ++i) {
                            double sv = b[i];
                            for (int kk = 0; kk < i; ++kk) sv -= A[i * 6 + kk] * b[kk];
                            b[i] = sv / A[i * 7];
                        }
                        for (int i = 5; i >= 0; --i) {
                            double sv = b[i];
                            for (int kk = i + 1; kk < 6; ++kk) sv -= A[kk * 6 + i] * b[kk];
                            b[i] = sv / A[i * 7];
                        }
                        for (int i = 0; i < 6; ++i) x[i] = b[i];
                        se3_oplus(q_cur, t_cur, x, q_trial, t_trial);
                    } else {
                        for (int i = 0; i < 4; ++i) q_trial[i] = q_cur[i];
                        for (int i = 0; i < 3; ++i) t_trial[i] = t_cur[i];
                    }
                    s_ok2 = ok2;
                    pose_rt(q_trial, t_trial, Rt_trial);
                }
                __syncthreads();
                double tacc[28];
                accumulate(Rt_trial, false, tacc);
                double chi1[1] = {tacc[27]};
                cta_sum<kPoseThreads>(chi1, red + 27, scratch);  // red[0..26] (H, b of the current state) stay valid for the next trial
                if (tid == 0) {
                    const bool ok2 = s_ok2 != 0;
                    const double temp_chi = ok2 ? red[27] : 1.7976931348623157e308;
                    double rho = s_cur_chi - temp_chi;
                    double scale = 0.0;  // computeScale
                    if (ok2)
                        for (int i = 0; i < 6; ++i) scale += x[i] * (s_lambda * x[i] + red[21 + i]);
                    scale += 1e-3;
                    rho /= scale;
                    bool broke = false;
                    if (rho > 0 && isfinite(temp_chi) && ok2) {
                        double alpha = 1. - pow(2 * rho - 1, 3.0);
                        alpha = fmin(alpha, 2. / 3.);
                        s_lambda *= fmax(1. / 3., alpha);
                        s_ni = 2.0;
                        s_cur_chi = temp_chi;
                        for (int i = 0; i < 4; ++i) q_cur[i] = q_trial[i];
                        for (int i = 0; i < 3; ++i) t_cur[i] = t_trial[i];
                    } else {
                        s_lambda *= s_ni;
                        s_ni *= 2.0;
                        if (!isfinite(s_lambda)) broke = true;
                    }
                    if (!broke) s_qmax++;
                    s_rho = rho;
                    const bool again = !broke && rho < 0 && s_qmax < 10 && !s_stop;
                    s_go_inner = again ? 1 : 0;
                    if (!again) {
                        if (s_qmax == 10 || rho == 0 || !isfinite(s_lambda)) s_ok = 0;
                        const double chi_now = s_cur_chi;
                        if (s_it == 0) {
                            s_last_chi = chi_now;
                        } else {
                            const double gain = (s_last_chi - chi_now) / chi_now;
                            s_last_chi = chi_now;
                            if (gain >= 0 && gain < 1e-3) s_stop = 1;
                        }
                        s_it++;
                        s_go_outer = (s_it < each_iter && !s_stop && s_ok) ? 1 : 0;
                    }
                }
                __syncthreads();
            }
        }
        // ---- :133-167 classify every observation at the optimised pose (inactive edges are re-evaluated, :137-139)
        if (tid == 0) {
            pose_rt(q_cur, t_cur, Rt);
            s_bad = 0;
        }
        __syncthreads();
        int bad = 0;
        for (int e = tid; e < n; e += kPoseThreads) {
            const PoseEdge pe = edges[e];
            EdgeS ed;
            ed.ox = pe.ox; ed.oy = pe.oy; ed.oxr = pe.oxr;
            double err[3], pc[3];
            edge_residual(ed, cam, Rt, pe.pw, err, pc);
            const double e2 = (double)pe.inv_sigma_sq * (err[0] * err[0] + err[1] * err[1] + err[2] * err[2]);
            const double thr = (pe.oxr < 0.f) ? (double)5.99146f : (double)7.81473f;
            const unsigned char o = thr < e2 ? 1 : 0;
            flags[e] = o;
            level[e] = o;
            bad += o;
        }
        atomicAdd(&s_bad, bad);
        if (trials != 0 && trial + 1 == trials_robust) robust_on = false;  // :164-166
        __syncthreads();
        bad_total = s_bad;
        __syncthreads();
        if (n - bad_total < 5) break;  // :169-171
    }
    if (tid == 0) {
        n_valid_out[blockIdx.x] = (unsigned)(n - bad_total);
        double Rm[9];
        quat_to_rot(q_cur, Rm);
        double* M = pose_out + 16 * (size_t)blockIdx.x;  // util::converter::to_eigen_mat
        M[0] = Rm[0]; M[1] = Rm[1]; M[2] = Rm[2]; M[3] = t_cur[0];
        M[4] = Rm[3]; M[5] = Rm[4]; M[6] = Rm[5]; M[7] = t_cur[1];
        M[8] = Rm[6]; M[9] = Rm[7]; M[10] = Rm[8]; M[11] = t_cur[2];
        M[12] = 0; M[13] = 0; M[14] = 0; M[15] = 1;
    }
}


// ---------------------------------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------------------------------
struct Solver {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    StagingArena arena;
    double* h_res = nullptr;           // pinned readback
    size_t h_res_cap = 0;
    float last_ms = 0.f;
    int last_launches = 0;
    cudaEvent_t ev_sync = nullptr;
    cudaEvent_t ev_ctl[2] = {nullptr, nullptr};  // completion of the two alternating control-block read-backs
    int* h_abort = nullptr;       // pinned, device-visible mirrors of the callers' force_stop flags (one word per window)
    int* d_abort = nullptr;
    int abort_cap = 0;
    // profiling mode (b200_lba_enable_profile): an event after every launch; per-kernel sums of the last batch
    bool profile = false;
    std::vector<cudaEvent_t> prof_ev;
    std::vector<int> prof_kind;
    float prof_ms[8] = {};
    int prof_n[8] = {};
    bool force_offchip = false;
    int chol_cluster = kCholCluster;  // CTAs sharing one factorisation (B200_LBA_CLUSTER overrides: 1, 2, 4 or 8)
    bool chol_cluster_pinned = false;
    // Waiting for the stream (a few times per batch).  B200_LBA_WAIT=spin|block|yield|nap overrides.
    bool last_gain_stop = false;  // the last window of the last batch ended on terminate_action's gain threshold
    int wait_mode = 3;  // 0 spin (cudaStreamSynchronize), 1 blocking event, 2 poll + sched_yield, 3 poll + 15 us sleep
    cudaError_t wait(cudaStream_t st) {
        if (wait_mode == 0) return cudaStreamSynchronize(st);
        if (wait_mode >= 2) {
            cudaError_t e;
            while ((e = cudaStreamQuery(st)) == cudaErrorNotReady) {
                if (wait_mode == 2) sched_yield();
                else std::this_thread::sleep_for(std::chrono::microseconds(15));
            }
            return e;
        }
        cudaError_t e = cudaEventRecord(ev_sync, st);
        return e != cudaSuccess ? e : cudaEventSynchronize(ev_sync);
    }
    cudaError_t wait_event(cudaEvent_t ev) {
        if (wait_mode < 2) return cudaEventSynchronize(ev);
        cudaError_t e;
        while ((e = cudaEventQuery(ev)) == cudaErrorNotReady) {
            if (wait_mode == 2) sched_yield();
            else std::this_thread::sleep_for(std::chrono::microseconds(15));
        }
        return e;
    }

    int ensure_res(size_t res_doubles) {
        if (res_doubles > h_res_cap) {
            if (h_res) B200_CUDA(cudaFreeHost(h_res));
            h_res = nullptr;
            h_res_cap = 0;
            B200_CUDA(cudaHostAlloc(&h_res, sizeof(double) * res_doubles * 2, cudaHostAllocDefault));
            h_res_cap = res_doubles * 2;
        }
        return B200_OK;
    }
    int ensure_abort(int n) {
        if (n <= abort_cap) return B200_OK;
        if (h_abort) B200_CUDA(cudaFreeHost(h_abort));
        h_abort = nullptr;
        abort_cap = 0;
        B200_CUDA(cudaHostAlloc((void**)&h_abort, sizeof(int) * (size_t)n * 2, cudaHostAllocMapped));
        B200_CUDA(cudaHostGetDevicePointer((void**)&d_abort, h_abort, 0));
        abort_cap = n * 2;
        return B200_OK;
    }
};

// per-window byte offsets into the arena
struct WinOff {
    size_t cams, e_pose, e_point, e_cam, e_robust, e_can, e_obs, e_isig, e_delta, pose_col, pt_col, q0, t0, Rt0, pts0;  // uploaded
    size_t pt_cnt, pose_cnt, level, chi0, fail, tickets, bad, blk_done;                                                                      // zeroed
    size_t pt_start, order, edges, epcol, pose_start, pose_edges, rowrec, lm_mask, blk_cnt, blk_pair_start, blk_chunk_start, pairs, blocks, chunks,
        chunk_part, robust, q1, t1, Rt1, pts1, chi1, Hpl, Hll, bl, Dinv, Hpp, bp, M, xp, r_chi,
        r_diag, r_scale, r_result, gP, gD, ginvd;                                                                     // scratch
    size_t exp_begin, qf, tf, pf, out, exp_end;                                                                       // export block
};

// Solves the windows ws[0..nw) (indices into the caller's arrays) in lockstep.  status[w] is set for every window.
static int solve_batch(Solver& S, int n_all, const b200_lba_problem_t* Ps, int iters1, int iters2, volatile uint8_t* const* stops,
                       double* const* pose_outs, double* const* points_outs, uint8_t* const* outlier_outs, b200_lba_stats_t* stats, int* status, int rounds = 2, double gain_thr = 1e-3, bool allow_large = false) {
    B200_RANGE("b200:lba:batch");
    const bool debug = getenv("B200_LBA_DEBUG") != nullptr;
    const auto t_begin = std::chrono::steady_clock::now();
    auto ms_since = [](std::chrono::steady_clock::time_point t) { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t).count(); };
    std::vector<int> act;  // windows that take part
    int ret = B200_OK;
    for (int w = 0; w < n_all; ++w) {
        if (stats) std::memset(&stats[w], 0, sizeof(stats[w]));
        status[w] = B200_OK;
        if (stops && stops[w] && *stops[w]) {
            status[w] = B200_ERR_ABORTED;  // local_bundle_adjuster_g2o.cc:308-310
            continue;
        }
        int n_free = 0;
        for (int k = 0; k < Ps[w].n_poses; ++k) n_free += Ps[w].pose_fixed[k] ? 0 : 1;
        // only FREE keyframes enter the reduced system; fixed ones are unlimited.  Up to 166 free keyframes it is factored on chip
        // (one cluster per window); beyond that -- global bundle adjustment -- panel by panel over the whole chip, dense in HBM
        if (6 * n_free > (allow_large ? kCholGlobalMax : kCholOnChipMax)) {
            set_error("b200_lba_solve: window %d has %d free keyframes; the limit of this entry point is %d", w, n_free,
                      (allow_large ? kCholGlobalMax : kCholOnChipMax) / 6);
            status[w] = B200_ERR_INVALID;
            ret = B200_ERR_INVALID;
            continue;
        }
        act.push_back(w);
    }
    const int nw = (int)act.size();
    S.last_ms = 0.f;
    S.last_launches = 0;
    if (nw == 0) return ret;
    // ---- per-window sizes and the free-vertex columns (O(K + L) on the host; everything O(E) happens on the device) ----------
    struct HostWin {
        int K, L, E, Kf, Lf, n, ld, lbc, mask_words, n_blocks, n_chunks_bound;
        size_t n_pairs;
        std::vector<int> pose_col, pt_col;
    };
    std::vector<HostWin> hw(nw);
    int maxE = 1, maxL = 1, maxKf = 1, maxK = 1, max_n = 0, max_lbc = 1, max_blocks = 1, max_chunk_warps = 1;
    std::vector<int> deg;
    for (int x = 0; x < nw; ++x) {
        const b200_lba_problem_t& P = Ps[act[x]];
        HostWin& h = hw[x];
        h.K = P.n_poses; h.L = P.n_points; h.E = P.n_edges;
        h.pose_col.resize(std::max(h.K, 1));
        h.pt_col.resize(std::max(h.L, 1));
        h.Kf = h.Lf = 0;
        for (int k = 0; k < h.K; ++k) h.pose_col[k] = P.pose_fixed[k] ? -1 : h.Kf++;
        if (P.point_fixed) {
            for (int l = 0; l < h.L; ++l) h.pt_col[l] = P.point_fixed[l] ? -1 : h.Lf++;
        } else {
            for (int l = 0; l < h.L; ++l) h.pt_col[l] = l;
            h.Lf = h.L;
        }
        h.n = 6 * h.Kf;
        h.ld = h.n + 2;
        h.lbc = std::max(1, ceil_div(h.L, 16));
        // pairs of the Schur complement: every landmark with m free-keyframe observations contributes m (m + 1) / 2 (one counting pass
        // over the observations; everything else that is O(E) happens on the device)
        h.mask_words = std::max(1, ceil_div(h.Kf, 64));
        h.n_blocks = h.Kf * (h.Kf + 1) / 2;
        h.n_pairs = 0;
        deg.assign(std::max(h.L, 1), 0);
        for (int e = 0; e < h.E; ++e) {
            const int p = P.e_point[e], k = P.e_pose[e];
            if (p >= 0 && p < h.L && k >= 0 && k < h.K && h.pose_col[k] >= 0 && h.pt_col[p] >= 0) deg[p]++;
        }
        for (int l = 0; l < h.L; ++l) h.n_pairs += (size_t)deg[l] * (deg[l] + 1) / 2;
        h.n_chunks_bound = (int)(h.n_pairs / kSchurChunk) + h.n_blocks + 1;
        max_blocks = std::max(max_blocks, h.n_blocks);
        max_chunk_warps = std::max(max_chunk_warps, h.n_chunks_bound + h.n_blocks);
        maxE = std::max(maxE, h.E); maxL = std::max(maxL, h.L); maxKf = std::max(maxKf, h.Kf); maxK = std::max(maxK, h.K);
        max_n = std::max(max_n, h.n); max_lbc = std::max(max_lbc, h.lbc);
    }
    // ---- arena layout -------------------------------------------------------------------------------------------------------
    std::vector<WinOff> wo(nw);
    Layout cv;
    const size_t o_wins = cv.take<WinDev>(nw), o_ctl = cv.take<LmCtl>(nw);
    for (int x = 0; x < nw; ++x) {
        const HostWin& h = hw[x];
        const b200_lba_problem_t& P = Ps[act[x]];
        WinOff& o = wo[x];
        const size_t E = h.E, K = h.K, L = h.L;
        o.cams = cv.take<Cam>(P.n_cams); o.e_pose = cv.take<int>(E); o.e_point = cv.take<int>(E); o.e_cam = cv.take<unsigned char>(E);
        o.e_robust = cv.take<unsigned char>(E); o.e_can = cv.take<unsigned char>(E); o.e_obs = cv.take<float>(3 * E); o.e_isig = cv.take<float>(E);
        o.e_delta = cv.take<float>(E); o.pose_col = cv.take<int>(K); o.pt_col = cv.take<int>(L); o.q0 = cv.take<double>(4 * K);
        o.t0 = cv.take<double>(3 * K); o.Rt0 = cv.take<double>(12 * K); o.pts0 = cv.take<double>(3 * L);
    }
    const size_t upload_bytes = cv.end;
    for (int x = 0; x < nw; ++x) {
        const HostWin& h = hw[x];
        WinOff& o = wo[x];
        o.pt_cnt = cv.take<int>(h.L); o.pose_cnt = cv.take<int>(h.Kf); o.level = cv.take<unsigned char>(h.E); o.chi0 = cv.take<double>(h.E);
        o.fail = cv.take<int>(1); o.tickets = cv.take<int>(2); o.bad = cv.take<int>(1); o.blk_done = cv.take<int>(h.n_blocks);
    }
    const size_t zero_end = cv.end;
    for (int x = 0; x < nw; ++x) {
        const HostWin& h = hw[x];
        WinOff& o = wo[x];
        const size_t E = h.E, K = h.K, L = h.L, Kf = h.Kf, Lf = h.Lf;
        o.pt_start = cv.take<int>(L + 1); o.order = cv.take<int>(E); o.edges = cv.take<EdgeS>(E); o.epcol = cv.take<int>(E);
        o.pose_start = cv.take<int>(Kf + 1); o.pose_edges = cv.take<int>(E); o.rowrec = cv.take<int4>(E);
        o.lm_mask = cv.take<unsigned long long>(L * (size_t)h.mask_words); o.blk_cnt = cv.take<int>(h.n_blocks);
        o.blk_pair_start = cv.take<int>(h.n_blocks + 1); o.blk_chunk_start = cv.take<int>(h.n_blocks + 1); o.pairs = cv.take<int4>(h.n_pairs);
        o.blocks = cv.take<SchurBlock>(h.n_blocks); o.chunks = cv.take<SchurChunk>(h.n_chunks_bound);
        o.chunk_part = cv.take<double>(42 * (size_t)h.n_chunks_bound); o.robust = cv.take<unsigned char>(E);
        o.q1 = cv.take<double>(4 * K); o.t1 = cv.take<double>(3 * K); o.Rt1 = cv.take<double>(12 * K); o.pts1 = cv.take<double>(3 * L);
        o.chi1 = cv.take<double>(E); o.Hpl = cv.take<double>(kHplStride * E); o.Hll = cv.take<double>(6 * Lf); o.bl = cv.take<double>(3 * Lf);
        o.Dinv = cv.take<double>(6 * Lf); o.Hpp = cv.take<double>(36 * Kf); o.bp = cv.take<double>(6 * Kf);
        o.M = cv.take<double>((size_t)(h.n + 1) * h.ld); o.xp = cv.take<double>(h.n);
        o.gP = o.gD = o.ginvd = 0;
        if (h.n > kCholOnChipMax || S.force_offchip) {
            o.gP = cv.take<double>((size_t)kNB * ((h.n + 1 + 3) & ~3));
            o.gD = cv.take<double>(kNB * (kNB + 1));
            o.ginvd = cv.take<double>(h.n);
        }
        o.r_chi = cv.take<double>(h.lbc); o.r_diag = cv.take<double>(h.lbc); o.r_scale = cv.take<double>(h.lbc); o.r_result = cv.take<double>(8);
    }
    const size_t export_begin = cv.end;
    for (int x = 0; x < nw; ++x) {
        const HostWin& h = hw[x];
        WinOff& o = wo[x];
        o.qf = cv.take<double>(4 * (size_t)h.K); o.tf = cv.take<double>(3 * (size_t)h.K); o.pf = cv.take<double>(3 * (size_t)h.L);
        o.out = cv.take<unsigned char>(h.E);
    }
    const size_t export_bytes = cv.end - export_begin;
    const size_t ctl_doubles = ceil_div(sizeof(LmCtl) * (size_t)nw, sizeof(double)) + 8;
    int rc = S.arena.reserve(cv.end + 512, upload_bytes, S.stream);
    if (rc) return rc;
    if ((rc = S.ensure_res(ceil_div(export_bytes, sizeof(double)) + 2 * ctl_doubles + 64))) return rc;
    if ((rc = S.ensure_abort(nw))) return rc;
    unsigned char* d = S.arena.d;
    unsigned char* hs = S.arena.h;
    LmCtl* h_ctl2[2] = {reinterpret_cast<LmCtl*>(S.h_res), reinterpret_cast<LmCtl*>(S.h_res + ctl_doubles)};  // read-back mirrors of the control blocks
    LmCtl* h_ctl = h_ctl2[0];
    unsigned char* h_export = reinterpret_cast<unsigned char*>(S.h_res + 2 * ctl_doubles + 8);
    // ---- staging: the caller's arrays as they are, the initial keyframe states, the descriptors -------------------------------
    WinDev* hwd = reinterpret_cast<WinDev*>(hs + o_wins);
    LmCtl* hctl0 = reinterpret_cast<LmCtl*>(hs + o_ctl);
    for (int x = 0; x < nw; ++x) {
        const HostWin& h = hw[x];
        const b200_lba_problem_t& P = Ps[act[x]];
        const WinOff& o = wo[x];
        const size_t E = h.E, K = h.K, L = h.L;
        Cam* cams = reinterpret_cast<Cam*>(hs + o.cams);
        for (int i = 0; i < P.n_cams; ++i) {
            const b200_camera_t& c = P.cams[i];
            cams[i] = Cam{c.model, c.fx, c.fy, c.cx, c.cy, c.fxb, c.cols, c.rows};
        }
        if (E) {
            std::memcpy(hs + o.e_pose, P.e_pose, sizeof(int) * E);
            std::memcpy(hs + o.e_point, P.e_point, sizeof(int) * E);
            std::memcpy(hs + o.e_cam, P.e_cam, E);
            if (P.e_robust) std::memcpy(hs + o.e_robust, P.e_robust, E);
            else std::memset(hs + o.e_robust, 1, E);
            if (P.e_can_be_outlier) std::memcpy(hs + o.e_can, P.e_can_be_outlier, E);
            else std::memset(hs + o.e_can, 1, E);
            std::memcpy(hs + o.e_obs, P.e_obs, sizeof(float) * 3 * E);
            std::memcpy(hs + o.e_isig, P.e_inv_sigma_sq, sizeof(float) * E);
            std::memcpy(hs + o.e_delta, P.e_delta, sizeof(float) * E);
        }
        if (K) std::memcpy(hs + o.pose_col, h.pose_col.data(), sizeof(int) * K);
        if (L) {
            std::memcpy(hs + o.pt_col, h.pt_col.data(), sizeof(int) * L);
            std::memcpy(hs + o.pts0, P.points, sizeof(double) * 3 * L);
        }
        double* q0 = reinterpret_cast<double*>(hs + o.q0);
        double* t0 = reinterpret_cast<double*>(hs + o.t0);
        double* Rt0 = reinterpret_cast<double*>(hs + o.Rt0);
        for (size_t k = 0; k < K; ++k) {  // util::converter::to_g2o_SE3 (util/converter.cc:17-21)
            const double* M = P.pose_cw + 16 * k;
            const double R[9] = {M[0], M[1], M[2], M[4], M[5], M[6], M[8], M[9], M[10]};
            rot_to_quat(R, &q0[4 * k]);
            quat_normalize(&q0[4 * k]);
            t0[3 * k] = M[3]; t0[3 * k + 1] = M[7]; t0[3 * k + 2] = M[11];
            quat_to_rot(&q0[4 * k], &Rt0[12 * k]);
            Rt0[12 * k + 9] = M[3]; Rt0[12 * k + 10] = M[7]; Rt0[12 * k + 11] = M[11];
        }
        WinDev& W = hwd[x];
        std::memset(&W, 0, sizeof(W));
        W.K = h.K; W.L = h.L; W.E = h.E; W.Kf = h.Kf; W.Lf = h.Lf; W.n = h.n; W.ld = h.ld; W.n_cams = P.n_cams; W.lbc = h.lbc;
        W.e_pose = (const int*)(d + o.e_pose); W.e_point = (const int*)(d + o.e_point); W.e_cam = d + o.e_cam; W.e_robust = d + o.e_robust;
        W.e_can_outlier = d + o.e_can; W.e_obs = (const float*)(d + o.e_obs); W.e_isig = (const float*)(d + o.e_isig);
        W.e_delta = (const float*)(d + o.e_delta); W.pose_col = (const int*)(d + o.pose_col); W.pt_col = (const int*)(d + o.pt_col);
        W.cams = (const Cam*)(d + o.cams);
        W.pt_cnt = (int*)(d + o.pt_cnt); W.pt_start = (int*)(d + o.pt_start); W.order = (int*)(d + o.order); W.edges = (EdgeS*)(d + o.edges);
        W.epcol = (int*)(d + o.epcol); W.pose_cnt = (int*)(d + o.pose_cnt); W.pose_start = (int*)(d + o.pose_start);
        W.pose_edges = (int*)(d + o.pose_edges); W.level = d + o.level; W.robust = d + o.robust;
        W.rowrec = (int4*)(d + o.rowrec);
        W.lm_mask = (unsigned long long*)(d + o.lm_mask); W.mask_words = h.mask_words; W.n_blocks = h.n_blocks; W.blk_cnt = (int*)(d + o.blk_cnt);
        W.blk_pair_start = (int*)(d + o.blk_pair_start); W.blk_chunk_start = (int*)(d + o.blk_chunk_start); W.pairs = (int4*)(d + o.pairs);
        W.blocks = (SchurBlock*)(d + o.blocks); W.chunks = (SchurChunk*)(d + o.chunks); W.chunk_part = (double*)(d + o.chunk_part);
        W.blk_done = (int*)(d + o.blk_done);
        W.q[0] = (double*)(d + o.q0); W.q[1] = (double*)(d + o.q1); W.t[0] = (double*)(d + o.t0); W.t[1] = (double*)(d + o.t1);
        W.Rt[0] = (double*)(d + o.Rt0); W.Rt[1] = (double*)(d + o.Rt1); W.pts[0] = (double*)(d + o.pts0); W.pts[1] = (double*)(d + o.pts1);
        W.chi[0] = (double*)(d + o.chi0); W.chi[1] = (double*)(d + o.chi1);
        W.Hpl = (double*)(d + o.Hpl); W.Hll = (double*)(d + o.Hll); W.bl = (double*)(d + o.bl); W.Dinv = (double*)(d + o.Dinv);
        W.Hpp = (double*)(d + o.Hpp); W.bp = (double*)(d + o.bp); W.M = (double*)(d + o.M); W.xp = (double*)(d + o.xp);
        W.gP = (double*)(d + o.gP); W.gD = (double*)(d + o.gD); W.ginvd = (double*)(d + o.ginvd);
        W.r_chi = (double*)(d + o.r_chi); W.r_diag = (double*)(d + o.r_diag); W.r_scale = (double*)(d + o.r_scale); W.r_result = (double*)(d + o.r_result);
        W.fail = (int*)(d + o.fail); W.tickets = (int*)(d + o.tickets); W.bad_input = (int*)(d + o.bad);
        W.ctl = (LmCtl*)(d + o_ctl) + x;
        W.qf = (double*)(d + o.qf); W.tf = (double*)(d + o.tf); W.pf = (double*)(d + o.pf); W.out = d + o.out;
        LmCtl& c = hctl0[x];
        std::memset(&c, 0, sizeof(c));
        c.ok = 1;
        S.h_abort[x] = 0;
        c.abort_word = (stops && stops[act[x]]) ? S.d_abort + x : nullptr;
    }
    if (debug) fprintf(stderr, "[lba] %d windows staged in %.3f ms (upload %.2f MB, arena %.1f MB)\n", nw, ms_since(t_begin), upload_bytes / 1e6, cv.end / 1e6);
    cudaStream_t st = S.stream;
    int launches = 0;
    S.prof_kind.clear();
    auto mark = [&](int kind) -> int {  // profiling: the time since the previous mark belongs to `kind`
        if (!S.profile) return B200_OK;
        const size_t idx = S.prof_kind.size();
        if (idx >= S.prof_ev.size()) {
            cudaEvent_t e;
            B200_CUDA(cudaEventCreate(&e));
            S.prof_ev.push_back(e);
        }
        B200_CUDA(cudaEventRecord(S.prof_ev[idx], st));
        S.prof_kind.push_back(kind);
        return B200_OK;
    };
    B200_CUDA(cudaEventRecord(S.ev0, st));
    B200_CUDA(S.arena.upload(upload_bytes, st));
    B200_CUDA(cudaMemsetAsync(d + upload_bytes, 0, zero_end - upload_bytes, st));
    if ((rc = mark(-1))) return rc;
    const WinDev* wins = (const WinDev*)(d + o_wins);
    const LmCtl* d_ctl = (const LmCtl*)(d + o_ctl);
    // ---- plan on the device ----------------------------------------------------------------------------------------------------
    plan_count_kernel<<<dim3(ceil_div(maxE, 256), nw), 256, 0, st>>>(wins);
    plan_scan_kernel<<<nw, 1024, 0, st>>>(wins);
    plan_place_kernel<<<dim3(ceil_div(maxE, 256), nw), 256, 0, st>>>(wins);
    plan_sort_kernel<<<dim3(ceil_div(maxL, 128), nw), 128, 0, st>>>(wins);
    plan_pose_lists_kernel<<<dim3(maxKf, nw), kListThreads, 0, st>>>(wins);
    plan_pairs_kernel<false><<<dim3(ceil_div(max_blocks, 4), nw), 128, 0, st>>>(wins);
    plan_pair_scan_kernel<<<nw, 1024, 0, st>>>(wins);
    plan_pairs_kernel<true><<<dim3(ceil_div(max_blocks, 4), nw), 128, 0, st>>>(wins);
    launches += 8;
    if ((rc = mark(0))) return rc;
    B200_RANGE("b200:lba:rounds+export");  // (the plan above is the part of b200:lba:batch outside this range)
    // ---- LM rounds in lockstep ---------------------------------------------------------------------------------------------------
    const bool large = max_n > kCholOnChipMax || S.force_offchip;  // (B200_LBA_FORCE_OFFCHIP: the panel-by-panel path on any size, for tests)
    const size_t chol_smem = sizeof(double) * ((size_t)kNB * (kNB + 1) + 4 + (size_t)((std::min(max_n, kCholOnChipMax) + 1 + 3) & ~3) * kNB);
    B200_CUDA(cudaFuncSetAttribute(chol_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)chol_smem));
    // 8-CTA clusters must sit inside one GPC, so not many of them are co-resident: batches use the smaller cluster (H100 SXM, four
    // windows per batch: 0.18 ms per factorisation with clusters of 4, 0.20 with 2, 0.28 with 8); B200_LBA_CLUSTER pins it
    const int chol_cluster = S.chol_cluster_pinned ? S.chol_cluster : (nw <= 2 ? 8 : 4);
    auto launch_rep = [&]() -> int {
        // computeActiveErrors + buildSystem (windows that start an iteration)
        int rcm;
        landmark_kernel<kBuild><<<dim3(max_lbc, nw), kLmThreads, 0, st>>>(wins);
        if ((rcm = mark(1))) return rcm;
        pose_rows_kernel<<<dim3(maxKf, nw), kRowThreads, 0, st>>>(wins);
        if ((rcm = mark(2))) return rcm;
        // one LM trial (every window that is still iterating)
        schur_mma_kernel<<<dim3(ceil_div(max_chunk_warps, 4), nw), 128, 4 * kSmmaWarpDoubles * sizeof(double), st>>>(wins);
        if ((rcm = mark(3))) return rcm;
        if (large) {  // panel by panel over the whole chip (every window of the batch takes this path; small ones finish early)
            for (int kb = 0; kb < max_n; kb += kNB) {
                const int m = max_n + 1 - std::min(kb + kNB, max_n);
                const long long tm = (m + 3) >> 2, n_tiles = tm * (tm + 1) / 2;
                gchol_panel_kernel<<<dim3(ceil_div(m + 4, kGcholThreads), nw), kGcholThreads, 0, st>>>(wins, kb);
                gchol_trail_kernel<<<dim3((unsigned)std::max<long long>(1, (n_tiles + kGcholThreads - 1) / kGcholThreads), nw), kGcholThreads, 0, st>>>(wins, kb);
                launches += 2;
            }
            gchol_finish_kernel<<<nw, kGfinThreads, 0, st>>>(wins);
        } else {
            cudaLaunchConfig_t cfg = {};
            cfg.gridDim = dim3(chol_cluster * nw);
            cfg.blockDim = dim3(kCholThreads);
            cfg.dynamicSmemBytes = chol_smem;
            cfg.stream = st;
            cudaLaunchAttribute attr[1];
            attr[0].id = cudaLaunchAttributeClusterDimension;
            attr[0].val.clusterDim.x = chol_cluster;
            attr[0].val.clusterDim.y = 1;
            attr[0].val.clusterDim.z = 1;
            cfg.attrs = attr;
            cfg.numAttrs = 1;
            B200_CUDA(cudaLaunchKernelEx(&cfg, chol_solve_kernel, wins));
        }
        if ((rcm = mark(4))) return rcm;
        backsub_kernel<<<dim3(max_lbc, nw), 128, 0, st>>>(wins);  // back-substitution + chi2 of the trial state + accept / reject
        if ((rcm = mark(5))) return rcm;
        launches += 5;
        return B200_OK;
    };
    // Read the control blocks back into mirror `b` (asynchronously) / wait for that copy.  The loop below always has the NEXT chunk
    // of repetitions enqueued before it waits for the read-back of the previous one, so the GPU never idles on a host decision; a
    // chunk enqueued for windows that have all finished costs a handful of empty launches.
    auto fetch_issue = [&](int b) -> int {
        B200_CUDA(cudaMemcpyAsync(h_ctl2[b], d_ctl, sizeof(LmCtl) * nw, cudaMemcpyDeviceToHost, st));
        B200_CUDA(cudaEventRecord(S.ev_ctl[b], st));
        return B200_OK;
    };
    auto fetch_wait = [&](int b) -> int {
        B200_CUDA(S.wait_event(S.ev_ctl[b]));
        h_ctl = h_ctl2[b];
        for (int x = 0; x < nw; ++x)  // the caller's flag may be raised by another thread meanwhile (mapping_module.cc:124)
            if (stops && stops[act[x]] && *stops[act[x]]) S.h_abort[x] = 1;
        return B200_OK;
    };
    auto fetch_ctl = [&]() -> int {
        int r_ = fetch_issue(0);
        return r_ ? r_ : fetch_wait(0);
    };
    const int iters[2] = {iters1, iters2};
    int rc2;
    for (int r = 0; r < rounds; ++r) {
        if (r == 1) {
            // local_bundle_adjuster_g2o.cc:317-321 reads the caller's flag, which the gain stop of round 1 has set through
            // terminate_action; the device takes the same decision from stop_flag / the mirrored word.  A round that does run starts
            // with terminate_action's reset of that flag (terminate_action.cc:46-51).
            if ((rc2 = fetch_ctl())) return rc2;
            for (int x = 0; x < nw; ++x) {
                volatile uint8_t* f = stops ? stops[act[x]] : nullptr;
                if (!f) continue;
                if (h_ctl[x].stop_flag || *f) {
                    S.h_abort[x] = 1;
                    *f = 1;
                } else {
                    S.h_abort[x] = 0;
                }
            }
        }
        lm_round_begin_kernel<<<ceil_div(nw, 64), 64, 0, st>>>(wins, nw, iters[r], r, gain_thr);
        ++launches;
        if (r == 1) {
            outlier_kernel<<<dim3(ceil_div(maxE, 128), nw), 128, 0, st>>>(wins, 0);  // :323-344 (skips itself after an abort)
            ++launches;
        }
        // repetitions of {build; trial}: a round of `iterations` LM iterations needs at least that many trials unless it stops early, so
        // that many repetitions are enqueued (in chunks of at most six) before the control blocks are read back; a window that stops
        // early lets the rest of its chunk run empty (every kernel returns on its control block) and only rejected trials need more.
        // (Round 2a enqueued speculative chunks ahead of every read-back: 5 of 20 repetitions of the bench window ran empty.)
        if (iters[r] > 0) {
            int need = iters[r];
            for (;;) {
                const int chunk = std::max(1, std::min(need, 6));  // (bounded: an early gain stop wastes at most five repetitions)
                for (int i = 0; i < chunk; ++i)
                    if ((rc2 = launch_rep())) return rc2;
                if ((rc2 = fetch_ctl())) return rc2;
                need = 0;
                for (int x = 0; x < nw; ++x)
                    if (h_ctl[x].outer_go) need = std::max(need, std::max(1, h_ctl[x].iterations - h_ctl[x].it));
                if (need == 0) break;
            }
        }
        landmark_kernel<kRoundEnd><<<dim3(max_lbc, nw), kLmThreads, 0, st>>>(wins);  // chi2 of every active edge at the final state
        lm_round_end_kernel<<<nw, 256, 0, st>>>(wins, r);
        launches += 2;
    }
    if (rounds == 2) outlier_kernel<<<dim3(ceil_div(maxE, 128), nw), 128, 0, st>>>(wins, 1);  // :354-375 (global BA marks nothing)
    lm_export_kernel<<<dim3(ceil_div(std::max(std::max(4 * maxK, 3 * maxL), 1), 256), nw), 256, 0, st>>>(wins);
    launches += 2;
    B200_CUDA(cudaGetLastError());
    if ((rc = mark(7))) return rc;
    B200_CUDA(cudaEventRecord(S.ev1, st));
    B200_CUDA(cudaMemcpyAsync(h_export, d + export_begin, export_bytes, cudaMemcpyDeviceToHost, st));
    std::vector<int> h_bad(nw, 0);
    if ((rc2 = fetch_ctl())) return rc2;
    for (int x = 0; x < nw; ++x) B200_CUDA(cudaMemcpyAsync(&h_bad[x], d + wo[x].bad, sizeof(int), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    B200_CUDA(cudaEventElapsedTime(&S.last_ms, S.ev0, S.ev1));
    S.last_launches = launches;
    for (int k2 = 0; k2 < 8; ++k2) {
        S.prof_ms[k2] = 0.f;
        S.prof_n[k2] = 0;
    }
    for (size_t m = 1; m < S.prof_kind.size(); ++m) {
        float ms = 0.f;
        B200_CUDA(cudaEventElapsedTime(&ms, S.prof_ev[m - 1], S.prof_ev[m]));
        const int kd = S.prof_kind[m];
        if (kd >= 0 && kd < 8) {
            S.prof_ms[kd] += ms;
            S.prof_n[kd] += 1;
        }
    }
    if (debug) fprintf(stderr, "[lba] batch of %d windows: %.3f ms wall, %.3f ms on the stream, %d launches\n", nw, ms_since(t_begin), S.last_ms, launches);
    // ---- results ----------------------------------------------------------------------------------------------------------------
    for (int x = 0; x < nw; ++x) {
        const int w = act[x];
        const HostWin& h = hw[x];
        const b200_lba_problem_t& P = Ps[w];
        const WinOff& o = wo[x];
        if (h_bad[x]) {
            set_error("b200_lba_solve: edge %d of window %d references an invalid vertex/camera", h_bad[x] - 1, w);
            status[w] = B200_ERR_INVALID;
            ret = B200_ERR_INVALID;
            continue;
        }
        const LmCtl& c = h_ctl[x];
        if (stats) {
            stats[w].lambda_init = c.lambda_init;
            for (int r = 0; r < 2; ++r) {
                stats[w].iterations[r] = c.iters_done[r];
                stats[w].chi2[r] = c.chi2[r];
                stats[w].lambda_final[r] = c.lambda_final[r];
            }
        }
        // terminate_action's gain-threshold stop writes the caller's flag (terminate_action.cc:66-70); an externally raised flag stays up
        if (stops && stops[w] && c.stop_flag) *stops[w] = 1;
        S.last_gain_stop = c.stop_flag != 0;
        const unsigned char* ex = h_export + (o.qf - export_begin);
        const double* qf = reinterpret_cast<const double*>(ex);
        const double* tf = reinterpret_cast<const double*>(h_export + (o.tf - export_begin));
        const double* pf = reinterpret_cast<const double*>(h_export + (o.pf - export_begin));
        const unsigned char* out = h_export + (o.out - export_begin);
        int n_out = 0;
        for (int e = 0; e < h.E && rounds == 2; ++e) n_out += out[e];
        if (rounds == 2 && outlier_outs && outlier_outs[w] && h.E) std::memcpy(outlier_outs[w], out, h.E);
        if (stats) stats[w].n_outliers = n_out;
        if (h.L) std::memcpy(points_outs[w], pf, sizeof(double) * 3 * (size_t)h.L);
        for (int k = 0; k < h.K; ++k) {  // util::converter::to_eigen_mat (util/converter.cc:23-25)
            double* M = pose_outs[w] + 16 * (size_t)k;
            if (P.pose_fixed[k]) {
                std::memcpy(M, P.pose_cw + 16 * (size_t)k, sizeof(double) * 16);
                continue;
            }
            double R[9];
            quat_to_rot(&qf[4 * k], R);
            M[0] = R[0]; M[1] = R[1]; M[2] = R[2]; M[3] = tf[3 * k];
            M[4] = R[3]; M[5] = R[4]; M[6] = R[5]; M[7] = tf[3 * k + 1];
            M[8] = R[6]; M[9] = R[7]; M[10] = R[8]; M[11] = tf[3 * k + 2];
            M[12] = 0; M[13] = 0; M[14] = 0; M[15] = 1;
        }
    }
    return ret;
}

// ---- stage C of b200_track_local_map (track_chain.cuh) -------------------------------------------------------------------------
// One CTA per frame: apply the matches of the search to the frame's landmark slots in the reference's order (frm.add_landmark,
// projection.cc:87: a later landmark replaces an earlier one on the same keypoint), then one edge per keypoint that carries a
// landmark, in keypoint order (pose_optimizer_g2o.cc:88-111).
constexpr int kTrackEdgeThreads = 256;
constexpr int kMatchedBias = 1 << 30;
__global__ void __launch_bounds__(kTrackEdgeThreads) track_edges_kernel(chain::TrackShared sh, const chain::TrackFrameDev* __restrict__ frames,
                                                                        PoseProb* __restrict__ probs, PoseEdge* __restrict__ edges_all,
                                                                        int* __restrict__ edge_kp_all, const int* __restrict__ gate) {
    __shared__ int warp_sum[kTrackEdgeThreads / 32];
    __shared__ int s_base;
    const chain::TrackFrameDev& F = frames[blockIdx.x];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = F.status[0];
    int* slot = F.kp_landmark_out;
    for (int i = tid; i < F.kp_cap; i += kTrackEdgeThreads) {
        int l = -1;
        if (i < n && F.kp_landmark && i < F.n_kp_in) {
            l = F.kp_landmark[i];
            if (l < 0 || l >= F.n_lm) l = -1;
        }
        slot[i] = l;
        F.kp_outlier[i] = 0;
    }
    __syncthreads();
    for (int q = tid; q < F.n_lm; q += kTrackEdgeThreads) {
        const int k = F.match_out[q];
        if (k >= 0 && k < n) atomicMax(&slot[k], q + kMatchedBias);
    }
    __syncthreads();
    if (tid == 0) s_base = 0;
    const PoseProb pb = probs[blockIdx.x];
    PoseEdge* __restrict__ edges = edges_all + pb.edge_off;
    int* __restrict__ edge_kp = edge_kp_all + pb.edge_off;
    __syncthreads();
    for (int i0 = 0; i0 < n; i0 += kTrackEdgeThreads) {
        const int i = i0 + tid;
        int l = -1;
        if (i < n) {
            l = slot[i];
            if (l >= kMatchedBias) l -= kMatchedBias;
            slot[i] = l;
        }
        const unsigned ballot = __ballot_sync(0xFFFFFFFFu, l >= 0);
        if (lane == 0) warp_sum[warp] = __popc(ballot);
        __syncthreads();
        int before = s_base;
        for (int w = 0; w < warp; ++w) before += warp_sum[w];
        if (l >= 0) {
            const int e = before + __popc(ballot & ((1u << lane) - 1u));
            const b200_keypoint_t kp = F.undist[i];
            PoseEdge pe;
            pe.pw[0] = F.pos_w[3 * (size_t)l];
            pe.pw[1] = F.pos_w[3 * (size_t)l + 1];
            pe.pw[2] = F.pos_w[3 * (size_t)l + 2];
            pe.ox = kp.x;
            pe.oy = kp.y;
            pe.oxr = F.kp_x_right ? F.kp_x_right[i] : -1.0f;  // stereo_x_right_.empty() ? -1 (:94)
            pe.inv_sigma_sq = sh.inv_level_sigma_sq[kp.octave & 31];
            pe.delta = sh.delta;
            pe.pad = 0;
            edges[e] = pe;
            edge_kp[e] = i;
        }
        __syncthreads();
        if (tid == 0) {
            int t = s_base;
            for (int w = 0; w < kTrackEdgeThreads / 32; ++w) t += warp_sum[w];
            s_base = t;
        }
        __syncthreads();
    }
    if (tid == 0) {  // a gated frame keeps its matches but gets no edge: pose_optimize_kernel returns before any iteration
        const int n_edges = (!gate || gate[blockIdx.x]) ? s_base : 0;
        probs[blockIdx.x].n = n_edges;
        F.status[2] = n_edges;
    }
}

__global__ void __launch_bounds__(256) track_scatter_kernel(const chain::TrackFrameDev* __restrict__ frames, const PoseProb* __restrict__ probs,
                                                            const unsigned char* __restrict__ flags_all, const int* __restrict__ edge_kp_all) {
    const PoseProb& pb = probs[blockIdx.y];
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= pb.n) return;
    frames[blockIdx.y].kp_outlier[edge_kp_all[pb.edge_off + e]] = flags_all[pb.edge_off + e];
}

}  // namespace lba
}  // namespace b200

struct b200_lba_s {
    b200::lba::Solver s;
};

namespace b200 {
namespace lba {
// For the entry points of other translation units that run on a handle's stream (PnP, essential and two-view RANSAC, pose graph,
// Sim3 refinement): its arena holds at least dev_bytes on the device and host_bytes in the mirror until the handle's next call.
int staging(b200_lba_t h, size_t dev_bytes, size_t host_bytes, cudaStream_t* stream, StagingArena** arena) {
    Solver& S = h->s;
    B200_CUDA(cudaSetDevice(S.device));
    const int rc = S.arena.reserve(dev_bytes, host_bytes, S.stream);
    if (rc) return rc;
    *stream = S.stream;
    *arena = &S.arena;
    return B200_OK;
}
}  // namespace lba
}  // namespace b200

static int lba_check_problem(const b200_lba_problem_t* P, const char* who) {
    if (P->n_poses < 0 || P->n_points < 0 || P->n_edges < 0 || P->n_cams < 0 || (P->n_poses > 0 && (!P->pose_cw || !P->pose_fixed))
        || (P->n_points > 0 && !P->points)
        || (P->n_edges > 0 && (!P->e_pose || !P->e_point || !P->e_cam || !P->e_obs || !P->e_inv_sigma_sq || !P->e_delta || !P->cams))) {
        b200::set_error("%s: inconsistent problem description", who);
        return B200_ERR_INVALID;
    }
    return B200_OK;
}

extern "C" {

int b200_lba_create(int device, b200_lba_t* out) {
    if (!out) return B200_ERR_INVALID;
    int rc = b200::require_device(device);
    if (rc) return rc;
    b200_lba_s* h = new (std::nothrow) b200_lba_s();
    if (!h) return B200_ERR_INVALID;
    h->s.device = device;
    // Local BA is the mapping thread's work (mapping_module.cc:63): tracking must not wait for it, so its stream has the LOWEST
    // priority (its CTAs fill the gaps the front end leaves; lowest == the default priority 0 of ordinary streams on this GPU, the
    // range is [0, -5]).  B200_LBA_PRIORITY=high|normal|low overrides.
    int prio_lo = 0, prio_hi = 0;
    cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
    int prio = prio_lo;
    if (const char* pe = getenv("B200_LBA_PRIORITY")) prio = (pe[0] == 'l') ? prio_lo : ((pe[0] == 'n') ? 0 : prio_hi);
    cudaError_t e = cudaStreamCreateWithPriority(&h->s.stream, cudaStreamNonBlocking, prio);
    if (e == cudaSuccess) e = cudaEventCreate(&h->s.ev0);
    if (e == cudaSuccess) e = cudaEventCreate(&h->s.ev1);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->s.ev_sync, cudaEventBlockingSync | cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->s.ev_ctl[0], cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->s.ev_ctl[1], cudaEventDisableTiming);
    if (const char* cc = getenv("B200_LBA_CLUSTER")) {
        const int c = atoi(cc);
        if (c == 1 || c == 2 || c == 4 || c == 8) {
            h->s.chol_cluster = c;
            h->s.chol_cluster_pinned = true;
        }
    }
    if (const char* fo = getenv("B200_LBA_FORCE_OFFCHIP")) h->s.force_offchip = fo[0] == '1';
    if (const char* w = getenv("B200_LBA_WAIT")) h->s.wait_mode = w[0] == 'b' ? 1 : (w[0] == 'y' ? 2 : (w[0] == 'n' ? 3 : 0));  // spin | block | yield | nap
    if (e != cudaSuccess) {
        delete h;
        return b200::cuda_fail(e, "stream/event creation", __FILE__, __LINE__);
    }
    *out = h;
    return B200_OK;
}

int b200_lba_destroy(b200_lba_t h) {
    if (!h) return B200_OK;
    cudaSetDevice(h->s.device);
    if (h->s.stream) cudaStreamSynchronize(h->s.stream);
    h->s.arena.release();
    if (h->s.h_res) cudaFreeHost(h->s.h_res);
    if (h->s.h_abort) cudaFreeHost(h->s.h_abort);
    if (h->s.ev0) cudaEventDestroy(h->s.ev0);
    if (h->s.ev1) cudaEventDestroy(h->s.ev1);
    if (h->s.ev_sync) cudaEventDestroy(h->s.ev_sync);
    for (cudaEvent_t e : h->s.prof_ev) cudaEventDestroy(e);
    if (h->s.ev_ctl[0]) cudaEventDestroy(h->s.ev_ctl[0]);
    if (h->s.ev_ctl[1]) cudaEventDestroy(h->s.ev_ctl[1]);
    if (h->s.stream) cudaStreamDestroy(h->s.stream);
    delete h;
    return B200_OK;
}

int b200_lba_solve_batch(b200_lba_t h, int n_windows, const b200_lba_problem_t* problems, int iters1, int iters2,
                         volatile uint8_t* const* force_stop, double* const* pose_cw_out, double* const* points_out, uint8_t* const* outlier_out,
                         b200_lba_stats_t* stats, int32_t* status) {
    if (!h || n_windows < 0 || iters1 < 0 || iters2 < 0) return B200_ERR_INVALID;
    if (n_windows == 0) return B200_OK;
    if (!problems || !pose_cw_out || !points_out || !status) {
        b200::set_error("b200_lba_solve_batch: null argument");
        return B200_ERR_INVALID;
    }
    for (int w = 0; w < n_windows; ++w) {
        if ((problems[w].n_poses > 0 && !pose_cw_out[w]) || (problems[w].n_points > 0 && !points_out[w])) {
            b200::set_error("b200_lba_solve_batch: window %d has no output buffers", w);
            return B200_ERR_INVALID;
        }
        const int rc = lba_check_problem(&problems[w], "b200_lba_solve_batch");
        if (rc) return rc;
    }
    B200_CUDA(cudaSetDevice(h->s.device));
    return b200::lba::solve_batch(h->s, n_windows, problems, iters1, iters2, force_stop, pose_cw_out, points_out, outlier_out, stats, status);
}

int b200_lba_solve(b200_lba_t h, const b200_lba_problem_t* P, int iters1, int iters2, volatile uint8_t* force_stop, double* pose_cw_out,
                   double* points_out, uint8_t* outlier_out, b200_lba_stats_t* stats) {
    if (!h || !P || !pose_cw_out || !points_out || iters1 < 0 || iters2 < 0) {
        b200::set_error("b200_lba_solve: null argument");
        return B200_ERR_INVALID;
    }
    int rc = lba_check_problem(P, "b200_lba_solve");
    if (rc) return rc;
    B200_CUDA(cudaSetDevice(h->s.device));
    int32_t status = B200_OK;
    volatile uint8_t* stops[1] = {force_stop};
    double* poses[1] = {pose_cw_out};
    double* pts[1] = {points_out};
    uint8_t* outl[1] = {outlier_out};
    rc = b200::lba::solve_batch(h->s, 1, P, iters1, iters2, stops, poses, pts, outl, stats, &status);
    return rc ? rc : status;
}

int b200_global_ba_solve(b200_lba_t h, const b200_lba_problem_t* P, int num_iter, double gain_threshold, volatile uint8_t* force_stop, double* pose_cw_out,
                         double* points_out, b200_lba_stats_t* stats) {
    if (!h || !P || !pose_cw_out || !points_out || num_iter < 0 || !(gain_threshold >= 0.0)) {
        b200::set_error("b200_global_ba_solve: null argument");
        return B200_ERR_INVALID;
    }
    B200_CUDA(cudaSetDevice(h->s.device));
    // optimizer.setForceStopFlag(force_stop_flag): a flag that is already up stops the optimisation before its first iteration; the
    // reference then reports "aborted" (:340-342)
    if (force_stop && *force_stop) return B200_ERR_ABORTED;
    volatile uint8_t* stops[1] = {force_stop};
    double* poses[1] = {pose_cw_out};
    double* pts[1] = {points_out};
    uint8_t* outl[1] = {nullptr};
    int status = B200_OK;
    b200_lba_stats_t local{};
    b200_lba_stats_t* st = stats ? stats : &local;
    const int rc = b200::lba::solve_batch(h->s, 1, P, num_iter, 0, stops, poses, pts, outl, st, &status, 1, gain_threshold, true);
    if (rc) return rc;
    if (status) return status;
    if (force_stop && *force_stop && !h->s.last_gain_stop) return B200_ERR_ABORTED;  // raised by the caller while the solve ran (:340-342)
    return B200_OK;
}

int b200_pose_optimize(b200_lba_t h, int n_problems, const b200_lba_problem_t* problems, int num_trials_robust, int num_trials, int num_each_iter,
                       double* pose_cw_out, uint8_t* outlier_flags, uint32_t* n_valid) {
    B200_RANGE("b200:lba:pose_optimize");
    using namespace b200::lba;
    if (!h || n_problems < 0 || num_trials_robust < 0 || num_trials < 0 || num_each_iter < 0) return B200_ERR_INVALID;
    if (n_problems == 0) return B200_OK;
    if (!problems || !pose_cw_out || !n_valid) {
        b200::set_error("b200_pose_optimize: null argument");
        return B200_ERR_INVALID;
    }
    Solver& S = h->s;
    B200_CUDA(cudaSetDevice(S.device));
    size_t total_edges = 0;
    for (int p = 0; p < n_problems; ++p) {
        const b200_lba_problem_t& P = problems[p];
        if (P.n_poses != 1 || P.n_edges < 0 || P.n_points < 0 || P.n_cams < 1 || !P.pose_cw || !P.cams
            || (P.n_edges > 0 && (!P.points || !P.e_point || !P.e_obs || !P.e_inv_sigma_sq || !P.e_delta))) {
            b200::set_error("b200_pose_optimize: problem %d must hold exactly one pose, its observed landmarks and one edge per observation", p);
            return B200_ERR_INVALID;
        }
        for (int e = 0; e < P.n_edges; ++e) {
            if (P.e_point[e] < 0 || P.e_point[e] >= P.n_points || (P.e_cam && P.e_cam[e] >= P.n_cams)) {
                b200::set_error("b200_pose_optimize: edge %d of problem %d references an invalid landmark/camera", e, p);
                return B200_ERR_INVALID;
            }
            // one frame, one camera (pose_optimizer_g2o.cc:38-43): the kernel projects every edge with the camera of edge 0
            if (P.e_cam && P.e_cam[e] != P.e_cam[0]) {
                b200::set_error("b200_pose_optimize: problem %d names camera %d on edge 0 and camera %d on edge %d; a frame has one camera", p,
                                (int)P.e_cam[0], (int)P.e_cam[e], e);
                return B200_ERR_INVALID;
            }
        }
        total_edges += (size_t)P.n_edges;
    }
    if (total_edges > 0 && !outlier_flags) return B200_ERR_INVALID;
    b200::Layout L;
    const size_t o_probs = L.take<PoseProb>(n_problems), o_edges = L.take<PoseEdge>(total_edges);
    const size_t upload_bytes = L.end;
    const size_t o_level = L.take<unsigned char>(total_edges), o_flags = L.take<unsigned char>(total_edges);
    const size_t o_pose = L.take<double>(16 * (size_t)n_problems), o_valid = L.take<unsigned>(n_problems);
    cudaStream_t st = S.stream;
    int rc = S.arena.reserve(L.end + 256, upload_bytes, st);
    if (rc) return rc;
    unsigned char* hs = S.arena.h;
    PoseProb* hp = reinterpret_cast<PoseProb*>(hs + o_probs);
    PoseEdge* he = reinterpret_cast<PoseEdge*>(hs + o_edges);
    size_t off = 0;
    for (int p = 0; p < n_problems; ++p) {
        const b200_lba_problem_t& P = problems[p];
        PoseProb pb{};
        pb.n = P.n_edges;
        pb.edge_off = (int)off;
        const b200_camera_t& c = P.cams[(P.e_cam && P.n_edges > 0) ? P.e_cam[0] : 0];
        pb.cam = Cam{c.model, c.fx, c.fy, c.cx, c.cy, c.fxb, c.cols, c.rows};
        const double* M = P.pose_cw;  // util::converter::to_g2o_SE3 (util/converter.cc:17-21)
        const double R[9] = {M[0], M[1], M[2], M[4], M[5], M[6], M[8], M[9], M[10]};
        rot_to_quat(R, pb.q);
        quat_normalize(pb.q);
        pb.t[0] = M[3]; pb.t[1] = M[7]; pb.t[2] = M[11];
        hp[p] = pb;
        for (int e = 0; e < P.n_edges; ++e) {
            PoseEdge pe{};
            const double* pw = P.points + 3 * (size_t)P.e_point[e];
            pe.pw[0] = pw[0]; pe.pw[1] = pw[1]; pe.pw[2] = pw[2];
            pe.ox = P.e_obs[3 * e]; pe.oy = P.e_obs[3 * e + 1]; pe.oxr = P.e_obs[3 * e + 2];
            pe.inv_sigma_sq = P.e_inv_sigma_sq[e];
            pe.delta = P.e_delta[e];
            he[off + e] = pe;
        }
        off += (size_t)P.n_edges;
    }
    unsigned char* d = S.arena.d;
    B200_CUDA(cudaEventRecord(S.ev0, st));
    B200_CUDA(S.arena.upload(upload_bytes, st));
    pose_optimize_kernel<<<n_problems, kPoseThreads, 0, st>>>((const PoseProb*)(d + o_probs), (const PoseEdge*)(d + o_edges), d + o_level, d + o_flags,
                                                             num_trials_robust, num_trials, num_each_iter, (double*)(d + o_pose),
                                                             (unsigned*)(d + o_valid));
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaEventRecord(S.ev1, st));
    B200_CUDA(cudaMemcpyAsync(pose_cw_out, d + o_pose, sizeof(double) * 16 * (size_t)n_problems, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaMemcpyAsync(n_valid, d + o_valid, sizeof(unsigned) * (size_t)n_problems, cudaMemcpyDeviceToHost, st));
    if (total_edges) B200_CUDA(cudaMemcpyAsync(outlier_flags, d + o_flags, total_edges, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    B200_CUDA(cudaEventElapsedTime(&S.last_ms, S.ev0, S.ev1));
    S.last_launches = 1;
    for (int p = 0; p < n_problems; ++p)  // fewer than five observations: the reference returns before touching the pose (:116-118)
        if (problems[p].n_edges < 5) std::memcpy(pose_cw_out + 16 * (size_t)p, problems[p].pose_cw, sizeof(double) * 16);
    return B200_OK;
}

int b200_lba_enable_profile(b200_lba_t h, int enable) {
    if (!h) return B200_ERR_INVALID;
    h->s.profile = enable != 0;
    return B200_OK;
}

int b200_lba_kernel_ms(b200_lba_t h, int kernel, float* total_ms, int* launches) {
    if (!h || kernel < 0 || kernel >= 8) return B200_ERR_INVALID;
    if (total_ms) *total_ms = h->s.prof_ms[kernel];
    if (launches) *launches = h->s.prof_n[kernel];
    return B200_OK;
}

int b200_lba_last_profile(b200_lba_t h, float* gpu_ms, int* launches) {
    if (!h) return B200_ERR_INVALID;
    if (gpu_ms) *gpu_ms = h->s.last_ms;
    if (launches) *launches = h->s.last_launches;
    return B200_OK;
}

}  // extern "C"

namespace b200 {
namespace chain {
int track_stage_c(b200_lba_t opt, cudaStream_t st, const TrackShared& sh, const TrackFrameDev* d_frames, const TrackFrameDev* h_frames,
                  const double* const* pose_cw, int n_frames, int max_kp, int trials_robust, int trials, int each_iter, double* d_pose_out,
                  unsigned* d_n_valid, cudaEvent_t ev_edges_done, const int* d_gate) {
    using namespace b200::lba;
    if (!opt) return B200_ERR_INVALID;
    Solver& S = opt->s;
    size_t total = 0;
    for (int f = 0; f < n_frames; ++f) total += (size_t)h_frames[f].kp_cap;
    Layout L;
    const size_t o_probs = L.take<PoseProb>(n_frames);
    const size_t upload_bytes = L.end;
    const size_t o_edges = L.take<PoseEdge>(total), o_kp = L.take<int>(total), o_level = L.take<unsigned char>(total), o_flags = L.take<unsigned char>(total);
    int rc = S.arena.reserve(L.end + 256, upload_bytes, st);
    if (rc) return rc;
    PoseProb* hp = S.arena.host<PoseProb>(o_probs);
    size_t off = 0;
    for (int f = 0; f < n_frames; ++f) {
        PoseProb pb{};
        pb.n = 0;
        pb.edge_off = (int)off;
        // fisheye and radial division use the perspective edges (reproj_edge_wrapper.h), i.e. edge model 0
        pb.cam = Cam{sh.model == 1 ? 1 : 0, sh.fx, sh.fy, sh.cx, sh.cy, sh.fxb, sh.cols, sh.rows};
        const double* M = pose_cw[f];  // util::converter::to_g2o_SE3 (util/converter.cc:17-21)
        const double R[9] = {M[0], M[1], M[2], M[4], M[5], M[6], M[8], M[9], M[10]};
        rot_to_quat(R, pb.q);
        quat_normalize(pb.q);
        pb.t[0] = M[3]; pb.t[1] = M[7]; pb.t[2] = M[11];
        hp[f] = pb;
        off += (size_t)h_frames[f].kp_cap;
    }
    unsigned char* d = S.arena.d;
    B200_CUDA(S.arena.upload(upload_bytes, st));
    PoseProb* dp = reinterpret_cast<PoseProb*>(d + o_probs);
    track_edges_kernel<<<n_frames, kTrackEdgeThreads, 0, st>>>(sh, d_frames, dp, (PoseEdge*)(d + o_edges), (int*)(d + o_kp), d_gate);
    if (ev_edges_done) B200_CUDA(cudaEventRecord(ev_edges_done, st));
    pose_optimize_kernel<<<n_frames, kPoseThreads, 0, st>>>(dp, (const PoseEdge*)(d + o_edges), d + o_level, d + o_flags, trials_robust, trials, each_iter,
                                                           d_pose_out, d_n_valid);
    if (max_kp > 0) track_scatter_kernel<<<dim3(ceil_div(max_kp, 256), n_frames), 256, 0, st>>>(d_frames, dp, d + o_flags, (const int*)(d + o_kp));
    B200_CUDA(cudaGetLastError());
    S.last_launches = 3;
    return B200_OK;
}
}  // namespace chain
}  // namespace b200
