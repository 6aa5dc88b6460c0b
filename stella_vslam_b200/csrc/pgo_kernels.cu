// pgo_kernels.cu -- optimize::graph_optimizer (Sim3 pose-graph optimisation of a loop closure) on sm_90a, fp64.
//
// Reference path (relative to the reference checkout):
//   graph_optimizer::optimize steps 4-5       src/stella_vslam/optimize/graph_optimizer.cc:254-302
//   graph_opt_edge / shot_vertex              optimize/internal/sim3/graph_opt_edge.h, shot_vertex.h
//   terminate_action (gain threshold 1e-3)    optimize/terminate_action.cc:36-76
// and upstream g2o (tag 20230223_git, not vendored): g2o::Sim3 (sim3.cuh), BaseFixedSizedEdge's numeric Jacobian (central
// difference, delta 1e-9, one vertex dimension at a time), BlockSolver_7_3, OptimizationAlgorithmLevenberg (tau 1e-5, rho rule,
// at most 10 trials).
//
// One call: one upload, then per LM iteration a linearisation pass (errors, one thread per (edge, vertex, dimension) for the
// Jacobian, each nonzero 7x7 block and b summed over its edges in edge order) and per trial one replay of a captured CUDA graph:
// scatter the blocks + lambda into the envelope, factor it panel by panel (right-looking, 32x32 tiles, an active-row list per panel),
// forward / backward substitution, trial oplus and chi2.  The LM decisions are taken on the host from one small read-back per
// trial.  The free vertices are ordered once per call by reverse Cuthill-McKee (ties by index), so the envelope of a map that
// revisits old ground stays narrow.  No floating-point atomics: repeated calls are bit-identical.
#include <algorithm>
#include <cfloat>
#include <chrono>
#include <cmath>
#include <cstring>
#include <map>
#include <vector>

#include "common.cuh"
#include "sim3.cuh"
#include "staging.cuh"

namespace b200 {

namespace pgo {

using sim3::Sim3;
constexpr int kT = 32;          // tile edge
constexpr int kTT = kT * kT;
constexpr double kDelta = 1e-9;  // BaseFixedSizedEdge::linearizeOplus

static_assert(sizeof(Sim3) == sizeof(b200_sim3_t), "Sim3 layout");

// ---------------------------------------------------------------------------------------------------------------
// host plan: validation, RCM order, envelope, block lists
// ---------------------------------------------------------------------------------------------------------------
struct Plan {
    int nv = 0, ne = 0, nf = 0, n = 0, nt = 0;   // vertices, edges, free vertices, unknowns, tiles
    std::vector<int> order;                        // position -> vertex
    std::vector<int> vpos;                         // vertex -> position or -1
    std::vector<int> ftile;                        // tile row -> first tile
    std::vector<long long> tile_off;               // tile row -> offset (doubles) of its first tile
    long long env = 0;                             // envelope doubles
    std::vector<int> rows_ptr, rows_idx;           // active rows (tile rows i > k with ftile[i] <= k) per panel k
    // nonzero 7x7 blocks of the lower triangle (permuted): first the nf diagonal blocks (position order), then the off-diagonal ones
    std::vector<int> blk_r, blk_c;                 // block row / column positions
    std::vector<int> blk_ptr, blk_con;             // contributions: edge * 4 + row side * 2 + column side, in edge order
    long long flops = 0;
};

static bool finite_sim3(const b200_sim3_t& x) { return sim3::well_formed(x.q, x.t, x.s); }

static int validate(const b200_pose_graph_t* g, const char* who) {
    if (!g || g->n_vertices <= 0 || g->n_edges < 0 || g->n_points < 0 || !g->estimate || !g->fixed
        || (g->n_edges > 0 && (!g->e_v1 || !g->e_v2 || !g->e_meas)) || (g->n_points > 0 && (!g->points || !g->point_ref))) {
        set_error("%s: inconsistent pose graph description", who);
        return B200_ERR_INVALID;
    }
    int n_free = 0;
    for (int v = 0; v < g->n_vertices; ++v) {
        if (!finite_sim3(g->estimate[v])) {
            set_error("%s: vertex %d has a non-finite estimate or a scale <= 0", who, v);
            return B200_ERR_INVALID;
        }
        n_free += g->fixed[v] ? 0 : 1;
    }
    if (n_free == 0) {
        set_error("%s: no free vertex", who);
        return B200_ERR_INVALID;
    }
    for (int e = 0; e < g->n_edges; ++e) {
        const int a = g->e_v1[e], b = g->e_v2[e];
        if (a < 0 || b < 0 || a >= g->n_vertices || b >= g->n_vertices || a == b) {
            set_error("%s: edge %d joins vertices %d and %d", who, e, a, b);
            return B200_ERR_INVALID;
        }
        if (!finite_sim3(g->e_meas[e])) {
            set_error("%s: edge %d has a non-finite measurement or a scale <= 0", who, e);
            return B200_ERR_INVALID;
        }
    }
    for (int i = 0; i < g->n_points; ++i) {
        if (g->point_ref[i] < 0 || g->point_ref[i] >= g->n_vertices || !std::isfinite(g->points[3 * i]) || !std::isfinite(g->points[3 * i + 1])
            || !std::isfinite(g->points[3 * i + 2])) {
            set_error("%s: landmark %d has a reference vertex out of range or a non-finite position", who, i);
            return B200_ERR_INVALID;
        }
    }
    return B200_OK;
}

// Reverse Cuthill-McKee over the free vertices: start at the unvisited vertex of least degree (ties: lowest index), breadth-first,
// neighbours by (degree, index); reversed.  Components one after another.
static void rcm(const b200_pose_graph_t* g, Plan& P, std::vector<std::vector<int>>& adj) {
    const int nv = g->n_vertices;
    adj.assign(nv, {});
    for (int e = 0; e < g->n_edges; ++e) {
        const int a = g->e_v1[e], b = g->e_v2[e];
        if (g->fixed[a] || g->fixed[b]) continue;
        adj[a].push_back(b);
        adj[b].push_back(a);
    }
    std::vector<int> deg(nv, 0);
    for (int v = 0; v < nv; ++v) {
        std::sort(adj[v].begin(), adj[v].end());
        adj[v].erase(std::unique(adj[v].begin(), adj[v].end()), adj[v].end());
        deg[v] = (int)adj[v].size();
    }
    std::vector<int> byd;
    for (int v = 0; v < nv; ++v)
        if (!g->fixed[v]) byd.push_back(v);
    std::stable_sort(byd.begin(), byd.end(), [&](int a, int b) { return deg[a] < deg[b]; });
    std::vector<char> seen(nv, 0);
    std::vector<int> ord;
    ord.reserve(byd.size());
    std::vector<int> nb;
    for (int st : byd) {
        if (seen[st]) continue;
        seen[st] = 1;
        size_t head = ord.size();
        ord.push_back(st);
        while (head < ord.size()) {
            const int u = ord[head++];
            nb.clear();
            for (int w : adj[u])
                if (!seen[w]) nb.push_back(w);
            std::stable_sort(nb.begin(), nb.end(), [&](int a, int b) { return deg[a] < deg[b]; });
            for (int w : nb) {
                seen[w] = 1;
                ord.push_back(w);
            }
        }
    }
    std::reverse(ord.begin(), ord.end());
    P.order = ord;
    P.vpos.assign(nv, -1);
    for (int p = 0; p < (int)ord.size(); ++p) P.vpos[ord[p]] = p;
}

static void envelope(Plan& P, const std::vector<std::vector<int>>& adj) {
    P.nf = (int)P.order.size();
    P.n = 7 * P.nf;
    P.nt = ceil_div(P.n, kT);
    P.ftile.assign(P.nt, 0);
    for (int t = 0; t < P.nt; ++t) P.ftile[t] = t;
    for (int p = 0; p < P.nf; ++p) {
        int fp = p;
        for (int w : adj[P.order[p]]) fp = std::min(fp, P.vpos[w]);
        const int fcol_tile = (7 * fp) / kT;
        for (int r = 7 * p; r < 7 * p + 7; ++r) P.ftile[r / kT] = std::min(P.ftile[r / kT], fcol_tile);
    }
    P.tile_off.assign(P.nt, 0);
    long long off = 0;
    for (int t = 0; t < P.nt; ++t) {
        P.tile_off[t] = off;
        off += (long long)(t - P.ftile[t] + 1) * kTT;
    }
    P.env = off;
}

static void structure(const b200_pose_graph_t* g, Plan& P) {
    P.rows_ptr.assign(P.nt + 1, 0);
    for (int i = 0; i < P.nt; ++i)
        for (int k = P.ftile[i]; k < i; ++k) P.rows_ptr[k + 1]++;
    for (int k = 0; k < P.nt; ++k) P.rows_ptr[k + 1] += P.rows_ptr[k];
    P.rows_idx.assign(P.rows_ptr[P.nt], 0);
    std::vector<int> fill(P.rows_ptr.begin(), P.rows_ptr.end() - 1);
    for (int i = 0; i < P.nt; ++i)
        for (int k = P.ftile[i]; k < i; ++k) P.rows_idx[fill[k]++] = i;
    const double T3 = (double)kT * kT * kT;
    double fl = 0;
    for (int k = 0; k < P.nt; ++k) {
        const double m = P.rows_ptr[k + 1] - P.rows_ptr[k];
        fl += T3 / 3 + m * T3 + m * (m + 1) / 2 * 2 * T3;
    }
    P.flops = (long long)fl;

    // blocks: diagonal ones first, then the off-diagonal ones in order of first appearance
    std::vector<std::vector<int>> con(P.nf);
    std::map<std::pair<int, int>, int> off_id;
    std::vector<std::pair<int, int>> off_rc;
    std::vector<std::vector<int>> off_con;
    for (int e = 0; e < g->n_edges; ++e) {
        const int v[2] = {g->e_v1[e], g->e_v2[e]};
        const int p[2] = {P.vpos[v[0]], P.vpos[v[1]]};
        for (int s = 0; s < 2; ++s)
            if (p[s] >= 0) con[p[s]].push_back(e * 4 + s * 2 + s);
        if (p[0] >= 0 && p[1] >= 0) {
            const int sr = p[0] > p[1] ? 0 : 1;  // the side whose position is larger is the block row
            const std::pair<int, int> key(p[sr], p[1 - sr]);
            auto it = off_id.find(key);
            int id;
            if (it == off_id.end()) {
                id = (int)off_rc.size();
                off_id.emplace(key, id);
                off_rc.push_back(key);
                off_con.emplace_back();
            } else {
                id = it->second;
            }
            off_con[id].push_back(e * 4 + sr * 2 + (1 - sr));
        }
    }
    const int nb = P.nf + (int)off_rc.size();
    P.blk_r.resize(nb);
    P.blk_c.resize(nb);
    P.blk_ptr.assign(nb + 1, 0);
    P.blk_con.clear();
    for (int b = 0; b < nb; ++b) {
        const std::vector<int>& c = b < P.nf ? con[b] : off_con[b - P.nf];
        P.blk_r[b] = b < P.nf ? b : off_rc[b - P.nf].first;
        P.blk_c[b] = b < P.nf ? b : off_rc[b - P.nf].second;
        P.blk_con.insert(P.blk_con.end(), c.begin(), c.end());
        P.blk_ptr[b + 1] = (int)P.blk_con.size();
    }
}

static int make_plan(const b200_pose_graph_t* g, Plan& P, const char* who) {
    int rc = validate(g, who);
    if (rc) return rc;
    P.nv = g->n_vertices;
    P.ne = g->n_edges;
    std::vector<std::vector<int>> adj;
    rcm(g, P, adj);
    envelope(P, adj);
    return B200_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// device
// ---------------------------------------------------------------------------------------------------------------
struct Dev {
    Sim3 *est, *est_trial, *est_init, *meas, *est_out;
    int *e_v, *vpos, *ftile, *rows_ptr, *rows_idx, *blk_r, *blk_c, *blk_ptr, *blk_con, *point_ref;
    long long* tile_off;
    double *J, *err, *chi_e, *blkH, *b, *x, *env, *diagL, *points, *points_out, *pose_out;
    double* ctl;  // [0] lambda
    double* res;  // [0] chi2, [1] max |H_aa| or scale, [2] factorisation failed
    int nv, ne, nf, n, nt, nb, np, fix_scale;
};

__device__ __forceinline__ Sim3 ld(const Sim3* p, int i) { return p[i]; }

// graph_opt_edge::computeError for every edge, and its chi2 e^T I e
__global__ void __launch_bounds__(256) pgo_error_kernel(const Sim3* __restrict__ est, const Sim3* __restrict__ meas, const int* __restrict__ e_v,
                                                        int ne, double* __restrict__ err, double* __restrict__ chi_e) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= ne) return;
    double r[7];
    sim3::edge_error(meas[e], est[e_v[2 * e]], est[e_v[2 * e + 1]], r);
    double c = 0;
    for (int k = 0; k < 7; ++k) {
        if (err) err[7 * e + k] = r[k];
        c += r[k] * r[k];
    }
    chi_e[e] = c;
}

// BaseFixedSizedEdge::linearizeOplus: one thread per (edge, vertex side, dimension); fixed vertices get no Jacobian
__global__ void __launch_bounds__(256) pgo_jacobian_kernel(const Sim3* __restrict__ est, const Sim3* __restrict__ meas, const int* __restrict__ e_v,
                                                           const int* __restrict__ vpos, int ne, int fix_scale, double* __restrict__ J) {
    const int gid = blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= 14 * ne) return;
    const int e = gid / 14, s = (gid % 14) / 7, d = gid % 7;
    const int v = e_v[2 * e + s];
    if (vpos[v] < 0) return;
    const Sim3 m = meas[e];
    Sim3 v1 = est[e_v[2 * e]], v2 = est[e_v[2 * e + 1]];
    double add[7] = {0, 0, 0, 0, 0, 0, 0};
    double ep[7], em[7];
    add[d] = kDelta;
    if (s == 0) sim3::edge_error(m, sim3::oplus(v1, add, fix_scale), v2, ep);
    else sim3::edge_error(m, v1, sim3::oplus(v2, add, fix_scale), ep);
    add[d] = -kDelta;
    if (s == 0) sim3::edge_error(m, sim3::oplus(v1, add, fix_scale), v2, em);
    else sim3::edge_error(m, v1, sim3::oplus(v2, add, fix_scale), em);
    const double scalar = 1 / (2 * kDelta);
    double* Jo = J + (size_t)(2 * e + s) * 49;
    for (int k = 0; k < 7; ++k) Jo[7 * k + d] = scalar * (ep[k] - em[k]);
}

// H blocks (A^T I A summed over the block's edges in edge order) and b (-A^T I e on the diagonal blocks)
__global__ void __launch_bounds__(256) pgo_block_kernel(const double* __restrict__ J, const double* __restrict__ err, const int* __restrict__ blk_ptr,
                                                        const int* __restrict__ blk_con, int nb, int nf, double* __restrict__ blkH, double* __restrict__ bvec) {
    const int gid = blockIdx.x * blockDim.x + threadIdx.x;
    const int blk = gid / 56, q = gid % 56;
    if (blk >= nb || (q >= 49 && blk >= nf)) return;
    double tot = 0;
    if (q < 49) {
        const int a = q / 7, c = q % 7;
        for (int i = blk_ptr[blk]; i < blk_ptr[blk + 1]; ++i) {
            const int con = blk_con[i], e = con >> 2, sr = (con >> 1) & 1, sc = con & 1;
            const double* A = J + (size_t)(2 * e + sr) * 49;
            const double* B = J + (size_t)(2 * e + sc) * 49;
            double acc = 0;
            for (int k = 0; k < 7; ++k) acc += A[7 * k + a] * B[7 * k + c];
            tot += acc;
        }
        blkH[(size_t)blk * 49 + q] = tot;
    } else {
        const int a = q - 49;
        for (int i = blk_ptr[blk]; i < blk_ptr[blk + 1]; ++i) {
            const int con = blk_con[i], e = con >> 2, s = con & 1;
            const double* A = J + (size_t)(2 * e + s) * 49;
            double acc = 0;
            for (int k = 0; k < 7; ++k) acc += A[7 * k + a] * (-err[7 * e + k]);
            tot += acc;
        }
        bvec[7 * blk + a] = tot;
    }
}

// fixed-order single-CTA reductions: res[0] = sum chi_e, res[1] = max |H_aa| (mode 0) or x^T (lambda x + b) (mode 1)
__global__ void __launch_bounds__(1024) pgo_reduce_kernel(const double* __restrict__ chi_e, int ne, const double* __restrict__ blkH, int nf,
                                                          const double* __restrict__ x, const double* __restrict__ bvec, int n,
                                                          const double* __restrict__ ctl, int mode, double* __restrict__ res) {
    __shared__ double s0[1024], s1[1024];
    const int t = threadIdx.x;
    double c = 0, m = 0;
    for (int i = t; i < ne; i += 1024) c += chi_e[i];
    if (mode == 0) {
        for (int i = t; i < 7 * nf; i += 1024) m = fmax(m, fabs(blkH[(size_t)(i / 7) * 49 + (i % 7) * 8]));
    } else {
        const double lambda = ctl[0];
        for (int i = t; i < n; i += 1024) m += x[i] * (lambda * x[i] + bvec[i]);
    }
    s0[t] = c;
    s1[t] = m;
    __syncthreads();
    for (int w = 512; w > 0; w >>= 1) {
        if (t < w) {
            s0[t] += s0[t + w];
            s1[t] = mode == 0 ? fmax(s1[t], s1[t + w]) : s1[t] + s1[t + w];
        }
        __syncthreads();
    }
    if (t == 0) {
        res[0] = s0[0];
        res[1] = s1[0];
    }
}

__device__ __forceinline__ double* tile_ptr(double* env, const long long* tile_off, const int* ftile, int i, int j) {
    return env + tile_off[i] + (long long)(j - ftile[i]) * kTT;
}

// H + lambda I into the (zeroed) envelope: one thread per block entry of the lower triangle; the padding rows get a unit diagonal
__global__ void __launch_bounds__(256) pgo_scatter_kernel(const double* __restrict__ blkH, const int* __restrict__ blk_r, const int* __restrict__ blk_c,
                                                          int nb, int n, int nt, const double* __restrict__ ctl, double* __restrict__ env,
                                                          const long long* __restrict__ tile_off, const int* __restrict__ ftile, double* __restrict__ res) {
    const int gid = blockIdx.x * blockDim.x + threadIdx.x;
    if (gid == 0) res[2] = 0.0;
    if (gid < nt * kT - n) {
        const int r = n + gid;
        tile_ptr(env, tile_off, ftile, r / kT, r / kT)[(r % kT) * kT + r % kT] = 1.0;
    }
    if (gid >= nb * 49) return;
    const int blk = gid / 49, a = (gid % 49) / 7, c = gid % 7;
    const int br = blk_r[blk], bc = blk_c[blk];
    if (br == bc && c > a) return;
    double v = blkH[gid];
    if (br == bc && a == c) v += ctl[0];  // setLambda: lambda on every diagonal entry of the free vertices
    const int r = 7 * br + a, col = 7 * bc + c;
    tile_ptr(env, tile_off, ftile, r / kT, col / kT)[(r % kT) * kT + col % kT] = v;
}

// panel k: every CTA factors the diagonal tile in shared memory (identically); CTA 0 stores it in diagL, CTA 1 + a solves the tile of
// active row a: L(i,k) = A(i,k) L(k,k)^-T
__global__ void __launch_bounds__(256) pgo_panel_kernel(double* __restrict__ env, double* __restrict__ diagL, const long long* __restrict__ tile_off,
                                                        const int* __restrict__ ftile, const int* __restrict__ rows_ptr, const int* __restrict__ rows_idx,
                                                        int k, double* __restrict__ res) {
    __shared__ double D[kTT];
    __shared__ double X[kT * (kT + 1)];
    __shared__ int s_bad;
    const int tid = threadIdx.x;
    const double* Akk = tile_ptr(env, tile_off, ftile, k, k);
    for (int i = tid; i < kTT; i += blockDim.x) D[i] = Akk[i];
    if (tid == 0) s_bad = 0;
    __syncthreads();
    for (int j = 0; j < kT; ++j) {
        if (tid == 0) {
            const double d = D[j * kT + j];
            if (!(d > 0)) s_bad = 1;
            D[j * kT + j] = sqrt(d);
        }
        __syncthreads();
        if (tid > j && tid < kT) D[tid * kT + j] /= D[j * kT + j];
        __syncthreads();
        for (int idx = tid; idx < kTT; idx += blockDim.x) {
            const int r = idx / kT, c = idx % kT;
            if (c > j && r >= c) D[idx] -= D[r * kT + j] * D[c * kT + j];
        }
        __syncthreads();
    }
    if (blockIdx.x == 0) {
        for (int i = tid; i < kTT; i += blockDim.x) diagL[(size_t)k * kTT + i] = D[i];
        if (tid == 0 && s_bad) res[2] = 1.0;
        return;
    }
    const int i = rows_idx[rows_ptr[k] + blockIdx.x - 1];
    double* A = tile_ptr(env, tile_off, ftile, i, k);
    for (int q = tid; q < kTT; q += blockDim.x) X[(q / kT) * (kT + 1) + q % kT] = A[q];
    __syncthreads();
    if (tid < kT) {
        double* xr = X + tid * (kT + 1);
        for (int c = 0; c < kT; ++c) {
            double v = xr[c];
            for (int j = 0; j < c; ++j) v -= xr[j] * D[c * kT + j];
            xr[c] = v / D[c * kT + c];
        }
    }
    __syncthreads();
    for (int q = tid; q < kTT; q += blockDim.x) A[q] = X[(q / kT) * (kT + 1) + q % kT];
}

// right-looking update of panel k: A(i,j) -= L(i,k) L(j,k)^T for every pair of active rows i >= j
__global__ void __launch_bounds__(256) pgo_update_kernel(double* __restrict__ env, const long long* __restrict__ tile_off, const int* __restrict__ ftile,
                                                         const int* __restrict__ rows_ptr, const int* __restrict__ rows_idx, int k) {
    __shared__ double Li[kT * (kT + 1)], Lj[kT * (kT + 1)];
    const long long p = blockIdx.x;
    long long a = (long long)((sqrt(8.0 * (double)p + 1.0) - 1.0) / 2.0);
    while (a * (a + 1) / 2 > p) --a;
    while ((a + 1) * (a + 2) / 2 <= p) ++a;
    const int b = (int)(p - a * (a + 1) / 2);
    const int i = rows_idx[rows_ptr[k] + a], j = rows_idx[rows_ptr[k] + b];
    const double* Ti = tile_ptr(env, tile_off, ftile, i, k);
    const double* Tj = tile_ptr(env, tile_off, ftile, j, k);
    for (int q = threadIdx.x; q < kTT; q += blockDim.x) {
        Li[(q / kT) * (kT + 1) + q % kT] = Ti[q];
        Lj[(q / kT) * (kT + 1) + q % kT] = Tj[q];
    }
    __syncthreads();
    double* T = tile_ptr(env, tile_off, ftile, i, j);
    for (int q = threadIdx.x; q < kTT; q += blockDim.x) {
        const int r = q / kT, c = q % kT;
        const double* li = Li + r * (kT + 1);
        const double* lj = Lj + c * (kT + 1);
        double acc = 0;
        for (int m = 0; m < kT; ++m) acc += li[m] * lj[m];
        T[q] -= acc;
    }
}

__device__ __forceinline__ double warp_sum(double v) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// L y = b, then L^T x = y, in one CTA of 32 warps (x overwrites the vector in place)
__global__ void __launch_bounds__(1024) pgo_substitute_kernel(const double* __restrict__ env, const double* __restrict__ diagL,
                                                              const long long* __restrict__ tile_off, const int* __restrict__ ftile,
                                                              const int* __restrict__ rows_ptr, const int* __restrict__ rows_idx, int nt, int n,
                                                              const double* __restrict__ bvec, double* __restrict__ z) {
    __shared__ double part[kT][kT + 1];
    __shared__ double v[kT];
    const int w = threadIdx.x / 32, l = threadIdx.x % 32;
    for (int i = threadIdx.x; i < nt * kT; i += blockDim.x) z[i] = i < n ? bvec[i] : 0.0;
    __syncthreads();
    for (int k = 0; k < nt; ++k) {
        double acc = 0;  // row w of tile row k, column lane l
        for (int p = ftile[k]; p < k; ++p) acc += env[tile_off[k] + (long long)(p - ftile[k]) * kTT + w * kT + l] * z[p * kT + l];
        acc = warp_sum(acc);
        if (l == 0) v[w] = z[k * kT + w] - acc;
        __syncthreads();
        if (w == 0) {
            const double* Dk = diagL + (size_t)k * kTT;
            double y = v[l];
            for (int c = 0; c < kT; ++c) {
                const double yc = __shfl_sync(0xffffffffu, y, c) / Dk[c * kT + c];
                if (l == c) y = yc;
                else if (l > c) y -= Dk[l * kT + c] * yc;
            }
            z[k * kT + l] = y;
        }
        __syncthreads();
    }
    for (int k = nt - 1; k >= 0; --k) {
        double acc = 0;  // sum over the active rows i of L(i,k)[w][l] x_i[w]
        for (int q = rows_ptr[k]; q < rows_ptr[k + 1]; ++q) {
            const int i = rows_idx[q];
            acc += env[tile_off[i] + (long long)(k - ftile[i]) * kTT + w * kT + l] * z[i * kT + w];
        }
        part[w][l] = acc;
        __syncthreads();
        if (w == 0) {
            double s = 0;
            for (int r = 0; r < kT; ++r) s += part[r][l];
            const double* Dk = diagL + (size_t)k * kTT;
            double x = z[k * kT + l] - s;
            for (int r = kT - 1; r >= 0; --r) {
                const double xr = __shfl_sync(0xffffffffu, x, r) / Dk[r * kT + r];
                if (l == r) x = xr;
                else if (l < r) x -= Dk[r * kT + l] * xr;
            }
            z[k * kT + l] = x;
        }
        __syncthreads();
    }
}

// trial oplus: est_trial = Sim3(x_v) * est for the free vertices, a copy for the fixed ones
__global__ void __launch_bounds__(256) pgo_oplus_kernel(const Sim3* __restrict__ est, const int* __restrict__ vpos, const double* __restrict__ x, int nv,
                                                        int fix_scale, Sim3* __restrict__ out) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nv) return;
    const int p = vpos[v];
    out[v] = p < 0 ? est[v] : sim3::oplus(est[v], x + 7 * p, fix_scale);
}

// write-back (:261-302): pose_cw = [R | t / (float)s]; landmarks corrected through their reference keyframe
__global__ void __launch_bounds__(256) pgo_export_kernel(const Sim3* __restrict__ est, const Sim3* __restrict__ est_init, int nv,
                                                         const double* __restrict__ pts, const int* __restrict__ pref, int np, double* __restrict__ pose,
                                                         double* __restrict__ pts_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nv) {
        const Sim3 g = est[i];
        double R[9];
        quat_to_rot(g.q, R);
        const float s = (float)g.s;
        double* P = pose + 16 * (size_t)i;
        for (int r = 0; r < 3; ++r) {
            P[4 * r] = R[3 * r]; P[4 * r + 1] = R[3 * r + 1]; P[4 * r + 2] = R[3 * r + 2];
            P[4 * r + 3] = g.t[r] / (double)s;
        }
        P[12] = 0; P[13] = 0; P[14] = 0; P[15] = 1;
    }
    if (pts_out && i < np) {
        const int ref = pref[i];
        double pc[3], pw[3];
        sim3::map(est_init[ref], pts + 3 * (size_t)i, pc);
        sim3::map(sim3::inverse(est[ref]), pc, pw);
        for (int k = 0; k < 3; ++k) pts_out[3 * (size_t)i + k] = pw[k];
    }
}

// ---------------------------------------------------------------------------------------------------------------
// host driver
// ---------------------------------------------------------------------------------------------------------------
struct GraphGuard {
    cudaGraph_t g = nullptr;
    cudaGraphExec_t x = nullptr;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    ~GraphGuard() {
        if (x) cudaGraphExecDestroy(x);
        if (g) cudaGraphDestroy(g);
        for (cudaEvent_t e : ev)
            if (e) cudaEventDestroy(e);
    }
};

static int grid(long long n, int b) { return (int)std::max<long long>(1, ceil_div<long long>(n, b)); }

// the factorisation: zero the envelope, scatter H + lambda I, then the panels
static int launch_factor(const Dev& d, const Plan& P, cudaStream_t st, int* launches) {
    B200_CUDA(cudaMemsetAsync(d.env, 0, sizeof(double) * P.env, st));
    const long long scat = std::max<long long>((long long)d.nb * 49, (long long)P.nt * kT - P.n);
    pgo_scatter_kernel<<<grid(scat, 256), 256, 0, st>>>(d.blkH, d.blk_r, d.blk_c, d.nb, d.n, d.nt, d.ctl, d.env, d.tile_off, d.ftile, d.res);
    ++*launches;
    for (int k = 0; k < P.nt; ++k) {
        const int m = P.rows_ptr[k + 1] - P.rows_ptr[k];
        pgo_panel_kernel<<<1 + m, 256, 0, st>>>(d.env, d.diagL, d.tile_off, d.ftile, d.rows_ptr, d.rows_idx, k, d.res);
        ++*launches;
        if (m > 0) {
            pgo_update_kernel<<<(unsigned)((long long)m * (m + 1) / 2), 256, 0, st>>>(d.env, d.tile_off, d.ftile, d.rows_ptr, d.rows_idx, k);
            ++*launches;
        }
    }
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

static int launch_solve(const Dev& d, const Plan& P, cudaStream_t st, int* launches) {
    pgo_substitute_kernel<<<1, 1024, 0, st>>>(d.env, d.diagL, d.tile_off, d.ftile, d.rows_ptr, d.rows_idx, d.nt, d.n, d.b, d.x);
    pgo_oplus_kernel<<<grid(d.nv, 256), 256, 0, st>>>(d.est, d.vpos, d.x, d.nv, d.fix_scale, d.est_trial);
    pgo_error_kernel<<<grid(d.ne, 256), 256, 0, st>>>(d.est_trial, d.meas, d.e_v, d.ne, nullptr, d.chi_e);
    pgo_reduce_kernel<<<1, 1024, 0, st>>>(d.chi_e, d.ne, d.blkH, d.nf, d.x, d.b, d.n, d.ctl, 1, d.res);
    *launches += 4;
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

static int capture(cudaStream_t st, GraphGuard& G, int (*fn)(const Dev&, const Plan&, cudaStream_t, int*), const Dev& d, const Plan& P,
                   int* nodes) {
    B200_CUDA(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    const int rc = fn(d, P, st, nodes);
    cudaGraph_t g = nullptr;
    const cudaError_t e = cudaStreamEndCapture(st, &g);
    if (rc) {
        if (g) cudaGraphDestroy(g);
        return rc;
    }
    B200_CUDA(e);
    G.g = g;
    B200_CUDA(cudaGraphInstantiate(&G.x, G.g, 0));
    return B200_OK;
}

static int solve(b200_lba_t h, const b200_pose_graph_t* g, const Plan& P, int max_iter, double gain_threshold, b200_pgo_stats_t* stats) {
    const auto t0 = std::chrono::steady_clock::now();
    const int nv = P.nv, ne = P.ne, np = g->n_points, nb = (int)P.blk_r.size();
    const bool want_pts = g->points_out && np > 0;
    Layout A;
    // inputs (uploaded in one copy from the staging buffer, laid out identically)
    const size_t o_est = A.take(sizeof(Sim3) * nv), o_meas = A.take(sizeof(Sim3) * ne), o_ev = A.take(sizeof(int) * 2 * ne),
                 o_vpos = A.take(sizeof(int) * nv), o_ftile = A.take(sizeof(int) * P.nt), o_toff = A.take(sizeof(long long) * P.nt),
                 o_rptr = A.take(sizeof(int) * (P.nt + 1)), o_ridx = A.take(sizeof(int) * P.rows_idx.size()), o_br = A.take(sizeof(int) * nb),
                 o_bc = A.take(sizeof(int) * nb), o_bptr = A.take(sizeof(int) * (nb + 1)), o_bcon = A.take(sizeof(int) * P.blk_con.size()),
                 o_pts = A.take(sizeof(double) * 3 * (want_pts ? np : 0)), o_pref = A.take(sizeof(int) * (want_pts ? np : 0)),
                 o_ctl = A.take(sizeof(double) * 4);
    const size_t in_bytes = A.end;
    // outputs (downloaded in one copy)
    const size_t o_eout = A.take(sizeof(Sim3) * nv), o_pose = A.take(sizeof(double) * 16 * nv), o_pout = A.take(sizeof(double) * 3 * (want_pts ? np : 0)),
                 o_res = A.take(sizeof(double) * 4);
    const size_t out_lo = o_eout, out_hi = A.end;
    // device-only work buffers
    const size_t o_etr = A.take(sizeof(Sim3) * nv), o_einit = A.take(sizeof(Sim3) * nv), o_J = A.take(sizeof(double) * 98 * (size_t)ne),
                 o_err = A.take(sizeof(double) * 7 * (size_t)ne), o_chi = A.take(sizeof(double) * ne), o_blkH = A.take(sizeof(double) * 49 * (size_t)nb),
                 o_b = A.take(sizeof(double) * P.nt * kT), o_x = A.take(sizeof(double) * P.nt * kT), o_diag = A.take(sizeof(double) * kTT * (size_t)P.nt),
                 o_env = A.take(sizeof(double) * (size_t)P.env);
    cudaStream_t st;
    StagingArena* S;
    int rc = lba::staging(h, A.end, out_hi, &st, &S);
    if (rc) return rc;
    unsigned char *db = S->d, *hb = S->h;
    S->put(o_est, g->estimate, sizeof(Sim3) * nv);
    S->put(o_meas, g->e_meas, sizeof(Sim3) * ne);
    int* ev = (int*)(hb + o_ev);
    for (int e = 0; e < ne; ++e) { ev[2 * e] = g->e_v1[e]; ev[2 * e + 1] = g->e_v2[e]; }
    S->put(o_vpos, P.vpos.data(), sizeof(int) * nv);
    S->put(o_ftile, P.ftile.data(), sizeof(int) * P.nt);
    S->put(o_toff, P.tile_off.data(), sizeof(long long) * P.nt);
    S->put(o_rptr, P.rows_ptr.data(), sizeof(int) * (P.nt + 1));
    S->put(o_ridx, P.rows_idx.data(), sizeof(int) * P.rows_idx.size());
    S->put(o_br, P.blk_r.data(), sizeof(int) * nb);
    S->put(o_bc, P.blk_c.data(), sizeof(int) * nb);
    S->put(o_bptr, P.blk_ptr.data(), sizeof(int) * (nb + 1));
    S->put(o_bcon, P.blk_con.data(), sizeof(int) * P.blk_con.size());
    if (want_pts) {
        S->put(o_pts, g->points, sizeof(double) * 3 * np);
        S->put(o_pref, g->point_ref, sizeof(int) * np);
    }
    Dev d;
    d.est = (Sim3*)(db + o_est); d.meas = (Sim3*)(db + o_meas); d.est_trial = (Sim3*)(db + o_etr); d.est_init = (Sim3*)(db + o_einit);
    d.est_out = (Sim3*)(db + o_eout);
    d.e_v = (int*)(db + o_ev); d.vpos = (int*)(db + o_vpos); d.ftile = (int*)(db + o_ftile); d.tile_off = (long long*)(db + o_toff);
    d.rows_ptr = (int*)(db + o_rptr); d.rows_idx = (int*)(db + o_ridx); d.blk_r = (int*)(db + o_br); d.blk_c = (int*)(db + o_bc);
    d.blk_ptr = (int*)(db + o_bptr); d.blk_con = (int*)(db + o_bcon); d.point_ref = (int*)(db + o_pref);
    d.J = (double*)(db + o_J); d.err = (double*)(db + o_err); d.chi_e = (double*)(db + o_chi); d.blkH = (double*)(db + o_blkH);
    d.b = (double*)(db + o_b); d.x = (double*)(db + o_x); d.env = (double*)(db + o_env); d.diagL = (double*)(db + o_diag);
    d.points = (double*)(db + o_pts); d.points_out = (double*)(db + o_pout); d.pose_out = (double*)(db + o_pose);
    d.ctl = (double*)(db + o_ctl); d.res = (double*)(db + o_res);
    d.nv = nv; d.ne = ne; d.nf = P.nf; d.n = P.n; d.nt = P.nt; d.nb = nb; d.np = want_pts ? np : 0; d.fix_scale = g->fix_scale ? 1 : 0;
    double* h_ctl = (double*)(hb + o_ctl);
    const double* h_res = (const double*)(hb + o_res);

    GraphGuard Gf, Gs;
    for (cudaEvent_t& e : Gf.ev) B200_CUDA(cudaEventCreate(&e));
    int launches = 0, nodes_f = 0, nodes_s = 0;
    B200_CUDA(S->upload(in_bytes, st));
    B200_CUDA(cudaMemcpyAsync(d.est_init, d.est, sizeof(Sim3) * nv, cudaMemcpyDeviceToDevice, st));
    rc = capture(st, Gf, launch_factor, d, P, &nodes_f);
    if (rc) return rc;
    rc = capture(st, Gs, launch_solve, d, P, &nodes_s);
    if (rc) return rc;

    float lin_ms = 0, fac_ms = 0, sol_ms = 0;
    auto elapsed = [&](cudaEvent_t a, cudaEvent_t b, float* acc) -> int {
        float ms = 0;
        B200_CUDA(cudaEventElapsedTime(&ms, a, b));
        *acc += ms;
        return B200_OK;
    };
    // errors, Jacobians, blocks, chi2 and max |H_aa| of the current estimate
    auto linearize = [&]() -> int {
        B200_CUDA(cudaEventRecord(Gf.ev[0], st));
        pgo_error_kernel<<<grid(ne, 256), 256, 0, st>>>(d.est, d.meas, d.e_v, ne, d.err, d.chi_e);
        pgo_jacobian_kernel<<<grid(14LL * ne, 256), 256, 0, st>>>(d.est, d.meas, d.e_v, d.vpos, ne, d.fix_scale, d.J);
        pgo_block_kernel<<<grid(56LL * nb, 256), 256, 0, st>>>(d.J, d.err, d.blk_ptr, d.blk_con, nb, d.nf, d.blkH, d.b);
        pgo_reduce_kernel<<<1, 1024, 0, st>>>(d.chi_e, ne, d.blkH, d.nf, d.x, d.b, d.n, d.ctl, 0, d.res);
        launches += 4;
        B200_CUDA(cudaGetLastError());
        B200_CUDA(cudaEventRecord(Gf.ev[1], st));
        B200_CUDA(cudaMemcpyAsync(hb + o_res, d.res, sizeof(double) * 4, cudaMemcpyDeviceToHost, st));
        B200_CUDA(cudaStreamSynchronize(st));
        return elapsed(Gf.ev[0], Gf.ev[1], &lin_ms);
    };

    // SparseOptimizer::optimize(max_iter) with OptimizationAlgorithmLevenberg and terminate_action (terminate_action.cc:36-76)
    double lambda = 0, ni = 2, last_chi = 0, chi2_init = 0, chi = 0, lambda_init = 0;
    int it = 0, trials = 0;
    bool ok = true, stop = false;
    for (; it < max_iter && !stop && ok; ++it) {
        if ((rc = linearize())) return rc;
        double current_chi = h_res[0];
        if (it == 0) {  // computeLambdaInit: tau * max |H_jj| over the free vertices
            chi2_init = current_chi;
            lambda = 1e-5 * h_res[1];
            lambda_init = lambda;
            ni = 2;
        }
        double rho = 0;
        int qmax = 0;
        do {
            h_ctl[0] = lambda;
            B200_CUDA(cudaMemcpyAsync(d.ctl, h_ctl, sizeof(double), cudaMemcpyHostToDevice, st));
            B200_CUDA(cudaEventRecord(Gf.ev[0], st));
            B200_CUDA(cudaGraphLaunch(Gf.x, st));
            B200_CUDA(cudaEventRecord(Gf.ev[2], st));
            B200_CUDA(cudaGraphLaunch(Gs.x, st));
            B200_CUDA(cudaEventRecord(Gf.ev[3], st));
            B200_CUDA(cudaMemcpyAsync(hb + o_res, d.res, sizeof(double) * 4, cudaMemcpyDeviceToHost, st));
            B200_CUDA(cudaStreamSynchronize(st));
            if ((rc = elapsed(Gf.ev[0], Gf.ev[2], &fac_ms)) || (rc = elapsed(Gf.ev[2], Gf.ev[3], &sol_ms))) return rc;
            launches += nodes_f + nodes_s;
            ++trials;
            const bool ok2 = h_res[2] == 0.0;
            const double temp_chi = ok2 ? h_res[0] : DBL_MAX;
            rho = current_chi - temp_chi;
            const double scale = ok2 ? h_res[1] + 1e-3 : 1;  // computeScale() + 1e-3
            rho /= scale;
            if (rho > 0 && std::isfinite(temp_chi) && ok2) {
                double alpha = 1. - pow((2 * rho - 1), 3);
                alpha = std::min(alpha, 2. / 3.);
                const double sf = std::max(1. / 3., alpha);
                lambda *= sf;
                ni = 2;
                current_chi = temp_chi;
                B200_CUDA(cudaMemcpyAsync(d.est, d.est_trial, sizeof(Sim3) * nv, cudaMemcpyDeviceToDevice, st));  // discardTop
            } else {
                lambda *= ni;  // pop
                ni *= 2;
                if (!std::isfinite(lambda)) break;
            }
            qmax++;
        } while (rho < 0 && qmax < 10);
        if (qmax == 10 || rho == 0 || !std::isfinite(lambda)) ok = false;  // SolverResult::Terminate
        chi = current_chi;  // chi2 of the state the iteration leaves
        if (it == 0) {
            last_chi = chi;
        } else {
            const double gain = (last_chi - chi) / chi;
            last_chi = chi;
            if (gain >= 0 && gain < gain_threshold) stop = true;
        }
    }
    if (it == 0) {
        if ((rc = linearize())) return rc;
        chi2_init = chi = h_res[0];
    }
    pgo_export_kernel<<<grid(std::max(nv, d.np), 256), 256, 0, st>>>(d.est, d.est_init, nv, d.points, d.point_ref, d.np, d.pose_out,
                                                                     want_pts ? d.points_out : nullptr);
    ++launches;
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaMemcpyAsync(d.est_out, d.est, sizeof(Sim3) * nv, cudaMemcpyDeviceToDevice, st));
    B200_CUDA(S->download(out_lo, out_hi, st));
    B200_CUDA(cudaStreamSynchronize(st));
    memcpy(g->estimate_out, hb + o_eout, sizeof(Sim3) * nv);
    memcpy(g->pose_cw_out, hb + o_pose, sizeof(double) * 16 * nv);
    if (want_pts) memcpy(g->points_out, hb + o_pout, sizeof(double) * 3 * np);
    if (stats) {
        stats->iterations = it;
        stats->trials = trials;
        stats->chi2_init = chi2_init;
        stats->chi2_final = chi;
        stats->lambda_init = lambda_init;
        stats->lambda_final = lambda;
        stats->envelope_doubles = P.env;
        stats->factor_flops = P.flops;
        stats->launches = launches;
        stats->lin_ms = lin_ms;
        stats->factor_ms = fac_ms;
        stats->solve_ms = sol_ms;
        stats->total_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    }
    return B200_OK;
}

}  // namespace pgo
}  // namespace b200

extern "C" {

int b200_pgo_envelope(const b200_pose_graph_t* g, int32_t* n_free, int32_t* order_out, int64_t* envelope_doubles) {
    b200::pgo::Plan P;
    const int rc = b200::pgo::make_plan(g, P, "b200_pgo_envelope");
    if (rc) return rc;
    if (n_free) *n_free = P.nf;
    if (order_out) memcpy(order_out, P.order.data(), sizeof(int32_t) * P.nf);
    if (envelope_doubles) *envelope_doubles = P.env;
    return B200_OK;
}

int b200_graph_optimize(b200_lba_t h, const b200_pose_graph_t* g, int max_iter, double gain_threshold, b200_pgo_stats_t* stats) {
    B200_RANGE("b200:lba:graph_optimize");
    if (!h || !g || !g->estimate_out || !g->pose_cw_out || max_iter < 0 || !(gain_threshold >= 0.0)) {
        b200::set_error("b200_graph_optimize: null argument");
        return B200_ERR_INVALID;
    }
    b200::pgo::Plan P;
    int rc = b200::pgo::make_plan(g, P, "b200_graph_optimize");
    if (rc) return rc;
    if (P.env > B200_PGO_MAX_ENVELOPE_DOUBLES) {
        b200::set_error("b200_graph_optimize: the envelope of %d free vertices needs %lld doubles, more than the bound of %lld", P.nf,
                        (long long)P.env, (long long)B200_PGO_MAX_ENVELOPE_DOUBLES);
        return B200_ERR_CAPACITY;
    }
    b200::pgo::structure(g, P);
    return b200::pgo::solve(h, g, P, max_iter, gain_threshold, stats);
}

}  // extern "C"
