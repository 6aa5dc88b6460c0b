// triangulate.cuh -- module::two_view_triangulator::triangulate (src/stella_vslam/module/two_view_triangulator.cc:18-122, .h:88-108)
// as a device function, with solve::triangulator::triangulate (solve/triangulator.h:77-90: null vector of a 4x4 by a two-sided
// Jacobi SVD in the manner of Eigen::JacobiSVD) and data::triangulate_stereo (data/common.cc:192-260).
//
// Every fp64 / fp32 operation is an explicit round-to-nearest intrinsic, so no multiply-add is contracted whatever the translation
// unit's -fmad setting: the arithmetic is the CPU restatement's (tests/mapping_oracle.c) operation for operation -- sums left to right
// in index order, float exactly where the reference stores float.  atan2 / cos (stereo parallax) and asin / atan2 (equirectangular
// reprojection) are CUDA's libm, within 1-2 ulp of glibc; they only feed accept / reject comparisons (DESIGN.md section 4).
#pragma once

#include "jacobi.cuh"

namespace b200 {
namespace tri {

// One keyframe as the triangulator reads it (device copy of b200_tri_keyframe_t with device pointers).
struct TriKfDev {
    double pose_cw[16], pose_wc[16];
    int model;  // 0 perspective family, 1 equirectangular
    double fx, fy, cx, cy, fx_inv, fy_inv, fxb, true_baseline, cols, rows;
    const float *x, *y, *x_right, *depth, *scale_factors, *level_sigma_sq;
    const int* octave;
    const double* bearings;
};

// Null vector (column of V for the smallest singular value) of the row-major 4x4 A.  Returns false when the sweeps did not converge.
__device__ __forceinline__ bool jacobi_svd4_null(const double (&A)[16], double (&v)[4]) {
    double W[16], V[16];
    double scale = 0.0;
#pragma unroll
    for (int k = 0; k < 16; ++k)
        if (fabs(A[k]) > scale) scale = fabs(A[k]);
    if (scale == 0.0) scale = 1.0;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        W[k] = dd(A[k], scale);
        V[k] = (k % 5 == 0) ? 1.0 : 0.0;
    }
    double max_diag = fabs(W[0]);
#pragma unroll
    for (int i = 1; i < 4; ++i)
        if (fabs(W[i * 5]) > max_diag) max_diag = fabs(W[i * 5]);
    const double precision = 2.0 * DBL_EPSILON;
    bool finished = false;
    int sweeps = 0;
    while (!finished) {
        if (sweeps == kMaxSweeps) return false;
        ++sweeps;
        finished = true;
#pragma unroll
        for (int p = 1; p < 4; ++p) {
#pragma unroll
            for (int q = 0; q < p; ++q) {
                const double pm = dm(precision, max_diag);
                const double threshold = DBL_MIN < pm ? pm : DBL_MIN;
                if (!(fabs(W[p * 4 + q]) > threshold || fabs(W[q * 4 + p]) > threshold)) continue;
                finished = false;
                double cl, sl, cr, sr;
                jacobi_2x2(W[p * 4 + p], W[p * 4 + q], W[q * 4 + p], W[q * 4 + q], cl, sl, cr, sr);
                if (!(cl == 1.0 && sl == 0.0)) {
#pragma unroll
                    for (int k = 0; k < 4; ++k) rot2(W[p * 4 + k], W[q * 4 + k], cl, sl);
                }
                if (!(cr == 1.0 && -sr == 0.0)) {
#pragma unroll
                    for (int k = 0; k < 4; ++k) rot2(W[k * 4 + p], W[k * 4 + q], cr, -sr);
#pragma unroll
                    for (int k = 0; k < 4; ++k) rot2(V[k * 4 + p], V[k * 4 + q], cr, -sr);
                }
                const double dp = fabs(W[p * 5]), dq = fabs(W[q * 5]);
                const double dmx = dp < dq ? dq : dp;
                if (max_diag < dmx) max_diag = dmx;
            }
        }
    }
    double sv[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) sv[i] = dm(fabs(W[i * 5]), scale);
    // descending selection sort, first maximum on ties, stop at a zero maximum; only the column that ends up last is needed
    // (register-resident: every array index below is a compile-time constant)
    int col[4] = {0, 1, 2, 3};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        int pos = i;
        double best = sv[i];
#pragma unroll
        for (int k = i + 1; k < 4; ++k)
            if (sv[k] > best) {
                best = sv[k];
                pos = k;
            }
        if (best == 0.0) break;
#pragma unroll
        for (int k = i + 1; k < 4; ++k)
            if (k == pos) {
                const double ts = sv[i];
                sv[i] = sv[k];
                sv[k] = ts;
                const int tc = col[i];
                col[i] = col[k];
                col[k] = tc;
            }
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        double x = 0.0;
#pragma unroll
        for (int c = 0; c < 4; ++c)
            if (col[3] == c) x = V[r * 4 + c];
        v[r] = x;
    }
    return true;
}

// R p + t of a row-major 4x4 pose, row r
__device__ __forceinline__ double transform_row(const double* P, int r, double p0, double p1, double p2) {
    return da(dot3(P[r * 4], P[r * 4 + 1], P[r * 4 + 2], p0, p1, p2), P[r * 4 + 3]);
}

__device__ __forceinline__ bool depth_is_positive(const TriKfDev& K, const double (&p)[3]) {
    return K.model == 1 || 0.0 < transform_row(K.pose_cw, 2, p[0], p[1], p[2]);
}

// check_reprojection_error (two_view_triangulator.cc:92-122); the visibility bool of reproject_to_image is ignored there
__device__ __forceinline__ bool reprojection_ok(const TriKfDev& K, const double (&p)[3], int idx, bool is_stereo) {
    const double pc0 = transform_row(K.pose_cw, 0, p[0], p[1], p[2]);
    const double pc1 = transform_row(K.pose_cw, 1, p[0], p[1], p[2]);
    const double pc2 = transform_row(K.pose_cw, 2, p[0], p[1], p[2]);
    double r0, r1;
    float x_right_c;
    if (K.model == 1) {  // equirectangular.cc:59-73
        const double n = dot3(pc0, pc1, pc2, pc0, pc1, pc2);
        double b0 = pc0, b1 = pc1, b2 = pc2;
        if (n > 0.0) {
            const double s = __dsqrt_rn(n);
            b0 = dd(pc0, s);
            b1 = dd(pc1, s);
            b2 = dd(pc2, s);
        }
        const double latitude = -asin(b1);
        const double longitude = atan2(b0, b2);
        r0 = dm(K.cols, da(0.5, dd(longitude, dm(2.0, M_PI))));
        r1 = dm(K.rows, ds(0.5, dd(latitude, M_PI)));
        x_right_c = 0.0f;
    } else {  // perspective.cc:130-148
        const double z_inv = dd(1.0, pc2);
        r0 = da(dm(dm(K.fx, pc0), z_inv), K.cx);
        r1 = da(dm(dm(K.fy, pc1), z_inv), K.cy);
        x_right_c = __double2float_rn(ds(r0, dm(K.fxb, z_inv)));
    }
    const float sigma_sq = K.level_sigma_sq[K.octave[idx]];
    const double e0 = ds(r0, (double)K.x[idx]), e1 = ds(r1, (double)K.y[idx]);
    const double sq = da(dm(e0, e0), dm(e1, e1));
    if (is_stereo) {
        const float exr = __fsub_rn(x_right_c, K.x_right[idx]);
        return !((double)__fmul_rn(7.81473f, sigma_sq) < da(sq, (double)__fmul_rn(exr, exr)));
    }
    return !((double)__fmul_rn(5.99146f, sigma_sq) < sq);
}

// data::triangulate_stereo, perspective family: unprojection in double stored as float, then rot_wc p + trans_wc
__device__ __forceinline__ void triangulate_stereo(const TriKfDev& K, int idx, double (&p)[3]) {
    const float depth = K.depth ? K.depth[idx] : -1.0f;
    if (!(0.0 < depth)) {
        p[0] = p[1] = p[2] = 0.0;
        return;
    }
    const double ux = (double)__double2float_rn(dm(dm(ds((double)K.x[idx], K.cx), (double)depth), K.fx_inv));
    const double uy = (double)__double2float_rn(dm(dm(ds((double)K.y[idx], K.cy), (double)depth), K.fy_inv));
#pragma unroll
    for (int r = 0; r < 3; ++r) p[r] = transform_row(K.pose_wc, r, ux, uy, (double)depth);
}

// two_view_triangulator::triangulate.  pos_w receives the triangulated point (zeros when no branch applies) whatever the outcome.
// Returns 1 accepted, 0 rejected, -1 the Jacobi sweeps did not converge.
__device__ __forceinline__ int two_view_triangulate(const TriKfDev& k1, const TriKfDev& k2, int i1, int i2, float cos_rays_thr,
                                                    float ratio_factor, double (&pos_w)[3]) {
    const float xr1 = k1.x_right ? k1.x_right[i1] : -1.0f, xr2 = k2.x_right ? k2.x_right[i2] : -1.0f;
    const bool st1 = 0 <= xr1, st2 = 0 <= xr2;
    const double b10 = k1.bearings[3 * (size_t)i1], b11 = k1.bearings[3 * (size_t)i1 + 1], b12 = k1.bearings[3 * (size_t)i1 + 2];
    const double b20 = k2.bearings[3 * (size_t)i2], b21 = k2.bearings[3 * (size_t)i2 + 1], b22 = k2.bearings[3 * (size_t)i2 + 2];
    const double* P1 = k1.pose_cw;
    const double* P2 = k2.pose_cw;
    double rw1[3], rw2[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        rw1[i] = dot3(P1[i], P1[4 + i], P1[8 + i], b10, b11, b12);
        rw2[i] = dot3(P2[i], P2[4 + i], P2[8 + i], b20, b21, b22);
    }
    const double cos_rays = dot3(rw1[0], rw1[1], rw1[2], rw2[0], rw2[1], rw2[2]);
    const float d1 = k1.depth ? k1.depth[i1] : -1.0f, d2 = k2.depth ? k2.depth[i2] : -1.0f;
    const double cs1 = st1 ? cos(dm(2.0, atan2(dd(k1.true_baseline, 2.0), (double)d1))) : 2.0;
    const double cs2 = st2 ? cos(dm(2.0, atan2(dd(k2.true_baseline, 2.0), (double)d2))) : 2.0;
    const double cs = cs2 < cs1 ? cs2 : cs1;
    pos_w[0] = pos_w[1] = pos_w[2] = 0.0;
    const bool two_cameras = ((!st1 && !st2) && 0.0 < cos_rays && cos_rays < (double)cos_rays_thr) || ((st1 || st2) && 0.0 < cos_rays && cos_rays < cs);
    if (two_cameras) {
        double A[16], v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            A[j] = ds(dm(b10, P1[8 + j]), dm(b12, P1[j]));
            A[4 + j] = ds(dm(b11, P1[8 + j]), dm(b12, P1[4 + j]));
            A[8 + j] = ds(dm(b20, P2[8 + j]), dm(b22, P2[j]));
            A[12 + j] = ds(dm(b21, P2[8 + j]), dm(b22, P2[4 + j]));
        }
        if (!jacobi_svd4_null(A, v)) return -1;
#pragma unroll
        for (int k = 0; k < 3; ++k) pos_w[k] = dd(v[k], v[3]);
    } else if (st1 && cs1 < cs2) {
        triangulate_stereo(k1, i1, pos_w);
    } else if (st2 && cs2 < cs1) {
        triangulate_stereo(k2, i2, pos_w);
    } else {
        return 0;
    }
    if (!depth_is_positive(k1, pos_w) || !depth_is_positive(k2, pos_w)) return 0;
    if (!reprojection_ok(k1, pos_w, i1, st1) || !reprojection_ok(k2, pos_w, i2, st2)) return 0;
    // check_scale_factors (.h:93-108)
    const double v10 = ds(pos_w[0], k1.pose_wc[3]), v11 = ds(pos_w[1], k1.pose_wc[7]), v12 = ds(pos_w[2], k1.pose_wc[11]);
    const double v20 = ds(pos_w[0], k2.pose_wc[3]), v21 = ds(pos_w[1], k2.pose_wc[7]), v22 = ds(pos_w[2], k2.pose_wc[11]);
    const double dist1 = __dsqrt_rn(dot3(v10, v11, v12, v10, v11, v12)), dist2 = __dsqrt_rn(dot3(v20, v21, v22, v20, v21, v22));
    if (dist1 == 0.0 || dist2 == 0.0) return 0;
    const double ratio_dists = dd(dist2, dist1);
    const double ratio_octave = (double)__fdiv_rn(k1.scale_factors[k1.octave[i1]], k2.scale_factors[k2.octave[i2]]);
    return dd(ratio_octave, ratio_dists) < (double)ratio_factor && dd(ratio_dists, ratio_octave) < (double)ratio_factor;
}

}  // namespace tri
}  // namespace b200
