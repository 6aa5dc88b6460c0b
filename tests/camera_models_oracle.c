/*
 * tests/camera_models_oracle.c -- TEST INFRASTRUCTURE.  CPU restatement of the fisheye and radial-division camera steps between the
 * extractor and the matchers, written from the reference and OpenCV's published algorithm, independently of the device code:
 *   camera::fisheye::undistort_keypoints          src/stella_vslam/camera/fisheye.cc:281-309
 *        = cv::fisheye::undistortPoints(pts, K, D, R = empty, P = K) with the default TermCriteria(MAX_ITER + EPS, 10, 1e-8)
 *          (EXT: OpenCV calib3d fisheye.cpp; pinned against cv2 by tests/test_camera_models_cpu.py).  K and D are cv::Mat_<float>
 *          (fisheye.cc:21-22): the caller passes their float values.
 *   camera::radial_division::undistort_point      src/stella_vslam/camera/radial_division.cc:83-98
 *   data::frame::can_observe                      data/frame.cc:59-84 with fisheye.cc:169-187 (strict bounds) or
 *                                                 radial_division.cc:113-133 (inclusive bounds)
 * Compiled without contraction (-ffp-contract=off), so every double operation is rounded as written.
 */
#include <math.h>
#include <stdint.h>

#define CMO_PI 3.1415926535897932384626433832795

void cmo_fisheye_undistort(const float* xy, int n, float fx_f, float fy_f, float cx_f, float cy_f, const float* d4_f, float* out) {
    /* OpenCV widens the CV_32F camera matrix and coefficients to double */
    const double f0 = fx_f, f1 = fy_f, c0 = cx_f, c1 = cy_f;
    const double k[4] = {d4_f[0], d4_f[1], d4_f[2], d4_f[3]};
    const double eps = 1e-8;
    const int max_count = 10;
    for (int i = 0; i < n; ++i) {
        const double pi0 = xy[2 * i], pi1 = xy[2 * i + 1];
        const double pw0 = (pi0 - c0) / f0, pw1 = (pi1 - c1) / f1;
        double theta_d = sqrt(pw0 * pw0 + pw1 * pw1);
        /* theta_d = min(max(-pi/2, theta_d), pi/2) */
        const double lo = -CMO_PI / 2., hi = CMO_PI / 2.;
        if (lo < theta_d) {
        } else {
            theta_d = lo;
        }
        if (hi < theta_d) theta_d = hi;
        int converged = 0;
        double theta = theta_d, scale = 0.0;
        if (fabs(theta_d) > eps) {
            for (int j = 0; j < max_count; j++) {
                const double theta2 = theta * theta, theta4 = theta2 * theta2, theta6 = theta4 * theta2, theta8 = theta6 * theta2;
                const double k0_theta2 = k[0] * theta2, k1_theta4 = k[1] * theta4, k2_theta6 = k[2] * theta6, k3_theta8 = k[3] * theta8;
                const double theta_fix = (theta * (1 + k0_theta2 + k1_theta4 + k2_theta6 + k3_theta8) - theta_d) /
                                         (1 + 3 * k0_theta2 + 5 * k1_theta4 + 7 * k2_theta6 + 9 * k3_theta8);
                theta = theta - theta_fix;
                if (fabs(theta_fix) < eps) {
                    converged = 1;
                    break;
                }
            }
            scale = tan(theta) / theta_d;
        } else {
            converged = 1;
        }
        const int flipped = (theta_d < 0 && theta > 0) || (theta_d > 0 && theta < 0);
        if (converged && !flipped) {
            const double pu0 = pw0 * scale, pu1 = pw1 * scale;
            /* pr = (P * R) * (pu, 1) with R = I, P = K: row sums of a 3x3 product, left to right from 0 */
            const double RR[9] = {f0, 0, c0, 0, f1, c1, 0, 0, 1};
            double pr[3];
            for (int r = 0; r < 3; ++r) {
                double s = 0;
                s += RR[3 * r] * pu0;
                s += RR[3 * r + 1] * pu1;
                s += RR[3 * r + 2] * 1.0;
                pr[r] = s;
            }
            out[2 * i] = (float)(pr[0] / pr[2]);
            out[2 * i + 1] = (float)(pr[1] / pr[2]);
        } else {
            out[2 * i] = (float)-1000000.0;
            out[2 * i + 1] = (float)-1000000.0;
        }
    }
}

void cmo_radial_undistort(const float* xy, int n, double fx, double fy, double cx, double cy, double distortion, float* out) {
    for (int i = 0; i < n; ++i) {
        const double pixel_x = (xy[2 * i] - cx) / fx;
        const double pixel_y = (xy[2 * i + 1] - cy) / fy;
        const double radius_distorted_squared = pixel_x * pixel_x + pixel_y * pixel_y;
        const double undistortion = 1.0 + distortion * radius_distorted_squared;
        const double ux = pixel_x / undistortion, uy = pixel_y / undistortion;
        out[2 * i] = (float)(ux * fx + cx);
        out[2 * i + 1] = (float)(uy * fy + cy);
    }
}

/* data::frame::can_observe for the perspective-family reprojection (fisheye: strict bounds, radial division: inclusive bounds).
 * Rt_cw: rot_cw row-major then trans_cw; trans_wc: camera centre; bounds: the camera's float img_bounds_. */
void cmo_can_observe(int inclusive, double fx, double fy, double cx, double cy, double fxb, const float* bounds, const double* Rt_cw,
                     const double* trans_wc, int n, const double* pos_w, const double* mean_normal, const float* min_valid_dist,
                     const float* max_valid_dist, float ray_cos_thr, unsigned num_levels, float log_scale_factor, uint8_t* observable,
                     double* reproj, float* x_right, uint32_t* pred_scale_level) {
    for (int i = 0; i < n; ++i) {
        const double* p = pos_w + 3 * i;
        observable[i] = 0;
        reproj[2 * i] = 0.0;
        reproj[2 * i + 1] = 0.0;
        x_right[i] = 0.f;
        pred_scale_level[i] = 0;
        const double pc[3] = {Rt_cw[0] * p[0] + Rt_cw[1] * p[1] + Rt_cw[2] * p[2] + Rt_cw[9],
                              Rt_cw[3] * p[0] + Rt_cw[4] * p[1] + Rt_cw[5] * p[2] + Rt_cw[10],
                              Rt_cw[6] * p[0] + Rt_cw[7] * p[1] + Rt_cw[8] * p[2] + Rt_cw[11]};
        if (pc[2] <= 0.0) continue;
        const double z_inv = 1.0 / pc[2];
        const double u = fx * pc[0] * z_inv + cx, v = fy * pc[1] * z_inv + cy;
        const float xr = (float)(u - fxb * z_inv);
        int visible;
        if (inclusive)
            visible = !(u < bounds[0] || u > bounds[1]) && !(v < bounds[2] || v > bounds[3]);
        else
            visible = bounds[0] < u && u < bounds[1] && bounds[2] < v && v < bounds[3];
        if (!visible) continue;
        /* landmark::is_inside_in_orb_scale (data/landmark.h:88-92) */
        const double d[3] = {p[0] - trans_wc[0], p[1] - trans_wc[1], p[2] - trans_wc[2]};
        const double dist = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
        const float distf = (float)dist;
        const float max_dist = (float)1.3 * max_valid_dist[i], min_dist = (float)(1.0 / 1.3) * min_valid_dist[i];
        if (!(min_dist <= distf && distf <= max_dist)) continue;
        const double* nm = mean_normal + 3 * i;
        if ((d[0] * nm[0] + d[1] * nm[1] + d[2] * nm[2]) / dist < ray_cos_thr) continue;
        /* landmark::predict_scale_level (data/landmark.cc:336-353) */
        const float ratio = max_valid_dist[i] / distf;
        const int level = (int)ceilf(logf(ratio) / log_scale_factor);
        const float levels = (float)num_levels;
        uint32_t lv = (uint32_t)level;
        if (level < 0) lv = 0;
        else if (levels <= (float)(unsigned)level) lv = (uint32_t)(levels - 1);
        observable[i] = 1;
        reproj[2 * i] = u;
        reproj[2 * i + 1] = v;
        x_right[i] = xr;
        pred_scale_level[i] = lv;
    }
}
