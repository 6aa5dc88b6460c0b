/*
 * tests/rgbd_oracle.c -- TEST INFRASTRUCTURE.  CPU restatement of the RGB-D frame step and of the depth-seeded landmarks, written from
 * the reference's behaviour, independently of the device code:
 *   system::create_RGBD_frame, the depth loop            src/stella_vslam/system.cc:494-511
 *   util::convert_to_true_depth                          util/image_converter.cc:41-43 = convertTo(CV_32F, 1.0 / factor), which OpenCV
 *                                                        evaluates as (float)v * (float)(1.0 / factor) and as a copy for 32F with factor 1
 *                                                        (pinned against cv2 by tests/test_rgbd_cpu.py)
 *   module::keyframe_inserter::create_new_keyframe       module/keyframe_inserter.cc:160-212 (mode 0)
 *   module::initializer::create_map_for_stereo           module/initializer.cc:363-387 (mode 1)
 *   data::triangulate_stereo                             data/common.cc:192-260
 *   data::landmark::update_mean_normal_and_obs_scale_variance with one observation (data/landmark.cc:256-311)
 * Compiled without contraction (-ffp-contract=off), so every operation is rounded as written.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>

/* img_depth.at<float>(y, x) after convert_to_true_depth, for the pixel (xi, yi) */
static float true_depth(const void* map, int depth_type, size_t pitch, int xi, int yi, double factor) {
    const unsigned char* row = (const unsigned char*)map + (size_t)yi * pitch;
    const float scale = (float)(1.0 / factor);
    if (depth_type == 2) return (float)((const uint16_t*)row)[xi] * scale;
    const float v = ((const float*)row)[xi];
    return factor == 1.0 ? v : v * scale;
}

/* one frame: kx, ky = keypts_[idx].pt (distorted), ux = undist_keypts_[idx].pt.x */
void rgo_depths(const float* kx, const float* ky, const float* ux, int n, const void* map, int depth_type, int w, int h, size_t pitch, double factor,
                double focal_x_baseline, float* depths, float* x_right) {
    for (int i = 0; i < n; ++i) {
        const int xi = (int)kx[i], yi = (int)ky[i]; /* the float -> int conversion of at<float>(y, x) truncates */
        const float depth = (0 <= xi && xi < w && 0 <= yi && yi < h) ? true_depth(map, depth_type, pitch, xi, yi, factor) : -1.f;
        if (!(0 < depth)) {
            depths[i] = -1.f;
            x_right[i] = -1.f;
            continue;
        }
        depths[i] = depth;
        x_right[i] = (float)((double)ux[i] - focal_x_baseline / (double)depth);
    }
}

typedef struct {
    float depth;
    unsigned idx;
} pair_t;

/* std::pair<float, unsigned>'s operator<: first, then second */
static int pair_cmp(const void* a, const void* b) {
    const pair_t *p = (const pair_t*)a, *q = (const pair_t*)b;
    if (p->depth < q->depth) return -1;
    if (q->depth < p->depth) return 1;
    return (p->idx > q->idx) - (p->idx < q->idx);
}

static void make_landmark(const double* pose_wc, double fx_inv, double fy_inv, double cx, double cy, float x, float y, float depth, float scale_factor,
                          float inv_scale_factor_last, double* pos_w, double* mean_normal, float* min_valid, float* max_valid) {
    const float unproj_x = (float)((x - cx) * depth * fx_inv);
    const float unproj_y = (float)((y - cy) * depth * fy_inv);
    const double pc[3] = {unproj_x, unproj_y, depth};
    const double c[3] = {pose_wc[3], pose_wc[7], pose_wc[11]};
    for (int r = 0; r < 3; ++r) pos_w[r] = pose_wc[4 * r] * pc[0] + pose_wc[4 * r + 1] * pc[1] + pose_wc[4 * r + 2] * pc[2] + c[r];
    /* one observation at the camera centre, which is also the reference keyframe */
    const double v[3] = {pos_w[0] - c[0], pos_w[1] - c[1], pos_w[2] - c[2]};
    const double nrm = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    double m[3];
    for (int k = 0; k < 3; ++k) m[k] = 0.0 + (nrm > 0 ? v[k] / nrm : v[k]);
    const double mn = sqrt(m[0] * m[0] + m[1] * m[1] + m[2] * m[2]);
    for (int k = 0; k < 3; ++k) mean_normal[k] = mn > 0 ? m[k] / mn : m[k];
    const float mx = (float)(nrm * scale_factor);
    *max_valid = mx;
    *min_valid = mx * inv_scale_factor_last;
}

/* Returns the number of landmarks created, in creation order.  has_landmark may be NULL (mode 0 only). */
int rgo_depth_landmarks(int mode, const double* pose_wc, double fx_inv, double fy_inv, double cx, double cy, double depth_thr, int n, const float* x,
                        const float* y, const int32_t* octave, const float* depth, const uint8_t* has_landmark, const float* scale_factors,
                        float inv_scale_factor_last, int32_t* idx_out, double* pos_w, double* mean_normal, float* min_valid, float* max_valid) {
    int k = 0;
    if (mode == 1) {
        for (int idx = 0; idx < n; ++idx) {
            const float z = depth[idx];
            if (z <= 0 || !(0 < z)) continue;
            make_landmark(pose_wc, fx_inv, fy_inv, cx, cy, x[idx], y[idx], z, scale_factors[octave[idx]], inv_scale_factor_last, pos_w + 3 * k,
                          mean_normal + 3 * k, min_valid + k, max_valid + k);
            idx_out[k++] = idx;
        }
        return k;
    }
    pair_t* pairs = (pair_t*)malloc(sizeof(pair_t) * (size_t)(n > 0 ? n : 1));
    int np = 0;
    for (int idx = 0; idx < n; ++idx)
        if (0 < depth[idx]) {
            pairs[np].depth = depth[idx];
            pairs[np].idx = (unsigned)idx;
            ++np;
        }
    qsort(pairs, (size_t)np, sizeof(pair_t), pair_cmp);
    const unsigned min_num_to_create = 100;
    for (unsigned count = 0; count < (unsigned)np; ++count) {
        const float z = pairs[count].depth;
        const unsigned idx = pairs[count].idx;
        if (min_num_to_create < count && depth_thr < z) break;
        if (has_landmark && has_landmark[idx]) continue;
        make_landmark(pose_wc, fx_inv, fy_inv, cx, cy, x[idx], y[idx], z, scale_factors[octave[idx]], inv_scale_factor_last, pos_w + 3 * k,
                      mean_normal + 3 * k, min_valid + k, max_valid + k);
        idx_out[k++] = (int32_t)idx;
    }
    free(pairs);
    return k;
}
